"""Every public module / function / class / method / constant of the reference python package
exists here under the same name, and reference argument names can be used as keywords.
(The reference's public surface - names and positional argument lists, parsed from its sources
with ``ast`` - is stored in tests/golden/reference_api.json; the reference is never imported.)"""
import importlib
import inspect
import json
import os

import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_api.json")

with open(GOLDEN) as _f:
  REF_API = json.load(_f)


@pytest.mark.parametrize("mod", sorted(REF_API))
def test_public_surface(mod):
  ref = REF_API[mod]
  m = importlib.import_module("tensorflowonspark_b200." + mod)
  alias = importlib.import_module("tensorflowonspark." + mod)   # reference-style import path
  assert alias is m or alias.__dict__.keys() >= {k for k in m.__dict__ if not k.startswith("_")}
  missing, renamed = [], []

  def check_sig(owner, name, want, label):
    obj = getattr(owner, name)
    try:
      sig = inspect.signature(obj)
    except (TypeError, ValueError):
      return
    mine = [p.name for p in sig.parameters.values()
            if p.kind in (p.POSITIONAL_ONLY, p.POSITIONAL_OR_KEYWORD)]
    if inspect.isclass(owner) and want[:1] in (["self"], ["cls"]) and mine[:1] not in (["self"], ["cls"]):
      want = want[1:]
    if mine[:len(want)] != want:
      renamed.append((label, want, mine))

  for const in ref["constants"]:
    if not hasattr(m, const):
      missing.append(const)
  for name, args in sorted(ref["functions"].items()):
    if not hasattr(m, name):
      missing.append(name)
    else:
      check_sig(m, name, args, name)
  for cname, methods in sorted(ref["classes"].items()):
    if not hasattr(m, cname):
      missing.append(cname)
      continue
    cls = getattr(m, cname)
    for name, args in sorted(methods.items()):
      if not hasattr(cls, name):
        missing.append(cname + "." + name)
      else:
        check_sig(cls, name, args, cname + "." + name)
  assert not missing, "missing from tensorflowonspark_b200.{}: {}".format(mod, missing)
  assert not renamed, "argument names differ in {}: {}".format(mod, renamed)


def test_version_and_logging_format():
  import tensorflowonspark_b200 as pkg
  assert isinstance(pkg.__version__, str) and pkg.__version__

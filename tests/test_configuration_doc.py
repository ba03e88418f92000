"""docs/configuration.md and the code agree on the TFOS_* environment variables: every variable
that the package, csrc/, bench.py or baseline/ reads is on the page, and every variable on the page
is read there (or, for the ones the node runtime exports to user code, set there)."""
import ast
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAGE = os.path.join(ROOT, "docs", "configuration.md")
NAME = re.compile(r"\bTFOS_[A-Z0-9_]*[A-Z0-9]\b")
CPP_READ = re.compile(r"\bgetenv\(\s*\"(TFOS_[A-Z0-9_]+)\"")


def _files():
  yield os.path.join(ROOT, "bench.py")
  for top in ("tensorflowonspark_b200", "csrc", "baseline"):
    for d, _, names in os.walk(os.path.join(ROOT, top)):
      for n in sorted(names):
        if n.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
          yield os.path.join(d, n)


def _is_environ(node):
  return (isinstance(node, ast.Attribute) and node.attr == "environ"
          and isinstance(node.value, ast.Name) and node.value.id == "os")


def _python_uses(src):
  """(read, set) TFOS_* names of one module: os.environ.get(k), os.environ[k], k in os.environ and
  os.getenv(k) read; os.environ[k] = v sets.  k is a string literal or a module-level constant."""
  tree = ast.parse(src)
  consts = {}
  for node in tree.body:
    if (isinstance(node, ast.Assign) and isinstance(node.value, ast.Constant)
        and isinstance(node.value.value, str)):
      for t in node.targets:
        if isinstance(t, ast.Name):
          consts[t.id] = node.value.value

  def key(node):
    if isinstance(node, ast.Constant) and isinstance(node.value, str):
      return node.value
    return consts.get(node.id) if isinstance(node, ast.Name) else None

  read, set_ = set(), set()
  for node in ast.walk(tree):
    k, dst = None, read
    if isinstance(node, ast.Call) and node.args:
      f = node.func
      if isinstance(f, ast.Attribute) and ((f.attr == "get" and _is_environ(f.value)) or (
          f.attr == "getenv" and isinstance(f.value, ast.Name) and f.value.id == "os")):
        k = key(node.args[0])
    elif isinstance(node, ast.Subscript) and _is_environ(node.value):
      k = key(node.slice)
      dst = set_ if isinstance(node.ctx, ast.Store) else read
    elif (isinstance(node, ast.Compare) and len(node.ops) == 1
          and isinstance(node.ops[0], (ast.In, ast.NotIn)) and _is_environ(node.comparators[0])):
      k = key(node.left)
    if k is not None and NAME.fullmatch(k):
      dst.add(k)
  return read, set_


def _code_uses():
  read, set_ = set(), set()
  for path in _files():
    with open(path, encoding="utf-8") as f:
      src = f.read()
    if path.endswith(".py"):
      r, s = _python_uses(src)
      read |= r
      set_ |= s
    else:
      read |= set(CPP_READ.findall(src))
  return read, set_


def _page_names():
  with open(PAGE, encoding="utf-8") as f:
    return set(NAME.findall(f.read()))


def test_every_variable_read_is_documented():
  read, _ = _code_uses()
  assert read, "found no environment reads: the scan is broken"
  missing = sorted(read - _page_names())
  assert not missing, "read by the code but missing from docs/configuration.md: {}".format(missing)


def test_every_documented_variable_is_used():
  read, set_ = _code_uses()
  stale = sorted(_page_names() - read - set_)
  assert not stale, "on docs/configuration.md but never read by the code: {}".format(stale)


def test_scan_sees_every_kind_of_read():
  src = ("import os\nK = 'TFOS_A'\nos.environ.get('TFOS_B')\nos.environ['TFOS_C']\n"
         "'TFOS_D' in os.environ\nos.getenv(K)\nos.environ['TFOS_E'] = '1'\n")
  assert _python_uses(src) == ({"TFOS_A", "TFOS_B", "TFOS_C", "TFOS_D"}, {"TFOS_E"})
  assert CPP_READ.findall('const char* e = getenv("TFOS_F");') == ["TFOS_F"]

"""Native sm_90a ops.  ``ops.C()`` is the loaded extension module (csrc/binding.cpp);
``ops.igemm`` builds wgmma implicit-GEMM plans; everything else is a thin call
into a fused elementwise / reduction / collective kernel.

No op here falls back to eager PyTorch: if the extension is missing the call
raises, so a silent CPU/library path can never be mistaken for the product.
"""
from .. import _build
from . import igemm  # noqa: F401

_count = 0


def C():
  return _build.load(required=True)


def count(n=1):
  """Account n native launches (bench.py reports the total as gpu_launches)."""
  global _count
  _count += n


def launch_count():
  return _count + igemm.launch_count()


class _Counted(object):
  """Attribute proxy over the extension that counts kernel launches."""

  def __getattr__(self, name):
    fn = getattr(C(), name)

    def call(*a, **k):
      count()
      return fn(*a, **k)

    call.__name__ = name
    setattr(self, name, call)
    return call


K = _Counted()

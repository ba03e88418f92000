"""In-tree build and loading of the native sm_90a extension.

The extension (`csrc/*.cu`, `csrc/*.cc`, `csrc/binding.cpp`) is compiled with
``-gencode arch=compute_90a,code=sm_90a`` into
``tensorflowonspark_b200/_ext/_tfos_b200_C.so``.  The ``.so`` is git-ignored but
is loaded from the tree as built, so nothing is JIT-compiled at run time.

GPU ops fail loudly when the extension is missing; there is no eager fallback
for them.  (Host-only helpers - TFRecord codec, the shared-memory ring - have a
pure-Python twin used only when the extension has not been built yet.)
"""
import importlib.util
import logging
import os
import sys
import threading

logger = logging.getLogger(__name__)

EXT_NAME = "_tfos_b200_C"
PKG_DIR = os.path.dirname(os.path.abspath(__file__))
REPO_DIR = os.path.dirname(PKG_DIR)
CSRC_DIR = os.path.join(REPO_DIR, "csrc")
EXT_DIR = os.path.join(PKG_DIR, "_ext")

SOURCES = ["binding.cpp", "igemm.cu", "igemm_wgrad.cu", "elementwise.cu", "bn_bwd.cu", "stem_fused.cu",
           "smallops.cu", "eval.cu", "optim_comm.cu", "mix.cu", "distill.cu", "feed.cc",
           "tfrecord.cc", "vmm.cc"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "--expt-relaxed-constexpr", "--use_fast_math"]

_lock = threading.Lock()
_module = None
_load_error = None


def so_path():
  return os.path.join(EXT_DIR, EXT_NAME + ".so")


def build(verbose=False):
  """Compile the extension in-tree (works on a CPU-only host: nvcc cross-compiles)."""
  from torch.utils import cpp_extension
  os.makedirs(EXT_DIR, exist_ok=True)
  os.environ.setdefault("MAX_JOBS", str(min(8, os.cpu_count() or 4)))
  sources = [os.path.join(CSRC_DIR, s) for s in SOURCES]
  mod = cpp_extension.load(
      name=EXT_NAME,
      sources=sources,
      extra_cflags=["-O3", "-std=c++17"],
      extra_cuda_cflags=NVCC_FLAGS,
      extra_include_paths=[CSRC_DIR],
      build_directory=EXT_DIR,
      with_cuda=True,
      verbose=verbose,
  )
  global _module, _load_error
  _module, _load_error = mod, None
  return mod


def _stale():
  so = so_path()
  if not os.path.exists(so):
    return True
  if not os.path.isdir(CSRC_DIR):   # installed without the sources: the shipped .so is the product
    return False
  t = os.path.getmtime(so)
  for s in os.listdir(CSRC_DIR):
    if os.path.getmtime(os.path.join(CSRC_DIR, s)) > t:
      return True
  return False


def load(required=True):
  """Return the extension module, importing the prebuilt in-tree ``.so``."""
  global _module, _load_error
  with _lock:
    if _module is not None:
      return _module
    so = so_path()
    if os.path.exists(so):
      try:
        import torch  # noqa: F401  (libtorch must be loaded before the extension)
        spec = importlib.util.spec_from_file_location(EXT_NAME, so)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        sys.modules[EXT_NAME] = mod
        _module = mod
        return mod
      except Exception as e:  # pragma: no cover - depends on the host
        _load_error = e
        logger.warning("failed to import %s: %s", so, e)
    elif os.environ.get("TFOS_AUTOBUILD", "0") == "1":
      try:
        return build()
      except Exception as e:  # pragma: no cover
        _load_error = e
    if required:
      raise RuntimeError(
          "tensorflowonspark_b200 native extension is not available ({}); run "
          "`python -c 'import __graft_entry__ as g; g.build()'` from the repo root".format(
              _load_error or "not built"))
    return None


def available():
  return load(required=False) is not None

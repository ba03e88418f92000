"""The implicit-GEMM kernels keep their accumulators in registers.

A wgmma accumulator that ptxas cannot keep in registers goes to local memory: every tile then
stores and reloads it, and ptxas serialises the wgmma pipeline around it.  This compiles
igemm.cu and igemm_wgrad.cu with the extension's own flags and checks ptxas' resource report.
Needs nvcc, not a GPU.
"""
import os
import re
import shutil
import subprocess

import pytest

from tensorflowonspark_b200 import _build

NVCC = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin",
                                            "nvcc")


def ptxas_report(source, tmp_path):
  out = tmp_path / (source + ".o")
  cmd = [NVCC] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", _build.CSRC_DIR, "-c",
                                      os.path.join(_build.CSRC_DIR, source), "-o", str(out)]
  r = subprocess.run(cmd, capture_output=True, text=True)
  assert r.returncode == 0, r.stderr[-4000:]
  kernels, cur = {}, None
  for line in r.stderr.splitlines():
    m = re.search(r"Compiling entry function '(\S+)'", line)
    if m:
      cur = m.group(1)
      continue
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                  line)
    if m and cur is not None:
      kernels[cur] = tuple(int(x) for x in m.groups())
    if "C7517" in line:   # ptxas serialised the wgmma pipeline (warpgroup.wait injected)
      kernels.setdefault("C7517", ())
  return kernels


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not found")
@pytest.mark.parametrize("source", ["igemm.cu", "igemm_wgrad.cu"])
def test_igemm_kernels_keep_accumulators_in_registers(source, tmp_path):
  kernels = ptxas_report(source, tmp_path)
  assert "C7517" not in kernels, "ptxas injected warpgroup.wait into a wgmma pipeline"
  igemm = {k: v for k, v in kernels.items() if "igemm_" in k}
  assert igemm, "no igemm kernels in the ptxas report of " + source
  bad = {k: v for k, v in igemm.items() if v != (0, 0, 0)}
  assert not bad, "stack frame / spill stores / spill loads (bytes): {}".format(bad)

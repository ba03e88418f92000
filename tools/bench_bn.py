"""Micro-benchmark of the batch-norm kernels on ResNet-50 activation shapes (batch 256).
Reports GB/s against the algorithmic bytes of each kernel."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from tensorflowonspark_b200 import ops  # noqa: E402

K = ops.K
SHAPES = [(256 * 56 * 56, 64), (256 * 56 * 56, 256), (256 * 28 * 28, 512), (256 * 14 * 14, 1024),
          (256 * 7 * 7, 2048)]


def timeit(fn, iters=10):
  for _ in range(2):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(iters):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / iters * 1e3


def main():
  tot = {}
  for P, C in SHAPES:
    x = torch.randn(P, C, device="cuda").bfloat16()
    dy = torch.randn(P, C, device="cuda").bfloat16()
    y = torch.relu(x)
    res = torch.randn(P, C, device="cuda").bfloat16()
    out = torch.empty_like(x)
    bits = torch.zeros(P * C // 8, dtype=torch.uint8, device="cuda")
    z = lambda: torch.zeros(C, device="cuda")  # noqa: E731
    mean, invstd, gamma, dg, db, sc, sh = z(), z() + 1, z() + 1, z(), z(), z() + 1, z()
    n = P * C * 2 / 1e3  # KB per tensor pass
    cases = [
        ("apply+res", lambda: K.bn_apply(x, res, sc, sh, out, 1), 3),
        ("bwd_reduce m2", lambda: K.bn_bwd_reduce(dy, x, None, mean, invstd, dg, db, 2, sc, sh), 2),
        ("bwd_reduce m1", lambda: K.bn_bwd_reduce(dy, x, y, mean, invstd, dg, db, 1, None, None), 3),
        ("bwd_apply m2", lambda: K.bn_bwd_apply(dy, x, None, gamma, mean, invstd, dg, db, out, None, 2, sc, sh), 3),
        ("bwd_apply m1+dres",
         lambda: K.bn_bwd_apply(dy, x, y, gamma, mean, invstd, dg, db, out, res, 1, None, None), 5),
        ("bwd_reduce m3", lambda: K.bn_bwd_reduce(dy, x, bits, mean, invstd, dg, db, 3, None, None), 2.0625),
        ("bwd_apply m3+dres",
         lambda: K.bn_bwd_apply(dy, x, bits, gamma, mean, invstd, dg, db, out, res, 3, None, None), 4.0625),
    ]
    for name, fn, passes in cases:
      us = timeit(fn)
      tot[name] = tot.get(name, 0) + us
      print("P={:8d} C={:5d} {:18s} {:8.1f} us  {:7.1f} GB/s".format(P, C, name, us, passes * n / us))
  print("totals:", {k: round(v) for k, v in tot.items()})


if __name__ == "__main__":
  main()

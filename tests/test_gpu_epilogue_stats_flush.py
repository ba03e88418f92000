"""Fused per-column statistics of the forward-like GEMM epilogue (csrc/igemm.cu): each CTA combines
its register partials with warp shuffles and one shared-memory slot per warp, then adds them to the
global sums.  The sums must equal the float64 sums of the stored bf16 output, for CTAs that stay on
one n tile for their whole tile list (the sums leave once per CTA) and for CTAs that change n tile
(once per tile), at 64, 128 and 256 columns per tile, with a ragged last tile, and on the direct
path (fp32 output) whose per-element sums meet in the same flush."""
import pytest

pytestmark = pytest.mark.gpu

# (N, H, W, Cin, Cout, k, out_fp32)
FPROP = [
    (8, 56, 56, 64, 64, 1, False),      # BN 64, one n tile
    (8, 28, 28, 512, 128, 1, False),    # BN 128
    (8, 28, 28, 128, 512, 1, False),    # BN 256, two n tiles: CTAs pinned to one
    (8, 14, 14, 256, 1024, 1, False),   # four n tiles
    (3, 7, 7, 512, 2048, 1, False),     # 147 pixels: few tiles, CTAs change n tile, ragged rows
    (8, 28, 28, 128, 128, 3, False),    # 3 x 3 pixel boxes
    (2, 14, 14, 64, 192, 1, True),      # fp32 output, ragged column tile: the direct path
]


def _ids(c):
  return "{}x{}x{}-{}to{}-k{}{}".format(c[0], c[1], c[2], c[3], c[4], c[5], "-fp32" if c[6] else "")


@pytest.mark.parametrize("case", FPROP, ids=[_ids(c) for c in FPROP])
def test_fprop_statistics_match_float64(case):
  import torch
  from tensorflowonspark_b200.ops import igemm
  N, H, W, Cin, Cout, k, fp32 = case
  torch.manual_seed(0)
  dev = "cuda"
  x = torch.randn(N, H, W, Cin, device=dev).bfloat16()
  w = (torch.randn(Cout, k, k, Cin, device=dev) * 0.05).bfloat16()
  y = torch.empty(N, H, W, Cout, device=dev, dtype=torch.float32 if fp32 else torch.bfloat16)
  sums = (torch.zeros(Cout, device=dev), torch.zeros(Cout, device=dev))
  plan = igemm.conv_fprop(x, w, y, 1, k // 2, stats=sums)
  plan.run()
  torch.cuda.synchronize()
  yd = y.double().view(-1, Cout)
  want_s, want_q = yd.sum(0), (yd * yd).sum(0)
  rows = yd.shape[0]
  # fp32 partial sums of up to ``rows`` terms: relative to the sum of magnitudes
  tol = 1e-5 * max(1.0, rows ** 0.5)
  assert float(((sums[0].double() - want_s).abs() / yd.abs().sum(0).clamp_min(1e-30)).max()) < tol
  assert float(((sums[1].double() - want_q).abs() / want_q.clamp_min(1e-30)).max()) < tol


def test_dgrad_bn_reduction_matches_float64():
  """The data-gradient batch-norm reduction (sum g, sum g x over the stored gradient) leaves
  through the same flush."""
  import torch
  from tensorflowonspark_b200.ops import igemm
  torch.manual_seed(0)
  dev = "cuda"
  N, H, W, Cin, Cout = 8, 28, 28, 256, 128
  dy = torch.randn(N, H, W, Cout, device=dev).bfloat16()
  w = (torch.randn(Cout, 1, 1, Cin, device=dev) * 0.05).bfloat16()
  x_raw = torch.randn(N, H, W, Cin, device=dev).bfloat16()
  dx = torch.empty(N, H, W, Cin, device=dev, dtype=torch.bfloat16)
  sg, sgx = torch.zeros(Cin, device=dev), torch.zeros(Cin, device=dev)
  igemm.conv_dgrad(dy, w, dx, 1, 0, bn_reduce=(x_raw, None, sg, sgx)).run()
  torch.cuda.synchronize()
  g, xr = dx.double().view(-1, Cin), x_raw.double().view(-1, Cin)
  mag_g, mag_gx = g.abs().sum(0), (g * xr).abs().sum(0)
  assert float(((sg.double() - g.sum(0)).abs() / mag_g).max()) < 1e-4
  assert float(((sgx.double() - (g * xr).sum(0)).abs() / mag_gx).max()) < 1e-4

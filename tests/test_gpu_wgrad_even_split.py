"""The generic weight-gradient kernel (csrc/igemm_wgrad.cu, igemm_wgrad_kernel) splits each launch's
(output tile, pixel box) iterations evenly over the SMs, so a CTA may start and stop anywhere in a
tile's pixels and cross several tiles.  dW accumulated onto a non-zero start must match the fp32
PyTorch reference for every shape of that split."""
import pytest

pytestmark = pytest.mark.gpu

# name, (N, H, W, Cin, Cout, k, stride), BN, what the split must show
#   "mid": some CTA starts inside a tile;  "span3": some CTA's slice touches three or more tiles
CASES = [
    ("1x1-wide", (64, 14, 14, 1024, 256, 1, 1), 256, "mid"),       # l3c1 at batch 64, 128 x 256
    ("1x1-bn128", (64, 14, 14, 256, 512, 1, 1), 128, "mid"),
    ("1x1-bn64", (32, 28, 28, 64, 256, 1, 1), 64, "mid"),
    ("1x1s2", (32, 28, 28, 512, 1024, 1, 2), 128, "mid"),          # projection shortcut, l3ds
    ("3x3s2", (16, 28, 28, 256, 256, 3, 2), 128, "mid"),           # l3c2s2: 9 taps, stride 2
    ("3x3s2-span3", (1, 8, 8, 1024, 1024, 3, 2), 128, "span3"),    # 576 tiles of one box each
    ("3x3s1-c96", (8, 28, 28, 96, 160, 3, 1), 128, "mid"),         # ragged n_valid / m_valid
]


def _rel(a, b):
  return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _check_split(plan, tiles, expect):
  from tensorflowonspark_b200.ops import igemm
  info = plan.info()[0]
  boxes = info["total_work"] // tiles
  assert boxes * tiles == info["total_work"], (info, tiles)
  slices = igemm._wgrad_slices(tiles, boxes, info["grid"])
  if expect == "mid":
    assert any(b0 != 0 for s in slices for (_, b0, _) in s), plan.desc
  else:
    assert max(len(s) for s in slices) >= 3, plan.desc
  return info


@pytest.mark.parametrize("name,shape,bn,expect", CASES, ids=[c[0] for c in CASES])
def test_even_split_wgrad_matches_fp32_reference(name, shape, bn, expect, monkeypatch):
  import torch
  from tensorflowonspark_b200.ops import igemm
  N, H, W, Cin, Cout, k, s = shape
  pad = k // 2
  OH, OW = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
  if bn == 256:
    monkeypatch.setattr(igemm, "_WGRAD_WIDE_MIN_PIXELS", 0)
  torch.manual_seed(0)
  dev = "cuda"
  x = torch.randn(N, H, W, Cin, device=dev).bfloat16()
  dy = torch.randn(N, OH, OW, Cout, device=dev).bfloat16()
  tf32 = torch.backends.cudnn.allow_tf32
  torch.backends.cudnn.allow_tf32 = False
  try:
    ref = torch.nn.grad.conv2d_weight(x.float().permute(0, 3, 1, 2), (Cout, Cin, k, k),
                                      dy.float().permute(0, 3, 1, 2), stride=s, padding=pad)
  finally:
    torch.backends.cudnn.allow_tf32 = tf32
  ref = ref.permute(0, 2, 3, 1).contiguous()             # KRSC
  dw0 = torch.randn_like(ref) * float(ref.abs().max())
  dw = dw0.clone()
  plan = igemm.conv_wgrad(dy, x, dw, s, pad)
  assert "onepass" not in plan.desc and plan.num_launches == 1, plan.desc
  info = _check_split(plan, k * k * -(-Cout // 128) * -(-Cin // bn), expect)
  assert info["bn"] == bn, (info, plan.desc)
  plan.run()
  torch.cuda.synchronize()
  err = _rel(dw - dw0, ref)
  assert err <= 2e-3, "rel err {:.3e} ({})".format(err, plan.desc)


@pytest.mark.parametrize("M", [256, 200])
def test_even_split_dense_head_matches_fp32_reference(M):
  """gemm_wgrad of the ResNet-50 head, 2048 -> 1000: ragged n tiles (1000 columns) and slices of
  one or two boxes that start mid-tile."""
  import torch
  from tensorflowonspark_b200.ops import igemm
  torch.manual_seed(0)
  dev = "cuda"
  Cin, Cout = 2048, 1000
  x = torch.randn(M, Cin, device=dev).bfloat16()
  dy = torch.randn(M, Cout, device=dev).bfloat16()
  tf32 = torch.backends.cuda.matmul.allow_tf32
  torch.backends.cuda.matmul.allow_tf32 = False
  try:
    ref = dy.float().t() @ x.float()
  finally:
    torch.backends.cuda.matmul.allow_tf32 = tf32
  dw0 = torch.randn_like(ref) * float(ref.abs().max())
  dw = dw0.clone()
  plan = igemm.gemm_wgrad(dy, x, dw)
  _check_split(plan, -(-Cout // 128) * -(-Cin // 128), "mid")
  plan.run()
  torch.cuda.synchronize()
  err = _rel(dw - dw0, ref)
  assert err <= 2e-3, "rel err {:.3e} ({})".format(err, plan.desc)

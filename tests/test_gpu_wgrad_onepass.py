"""3x3 weight gradients with all nine taps from one pass over the pixels (csrc/igemm_wgrad.cu,
igemm_wgrad_halo_kernel): conv_wgrad must pick the one-pass plan for these shapes and accumulate the
same dW as the fp32 PyTorch reference onto a non-zero dW."""
import pytest

pytestmark = pytest.mark.gpu

# (N, H, W, Cin, Cout); 3x3, stride 1, pad 1; every case has >= 16384 output pixels
CASES = [
    (8, 56, 56, 64, 64),      # layer1 conv2
    (32, 28, 28, 128, 128),   # layer2 conv2: four 64-channel slice pairs
    (128, 14, 14, 256, 256),  # layer3 conv2: two 8 x 14 boxes per image
    (512, 7, 7, 512, 512),    # layer4 conv2: two images per 8 x 8 box
    (512, 7, 7, 512, 256),    # Cout != Cin
    (128, 13, 11, 128, 64),   # ragged map
]


def _ids(c):
  return "{}x{}x{}-{}to{}".format(c[0], c[1], c[2], c[3], c[4])


def _rel(a, b):
  return float((a - b).abs().max() / (b.abs().max() + 1e-12))


@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
def test_onepass_wgrad_matches_fp32_reference(case):
  import torch
  from tensorflowonspark_b200.ops import igemm
  N, H, W, Cin, Cout = case
  torch.manual_seed(0)
  dev = "cuda"
  x = torch.randn(N, H, W, Cin, device=dev).bfloat16()
  dy = torch.randn(N, H, W, Cout, device=dev).bfloat16()
  tf32 = torch.backends.cudnn.allow_tf32
  torch.backends.cudnn.allow_tf32 = False
  try:
    ref = torch.nn.grad.conv2d_weight(x.float().permute(0, 3, 1, 2), (Cout, Cin, 3, 3),
                                      dy.float().permute(0, 3, 1, 2), stride=1, padding=1)
  finally:
    torch.backends.cudnn.allow_tf32 = tf32
  ref = ref.permute(0, 2, 3, 1).contiguous()             # KRSC
  dw0 = torch.randn_like(ref) * float(ref.abs().max())
  dw = dw0.clone()
  plan = igemm.conv_wgrad(dy, x, dw, 1, 1)
  assert "onepass" in plan.desc and plan.num_launches == 1, plan.desc
  plan.run()
  torch.cuda.synchronize()
  err = _rel(dw - dw0, ref)
  assert err <= 2e-3, "rel err {:.3e} ({})".format(err, plan.desc)

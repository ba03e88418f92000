"""Data-gradient epilogues that read operands (accumulate, fused BN-backward reduction): the plan
that prefetches those operands into shared memory must store the same dx, bit for bit, as the plan
that loads them in the copy-out pass, and the same per-channel sums up to the order of the fp32
atomics (csrc/igemm.cu, kEpiPrefetch)."""
import pytest

pytestmark = pytest.mark.gpu

# (N, H, W, Cin, Cout, k, stride, accumulate, acc_mask, bn_reduce); dx is [N, H, W, Cin]
CASES = [
    # identity-block conv1 data gradient: BN = 256, accumulate with mask and reduction
    (4, 56, 56, 256, 64, 1, 1, True, True, True),
    # 3 x 49 pixels: the last 128-row tile is ragged
    (3, 7, 7, 2048, 512, 1, 1, True, True, True),
    # conv2 data gradient with the reduction: 3 x 3 taps, 28 x 4 pixel boxes
    (4, 28, 28, 128, 128, 3, 1, False, True, True),
    # 64 channels (BN = 64): the plan keeps the loads in the copy-out pass
    (4, 56, 56, 64, 64, 3, 1, False, True, True),
    # stride 2: parity classes whose output pixels are strided
    (4, 28, 28, 256, 128, 3, 2, False, False, True),
    # projection-shortcut data gradient: strided 1x1, plain accumulate
    (4, 28, 28, 512, 256, 1, 2, True, False, False),
    # reduction with accumulate but no masks, BN = 128
    (4, 14, 14, 128, 256, 1, 1, True, False, True),
]


def _ids(c):
  return "{}x{}s{}-{}to{}{}{}{}".format(c[5], c[5], c[6], c[4], c[3], "-acc" if c[7] else "",
                                       "-mask" if c[8] else "", "-red" if c[9] else "")


def _rel(a, b):
  return float((a - b).abs().max() / (b.abs().max() + 1e-12))


@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
def test_prefetch_matches_register_path(case):
  import torch
  from tensorflowonspark_b200.ops import igemm
  N, H, W, Cin, Cout, k, stride, acc, use_mask, red = case
  torch.manual_seed(0)
  dev = "cuda"
  pad = k // 2
  OH, OW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
  dy = torch.randn(N, OH, OW, Cout, device=dev).bfloat16()
  w = (torch.randn(Cout, k, k, Cin, device=dev) * 0.05).bfloat16()
  nbits = N * H * W * Cin // 8
  amask = torch.randint(0, 256, (nbits,), device=dev, dtype=torch.uint8) if acc and use_mask \
      else None
  x_raw = (torch.randn(N, H, W, Cin, device=dev) * 1.5 + 0.3).bfloat16()
  rbits = torch.randint(0, 256, (nbits,), device=dev, dtype=torch.uint8) if use_mask else None
  dx0 = torch.randn(N, H, W, Cin, device=dev).bfloat16()
  out = {}
  for pf in (True, False):
    dx = dx0.clone()
    sums = (torch.zeros(Cin, device=dev), torch.zeros(Cin, device=dev))
    plan = igemm.conv_dgrad(dy, w, dx, stride, pad, accumulate=acc, acc_mask=amask,
                            bn_reduce=(x_raw, rbits, sums[0], sums[1]) if red else None,
                            epi_prefetch=pf)
    want = int(pf and Cin >= 128)   # BN = 64 plans keep the loads in the copy-out pass
    assert [i["epi_prefetch"] for i in plan.info()] == [want] * plan.num_launches
    plan.run()
    torch.cuda.synchronize()
    out[pf] = (dx, sums)
  dx_pf, (sg_pf, sgx_pf) = out[True]
  dx_reg, (sg_reg, sgx_reg) = out[False]
  assert torch.equal(dx_pf.view(torch.int16), dx_reg.view(torch.int16)), \
      "{} of {} elements differ".format(int((dx_pf != dx_reg).sum()), dx_pf.numel())
  if red:
    assert _rel(sg_pf, sg_reg) < 2e-4
    assert _rel(sgx_pf, sgx_reg) < 2e-4

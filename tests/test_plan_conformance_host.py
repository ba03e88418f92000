"""CPU tier: the element-wise bounds, rounding-bias statistic, row sampling, signature
de-duplication and guard bands of tools/plan_conformance.py (used by
tests/test_gpu_plan_conformance.py) accept exact results and reject subtly wrong ones."""
import importlib.util
import os

import pytest
import torch

_spec = importlib.util.spec_from_file_location(
    "plan_conformance", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                     "tools", "plan_conformance.py"))
pc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(pc)


def _problem(seed=0, P=512, K=576, N=64):
  """A float64 GEMM of bf16-representable operands: (x, w, ref, M, n)."""
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(P, K, generator=g).bfloat16().double()
  w = (torch.randn(K, N, generator=g) * 3 / K ** 0.5).bfloat16().double()
  return x, w, x @ w, x.abs() @ w.abs(), K + 1


def _rejects(out, ref, M, n):
  try:
    pc.check_close(out, ref, pc.elem_bound(ref, M, n), "t")
  except AssertionError:
    return True
  return False


def test_accepts_round_to_nearest_even():
  x, w, ref, M, n = _problem()
  out = pc.bf16_rne(ref)
  pc.check_close(out, ref, pc.elem_bound(ref, M, n), "rne")
  mean, cnt = pc.check_no_bias(out, ref, M, n, "rne")
  assert cnt > 1000 and abs(mean) < 0.05, (mean, cnt)


def test_accepts_fp32_accumulation_error_within_gamma():
  # a sequential fp32 sum: every partial sum rounded
  x, w, ref, M, n = _problem(P=64)
  acc = torch.zeros(64, 64, dtype=torch.float32)
  for k in range(x.shape[1]):
    acc = (acc.double() + x[:, k:k + 1] * w[k:k + 1, :]).float()
  out = pc.bf16_rne(acc.double())
  pc.check_close(out, ref, pc.elem_bound(ref, M, n), "fp32 chain")


def test_rejects_truncation():
  x, w, ref, M, n = _problem()
  out = pc.bf16_trunc(ref)
  mean, cnt = pc.rounding_bias(out, ref, M, n)
  assert cnt > 1000 and mean < -0.35, (mean, cnt)
  with pytest.raises(AssertionError, match="systematic rounding"):
    pc.check_no_bias(out, ref, M, n, "trunc")


def test_rejects_one_element_one_ulp_off():
  x, w, ref, M, n = _problem()
  out = pc.bf16_rne(ref)
  # an element whose accumulation error is far below its rounding error
  # (just above a power of two, where u |ref| is half an ulp)
  r = ref.reshape(-1)
  frac = pc.U_BF16 * r.abs() / pc.ulp_bf16(r)
  ok = (pc.gamma(n) * M * 8 <= pc.U_BF16 * ref.abs()).reshape(-1)
  i = int(torch.where(ok, frac, torch.full_like(frac, 9.0)).argmin())
  assert bool(ok[i])
  bad = out.clone().reshape(-1)
  bad[i] += torch.sign(bad[i] - ref.reshape(-1)[i] + 1e-300) * pc.ulp_bf16(bad[i:i + 1])[0]
  assert not _rejects(out, ref, M, n)
  assert _rejects(bad.view_as(out), ref, M, n)


def test_rejects_missing_tap():
  x, w, ref, M, n = _problem(K=9 * 64)
  w2 = w.clone()
  w2[64:128] = 0   # tap 1 of a 3x3 filter with 64 input channels
  out = pc.bf16_rne(x @ w2)
  assert _rejects(out, ref, M, n)


def test_rejects_missing_relu6_clamp():
  x, w, ref, M, n = _problem()
  want = ref.clamp(0, 6)
  out = pc.bf16_rne(ref.clamp_min(0))
  assert (ref > 6.5).any()
  assert _rejects(out, want, M, n)


def test_accumulate_bound_allows_double_rounding():
  x, w, ref, M, n = _problem()
  g = torch.Generator().manual_seed(1)
  prev = torch.randn(ref.shape, generator=g).bfloat16().double() * 2
  out = pc.bf16_rne(pc.bf16_rne(ref) + prev)
  want = ref + prev
  pc.check_close(out, want, pc.elem_bound(want, M, n, partial=ref, prev=prev), "acc")
  # without the partial term the double rounding can exceed the single-rounding bound
  assert _rejects(out, want, M, n)


def test_guard_band_detects_a_changed_word():
  for dtype in (torch.bfloat16, torch.float32, torch.uint8):
    view, back = pc.guarded((5, 24), dtype, "cpu")
    view.zero_()
    assert view.data_ptr() % 1024 == back.data_ptr() % 1024
    assert pc.guard_intact(view, back)
    for idx in (0, back.numel() - 1, (view.data_ptr() - back.data_ptr()) // back.element_size() - 1,
                (view.data_ptr() - back.data_ptr()) // back.element_size() + view.numel()):
      b2 = back.clone()
      v2 = b2[(view.data_ptr() - back.data_ptr()) // back.element_size():][:view.numel()]
      pc._int_view(b2)[idx] += 1
      assert not pc.guard_intact(v2, b2), (dtype, idx)


def test_unwritten_pattern_is_nan_and_detected():
  for dtype, bits in ((torch.bfloat16, pc.UNWRITTEN_BF16), (torch.float32, pc.UNWRITTEN_FP32)):
    view, _ = pc.guarded((4, 8), dtype, "cpu", bits)
    assert bool(torch.isnan(view.float()).all())
    view[1, 3] = 1.0
    un = pc.unwritten(view)
    assert int(un.sum()) == 31 and not bool(un[1, 3])
  # and a NaN output fails the element check
  ref = torch.ones(4)
  with pytest.raises(AssertionError):
    pc.check_close(torch.tensor([1.0, float("nan"), 1.0, 1.0]), ref, torch.full((4,), 0.1), "nan")


def test_signature_dedup_keeps_first_seen_order():
  a = pc.freeze({"x": ("T", (2, 3), "bfloat16"), "relu": 1})
  b = pc.freeze({"relu": 1, "x": ("T", (2, 3), "bfloat16")})
  c = pc.freeze({"x": ("T", (2, 3), "bfloat16"), "relu": 2})
  assert a == b and hash(a) == hash(b)
  assert pc.dedup([a, c, b, a, c]) == [a, c]
  assert pc.freeze([{"k": [1, 2]}]) == ((("k", (1, 2)),),)


def _info(tw, th, tn, bw, bh, bn, lim):
  return {"tiles_w": tw, "tiles_h": th, "tiles_n": tn, "box_w": bw, "box_h": bh, "box_n": bn,
          "lim_w": lim[0], "lim_h": lim[1], "lim_n": lim[2], "osw": 1, "oow": 0, "osh": 1,
          "ooh": 0}


def test_row_sampling_covers_every_box_and_all_128_rows():
  # 300 boxes of 128 rows (a GEMM with a ragged last box), then a conv launch of 16 x 8 boxes
  infos = [_info(300, 1, 1, 128, 1, 1, (300 * 128 - 77, 1, 1)),
           _info(4, 7, 3, 16, 8, 1, (60, 50, 3))]
  n, h, w, launch, box, row = pc.sample_pixels(infos)
  for li, info in enumerate(infos):
    boxes = info["tiles_w"] * info["tiles_h"] * info["tiles_n"]
    sel = launch == li
    counts = torch.bincount(box[sel], minlength=boxes)
    assert int(counts.min()) >= 1
  full = (launch == 0) & (box < 299)
  assert int(torch.bincount(box[full]).min()) == 2
  assert set(row[launch == 0].tolist()) == set(range(128))
  # both warpgroups of every full box
  r0 = row[full].view(-1, 2)
  assert bool(((r0[:, 0] < 64) != (r0[:, 1] < 64)).all())
  # every sample lies inside the tensor, and matches the scalar rule
  assert bool((w[launch == 1] < 60).all()) and bool((h[launch == 1] < 50).all())
  assert bool((w[launch == 0] < 300 * 128 - 77).all())
  gbox = 0
  for li, info in enumerate(infos):
    boxes = info["tiles_w"] * info["tiles_h"] * info["tiles_n"]
    for b in (0, 1, boxes - 1):
      px = pc.box_pixels(info, b)
      want = pc.sample_box_rows(gbox + b, len(px), lambda r: px[r] is not None)
      got = row[(launch == li) & (box == b)].tolist()
      assert sorted(got) == sorted(want), (li, b)
      for r in got:
        i = int(((launch == li) & (box == b) & (row == r)).nonzero()[0])
        assert (int(n[i]), int(h[i]), int(w[i])) == px[r]
    gbox += boxes


# ---------------------------------------------------------- long sums at the largest recorded P
def _rejects_bound(out, ref, bound):
  try:
    pc.check_close(out, ref, bound, "t")
  except AssertionError:
    return True
  return False


def _pos(n, cols, seed):
  """bf16 values of mean 1, sd 0.5 (the replay's operands for plans without activation)."""
  g = torch.Generator().manual_seed(seed)
  return (torch.randn(n, cols, generator=g) * 0.5 + 1).bfloat16().double()


# the ResNet-50 stem at batch 256 / 224^2: 112 x 112 outputs per image
_STEM_P = 256 * 112 * 112
_STEM_WGRAD = {"stem": 1, "k_splits": 132, "grid": 132, "total_work": 132, "box_rows": 128,
               "tiles_w": 7, "tiles_h": 14, "tiles_n": 256}
# layer-1 1x1 weight gradient 64 -> 256 at batch 256 / 56^2 (generic kernel, 2 x 1 tiles)
_L1_WGRAD = {"stem": 0, "k_splits": 1, "grid": 132, "total_work": 2 * 6272, "box_rows": 128,
             "tiles_w": 6272, "tiles_h": 1, "tiles_n": 1}


@pytest.mark.parametrize("info", [_STEM_WGRAD, _L1_WGRAD], ids=["stem_halo", "generic_1x1"])
def test_wgrad_bound_rejects_untouched_dw_and_a_missing_split(info):
  P = info["tiles_w"] * info["tiles_h"] * info["tiles_n"] * info["box_rows"]
  assert P in (_STEM_P, 256 * 56 * 56)
  dy, x = _pos(P, 2, 1), _pos(P, 2, 2)
  dw0 = torch.randn(2, 2, generator=torch.Generator().manual_seed(3)).float().double()
  ref = dw0 + dy.t() @ x
  bound = pc.wgrad_bound(dy.abs().t() @ x.abs(), dw0.abs(), info)
  assert not _rejects_bound(ref.float().double(), ref, bound)
  assert _rejects_bound(dw0, ref, bound)            # the kernel wrote nothing
  L, S = pc.wgrad_chain(info)
  part = dy[:L].t() @ x[:L]                          # one CTA's partial sum
  assert _rejects_bound(ref - part, ref, bound)      # one k split / slice never added


def test_column_sum_bound_rejects_one_missing_m_box():
  # stem forward with fused statistics at batch 256: 25088 boxes of 8 x 16 pixels, BN = 64,
  # 132 CTAs each on the one n tile
  info = {"bn": 64, "tiles_w": 14, "tiles_h": 7, "tiles_n": 256, "n_tiles": 1, "grid": 132,
          "total_work": 25088}
  v = _pos(_STEM_P, 2, 4) * 3
  ref = v.sum(0)
  bound = pc.gamma_prob(pc.fwd_stat_depth([info], True)) * v.abs().sum(0)
  assert not _rejects_bound(v.float().sum(0).double(), ref, bound)
  assert _rejects_bound(ref - v[:128].sum(0), ref, bound)
  sq = v * v
  bound2 = pc.gamma_prob(pc.fwd_stat_depth([info], True)) * sq.sum(0)
  assert _rejects_bound(sq.sum(0) - sq[:128].sum(0), sq.sum(0), bound2)


def test_bn_reduce_bound_rejects_one_missing_block():
  P, C = 256 * 56 * 56, 64
  g = _pos(P, 2, 5)
  depth = pc.red_grid_depth(P, C, 2)
  bound = pc.gamma_prob(depth) * g.abs().sum(0)
  ref = g.sum(0)
  assert not _rejects_bound(g.float().sum(0).double(), ref, bound)
  # one thread's rows (every (gridDim.x * rl)-th row of a column): the smallest unit a lost
  # register sum would remove
  rows = -(-P // (264 * 32))
  assert depth == rows + 32 + 264 + 1
  assert _rejects_bound(ref - g[:rows].sum(0), ref, bound)

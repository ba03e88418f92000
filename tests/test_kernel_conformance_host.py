"""CPU tier: the float64 references and ambiguity masks of tools/kernel_conformance.py (used by
tests/test_gpu_kernel_conformance.py) against PyTorch's pooling, autograd and convolution on the
CPU, at ties, all-negative border windows, NaN and odd sizes."""
import importlib.util
import os

import pytest
import torch
import torch.nn.functional as F

_spec = importlib.util.spec_from_file_location(
    "kernel_conformance", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                       "tools", "kernel_conformance.py"))
kc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(kc)

POOLS = [(3, 2, 1, 37, 41), (3, 2, 1, 1, 1), (3, 2, 1, 2, 3), (2, 2, 0, 26, 26), (2, 2, 0, 27, 9),
         (3, 1, 1, 7, 10), (5, 3, 2, 11, 8)]


def _nchw(t):
  return t.permute(0, 3, 1, 2)


def _torch_pool(x, k, s, p):
  """(y, tap) of F.max_pool2d, NHWC, the flat input index turned into the window tap."""
  N, H, W, C = x.shape
  y, ind = F.max_pool2d(_nchw(x), k, s, p, return_indices=True)
  y, ind = y.permute(0, 2, 3, 1), ind.permute(0, 2, 3, 1)
  OH, OW = y.shape[1], y.shape[2]
  oh = torch.arange(OH).view(1, OH, 1, 1)
  ow = torch.arange(OW).view(1, 1, OW, 1)
  return y, (ind // W - (oh * s - p)) * k + (ind % W - (ow * s - p))


def _few_values(shape, seed, negative=False):
  """bf16-representable values drawn from 24 levels: ties are common."""
  g = torch.Generator().manual_seed(seed)
  v = torch.randint(0, 24, shape, generator=g).double() / 8 - 1.5
  return -(v.abs() + 0.125) if negative else v


@pytest.mark.parametrize("k,s,p,H,W", POOLS)
@pytest.mark.parametrize("case", ["ties", "negative", "nan"])
def test_maxpool_ref_is_torch_max_pool2d(k, s, p, H, W, case):
  x = _few_values((2, H, W, 8), H * 100 + W, negative=case == "negative")
  if case == "nan":
    g = torch.Generator().manual_seed(7)
    x[torch.rand(x.shape, generator=g) < 0.15] = float("nan")
    x[0, :min(H, k), :min(W, k)] = float("nan")   # whole windows of NaN
  y, idx = kc.maxpool_ref(x, k, s, p)
  ty, tidx = _torch_pool(x, k, s, p)
  assert torch.equal(torch.isnan(y), torch.isnan(ty))
  assert torch.equal(torch.nan_to_num(y, 9.0), torch.nan_to_num(ty, 9.0))
  assert torch.equal(idx, tidx)
  if case == "negative" and p > 0:
    # border windows are all negative: a zero padding would have been picked
    assert bool((y[:, 0] < 0).all())
  if case == "ties" and H * W >= 16:
    # windows whose maximum sits at more than one tap: the first one must win
    hits = sum((v == y) & ok for _, v, ok in kc.pool_taps(x, k, s, p, fill=float("nan")))
    assert int((hits > 1).sum()) > 0
  assert bool(((idx >= 0) & (idx < k * k)).all())
  # at_tap reads the chosen value back
  v = kc.at_tap(x, idx, k, s, p)
  assert torch.equal(torch.nan_to_num(v, 9.0), torch.nan_to_num(y, 9.0))


@pytest.mark.parametrize("k,s,p,H,W", POOLS)
def test_maxpool_bwd_ref_is_autograd(k, s, p, H, W):
  x = torch.randn(2, H, W, 8, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
  xr = _nchw(x).clone().requires_grad_(True)
  y = F.max_pool2d(xr, k, s, p)
  dy = torch.randn(y.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(4))
  y.backward(dy)
  _, idx = kc.maxpool_ref(x, k, s, p)
  dx, mag, cnt = kc.maxpool_bwd_ref(dy.permute(0, 2, 3, 1), idx, H, W, k, s, p)
  assert torch.allclose(dx, xr.grad.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
  assert bool((mag >= dx.abs()).all()) and float(cnt.max()) <= (-(-k // s)) ** 2
  if (k, s, p) == (2, 2, 0) and H % 2:
    assert bool((dx[:, -1] == 0).all()) and bool((cnt[:, -1] == 0).all())


def test_stem_reference_and_ambiguity():
  g = torch.Generator().manual_seed(11)
  x = torch.randn(2, 37, 41, 16, generator=g).bfloat16().double()
  scale = (torch.rand(16, generator=g) + 0.5).float().double()
  shift = (torch.randn(16, generator=g) * 0.5).float().double()
  lo, hi = kc.stem_act_bounds(x, scale, shift)
  # the activation of an fp32 fma, computed exactly in float64 on the CPU
  act = (x * scale + shift).float().clamp_min(0).bfloat16().double()
  assert bool((lo <= act).all() and (act <= hi).all())
  ref = F.relu(x * scale + shift)
  y, idx, amb = kc.stem_pool_ref(lo, hi)
  ty, tidx = _torch_pool(act, 3, 2, 1)
  assert torch.equal(y[~amb], ty[~amb]) and torch.equal(idx[~amb], tidx[~amb])
  assert float((y - F.max_pool2d(_nchw(ref), 3, 2, 1).permute(0, 2, 3, 1)).abs().max()) < 0.05
  # a pixel whose interval is open near the window maximum makes the window ambiguous
  hi2 = lo.clone()
  hi2[0, 0, 0, 0] = lo[0, 0, 0, 0] + 1.0
  _, _, amb2 = kc.stem_pool_ref(lo, hi2)
  assert bool(amb2[0, 0, 0, 0]) and int(amb2.sum()) == 1


def test_relu_mask_ambiguity():
  x = torch.tensor([1.0, -1.0, 1.0, 2.0], dtype=torch.float64)
  scale = torch.tensor([1.0, 1.0, 1.0, 0.5], dtype=torch.float64)
  shift = torch.tensor([0.5, 0.5, -1.0, -1.0], dtype=torch.float64)
  keep, amb = kc.relu_mask(x, scale, shift)
  assert keep.tolist() == [True, False, False, False]
  assert amb.tolist() == [False, False, True, True]


@pytest.mark.parametrize("hw", [1, 4, 49, 64])
def test_avgpool_ref_is_avg_pool2d(hw):
  g = torch.Generator().manual_seed(hw)
  x = torch.randn(3, hw, 1, 16, dtype=torch.float64, generator=g)
  m, mag = kc.avgpool_ref(x)
  t = F.adaptive_avg_pool2d(_nchw(x), 1).reshape(3, 16)
  assert torch.allclose(m, t, rtol=1e-13, atol=0)
  xr = x.clone().requires_grad_(True)
  dy = torch.randn(3, 16, dtype=torch.float64, generator=g)
  xr.mean((1, 2)).backward(dy)
  assert torch.allclose(xr.grad, (dy / hw)[:, None, None, :].expand_as(x), rtol=1e-15)
  assert bool((mag >= m.abs()).all())


@pytest.mark.parametrize("C,Cp,wofs,Wp", [(3, 8, 0, 9), (3, 8, 3, 15), (3, 16, 2, 12),
                                          (6, 8, 0, 9), (1, 8, 1, 11)])
def test_decode_ref(C, Cp, wofs, Wp):
  g = torch.Generator().manual_seed(C * 100 + Cp)
  img = torch.randint(0, 256, (2, 5, 9, C), generator=g, dtype=torch.uint8)
  mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
  out, mag = kc.decode_ref(img, Wp, Cp, wofs, mean, std)
  m = torch.tensor([mean[c % 3] for c in range(C)], dtype=torch.float64)
  s = torch.tensor([std[c % 3] for c in range(C)], dtype=torch.float64)
  want = (img.double() / 255 - m) / s
  assert torch.allclose(out[:, :, wofs:wofs + 9, :C], want, rtol=1e-6, atol=1e-6)
  assert bool((out[:, :, :wofs] == 0).all() and (out[:, :, wofs + 9:] == 0).all())
  assert bool((out[..., C:] == 0).all()) and bool((mag >= out.abs()).all())


def test_conv3x3_c1_refs_are_conv2d_and_autograd():
  g = torch.Generator().manual_seed(5)
  x = torch.randn(2, 9, 11, dtype=torch.float64, generator=g)
  w = torch.randn(16, 9, dtype=torch.float64, generator=g)
  b = torch.randn(16, dtype=torch.float64, generator=g)
  y, mag = kc.conv3x3_c1_ref(x, w, b)
  xr = x.clone().requires_grad_(True)
  wr = w.clone().requires_grad_(True)
  br = b.clone().requires_grad_(True)
  t = F.conv2d(xr[:, None], wr.view(16, 1, 3, 3), br).permute(0, 2, 3, 1)
  assert torch.allclose(y, t, rtol=1e-12, atol=1e-12) and bool((mag >= y.abs()).all())
  dy = torch.randn(t.shape, dtype=torch.float64, generator=g)
  t.backward(dy)
  dw, dwm, db, dbm = kc.conv3x3_c1_wgrad_ref(x, dy)
  assert torch.allclose(dw, wr.grad, rtol=1e-12, atol=1e-12)
  assert torch.allclose(db, br.grad, rtol=1e-12, atol=1e-12)
  assert bool((dwm >= dw.abs()).all() and (dbm >= db.abs()).all())


# ------------------------------------------------------------------ gradient accumulation
def test_accumulated_check_rejects_overwrite_and_double_add():
  g = torch.Generator().manual_seed(3)
  A, v = torch.randn(200, generator=g), torch.randn(200, generator=g)
  kc.check_accumulated(A + v, A, v, "fl(A + v)")
  for wrong, name in ((v.clone(), "overwrites"), (A + v + v, "adds twice"),
                      ((A.double() + v.double()).float().nextafter(torch.tensor(float("inf"))),
                       "one ulp off")):
    with pytest.raises(AssertionError, match="not fl"):
      kc.check_accumulated(wrong, A, v, name)


# ------------------------------------------------------------------ batch-norm folding
def _fold_problem(seed=0, eps=1e-3):
  """Three folded units followed by a 10-row head the fold must not touch, as fold_table lays
  them out: (tab, eps, row0, w, aux32, running).  The variances span 1e-6 .. 1e3, so eps matters
  for some channels and var + eps is far above eps for others."""
  g = torch.Generator().manual_seed(seed)
  units = [(16, 8), (24, 16), (8, 72)]
  rows, woff, aoff, roff, boff = [], 0, 0, 0, 0
  for cout, per in units:
    rows.append([woff, cout, per, aoff, aoff + cout, roff, roff + cout, boff])
    woff += cout * per
    aoff += 2 * cout
    roff += 2 * cout
    boff += (cout + 7) // 8 * 8
  w = torch.randn(woff + 10 * 16, generator=g).to(torch.bfloat16)
  aux32 = torch.randn(aoff, generator=g)
  running = torch.randn(roff, generator=g)
  for r in rows:   # variances: positive, log-uniform
    running[r[6]:r[6] + r[1]] = torch.pow(10.0, torch.rand(r[1], generator=g) * 9 - 6)
  tab = torch.tensor(rows, dtype=torch.int64)
  row0 = torch.tensor([0, 16, 40, 48], dtype=torch.int64)
  return tab, torch.full((3,), eps, dtype=torch.float32), row0, w, aux32, running


def _fold_like_the_kernel(tab, eps, row0, w, aux32, running, drop_eps=False, mean_as_var=False,
                          extra_row=False):
  """fp32 s = gamma * rsqrt(var + eps), bf16(fp32(w s)), fp32 beta - mean s; and the faults."""
  wf = torch.randn(w.shape, generator=torch.Generator().manual_seed(9)).to(torch.bfloat16)
  nb = 48
  bias = torch.randn(nb + 8, generator=torch.Generator().manual_seed(10))
  wf0, bias0 = wf.clone(), bias.clone()
  for u, (wo, cout, per, go, bo, mo, vo, fo) in enumerate(tab.tolist()):
    var = running[mo:mo + cout] if mean_as_var else running[vo:vo + cout]
    s = aux32[go:go + cout] * torch.rsqrt(var if drop_eps else var + eps[u])
    wf[wo:wo + cout * per] = (w[wo:wo + cout * per].float().view(cout, per) * s[:, None]) \
        .to(torch.bfloat16).view(-1)
    bias[fo:fo + cout] = aux32[bo:bo + cout] - running[mo:mo + cout] * s
    if extra_row and u == len(tab) - 1:   # one row past the unit: the head's first row
      e = wo + cout * per
      wf[e:e + per] = (w[e:e + per].float() * s[-1]).to(torch.bfloat16)
  return wf, bias, wf0, bias0


def test_fold_ref_is_eval_batch_norm_after_the_layer():
  tab, eps, row0, w, aux32, running = _fold_problem()
  s, wf, bias, wmask, bmask = kc.fold_ref(tab, eps, row0, w, aux32, running)
  x = torch.randn(5, 72, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
  for (wo, cout, per, go, bo, mo, vo, fo), e in zip(tab.tolist(), eps.tolist()):
    W = w[wo:wo + cout * per].double().view(cout, per)
    ref = F.batch_norm(x[:, :per] @ W.t(), running[mo:mo + cout].double(),
                       running[vo:vo + cout].double(), aux32[go:go + cout].double(),
                       aux32[bo:bo + cout].double(), False, 0.0, e)
    got = x[:, :per] @ wf[wo:wo + cout * per].view(cout, per).t() + bias[fo:fo + cout]
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)
  assert int(wmask.sum()) == 16 * 8 + 24 * 16 + 8 * 72 and not bool(wmask[-160:].any())
  assert int(bmask.sum()) == 48


def test_check_bn_fold_accepts_the_kernels_rounding():
  for seed in range(3):
    p = _fold_problem(seed)
    kc.check_bn_fold(*_fold_like_the_kernel(*p), *p, "fold")


@pytest.mark.parametrize("fault", ["drop_eps", "mean_as_var", "extra_row"])
def test_check_bn_fold_rejects_a_wrong_fold(fault):
  p = _fold_problem(1)
  with pytest.raises(AssertionError):
    kc.check_bn_fold(*_fold_like_the_kernel(*p, **{fault: True}), *p, fault)


def test_check_bn_fold_rejects_one_bf16_step():
  p = _fold_problem(2)
  wf, bias, wf0, bias0 = _fold_like_the_kernel(*p)
  i = 200   # a filter element of the second unit
  wf.view(torch.int16)[i] += 1
  with pytest.raises(AssertionError, match="folded filter"):
    kc.check_bn_fold(wf, bias, wf0, bias0, *p, "one step")

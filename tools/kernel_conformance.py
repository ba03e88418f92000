"""Float64 references for the pooling, fused-stem, input-decode and small MNIST kernels, the
batch-norm fold of evaluation and serving, and the accumulators of gradient accumulation.

Shared by tests/test_gpu_kernel_conformance.py and tests/test_gpu_option_conformance.py (replay
what the models launch) and tests/test_kernel_conformance_host.py (checks these references against
PyTorch on the CPU, and the checkers against deliberately wrong results).
Everything works on torch tensors of any device, NHWC, float64.

Max pool selection (maxpool_fwd, PyTorch's max_pool2d): the taps of a window are visited in
row-major order; a tap replaces the running maximum when its value is larger or NaN.  Ties keep
the first maximal tap, and a window holding NaN gives NaN at its last NaN tap.  Padding is never a
candidate.

Fused stem (stem_bn_relu_pool_fwd): the kernel pools a = bf16(relu(fp32(fma(x, scale, shift)))).
The fp32 fma is one rounding of the exact pre-activation; its float64 value lies within
``STEM_PRE_REL`` (relative to |x scale| + |shift|) of the exact one, and a = A(pre) is monotone
in pre.  So a lies in [A(lo), A(hi)] with lo / hi the float64 value minus / plus that margin.  The
interval is a single value except where an fp32 rounding boundary lies inside it (about one pixel
in 10^4); a window is ambiguous when such a pixel could be its maximum.  Everywhere else the
pooled value and the first maximal tap are exact.
"""
import torch
import torch.nn.functional as F

STEM_PRE_REL = 2.0 ** -48


def pool_out(n, k, s, p):
  """Output extent of a k-wide window at stride s and padding p (floor mode)."""
  return (n + 2 * p - k) // s + 1


def pool_taps(x, k, s, p, fill=0.0):
  """(tap, values [N, OH, OW, C], valid [1, OH, OW, 1]) for each tap kh * k + kw of every window
  of a k x k / s / p pool over x [N, H, W, C]; ``valid`` is False where the tap is padding."""
  N, H, W, C = x.shape
  OH, OW = pool_out(H, k, s, p), pool_out(W, k, s, p)
  xp = F.pad(x, (0, 0, p, p, p, p), value=fill)
  valid = torch.zeros(H + 2 * p, W + 2 * p, dtype=torch.bool, device=x.device)
  valid[p:p + H, p:p + W] = True
  for kh in range(k):
    for kw in range(k):
      hs = slice(kh, kh + (OH - 1) * s + 1, s)
      ws = slice(kw, kw + (OW - 1) * s + 1, s)
      yield kh * k + kw, xp[:, hs, ws], valid[hs, ws][None, :, :, None]


def maxpool_ref(x, k, s, p):
  """(y, idx): the maximum of every window and its tap (int64), with the selection rule of the
  module docstring."""
  best = idx = seen = None
  for t, v, ok in pool_taps(x, k, s, p, fill=float("nan")):
    if best is None:
      best = torch.full_like(v, float("-inf"))
      idx = torch.zeros(v.shape, dtype=torch.int64, device=v.device)
      seen = torch.zeros_like(ok)
    upd = ok & ((v > best) | torch.isnan(v) | ~seen)
    best = torch.where(upd, v, best)
    idx = torch.where(upd, torch.full_like(idx, t), idx)
    seen = seen | ok
  return best, idx


def maxpool_bwd_ref(dy, idx, H, W, k, s, p):
  """(dx, mag, terms): the sum of the gradients each input pixel receives through ``idx``, the sum
  of their magnitudes, and how many there are (float64, [N, H, W, C])."""
  N, OH, OW, C = dy.shape
  Hp, Wp = max(H + 2 * p, (OH - 1) * s + k), max(W + 2 * p, (OW - 1) * s + k)
  acc = torch.zeros(N, Hp, Wp, C, dtype=torch.float64, device=dy.device)
  mag, cnt = torch.zeros_like(acc), torch.zeros_like(acc)
  for kh in range(k):
    for kw in range(k):
      sel = idx == kh * k + kw
      hs = slice(kh, kh + (OH - 1) * s + 1, s)
      ws = slice(kw, kw + (OW - 1) * s + 1, s)
      g = torch.where(sel, dy, torch.zeros_like(dy))
      acc[:, hs, ws] += g
      mag[:, hs, ws] += g.abs()
      cnt[:, hs, ws] += sel.to(torch.float64)
  crop = (slice(None), slice(p, p + H), slice(p, p + W))
  return acc[crop], mag[crop], cnt[crop]


def _stem_act(pre):
  return pre.clamp_min(0).to(torch.float32).to(torch.bfloat16).to(torch.float64)


def stem_act_bounds(x, scale, shift):
  """(lo, hi): the activation bf16(relu(fp32(x scale + shift))) of every pixel lies in [lo, hi]
  (see the module docstring); lo == hi almost everywhere."""
  xs = x * scale
  pre = xs + shift
  d = STEM_PRE_REL * (xs.abs() + shift.abs())
  return _stem_act(pre - d), _stem_act(pre + d)


def stem_pool_ref(lo, hi):
  """(y, idx, ambiguous) of the 3x3/2/1 pool over activations known to lie in [lo, hi]: y and idx
  from ``lo``, exact where ``ambiguous`` is False."""
  y, idx = maxpool_ref(lo, 3, 2, 1)
  amb = torch.zeros(y.shape, dtype=torch.bool, device=y.device)
  for (_, vl, ok), (_, vh, _) in zip(pool_taps(lo, 3, 2, 1), pool_taps(hi, 3, 2, 1)):
    amb |= ok & (vl != vh) & (vh >= y)
  return y, idx, amb


def at_tap(x, idx, k, s, p):
  """x's value at tap ``idx`` of every window (NaN where idx names padding or no tap)."""
  out = torch.full(idx.shape, float("nan"), dtype=torch.float64, device=x.device)
  for t, v, ok in pool_taps(x, k, s, p, fill=float("nan")):
    out = torch.where((idx == t) & ok, v, out)
  return out


def relu_mask(x, scale, shift, u=2.0 ** -24):
  """(keep, ambiguous) of the backward's recomputed ReLU mask fma(x, scale, shift) > 0: the sign
  of a value within two fp32 roundings (flush to zero included) of 0 is not decided."""
  xs = x * scale
  pre = xs + shift
  return pre > 0, pre.abs() <= 2 * u * (xs.abs() + shift.abs())


def stem_bwd_depth(N, H, W, C, sms=132):
  """Roundings of one pixel's term in stem_pool_bn_bwd's dgamma / dbeta sums over an N x H x W
  x C stem output: a thread's chain of 4 pixels per grid-stride iteration (each pixel up to 4
  routed terms), the block's threads of one channel group in shared memory, one atomic per
  block (the grid is capped at 8 blocks per SM)."""
  groups = C // 8
  threads = N * (((H + 1) // 2 + 3) // 4) * (((W + 1) // 2 + 7) // 8) * 32 * groups
  grid = max(1, min(-(-threads // 256), sms * 8))
  return 4 * -(-threads // (grid * 256)) + 4 + 256 // groups + grid + 3


def avgpool_ref(x):
  """(mean over the pixels, mean of magnitudes) of x [N, HW..., C] per image and channel."""
  N, C = x.shape[0], x.shape[-1]
  xx = x.reshape(N, -1, C)
  return xx.mean(1), xx.abs().mean(1)


def decode_ref(img, Wp, Cp, wofs, mean, std):
  """(out, mag): uint8 [N, H, W, C] normalised with fp32 constants as the kernel holds them (mean,
  1 / std) into [N, H, Wp, Cp]; channels >= C and the columns outside [wofs, wofs + W) are 0.
  ``mag`` bounds the terms: (x / 255 + |mean|) / std."""
  N, H, W, C = img.shape
  f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))  # noqa: E731
  m = torch.tensor([f32(mean[c % len(mean)]) for c in range(3)], dtype=torch.float64)
  si = torch.tensor([f32(1.0 / std[c % len(std)]) for c in range(3)], dtype=torch.float64)
  ch = torch.arange(C) % 3
  m, si = m[ch].to(img.device), si[ch].to(img.device)
  v = img.to(torch.float64) / 255.0
  out = torch.zeros(N, H, Wp, Cp, dtype=torch.float64, device=img.device)
  mag = torch.zeros_like(out)
  out[:, :, wofs:wofs + W, :C] = (v - m) * si
  mag[:, :, wofs:wofs + W, :C] = (v + m.abs()) * si.abs()
  return out, mag


def conv3x3_c1_ref(x, w, bias):
  """(y before the activation, sum of magnitudes): valid 3x3 convolution of x [N, H, W] with
  w [Cout, 9] plus bias [Cout] -> [N, H - 2, W - 2, Cout]."""
  N, H, W = x.shape
  cols = torch.stack([x[:, kh:kh + H - 2, kw:kw + W - 2] for kh in range(3) for kw in range(3)], -1)
  y = cols @ w.t()
  mag = cols.abs() @ w.abs().t()
  if bias is not None:
    y = y + bias
    mag = mag + bias.abs()
  return y, mag


def conv3x3_c1_wgrad_ref(x, dy):
  """(dw [Cout, 9], |dw| terms, dbias [Cout], |dbias| terms) of the valid 3x3 convolution."""
  N, H, W = x.shape
  Cout = dy.shape[-1]
  cols = torch.stack([x[:, kh:kh + H - 2, kw:kw + W - 2] for kh in range(3) for kw in range(3)], -1)
  cols, g = cols.reshape(-1, 9), dy.reshape(-1, Cout)
  return g.t() @ cols, g.abs().t() @ cols.abs(), g.sum(0), g.abs().sum(0)


# ------------------------------------------------------------------ gradient accumulation
def check_accumulated(acc, prefill, v, what):
  """An accumulating kernel's parameter gradient: exactly one fp32 round-to-nearest addition of
  this micro-batch's value ``v`` to the ``prefill`` A, fl(A + v), bit for bit."""
  want = (prefill.to(torch.float32) + v.to(torch.float32)).contiguous().view(torch.int32)
  got = acc.to(torch.float32).contiguous().view(torch.int32)
  bad = got != want
  if bool(bad.any()):
    i = int(bad.reshape(-1).nonzero()[0])
    raise AssertionError("{}: {} of {} accumulated elements are not fl(A + v); first at {}: "
                         "got {!r}"
                         " A {!r} v {!r}".format(what, int(bad.sum()), bad.numel(), i,
                                                 float(acc.reshape(-1)[i]),
                                                 float(prefill.reshape(-1)[i]),
                                                 float(v.reshape(-1)[i])))


# ------------------------------------------------------------------ batch-norm folding
# bn_fold (csrc/eval.cu) per output channel c of a unit: s = gamma * rsqrtf(var + eps) in fp32,
# wf = bf16(fp32(w * s)), bias = beta - mean * s.  The sum var + eps is one rounding (half an ulp
# of the result after the square root), rsqrtf is within 2 ulp (CUDA Programming Guide, the
# --use_fast_math table) and the product with gamma one rounding: |s - s64| <= FOLD_S_REL |s64|.
FOLD_S_REL = 7 * 2.0 ** -24
FOLD_COLS = 8   # kFold*: weight, cout, per_channel, gamma, beta, mean, var, bias


def fold_ref(tab, eps, row0, w, aux32, running):
  """float64 s = gamma / sqrt(var + eps) [rows], the folded filter w * s and bias beta - mean * s
  (flat, in the layouts of w and of the bias vector), and boolean masks of the filter / bias
  elements some unit writes.  Inputs: the host table, its fp32 eps and row0, the bf16 filters,
  aux32 (gamma, beta) and the running-statistics buffer."""
  f64 = lambda t: t.to(torch.float64)  # noqa: E731
  tab, row0 = tab.cpu().tolist(), row0.cpu().tolist()
  eps = f64(eps.cpu())
  wflat = w.reshape(-1)
  wf = torch.zeros(wflat.shape, dtype=torch.float64, device=w.device)
  wmask = torch.zeros(wflat.shape, dtype=torch.bool, device=w.device)
  nb = max(r[7] + (r[1] + 7) // 8 * 8 for r in tab)
  bias = torch.zeros(nb, dtype=torch.float64, device=w.device)
  bmask = torch.zeros(nb, dtype=torch.bool, device=w.device)
  s_all = torch.zeros(row0[-1], dtype=torch.float64, device=w.device)
  for u, (wo, cout, per, go, bo, mo, vo, fo) in enumerate(tab):
    gam, bet = f64(aux32[go:go + cout]), f64(aux32[bo:bo + cout])
    mean, var = f64(running[mo:mo + cout]), f64(running[vo:vo + cout])
    # var + eps with eps as the fp32 value the kernel adds
    s = gam / torch.sqrt(var + float(eps[u]))
    s_all[row0[u]:row0[u] + cout] = s
    sl = slice(wo, wo + cout * per)
    wf[sl] = (f64(wflat[sl]).reshape(cout, per) * s[:, None]).reshape(-1)
    wmask[sl] = True
    bias[fo:fo + cout] = bet - mean * s
    bmask[fo:fo + cout] = True
  return s_all, wf, bias, wmask, bmask


def check_bn_fold(wf, bias, wf0, bias0, tab, eps, row0, w, aux32, running, what):
  """bn_fold's outputs ``wf`` (bf16, layout of w) and ``bias`` (fp32) against float64, given what
  they held before the launch (``wf0``, ``bias0``):
    * wf: the float64 product t = w s64 rounded to bf16, exactly, unless t lies within the error
      of the fp32 product (FOLD_S_REL + one rounding) of a bf16 rounding boundary; there either
      neighbour (rounding is monotone, so wf must lie in [bf16(t - e), bf16(t + e)]);
    * bias: within fp32 bounds of beta - mean s64: the scale's error on mean s and two roundings;
    * every element no unit covers (the head's rows, the bias padding) exactly as it was."""
  u = 2.0 ** -24
  s64, t, b64, wmask, bmask = fold_ref(tab, eps, row0, w, aux32, running)
  e = (FOLD_S_REL + 2 * u) * t.abs()
  rne = lambda v: v.to(torch.float32).to(torch.bfloat16).to(torch.float64)  # noqa: E731
  lo, hi = rne(t - e), rne(t + e)
  got = wf.reshape(-1).to(torch.float64)
  bad = wmask & ~((got >= lo) & (got <= hi))
  if bool(bad.any()):
    i = int(bad.nonzero()[0])
    raise AssertionError("{}: {} of {} folded filter elements wrong; first at {}: got {!r} "
                         "float64 {!r}".format(what, int(bad.sum()), int(wmask.sum()), i,
                                               float(got[i]), float(t[i])))
  b = bias.reshape(-1)[:b64.numel()].to(torch.float64)
  ms = (b64 - _fold_beta(tab, aux32, b64)).abs()   # |mean s64|
  bound = (FOLD_S_REL + 2 * u) * ms + 2 * u * b64.abs()
  err = (b - b64).abs()
  badb = bmask & ~(err <= bound)
  if bool(badb.any()):
    i = int(badb.nonzero()[0])
    raise AssertionError("{}: {} of {} folded biases out of bound; first at {}: got {!r} float64 "
                         "{!r} bound {!r}".format(what, int(badb.sum()), int(bmask.sum()), i,
                                                  float(b[i]), float(b64[i]), float(bound[i])))
  keep = ~wmask
  assert _same_bits(wf.reshape(-1)[keep], wf0.reshape(-1)[keep]), \
      what + ": filter elements of no folded unit changed"
  bk = torch.ones(bias.numel(), dtype=torch.bool, device=bias.device)
  bk[:bmask.numel()] = ~bmask
  assert _same_bits(bias.reshape(-1)[bk], bias0.reshape(-1)[bk]), \
      what + ": bias elements of no folded unit changed"


def _same_bits(a, b):
  iv = {torch.bfloat16: torch.int16, torch.float32: torch.int32}
  return torch.equal(a.contiguous().view(iv[a.dtype]), b.contiguous().view(iv[b.dtype]))


def _fold_beta(tab, aux32, like):
  """beta of every bias slot the table covers, in the bias vector's layout (0 elsewhere)."""
  out = torch.zeros_like(like)
  for wo, cout, per, go, bo, mo, vo, fo in tab.cpu().tolist():
    out[fo:fo + cout] = aux32[bo:bo + cout].to(torch.float64)
  return out

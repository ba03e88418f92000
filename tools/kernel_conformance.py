"""Float64 references for the pooling, fused-stem, input-decode and small MNIST kernels.

Shared by tests/test_gpu_kernel_conformance.py (replays what the models launch) and
tests/test_kernel_conformance_host.py (checks these references against PyTorch on the CPU).
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

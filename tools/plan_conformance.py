"""Element-wise float64 checks for the implicit-GEMM plans and the batch-norm / elementwise kernels.

Shared by tests/test_gpu_plan_conformance.py (replays what the models build) and
tests/test_plan_conformance_host.py (checks this checker on the CPU).  Everything works on torch
tensors of any device; references are float64.

Error bound of one output element (``elem_bound``)
-------------------------------------------------
A forward-like kernel computes ``f = sum_k x_k w_k (+ bias)`` in fp32 and stores ``RN(act(f))``.
The products of two bf16 values are exact in fp32.  The sum is a chain of n = K + 1 additions
(K products, then the bias) in an order the wgmma unit and the K loop decide.  Whatever the order,
each addition adds a relative error of at most u_acc to a partial sum whose magnitude is at most
``M = sum_k |x_k||w_k| (+ |bias|)``, so (Higham, Accuracy and Stability, Lemma 3.1 / eq. 3.5)

    |f - ref| <= gamma_n * M,    gamma_n = n u_acc / (1 - n u_acc).

u_acc is 2^-23, not the 2^-24 of round-to-nearest: the tensor cores align and add significands
with truncation (Fasi, Higham, Mikaitis, Pranesh, "Numerical behavior of NVIDIA tensor cores",
PeerJ CS 2021), which is one full ulp per addition at worst.  The activations (ReLU, ReLU6) are
1-Lipschitz and monotone, so ``|act(f) - act(ref)| <= gamma_n M``.  The final rounding to the
output type (unit roundoff u_out = 2^-8 for bf16, 2^-24 for fp32) adds ``u_out |act(f)|``:

    |out - act(ref)| <= u_out |act(ref)| + (1 + u_out) gamma_n M.

The staged accumulate epilogue rounds twice: ``out = RN(act(RN(f) + prev))``.  The inner rounding
adds ``u_out |partial|`` with ``partial = conv + bias``, and the fp32 addition of two bf16 values
at most ``2^-24 (|partial| + |prev|)``; both are added to the bound (``partial=``, ``prev=``).

Systematic rounding (``rounding_bias``): where ``gamma_n M`` is far below ``u_out |ref|`` the error
is dominated by the final rounding, and ``sign(ref) (out - ref) / ulp(ref)`` averages to 0 under
round-to-nearest-even and to about -0.5 under truncation.
"""
import math

import torch

U_BF16 = 2.0 ** -8
U_FP32 = 2.0 ** -24
U_ACC = 2.0 ** -23   # per addition of the tensor-core fp32 accumulation (truncating, see above)

# guard-band pattern: bf16 0x7fc1 / fp32 0x7fc17fc1 (NaN payloads no kernel produces)
GUARD_BF16 = 0x7FC1
GUARD_FP32 = 0x7FC17FC1
# fill of outputs a kernel must overwrite completely: another NaN payload
UNWRITTEN_BF16 = 0x7FA5
UNWRITTEN_FP32 = 0x7FA57FA5
GUARD_BYTES = 4096   # a multiple of 1024: a view at this offset keeps the allocation's alignment


def gamma(n, u=U_ACC):
  """Higham's gamma_n = n u / (1 - n u) for a chain of n roundings of unit u."""
  nu = n * u
  assert nu < 0.5, "accumulation chain too long for a first-order bound"
  return nu / (1.0 - nu)


def bf16_rne(x):
  """Round float64 values to bf16 with round-to-nearest-even; returned as float64."""
  return x.to(torch.float32).to(torch.bfloat16).to(torch.float64)


def bf16_trunc(x):
  """Round float64 values toward zero to bf16 (what a wrong epilogue would store)."""
  bits = x.to(torch.float32).contiguous().view(torch.int32) & ~0xFFFF
  return bits.view(torch.float32).to(torch.float64)


def ulp_bf16(x):
  """Spacing of bf16 values at |x| (x != 0)."""
  e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
  return torch.pow(2.0, e - 7)


def elem_bound(ref, M, n, u_out=U_BF16, partial=None, prev=None):
  """Allowed |out - ref| per element (see the module docstring)."""
  g = gamma(n) * M
  b = u_out * ref.abs() + (1.0 + u_out) * g
  if partial is not None:
    b = b + (1.0 + u_out) * (u_out * (partial.abs() + g) + U_FP32 * (partial.abs() + g))
  if prev is not None:
    b = b + (1.0 + u_out) * U_FP32 * prev.abs()
  return b


def gamma_prob(d, u=U_FP32, lam=8.0):
  """Probabilistic counterpart of gamma_d for round-to-nearest (Higham and Mary, "A new approach
  to probabilistic rounding error analysis", SIAM J. Sci. Comput. 41(5), 2019): a term that
  passes through d roundings carries a relative error of at most
  exp(lam sqrt(d) u + d u^2 / (1 - u)) - 1 with probability >= 1 - 2 exp(-lam^2 (1 - u)^2 / 2),
  i.e. >= 1 - 3e-14 for lam = 8.  Used for the fp32 round-to-nearest column sums (statistics,
  batch-norm reductions), whose worst-case gamma_d cannot see one M box missing from a sum of
  millions of terms."""
  return math.expm1(lam * math.sqrt(d) * u + d * u * u / (1.0 - u))


def wgrad_chain(info):
  """(L, S): the longest run of pixels one CTA accumulates in its wgmma accumulator for one dW
  entry before adding it to dW, and how many such partial sums reach one entry with red.global.add.
    generic kernel (igemm_wgrad_kernel): CTA c takes iterations [c T / G, (c + 1) T / G) of the
      T = total_work (tile, pixel box) iterations and adds its partial once per tile it touches:
      L <= ceil(T / G) boxes, S <= G;
    halo kernels (stem 1 / 2): a work item is a slice pair and ceil(boxes / k_splits) boxes:
      L = that many boxes, S = k_splits."""
  boxes = info["tiles_w"] * info["tiles_h"] * info["tiles_n"]
  if info["stem"]:
    per = -(-boxes // info["k_splits"])
    return per * info["box_rows"], info["k_splits"]
  per = min(boxes, -(-info["total_work"] // info["grid"]))
  return per * info["box_rows"], info["grid"]


def wgrad_bound(M, dw0_abs, info):
  """Allowed |dW - (dW0 + ref)| for one entry: each partial carries gamma_L(u_acc) of its terms
  (the tensor-core accumulation, see the module docstring); dW0 and the S partials then meet in
  S fp32 round-to-nearest atomic additions, gamma_{S+1}(2^-24) of their magnitudes."""
  L, S = wgrad_chain(info)
  gl = gamma(L + 1)
  return gl * M + gamma(S + 1, U_FP32) * ((1.0 + gl) * M + dw0_abs)


def fwd_stat_depth(infos, staged):
  """Roundings one stored value passes through on its way into the per-column sums of the
  forward-like epilogue (col_sum / col_sumsq, and the fused BN-backward sums):
    staged copy-out: the thread's register sum over its copy-out rows (fwd_rows_per = min(BN, 128)
      / 16 per tile, for every tile the CTA runs before it flushes), then the shared-memory sum of
      the 2 * 128 / (kOutCols / 8) threads that own the column's chunk;
    direct path: red.shared of every row (128 per tile) of the tiles before a flush;
  then one global atomic per flush.  A CTA whose grid is a multiple of n_tiles keeps its n tile
  and flushes once (grid / n_tiles flushes per column); otherwise it flushes after every tile
  (one flush per M box).  All launches of a plan add into the same sums."""
  chain, flushes = 0, 0
  for i in infos:
    bn = i["bn"]
    boxes = i["tiles_w"] * i["tiles_h"] * i["tiles_n"]
    pinned = i["grid"] % i["n_tiles"] == 0
    tiles = -(-i["total_work"] // i["grid"]) if pinned else 1
    if staged:
      out_cols = min(bn, 128)
      c = tiles * out_cols // 16 + 2 * 128 // (out_cols // 8)
    else:
      c = tiles * 128
    chain = max(chain, c)
    flushes += i["grid"] // i["n_tiles"] if pinned else boxes
  return chain + flushes + 1


def red_grid_depth(P, C, waves, sms=132, threads=256):
  """Roundings of one row's term in the column reductions of bn_bwd.cu / elementwise.cu
  (red_grid and the thread geometry there): a thread sums every (gridDim.x * rl)-th row, the
  block sums its rl row lanes, and each block adds one atomic."""
  groups = C // 8
  cg = min(groups, threads)
  rl = threads // cg
  gy = -(-groups // cg)
  bx = max(1, min(-(-P // rl), (sms * waves + gy - 1) // gy))
  return -(-P // (bx * rl)) + rl + bx + 1


def check_close(out, ref, bound, what):
  """Raise AssertionError naming the worst element where |out - ref| > bound (NaN fails)."""
  out = out.to(torch.float64)
  err = (out - ref).abs()
  bad = ~(err <= bound)
  if bool(bad.any()):
    excess = torch.where(bad, torch.nan_to_num(err - bound, nan=float("inf")),
                         torch.zeros_like(err))
    i = int(excess.reshape(-1).argmax())
    raise AssertionError(
        "{}: {} of {} elements out of bound; worst at flat index {}: out {!r} ref {!r} bound {!r}"
        .format(what, int(bad.sum()), bad.numel(), i, float(out.reshape(-1)[i]),
                float(ref.reshape(-1)[i]), float(bound.reshape(-1)[i])))


def rounding_bias(out, ref, M, n, u_out=U_BF16, min_count=256):
  """Mean of sign(ref) (out - ref) / ulp(ref) over the elements whose accumulation error is far
  below the output rounding: gamma_n M <= u_out |ref| / 8, so that the accumulation moves an element
  by at most 1/8 ulp (u_out |ref| < 1 ulp).  Round-to-nearest-even then averages within 1/8 ulp of
  0 (plus sampling noise) and truncation within 1/8 ulp of -1/2.  Returns (mean, count); mean is
  None when fewer than ``min_count`` elements qualify."""
  out = out.to(torch.float64)
  sel = (gamma(n) * M * 8 <= u_out * ref.abs()) & (ref != 0)
  cnt = int(sel.sum())
  if cnt < min_count:
    return None, cnt
  r = ref[sel]
  if u_out == U_BF16:
    ulp = ulp_bf16(r)
  else:
    ulp = torch.pow(2.0, torch.floor(torch.log2(r.abs())) - 23)
  d = torch.sign(r) * (out[sel] - r) / ulp
  return float(d.mean()), cnt


def check_no_bias(out, ref, M, n, what, u_out=U_BF16, tol=0.25):
  mean, cnt = rounding_bias(out, ref, M, n, u_out)
  if mean is not None:
    assert abs(mean) <= tol, "{}: systematic rounding error {:+.3f} ulp over {} elements".format(
        what, mean, cnt)
  return mean, cnt


# ------------------------------------------------------------------ batch norm
# Bounds of the batch-norm kernels (csrc/bn_bwd.cu, csrc/elementwise.cu), shared by the plan
# suite's replays and the step suite (tools/step_conformance.py).  Everything is float64; per-
# channel vectors are [C], per-element tensors [P, C].  The extension is built with
# --use_fast_math: an fp32 division is within 2 ulp (4 u), a multiply or add within u, rsqrtf
# within 2 ulp.
def bn_finalize_refs(s_sum, s_sq, gam, bet, rm0, rv0, cnt, eps, mom, u=U_FP32):
  """{output: (float64 reference, bound)} of the statistics finalisation (bn_apply_finalize,
  bn_finalize, the fused stem) from the fp32 sums it read, the parameters and the running
  statistics before the launch."""
  m64 = s_sum / cnt
  ex2 = s_sq / cnt
  var = (ex2 - m64 * m64).clamp_min(0)
  is64 = 1.0 / torch.sqrt(var + eps)
  e_var = gamma(10, u) * (ex2 + m64 * m64)
  rel_is = 0.5 * e_var / (var + eps) + 5 * u
  sc64 = gam * is64
  sh64 = bet - m64 * sc64
  unb = var * cnt / (cnt - 1) if cnt > 1 else var
  fac = cnt / (cnt - 1) if cnt > 1 else 1.0
  return {
      "mean": (m64, 4 * u * m64.abs()),
      "invstd": (is64, rel_is * is64),
      "scale": (sc64, (rel_is + 2 * u) * sc64.abs()),
      "shift": (sh64, (rel_is + 8 * u) * (m64 * sc64).abs() + 2 * u * sh64.abs()),
      "running_mean": ((1 - mom) * rm0 + mom * m64,
                       gamma(8, u) * ((1 - mom) * rm0.abs() + mom * m64.abs())),
      "running_var": ((1 - mom) * rv0 + mom * unb,
                      gamma(10, u) * ((1 - mom) * rv0.abs() + mom * unb) +
                      mom * (e_var + u * var) * fac),
  }


def bn_apply_ref(x, scale, shift, res=None, act=1, u=U_FP32, sample_scale=None):
  """(y reference, bound, pre-activation, ambiguous) of the apply y = bf16(act(x scale + shift
  (+ res))): one fma and one add in fp32, then the bf16 rounding.  ``ambiguous``: elements whose
  pre-activation lies within those roundings of 0, where the ReLU mask bit is not decided.
  ``sample_scale`` (stochastic depth; per row, broadcast against x): y = act(s (x scale + shift)
  (+ res)), one more fp32 multiply."""
  xs = x * scale
  pre = xs + shift
  Mv = xs.abs() + shift.abs()
  n = 2
  if sample_scale is not None:
    pre = pre * sample_scale
    Mv = Mv * sample_scale.abs()
    n = 3
  if res is not None:
    pre = pre + res
    Mv = Mv + res.abs()
  ref = pre.clamp_min(0.0) if act else pre
  if act == 2:
    ref = ref.clamp_max(6.0)
  bound = U_BF16 * ref.abs() + (1 + U_BF16) * gamma(n, u) * Mv
  return ref, bound, pre, pre.abs() <= gamma(n, u) * Mv


def bn_bwd_reduce_refs(g, xm, invstd, depth, d0=0.0, b0=0.0, amb_mag=None):
  """((dgamma ref, bound), (dbeta ref, bound)) of bn_bwd_reduce: column sums of the masked
  gradient g and of g (x - mean) invstd added to d0 / b0, fp32 round-to-nearest along a tree of
  ``depth`` roundings (red_grid_depth), plus x - mean and the invstd product for dgamma.
  ``amb_mag``: |dy| where the recomputed mask is ambiguous (either bit is right there)."""
  d0 = torch.as_tensor(d0, dtype=torch.float64, device=g.device)
  b0 = torch.as_tensor(b0, dtype=torch.float64, device=g.device)
  ref_g = d0 + (g * xm).sum(0) * invstd
  bnd_g = gamma_prob(depth + 2) * (d0.abs() + (g.abs() * xm.abs()).sum(0) * invstd)
  ref_b = b0 + g.sum(0)
  bnd_b = gamma_prob(depth) * (b0.abs() + g.abs().sum(0))
  if amb_mag is not None:
    bnd_g = bnd_g + (amb_mag * xm.abs()).sum(0) * invstd
    bnd_b = bnd_b + amb_mag.sum(0)
  return (ref_g, bnd_g), (ref_b, bnd_b)


def bn_bwd_fused_dgamma_ref(sum_g, sum_gx, mean, invstd, u=U_FP32):
  """(dgamma reference, bound) of the apply kernel that finishes a reduction fused into a data
  gradient's epilogue: invstd (sum(g x) - mean sum(g)), three fp32 roundings."""
  return invstd * (sum_gx - mean * sum_g), gamma(3, u) * invstd * (sum_gx.abs() +
                                                                  (mean * sum_g).abs())


def bn_bwd_dx_ref(g, x, gam, mean, invstd, dg, db, amb=None, gmag=None, u=U_FP32, roundings=10):
  """(dx reference, bound) of bn_bwd_apply: dx = gamma invstd (g - dbeta / P - (x - mean) invstd
  dgamma / P) from the dgamma / dbeta the kernel read, ten fp32 roundings, then bf16; infinite
  where ``amb`` (the mask bit is not decided).  ``gmag``: sum of the magnitudes behind g, where g
  is itself a sum (the stem's routed max-pool gradient); |g| otherwise.  ``roundings``: 11 where
  g is itself an fp32 product (the stochastic-depth factor times the masked gradient)."""
  P = x.shape[0]
  A = gam * invstd
  ref = A * (g - db / P - (x - mean) * invstd * dg / P)
  Mv = (A * (g.abs() if gmag is None else gmag)).abs() + \
      (A * invstd * dg / P).abs() * (x.abs() + mean.abs()) + (A * db / P).abs()
  bound = U_BF16 * ref.abs() + (1 + U_BF16) * gamma(roundings, u) * Mv
  if amb is not None:
    bound = torch.where(amb, torch.full_like(bound, float("inf")), bound)
  return ref, bound


# ------------------------------------------------------------------ row sampling
def sample_box_rows(box_index, rows, valid):
  """Rows of M box ``box_index`` (``rows`` rows, ``valid(r)``: row r maps to a pixel inside the
  tensor) that the check samples: two rows 64 apart (one per consumer warpgroup of a 128-row box)
  that rotate with the box index, so that over >= 128 boxes every row position - every copy-out
  chunk owner and both warpgroups - is sampled.  An invalid row moves to the next valid one."""
  out = []
  for start in (box_index % rows, (box_index + 64) % rows):
    for k in range(rows):
      r = (start + k) % rows
      if valid(r):
        if r not in out:
          out.append(r)
        break
  return out


def box_pixels(info, box):
  """Output pixels (n, oh, ow) of every row of M box ``box`` of a forward-like launch, None where
  the row lies outside the tensor (igemm_fwd_kernel: tile origin and org_pixel_off)."""
  tw = box % info["tiles_w"]
  th = (box // info["tiles_w"]) % info["tiles_h"]
  tn = box // (info["tiles_w"] * info["tiles_h"])
  bw, bh, bn = info["box_w"], info["box_h"], info["box_n"]
  out = []
  for pr in range(bw * bh * bn):
    w, h, n = tw * bw + pr % bw, th * bh + (pr // bw) % bh, tn * bn + pr // (bw * bh)
    if w < info["lim_w"] and h < info["lim_h"] and n < info["lim_n"]:
      out.append((n, h * info["osh"] + info["ooh"], w * info["osw"] + info["oow"]))
    else:
      out.append(None)
  return out


def all_pixels(infos, device="cpu"):
  """Every output pixel (n, oh, ow) the launches of a plan cover (small plans are checked in
  full)."""
  cols = [[], [], []]
  for info in infos:
    bw, bh, bn = info["box_w"], info["box_h"], info["box_n"]
    w = torch.arange(info["tiles_w"] * bw, device=device)
    h = torch.arange(info["tiles_h"] * bh, device=device)
    n = torch.arange(info["tiles_n"] * bn, device=device)
    n, h, w = torch.meshgrid(n[n < info["lim_n"]], h[h < info["lim_h"]], w[w < info["lim_w"]],
                             indexing="ij")
    cols[0].append(n.reshape(-1))
    cols[1].append(h.reshape(-1) * info["osh"] + info["ooh"])
    cols[2].append(w.reshape(-1) * info["osw"] + info["oow"])
  return tuple(torch.cat(c) for c in cols)


def sample_pixels(infos, device="cpu"):
  """Sampled output pixels of a plan (all its launches): the rows ``sample_box_rows`` picks in
  every M box, computed for all boxes at once.  Returns int64 tensors (n, oh, ow, launch, box,
  row), one entry per sample; a box whose two picks coincide contributes one."""
  cols = [[] for _ in range(6)]
  gbox = 0
  for li, info in enumerate(infos):
    bw, bh, bn = info["box_w"], info["box_h"], info["box_n"]
    rows = bw * bh * bn
    boxes = info["tiles_w"] * info["tiles_h"] * info["tiles_n"]
    b = torch.arange(boxes, device=device).unsqueeze(1)
    r = torch.arange(rows, device=device).unsqueeze(0)
    tw, th, tn = b % info["tiles_w"], (b // info["tiles_w"]) % info["tiles_h"], \
        b // (info["tiles_w"] * info["tiles_h"])
    w, h, n = tw * bw + r % bw, th * bh + (r // bw) % bh, tn * bn + r // (bw * bh)
    valid = (w < info["lim_w"]) & (h < info["lim_h"]) & (n < info["lim_n"])
    picks = []
    for off in (0, 64):
      start = (b[:, 0] + gbox + off) % rows
      order = (start.unsqueeze(1) + r) % rows                  # rows from `start` on, cyclically
      first = torch.gather(valid, 1, order).to(torch.int8).argmax(1)
      picks.append(torch.gather(order, 1, first.unsqueeze(1))[:, 0])
    rr = torch.stack(picks, 1)                                   # [boxes, 2]
    bb = b.expand(-1, 2)
    keep = torch.ones_like(rr, dtype=torch.bool)
    keep[:, 1] = rr[:, 1] != rr[:, 0]
    rr, bb = rr[keep], bb[keep]
    ww, hh, nn = (x.expand(boxes, rows)[bb, rr] for x in (w, h, n))
    cols[0].append(nn)
    cols[1].append(hh * info["osh"] + info["ooh"])
    cols[2].append(ww * info["osw"] + info["oow"])
    cols[3].append(torch.full_like(rr, li))
    cols[4].append(bb)
    cols[5].append(rr)
    gbox += boxes
  return tuple(torch.cat(c) for c in cols)


# ------------------------------------------------------------------ signatures
def dedup(signatures):
  """Signatures (hashable) in first-seen order without repeats."""
  seen, out = set(), []
  for s in signatures:
    if s not in seen:
      seen.add(s)
      out.append(s)
  return out


def freeze(v):
  """A hashable form of nested dicts / lists / tuples."""
  if isinstance(v, dict):
    return tuple(sorted((k, freeze(x)) for k, x in v.items()))
  if isinstance(v, (list, tuple)):
    return tuple(freeze(x) for x in v)
  return v


# ------------------------------------------------------------------ guard bands
def guarded(shape, dtype, device, fill_bits=None, margin=GUARD_BYTES):
  """A tensor of ``shape`` that is a view into a larger allocation with ``margin`` bytes before
  and after it, filled with the guard pattern.  ``fill_bits``: initial bit pattern of the view
  (e.g. UNWRITTEN_*), else the caller fills it.  Returns (view, backing)."""
  es = torch.empty((), dtype=dtype).element_size()
  assert margin % 1024 == 0 and margin % es == 0
  numel = int(math.prod(shape))
  pad = margin // es
  back = torch.empty(numel + 2 * pad, dtype=dtype, device=device)
  ib = _int_view(back)
  ib.fill_(_guard(dtype))
  view = back[pad:pad + numel].view(shape)
  if fill_bits is not None:
    _int_view(view).fill_(fill_bits)
  return view, back


def _int_view(t):
  if t.dtype == torch.bfloat16:
    return t.view(torch.int16)
  if t.dtype == torch.float32:
    return t.view(torch.int32)
  return t.view(torch.uint8)


def _guard(dtype):
  if dtype == torch.bfloat16:
    return GUARD_BF16 - 0x10000 if GUARD_BF16 >= 0x8000 else GUARD_BF16
  if dtype == torch.float32:
    return GUARD_FP32
  return 0xA5


def guard_intact(view, back, margin=GUARD_BYTES):
  """True when both margins around ``view`` still hold the guard pattern."""
  es = back.element_size()
  pad = margin // es
  ib = _int_view(back)
  g = _guard(back.dtype)
  return bool((ib[:pad] == g).all()) and bool((ib[pad + view.numel():] == g).all())


def unwritten(t):
  """Mask of elements that still hold the UNWRITTEN pattern."""
  if t.dtype == torch.bfloat16:
    return t.view(torch.int16) == UNWRITTEN_BF16
  return t.view(torch.int32) == UNWRITTEN_FP32

"""Plans for the wgmma implicit-GEMM kernels (csrc/igemm.cu, csrc/igemm_wgrad.cu).

A *plan* binds fixed device buffers to one kernel launch: two TMA tensor maps
plus the tile/tap tables.  Layers build their plans once (buffers are static,
which is also what CUDA-graph capture wants) and then only call ``run()``.

Layout conventions (all bf16 unless noted):
  activations  NHWC  ``[N, H, W, C]``        C % 8 == 0
  weights      KRSC  ``[Cout, R, S, Cin]``   (a dense layer is R = S = 1)
  weight grads KRSC  fp32, accumulated with red.global.add (zero them first)

These replace the cuDNN/cuBLAS calls the reference reaches through TensorFlow
(SURVEY.md section 2.6(b)).
"""
from .. import _build

BLOCK_M = 128
BLOCK_K = 64
_launches = 0
# 128 x 256-tile weight gradients from this many pixels on (_wgrad_plan)
_WGRAD_WIDE_MIN_PIXELS = 32768
# 3x3 / stride 1 weight gradients with 64-channel multiples: all nine taps from one pass over the
# pixels (_wgrad3x3_onepass_plan) once the layer has this many output pixels
_WGRAD_HALO_MIN_PIXELS = 8192
_SMS = 132   # H100 SXM; the halo kernels' work-item counts below are multiples of it


def launch_count():
  """Number of native kernel launches issued through this module (bench accounting)."""
  return _launches


def _C():
  return _build.load(required=True)


class Plan(object):
  """One or more prepared igemm launches; ``run()`` enqueues them on the current stream."""

  def __init__(self, handles, keep, desc=""):
    self.handles = list(handles)
    self.keep = keep  # tensors that must outlive the plan
    self.desc = desc

  def run(self):
    global _launches
    C = _C()
    for h in self.handles:
      C.igemm_run(h)
    _launches += len(self.handles)

  @property
  def num_launches(self):
    return len(self.handles)

  def set_reverse(self, flag):
    """Walk the pixel tiles last-to-first (forward-like plans): an L2 hand-over hint - start where
    the kernel that produced this plan's input stopped writing (models/resnet.py)."""
    C = _C()
    for h in self.handles:
      C.igemm_set_reverse(h, bool(flag))

  def info(self):
    return [_C().igemm_info(h) for h in self.handles]

  def __del__(self):
    try:
      C = _build.load(required=False)
      if C is not None:
        for h in self.handles:
          C.igemm_free(h)
    except Exception:
      pass
    self.handles = []


def _bn_for(n):
  if n <= 64:
    return 64
  if n <= 128:
    return 128
  return 256 if n % 256 == 0 else 128


def _tmap4(t, dims_whn, c, box, es=None, c_box=64):
  """Tensor map (C, W, H, N) over an NHWC tensor (or any tensor addressed that way)."""
  W, H, N = dims_whn
  d = {
      "base": t.data_ptr(),
      "dims": [c, W, H, N],
      "strides": [c * 2, W * c * 2, H * W * c * 2],
      "box": [c_box] + list(box),
  }
  if es is not None:
    d["elem_strides"] = [1] + list(es)
  return d


def _tmap2(t, rows, cols, box_rows, ld=None):
  """Tensor map over a row-major [rows, cols] matrix; box = 64 columns x box_rows rows."""
  ld = cols if ld is None else ld
  return {"base": t.data_ptr(), "dims": [cols, rows], "strides": [ld * 2], "box": [64, box_rows]}


def choose_box(OW, OH, N, multiple_of=1, allow_pad=False, max_rows=128, min_rows=1):
  """Pick the pixel box (bw, bh, bn) with bw*bh*bn <= max_rows that wastes the fewest MMA rows.

  ``multiple_of`` constrains the row count (the weight-gradient kernel needs a
  multiple of 16 because pixels are its K dimension); ``allow_pad`` lets the box
  overhang the tensor (TMA zero-fills the overhang).
  """
  best = None
  max_bw = min(max_rows, OW + (7 if allow_pad else 0))
  for bw in range(1, max_bw + 1):
    tw = -(-OW // bw)
    if not allow_pad and bw > OW:
      break
    for bh in range(1, min(max_rows // bw, OH + (15 if allow_pad else 0)) + 1):
      th = -(-OH // bh)
      full_img = tw == 1 and th == 1
      for bn in ([1] + ([b for b in range(2, max_rows // (bw * bh) + 1)] if full_img else [])):
        if bn > N:
          break
        rows = bw * bh * bn
        if rows % multiple_of or rows < min_rows:
          continue
        tn = -(-N // bn)
        denom = 128 if multiple_of == 1 else rows
        eff = float(OW * OH * N) / (tw * th * tn * denom)
        # prefer efficient, then wide rows (longer contiguous TMA segments)
        key = (round(eff, 4), bw, bh)
        if best is None or key > best[0]:
          best = (key, (bw, bh, bn, tw, th, tn))
  if best is None:
    raise ValueError("no box for {}x{}x{}".format(OW, OH, N))
  return best[1]


def _stats_args(g, stats):
  if stats is not None:
    g["col_sum"] = stats[0].data_ptr()
    g["col_sumsq"] = stats[1].data_ptr()


# --------------------------------------------------------------------- GEMM
def gemm(a, b, out, b_layout="nk", bias=None, relu=False, accumulate=False, stats=None):
  """out[M, N] = a[M, K] @ B (+bias)(relu).  b_layout 'nk': b is [N, K]; 'kn': b is [K, N]."""
  import torch
  M, K = a.shape
  N = b.shape[0] if b_layout == "nk" else b.shape[1]
  assert K % 8 == 0 and a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
  assert a.is_contiguous() and b.is_contiguous() and out.is_contiguous()
  bn = _bn_for(N)
  ta = _tmap4(a, (M, 1, 1), K, (128, 1, 1))
  if b_layout == "nk":
    assert b.shape[1] == K
    tb = _tmap2(b, N, K, bn)
  else:
    assert b.shape[0] == K and N % 8 == 0
    tb = _tmap2(b, K, N, 64)
  g = {
      "tiles_w": -(-M // 128), "n_tiles": -(-N // bn), "box_w": 128,
      "num_taps": 1, "k_chunks": -(-K // 64),
      "lim_w": M, "lim_h": 1, "lim_n": 1, "OW": M, "OH": 1,
      "ldo": out.shape[1], "n_valid": N, "relu": int(relu),
      "out_fp32": int(out.dtype == torch.float32), "accumulate": int(accumulate),
      "bias": bias.data_ptr() if bias is not None else 0, "out": out.data_ptr(),
  }
  _stats_args(g, stats)
  h = _C().igemm_plan_fwd(ta, tb, g, bn, b_layout == "kn")
  return Plan([h], (a, b, out, bias, stats), "gemm M{} N{} K{}".format(M, N, K))


def gemm_wgrad(dy, x, dw):
  """dw[N_out, K_in] (fp32, +=) = dy[M, N_out]^T @ x[M, K_in]."""
  M, Cout = dy.shape
  Cin = x.shape[1]
  return _wgrad_plan(dy, (M, 1, 1), Cout, x, (M, 1, 1), Cin, dw, Cin, [(0, 0, 0, 0)], 1, 1,
                     box=(128, 1, 1, -(-M // 128), 1, 1))


# --------------------------------------------------------------------- conv
def conv_fprop(x, w, y, stride=1, pad=0, bias=None, relu=False, stats=None, accumulate=False):
  """y[N,OH,OW,Cout] (=|+=) conv(x[N,H,W,Cin], w[Cout,R,S,Cin]) with fused bias/ReLU/BN statistics.
  ``accumulate``: y = act(y + conv + bias) - the residual add of an inference network whose batch
  norms are folded into the filters (models/resnet.py: build_folded_inference)."""
  N, H, W, Cin = x.shape
  Cout, R, S, _ = w.shape
  _, OH, OW, _ = y.shape
  assert Cin % 8 == 0 and w.shape[3] == Cin and R * S <= 9
  bn = _bn_for(Cout)
  if R == 1 and S == 1 and stride == 1 and pad == 0:
    return gemm(x.view(-1, Cin), w.view(Cout, Cin), y.view(-1, Cout), "nk", bias, relu, accumulate,
                stats)
  bw, bh, bnn, tw, th, tn = choose_box(OW, OH, N)
  if stride == 1:
    ta = _tmap4(x, (W, H, N), Cin, (bw, bh, bnn))
  else:
    ta = _tmap4(x, (W, H, N), Cin, (bw * stride, bh * stride, bnn), es=(stride, stride, 1))
  tb = _tmap2(w, Cout, R * S * Cin, bn)
  taps = [(r, s) for r in range(R) for s in range(S)]
  g = {
      "tiles_w": tw, "tiles_h": th, "tiles_n": tn, "n_tiles": -(-Cout // bn),
      "box_w": bw, "box_h": bh, "box_n": bnn, "mul_w": stride, "mul_h": stride,
      "num_taps": len(taps), "k_chunks": -(-Cin // 64),
      "tap_dw": [s - pad for (r, s) in taps], "tap_dh": [r - pad for (r, s) in taps],
      "tap_bk": [(r * S + s) * Cin for (r, s) in taps],
      "lim_w": OW, "lim_h": OH, "lim_n": N, "OW": OW, "OH": OH,
      "ldo": Cout, "n_valid": Cout, "relu": int(relu), "accumulate": int(accumulate),
      "bias": bias.data_ptr() if bias is not None else 0, "out": y.data_ptr(),
  }
  _stats_args(g, stats)
  h = _C().igemm_plan_fwd(ta, tb, g, bn, False)
  return Plan([h], (x, w, y, bias, stats), "fprop {}x{} s{} {}->{} @{}x{}".format(
      R, S, stride, Cin, Cout, OH, OW))


def conv_dgrad(dy, w, dx, stride=1, pad=0, accumulate=False, relu=False, bias=None, stats=None,
               acc_mask=None, bn_reduce=None, epi_prefetch=True):
  """dx[N,H,W,Cin] (=|+=) conv_transpose(dy[N,OH,OW,Cout], w[Cout,R,S,Cin]).

  Also the forward of a transposed convolution (Keras Conv2DTranspose) when
  ``w`` is laid out [Cin_of_the_transposed_conv, R, S, Cout_of_it].
  For stride 2 the output is split in four parity classes, each a small
  stride-1 convolution over dy with the taps of matching parity.

  ``bn_reduce = (x_raw, mask_bits | None, sum_g, sum_gx)``: dx is the gradient entering the batch
  norm whose input was ``x_raw`` (shape of dx); the epilogue accumulates the two per-channel sums
  of that batch norm's backward reduction while it stores dx (csrc/igemm.h: red_x).  Requires
  that this call writes EVERY pixel of dx (raises ValueError otherwise: a strided 1x1 does not).

  ``epi_prefetch``: whether the accumulate / ``bn_reduce`` epilogue prefetches the values it reads
  into shared memory while the main loop runs (False: it loads them in the copy-out pass).  Both
  give the same dx bit for bit.  The plan falls back to the loads in the copy-out pass where it
  cannot prefetch (``Plan.info()``: ``epi_prefetch``).
  """
  N, OH, OW, Cout = dy.shape
  _, R, S, Cin = w.shape
  _, H, W, _ = dx.shape
  assert Cout % 8 == 0 and Cin % 8 == 0
  bn = _bn_for(Cin)
  tb = _tmap2(w, Cout, R * S * Cin, 64)
  handles = []
  classes = [(0, 0)] if stride == 1 else [(ph, pw) for ph in range(stride) for pw in range(stride)]
  for (ph, pw) in classes:
    taps = [(r, s) for r in range(R) for s in range(S)
            if (ph + pad - r) % stride == 0 and (pw + pad - s) % stride == 0]
    if not taps:
      assert accumulate, "strided dgrad class without taps needs accumulate=True (or a pre-zeroed dx)"
      if bn_reduce is not None:
        raise ValueError("fused BN reduction: this data gradient does not write every pixel")
      continue
    ch, cw = -(-(H - ph) // stride), -(-(W - pw) // stride)  # pixels of this class
    if ch <= 0 or cw <= 0:
      continue
    bw, bh, bnn, tw, th, tn = choose_box(cw, ch, N)
    ta = _tmap4(dy, (OW, OH, N), Cout, (bw, bh, bnn))
    g = {
        "tiles_w": tw, "tiles_h": th, "tiles_n": tn, "n_tiles": -(-Cin // bn),
        "box_w": bw, "box_h": bh, "box_n": bnn,
        "num_taps": len(taps), "k_chunks": -(-Cout // 64),
        "tap_dw": [(pw + pad - s) // stride for (r, s) in taps],
        "tap_dh": [(ph + pad - r) // stride for (r, s) in taps],
        "tap_bn": [(r * S + s) * Cin for (r, s) in taps],
        "lim_w": cw, "lim_h": ch, "lim_n": N, "OW": W, "OH": H,
        "osw": stride, "oow": pw, "osh": stride, "ooh": ph,
        "ldo": Cin, "n_valid": Cin, "accumulate": int(accumulate), "relu": int(relu),
        "acc_mask": acc_mask.data_ptr() if acc_mask is not None else 0,
        "bias": bias.data_ptr() if bias is not None else 0, "out": dx.data_ptr(),
        "epi_prefetch": int(bool(epi_prefetch)),
    }
    _stats_args(g, stats)  # transposed-conv *forward* feeding a batch norm
    if bn_reduce is not None:
      rx, rmask, sum_g, sum_gx = bn_reduce
      assert stats is None and tuple(rx.shape) == tuple(dx.shape) and Cin % bn == 0
      g["red_x"] = rx.data_ptr()
      g["red_mask"] = rmask.data_ptr() if rmask is not None else 0
      g["col_sum"], g["col_sumsq"] = sum_g.data_ptr(), sum_gx.data_ptr()
    handles.append(_C().igemm_plan_fwd(ta, tb, g, bn, True))
  return Plan(handles, (dy, w, dx, bias, stats, acc_mask, bn_reduce),
              "dgrad {}x{} s{} {}->{} @{}x{}{}".format(R, S, stride, Cout, Cin, H, W,
                                                      " +bnred" if bn_reduce is not None else ""))


def _wgrad_plan(dy, dy_whn, Cout, x, x_whn, Cin, dw, ldw, taps, mul, es, box=None):
  OW, OH, N = dy_whn
  # 128 x 256 tile per CTA (wgmma N = 256): fewer operand bytes per MAC than 128 x 128; it only
  # pays when both channel counts fill the tile and there are enough pixels to split over
  wide = (Cout % 256 == 0 and Cin % 256 == 0 and es == 1
          and OW * OH * N >= _WGRAD_WIDE_MIN_PIXELS)
  if box is None:
    box = choose_box(OW, OH, N, multiple_of=16, allow_pad=True)
  bw, bh, bnn, tw, th, tn = box
  assert (bw * bh * bnn) % 16 == 0 and bw * bh * bnn <= 128
  bn = 64 if Cin <= 64 else 128
  if wide:
    bn = 256
  ta = _tmap4(dy, dy_whn, Cout, (bw, bh, bnn))
  if es == 1:
    tb = _tmap4(x, x_whn, Cin, (bw, bh, bnn))
  else:
    tb = _tmap4(x, x_whn, Cin, (bw * es, bh * es, bnn), es=(es, es, 1))
  m_tiles, n_tiles = -(-Cout // 128), -(-Cin // bn)
  g = {
      "tiles_w": tw, "tiles_h": th, "tiles_n": tn, "box_w": bw, "box_h": bh, "box_n": bnn,
      "mul_w": mul, "mul_h": mul, "num_taps": len(taps),
      "tap_dw": [t[0] for t in taps], "tap_dh": [t[1] for t in taps],
      "tap_out": [t[2] for t in taps],
      "m_tiles": m_tiles, "n_tiles": n_tiles,
      "m_valid": Cout, "n_valid": Cin, "ldw": ldw, "dw": dw.data_ptr(),
  }
  h = _C().igemm_plan_wgrad(ta, tb, g, bn)
  return Plan([h], (dy, x, dw), "wgrad{} {}->{} taps{} {}".format(
      " wide" if wide else "", Cin, Cout, len(taps),
      _slices_desc(len(taps) * m_tiles * n_tiles, tw * th * tn, _C().igemm_info(h)["grid"])))


def _wgrad_slices(tiles, boxes, ctas):
  """The pixel split of the generic weight-gradient kernel (csrc/igemm_wgrad.cu,
  igemm_wgrad_kernel).  The ``tiles * boxes`` (output tile, pixel box) iterations, tiles outermost,
  go to ``min(ctas, tiles * boxes)`` CTAs in contiguous slices whose lengths differ by at most one
  box.  Returns one list per CTA of the segments ``(tile, first box, end box)`` of its slice, one
  per tile it touches, in the order the CTA walks them: last first.  The CTA adds its partial dW
  to the tile once per segment."""
  total = tiles * boxes
  grid = min(ctas, total)
  out = []
  for c in range(grid):
    start, it = c * total // grid, (c + 1) * total // grid
    segs = []
    while it > start:
      t = (it - 1) // boxes
      b0 = max(start, t * boxes) - t * boxes
      segs.append((t, b0, it - t * boxes))
      it = t * boxes + b0
    out.append(segs)
  return out


def _slices_desc(tiles, boxes, ctas):
  slices = _wgrad_slices(tiles, boxes, ctas)
  lens = [sum(b1 - b0 for (_, b0, b1) in s) for s in slices]
  lo, hi = min(lens), max(lens)
  mid = sum(1 for s in slices if s[-1][1] != 0)
  return "slice {} boxes, {}/{} CTAs start mid-tile".format(
      lo if lo == hi else "{}-{}".format(lo, hi), mid, len(slices))


# three ring stages of igemm_wgrad_halo_kernel: the 7 x 7 layers measured 17 % slower with two stages
# of 8 x 8 x 2 pixels than with three of 8 x 8 x 1
_HALO_STAGE_BYTES = 216 * 1024 // 3


def onepass_box(OW, OH, N):
  """dY box (8, bh, bn) of the one-pass 3x3 weight gradient: 8 x bh pixels (bh even: a K slice is
  two 8-pixel rows) of bn images, several images only when one image fits in bh rows.  Picks the
  largest fraction of useful (non-padding) pixels, then the most pixels per stage.
  Returns (bh, bn, tiles_w, tiles_h, tiles_n, useful fraction)."""
  best = None
  tw = -(-OW // 8)
  for bh in range(2, 17, 2):
    th = -(-OH // bh)
    for bn in range(1, 128 // (8 * bh) + 1):
      if bn > N or (bn > 1 and th > 1):
        break
      if 16384 + 3 * 8 * (bh + 2) * bn * 128 > _HALO_STAGE_BYTES:
        break
      tn = -(-N // bn)
      useful = float(OW * OH * N) / (tw * 8 * th * bh * tn * bn)
      key = (round(useful, 4), bh * bn)
      if best is None or key > best[0]:
        best = (key, (bh, bn, tw, th, tn, useful))
  return best[1]


def _wgrad3x3_onepass_plan(dy, x, dw):
  """3x3 / stride 1 / pad 1 with Cin and Cout multiples of 64: all nine taps from one pass over the
  pixels (csrc/igemm_wgrad.cu igemm_wgrad_halo_kernel).  A work item is a 64 x 64 channel slice
  pair and a range of pixel boxes; each box of dY comes with three w-shifted X boxes (dw = -1, 0,
  +1) that also hold the rows above and below, and a filter tap selects rows of one of them."""
  N, OH, OW, Cout = dy.shape
  _, H, W, Cin = x.shape
  bh, bn, tw, th, tn, useful = onepass_box(OW, OH, N)
  ta = _tmap4(dy, (OW, OH, N), Cout, (8, bh, bn))
  tb = _tmap4(x, (W, H, N), Cin, (8, bh + 2, bn))
  taps = [(dh, dw_) for dh in (-1, 0, 1) for dw_ in (-1, 0, 1)]
  # K slice j (16 pixels: output rows 2j', 2j'+1 of image i) reads the B rows of image i starting
  # at output row 2j' (+ dh + 1 for the tap)
  jpi = bh // 2
  pairs = (Cout // 64) * (Cin // 64)
  total_boxes = tw * th * tn
  # one wave of work items: two waves measured 3-10 % slower (twice the fp32 atomics of dW)
  k_splits = max(1, min(_SMS // pairs, total_boxes // 2))
  g = {
      "tiles_w": tw, "tiles_h": th, "tiles_n": tn, "box_w": 8, "box_h": bh, "box_n": bn,
      "num_taps": 1, "stem": 2,
      "halo_boxes": 3, "box_dw": [-1, 0, 1], "halo_rows": bh + 2, "halo_hmul": 1, "halo_h0": -1,
      "halo_rowbytes": 1024, "halo_nacc": 9,
      "halo_jrow": [(j // jpi) * (bh + 2) + 2 * (j % jpi) for j in range(bh * bn // 2)],
      "acc_box": [d + 1 for (_, d) in taps], "acc_row": [dh + 1 for (dh, _) in taps],
      "tap_out": [((dh + 1) * 3 + (d + 1)) * Cin for (dh, d) in taps],
      "m_tiles": Cout // 64, "n_tiles": Cin // 64, "k_splits": k_splits,
      "m_valid": Cout, "n_valid": Cin, "ldw": 9 * Cin, "dw": dw.data_ptr(),
  }
  h = _C().igemm_plan_wgrad(ta, tb, g, 64)
  return Plan([h], (dy, x, dw), "wgrad 3x3 onepass {}->{} box 8x{}x{} useful {:.0%} splits{}".format(
      Cin, Cout, bh, bn, useful, k_splits))


def conv_wgrad(dy, x, dw, stride=1, pad=0):
  """dw[Cout,R,S,Cin] (fp32, +=) = sum_pixels dy[.,Cout]^T x_shifted[.,Cin]."""
  N, OH, OW, Cout = dy.shape
  _, H, W, Cin = x.shape
  _, R, S, _ = dw.shape
  if R == 1 and S == 1 and stride == 1 and pad == 0:
    return gemm_wgrad(dy.view(-1, Cout), x.view(-1, Cin), dw.view(Cout, Cin))
  if (R == 3 and S == 3 and stride == 1 and pad == 1 and Cin % 64 == 0
      and Cout % 64 == 0 and N * OH * OW >= _WGRAD_HALO_MIN_PIXELS):
    return _wgrad3x3_onepass_plan(dy, x, dw)
  taps = [(s - pad, r - pad, (r * S + s) * Cin) for r in range(R) for s in range(S)]
  return _wgrad_plan(dy, (OW, OH, N), Cout, x, (W, H, N), Cin, dw, R * S * Cin, taps, stride,
                     stride)


# --------------------------------------------------------------- ResNet stem
# 7x7 / stride-2 convolution on a 3-channel image.  The input is stored as
# [N, H, Wp, 8] (3 real + 5 zero channels, zero columns left and right) so that
# one filter ROW - 7 taps x 8 channels = 56 values, padded to 64 - is a single
# contiguous 128-byte TMA row; an overlapping tensor map (W stride = 2 pixels)
# turns the whole 7x7 window into 7 K-blocks of 64.
STEM_K, STEM_PAD, STEM_CP = 7, 3, 8


def stem_geometry(H, W):
  OH, OW = (H + 2 * STEM_PAD - STEM_K) // 2 + 1, (W + 2 * STEM_PAD - STEM_K) // 2 + 1
  Wp = 2 * (OW - 1) + 8 + 0  # last window start + 8 pixels
  Wp = max(Wp, W + STEM_PAD + 1)
  Wp = (Wp + 1) // 2 * 2
  return OH, OW, Wp


def _stem_halo_tmap(xp, N, H, Wp, OW, bw, rows):
  """Window-row view of xp with input rows at stride 1: one box = bw window columns x rows."""
  return {
      "base": xp.data_ptr(),
      "dims": [64, OW, H, N],
      "strides": [2 * STEM_CP * 2, Wp * STEM_CP * 2, H * Wp * STEM_CP * 2],
      "box": [64, bw, rows, 1],
  }


def stem_fprop(xp, w, y, bias=None, relu=False, stats=None):
  """xp [N,H,Wp,8] (image at column offset 3), w [Cout, 7, 64] (row-major taps, 8 ch each), y [N,OH,OW,Cout]."""
  N, H, Wp, _ = xp.shape
  Cout = w.shape[0]
  _, OH, OW, _ = y.shape
  if Cout > 64:
    raise ValueError("stem_fprop: Cout {} > 64 (the stem kernel computes one 64-channel tile)"
                     .format(Cout))
  # halo mode (csrc/igemm.cu "stem mode"): 8 x 16 output pixels per tile, one 8 x 37 box of
  # input rows serves all seven filter rows, the packed filter stays resident in smem
  ta = _stem_halo_tmap(xp, N, H, Wp, OW, 8, 2 * 16 + 5)
  tb = _tmap2(w, Cout, 7 * 64, 64)
  g = {
      "tiles_w": -(-OW // 8), "tiles_h": -(-OH // 16), "tiles_n": N, "n_tiles": 1,
      "box_w": 8, "box_h": 16, "box_n": 1, "mul_w": 1, "mul_h": 2,
      "num_taps": 7, "k_chunks": 1, "stem": 1,
      "tap_dw": [0] * 7, "tap_dh": [-STEM_PAD] * 7, "tap_bk": [r * 64 for r in range(7)],
      "lim_w": OW, "lim_h": OH, "lim_n": N, "OW": OW, "OH": OH,
      "ldo": Cout, "n_valid": Cout, "relu": int(relu),
      "bias": bias.data_ptr() if bias is not None else 0, "out": y.data_ptr(),
  }
  _stats_args(g, stats)
  h = _C().igemm_plan_fwd(ta, tb, g, 64, False)
  return Plan([h], (xp, w, y, bias, stats), "stem fprop (halo)")


def stem_wgrad(dy, xp, dw):
  """dw [Cout, 7, 64] fp32 += dy[N,OH,OW,Cout]^T windows(xp)."""
  N, OH, OW, Cout = dy.shape
  _, H, Wp, _ = xp.shape
  if Cout > 64:
    raise ValueError("stem_wgrad: Cout {} > 64 (the stem kernel computes one 64-channel tile)"
                     .format(Cout))
  # all seven filter rows from one 16 x 21 halo box per 16 x 8 output pixels
  # (csrc/igemm_wgrad.cu igemm_wgrad_halo_kernel)
  ta = _tmap4(dy, (OW, OH, N), Cout, (16, 8, 1))
  tb = _stem_halo_tmap(xp, N, H, Wp, OW, 16, 2 * 8 + 5)
  tw, th = -(-OW // 16), -(-OH // 8)
  g = {
      "tiles_w": tw, "tiles_h": th, "tiles_n": N, "box_w": 16, "box_h": 8, "box_n": 1,
      "num_taps": 1, "stem": 1,
      "halo_boxes": 1, "box_dw": [0], "halo_rows": 2 * 8 + 5, "halo_hmul": 2,
      "halo_h0": -STEM_PAD, "halo_jrow": [2 * j for j in range(8)], "halo_rowbytes": 2048,
      "halo_nacc": 7,
      "acc_box": [0] * 7, "acc_row": list(range(7)), "tap_out": [r * 64 for r in range(7)],
      "m_tiles": 1, "n_tiles": 1, "k_splits": max(1, min(_SMS, tw * th * N)),
      "m_valid": Cout, "n_valid": 64, "ldw": 7 * 64, "dw": dw.data_ptr(),
  }
  h = _C().igemm_plan_wgrad(ta, tb, g, 64)
  return Plan([h], (dy, xp, dw), "stem wgrad (halo)")


def pack_stem_weight(w_krsc):
  """[Cout, 7, 7, 3] float -> [Cout, 7, 64] (7 taps x 8 channels + 8 zeros per filter row)."""
  import torch
  Cout = w_krsc.shape[0]
  out = torch.zeros(Cout, 7, 64, dtype=w_krsc.dtype, device=w_krsc.device)
  out[:, :, :56].view(Cout, 7, 7, 8)[..., :3] = w_krsc
  return out


def unpack_stem_weight(w_packed):
  Cout = w_packed.shape[0]
  return w_packed[:, :, :56].reshape(Cout, 7, 7, 8)[..., :3].contiguous()

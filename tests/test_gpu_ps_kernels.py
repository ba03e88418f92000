"""The six parameter-server kernels of csrc/optim_comm.cu (ps_push_dense, ps_push_sparse, ps_pull,
ps_apply, ps_push_slot, ps_pull_model) element by element against float64 / fp32 references, on
one GPU: servers and clients share the process, so the kernels that run across NVLink address
local memory here.

  * pushes: one red.add per element is fl32(w + fl32(k g)), k = fl32(-lr scale), bit for bit;
    rows pushed d times are within gamma(d + 1) of the float64 sum (the atomics' order is free);
  * pull: the fp32 copy is bitwise, the bf16 copy is bitwise round-to-nearest-even (ties, +-0,
    subnormals, +-Inf, values past the bf16 maximum; NaN stays NaN);
  * apply: SGD and momentum within a per-element bound derived from the fp32 operation chain,
    Adam's master, m and v within a relative 1e-5 of the float64 step taken from the kernel's own
    state (its __powf bias corrections carry ~1e-4 relative error), the non-trainable tail
    w -= g bit for bit, decided per element at any ema_begin;
  * push_slot / pull_model: bitwise copies, flags and counters;
  * every output lives between guard bands (tools/plan_conformance.py), outputs a kernel must
    write start as NaN, and the entry points refuse null or misaligned arguments before any launch.

Every ps_push_slot launch here has its need_applied already met when it is enqueued (the applied
word is written first on the same stream, or the previous push was applied by poll_once), so no
launch ever waits on the device."""
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location(
    "plan_conformance", os.path.join(_ROOT, "tools", "plan_conformance.py"))
pc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(pc)

U = pc.U_FP32
BIG = (1 << 20)


def _K():
  from tensorflowonspark_b200 import ops
  return ops.K


def _gen(seed):
  return torch.Generator().manual_seed(seed)


def _hyper(lr=0.1, momentum=0.9, wd=0.0, scale=1.0, b1=0.9, b2=0.999, eps=1e-7, step=0.0):
  return torch.tensor([lr, momentum, wd, scale, b1, b2, eps, step], dtype=torch.float32,
                      device="cuda")


def _guarded(values, off=0, dtype=torch.float32):
  """A view holding ``values`` (a CPU tensor) ``off`` elements into a guarded region, the
  elements before it filled with the guard pattern too.  Returns (view, region, backing)."""
  region, back = pc.guarded((values.numel() + off,), dtype, "cuda")
  view = region[off:]
  view.copy_(values.to(dtype))
  if off:
    pc._int_view(region[:off]).fill_(pc._guard(dtype))
  return view, region, back


def _unwritten(n, dtype=torch.float32, off=0):
  region, back = pc.guarded((n + off,), dtype, "cuda")
  view = region[off:]
  pc._int_view(view).fill_(pc.UNWRITTEN_BF16 if dtype == torch.bfloat16 else pc.UNWRITTEN_FP32)
  if off:
    pc._int_view(region[:off]).fill_(pc._guard(dtype))
  return view, region, back


def _intact(region, back, off=0):
  assert pc.guard_intact(region, back), "guard band overwritten"
  if off:
    assert bool((pc._int_view(region[:off]) == pc._guard(region.dtype)).all()), "guard overwritten"


def _bits(t):
  t = t.detach().cpu()
  return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _same(a, b):
  """Element-wise: same bits, or both NaN (NaN payloads differ between the GPU and the CPU)."""
  a, b = a.detach().cpu(), b.detach().cpu()
  return (_bits(a) == _bits(b)) | (torch.isnan(a.float()) & torch.isnan(b.float()))


def _assert_same(a, b, what):
  ok = _same(a, b)
  bad = torch.nonzero(~ok).flatten()[:5].tolist()
  assert bool(ok.all()), "{}: {} elements differ, first {}: got {} want {}".format(
      what, int((~ok).sum()), bad, a.detach().cpu().flatten()[bad].tolist(),
      b.detach().cpu().flatten()[bad].tolist())


def _k_of(h):
  """The kernels' step factor fl32(-lr * scale), from the hyper-parameters as stored."""
  hc = h.cpu()
  return -hc[0] * hc[3]


# -------------------------------------------------------------------------------- ps_push_dense
@pytest.mark.parametrize("n", [1, 3, 4, 5, 4099, BIG + 5])
@pytest.mark.parametrize("off", [0, 1, 2, 3])
def test_push_dense_is_bit_exact(n, off):
  """off = 0: 16-byte reductions (and the scalar tail); off 1..3 floats: the scalar path."""
  g0 = torch.randn(n, generator=_gen(n + off))
  w0 = torch.randn(n, generator=_gen(n + off + 7)) * 4
  w, wr, wb = _guarded(w0, off)
  g, gr, gb = _guarded(g0, off)
  h = _hyper(lr=0.1, scale=0.3)
  _K().ps_push_dense(w.data_ptr(), g, h)
  torch.cuda.synchronize()
  k = _k_of(h)
  _assert_same(w, w0 + k * g0, "push_dense n={} off={}".format(n, off))
  _intact(wr, wb, off)
  _intact(gr, gb, off)
  assert torch.equal(g.cpu(), g0)


def test_push_dense_zero_lr_and_non_finite_gradients():
  n = 4099
  w0 = torch.randn(n, generator=_gen(1)) + 0.5
  g0 = torch.randn(n, generator=_gen(2))
  for off in (0, 1):
    w, wr, wb = _guarded(w0, off)
    g, _, _ = _guarded(g0, off)
    _K().ps_push_dense(w.data_ptr(), g, _hyper(lr=0.0, scale=0.7))
    torch.cuda.synchronize()
    assert torch.equal(_bits(w), _bits(w0)), "lr 0 moved the weights"
    _intact(wr, wb, off)
  gs = g0.clone()
  gs[[0, 5, 4096, 4098]] = float("nan")
  gs[[1, 6, 4097]] = float("inf")
  gs[[2, 7]] = float("-inf")
  for off in (0, 2):
    w, wr, wb = _guarded(w0, off)
    g, _, _ = _guarded(gs, off)
    h = _hyper(lr=0.25, scale=1.0)
    _K().ps_push_dense(w.data_ptr(), g, h)
    torch.cuda.synchronize()
    want = w0 + _k_of(h) * gs
    _assert_same(w, want, "non-finite gradients off={}".format(off))
    got = w.cpu()
    assert bool(torch.isnan(got[[0, 5, 4096, 4098]]).all())
    assert got[1] == float("-inf") and got[2] == float("inf")
    _intact(wr, wb, off)


# ------------------------------------------------------------------------------- ps_push_sparse
@pytest.mark.parametrize("width", [1, 3, 4, 5, 8, 64])
@pytest.mark.parametrize("off", [0, 3])
def test_push_sparse_against_float64(width, off):
  """Rows without duplicates bit for bit; rows pushed d times within gamma(d + 1) of the float64
  sum; nothing outside the addressed rows changes.  off = 3: a table at a base that is not a
  multiple of 4 (the scalar path even for widths that are)."""
  rows = 300
  t0 = torch.randn(rows * width, generator=_gen(width)) * 2
  h = _hyper(lr=0.1, scale=0.3)
  k = _k_of(h).double()
  # unique rows
  idx = torch.randperm(rows, generator=_gen(width + 1))[:200].to(torch.int32)
  gr = torch.randn(200, width, generator=_gen(width + 2))
  t, tr, tb = _guarded(t0, off)
  _K().ps_push_sparse(t.data_ptr(), gr.cuda(), idx.cuda(), h)
  torch.cuda.synchronize()
  want = t0.clone().view(rows, width)
  want[idx.long()] = want[idx.long()] + _k_of(h) * gr
  _assert_same(t, want.view(-1), "push_sparse unique width={} off={}".format(width, off))
  _intact(tr, tb, off)
  # duplicate rows: 400 pushes into rows 0..59
  idx = torch.randint(0, 60, (400,), generator=_gen(width + 3), dtype=torch.int32)
  gr = torch.randn(400, width, generator=_gen(width + 4))
  t, tr, tb = _guarded(t0, off)
  _K().ps_push_sparse(t.data_ptr(), gr.cuda(), idx.cuda(), h)
  torch.cuda.synchronize()
  ref = t0.double().view(rows, width).clone()
  mag = ref.abs()
  ref.index_add_(0, idx.long(), k * gr.double())
  mag.index_add_(0, idx.long(), (k * gr.double()).abs())
  d = torch.bincount(idx.long(), minlength=rows).double()
  bound = torch.tensor([pc.gamma(int(c) + 1, U) for c in d.tolist()], dtype=torch.float64)
  bound = bound[:, None] * mag
  err = (t.cpu().double().view(rows, width) - ref).abs()
  assert bool((err <= bound).all()), "duplicates: max err / bound {}".format(
      float((err / bound.clamp_min(1e-300)).max()))
  untouched = d == 0
  assert torch.equal(_bits(t.view(rows, width)[untouched.cuda()]),
                     _bits(t0.view(rows, width)[untouched])), "rows nobody pushed changed"
  _intact(tr, tb, off)


def test_push_sparse_refusals():
  K = _K()
  t, _, _ = _guarded(torch.zeros(64))
  before = _bits(t)
  h = _hyper()
  g = torch.ones(4, 8, device="cuda")
  for what, call in [
      ("idx shorter than the rows", lambda: K.ps_push_sparse(
          t.data_ptr(), g, torch.zeros(3, dtype=torch.int32, device="cuda"), h)),
      ("idx longer than the rows", lambda: K.ps_push_sparse(
          t.data_ptr(), g, torch.zeros(5, dtype=torch.int32, device="cuda"), h)),
      ("2-D idx", lambda: K.ps_push_sparse(
          t.data_ptr(), g, torch.zeros(4, 1, dtype=torch.int32, device="cuda"), h)),
      ("1-D rows", lambda: K.ps_push_sparse(
          t.data_ptr(), g.view(-1), torch.zeros(32, dtype=torch.int32, device="cuda"), h)),
      ("int64 idx", lambda: K.ps_push_sparse(
          t.data_ptr(), g, torch.zeros(4, dtype=torch.int64, device="cuda"), h)),
      ("bf16 hyper", lambda: K.ps_push_sparse(
          t.data_ptr(), g, torch.zeros(4, dtype=torch.int32, device="cuda"), h.bfloat16())),
      ("short hyper", lambda: K.ps_push_sparse(
          t.data_ptr(), g, torch.zeros(4, dtype=torch.int32, device="cuda"), h[:2])),
      ("null table", lambda: K.ps_push_sparse(
          0, g, torch.zeros(4, dtype=torch.int32, device="cuda"), h)),
      ("dense: short hyper", lambda: K.ps_push_dense(t.data_ptr(), g.view(-1), h[:3])),
      ("dense: null", lambda: K.ps_push_dense(0, g.view(-1), h)),
  ]:
    with pytest.raises((ValueError, RuntimeError)):
      call()
  torch.cuda.synchronize()
  assert torch.equal(_bits(t), before), "a refused push wrote"


# ------------------------------------------------------------------------------------- ps_pull
def _pull_source(n, seed):
  """fp32 values with the bf16 rounding edges mixed in."""
  v = torch.randn(n, generator=_gen(seed)) * 3
  special = torch.tensor([
      0x3F808000, 0x3F818000,              # ties: to the even below / the even above
      0x3F808001, 0x3F817FFF,              # just past / just below a tie
      0x00000000, 0x80000000,              # +0, -0
      0x00000001, 0x807FFFFF, 0x00408000, 0x00418000,   # fp32 subnormals (and subnormal ties)
      0x7F800000, 0xFF800000,              # +-Inf
      0x7FC00000, 0x7FA00001, 0xFFC12345,  # NaNs
      0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF,  # past the bf16 maximum: stays, tie to Inf, Inf
      0xFF7F8000, 0x7F7F0000,              # -Inf by the tie; the bf16 maximum itself
  ], dtype=torch.int64).to(torch.int32).view(torch.float32)
  for i in range(0, n, 97):
    v[i] = special[(i // 97) % special.numel()]
  if n >= special.numel():
    v[-special.numel():] = special      # (also through the scalar tail of the vector loop)
  return v


@pytest.mark.parametrize("n", [0, 1, 3, 4, 7, BIG + 3])
@pytest.mark.parametrize("mode", ["both", "fp32", "bf16"])
def test_pull_copies_bitwise(n, mode):
  src0 = _pull_source(n, n + 3)
  src, sr, sb = _guarded(src0)
  f32, fr, fb = _unwritten(n) if mode != "bf16" else (None, None, None)
  b16, br, bb = _unwritten(n, torch.bfloat16) if mode != "fp32" else (None, None, None)
  _K().ps_pull(src.data_ptr(), f32, b16, n)
  torch.cuda.synchronize()
  if f32 is not None:
    assert torch.equal(_bits(f32), _bits(src0)), "fp32 copy not bitwise"
    _intact(fr, fb)
  if b16 is not None:
    want = src0.to(torch.bfloat16)            # PyTorch's round-to-nearest-even
    _assert_same(b16, want, "bf16 copy n={}".format(n))
    assert bool(torch.isnan(b16.cpu()).eq(torch.isnan(src0)).all())
    _intact(br, bb)
  assert torch.equal(_bits(src), _bits(src0))
  _intact(sr, sb)


def test_pull_bf16_rounding_edges_explicitly():
  src0 = torch.tensor([0x3F808000, 0x3F818000, 0x00408000, 0x7F7F8000, 0x7F7F7FFF, 0x80000000,
                       0x00000001, 0x3F808001], dtype=torch.int64).to(torch.int32)
  src, _, _ = _guarded(src0.view(torch.float32))
  b16, _, _ = _unwritten(8, torch.bfloat16)
  _K().ps_pull(src.data_ptr(), None, b16, 8)
  torch.cuda.synchronize()
  want = [0x3F80, 0x3F82, 0x0040, 0x7F80, 0x7F7F, -0x8000, 0x0000, 0x3F81]
  assert _bits(b16).tolist() == want


def test_pull_refusals():
  """ps_pull checks its outputs' dtype, length and alignment before any launch."""
  K = _K()
  n = 64
  src, _, _ = _guarded(torch.randn(n, generator=_gen(3)))
  f32, _, _ = _unwritten(n + 1)
  b16, _, _ = _unwritten(n + 2, torch.bfloat16)
  cases = [
      ("fp32 too long", lambda: K.ps_pull(src.data_ptr(), f32, None, n)),
      ("fp32 too short", lambda: K.ps_pull(src.data_ptr(), f32[:n - 1], None, n)),
      ("fp32 misaligned", lambda: K.ps_pull(src.data_ptr(), f32[1:], None, n)),
      ("bf16 given as fp32", lambda: K.ps_pull(src.data_ptr(), None, f32[:n], n)),
      ("bf16 given as fp16", lambda: K.ps_pull(
          src.data_ptr(), None, b16[:n].view(torch.float16), n)),
      ("bf16 too long", lambda: K.ps_pull(src.data_ptr(), None, b16[:n + 1], n)),
      ("bf16 misaligned", lambda: K.ps_pull(src.data_ptr(), None, b16[1:n + 1], n)),
      ("source misaligned", lambda: K.ps_pull(src.data_ptr() + 4, f32[:n], None, n)),
      ("null source", lambda: K.ps_pull(0, f32[:n], None, n)),
      ("negative n", lambda: K.ps_pull(src.data_ptr(), None, None, -4)),
  ]
  for what, call in cases:
    with pytest.raises((ValueError, RuntimeError)):
      call()
  torch.cuda.synchronize()
  assert bool(pc.unwritten(f32).all()) and bool(pc.unwritten(b16).all()), "a refused pull wrote"


# ------------------------------------------------------------------------------------ ps_apply
OPTS = {"sgd": 0, "momentum": 1, "adam": 2}


def _apply_ref(opt, w, s1, s2, g, lo, decay_end, ema_begin, h):
  """ps.apply_numpy in float64 on copies: (w, s1, s2) after the step, hyper as it was before
  (apply_numpy advances Adam's step itself, as the server does before it launches)."""
  from tensorflowonspark_b200.parallel import ps
  w, s1, s2 = w.copy(), s1.copy(), s2.copy()
  hh = h.copy()
  ps.apply_numpy(w, s1, s2, hh, g.copy(), lo, decay_end, ema_begin, OPTS[opt])
  return w, s1, s2


def _sgd_bounds(opt, w, s1, g, lo, decay_end, h):
  """Per-element bounds on |master - ref| and |state1 - ref| for SGD and momentum: the fp32 chain
  g h3 (+ wd w) -> (m s1 +) -> w - lr d has at most two roundings per operand, each of unit u
  relative to the magnitude it sees."""
  idx = np.arange(lo, lo + g.size)
  mg = np.abs(h[3] * g) + np.abs(h[2] * w) * (idx < decay_end)
  md = mg + (np.abs(h[1] * s1) if opt == "momentum" else 0.0)
  bd = pc.gamma(4, U) * md
  bw = pc.gamma(3, U) * (np.abs(w) + abs(h[0]) * md) + abs(h[0]) * bd
  return bw, bd


def _check_apply(opt, before, after, g, lo, decay_end, ema_begin, h, what):
  """before / after: (master, s1, s2) float64 numpy arrays of the slice; h: float64 hyper as
  the kernel read it (Adam's step already advanced)."""
  w0, m0, v0 = before
  w1, m1, v1 = after
  n = g.size
  href = h.copy()
  if opt == "adam":
    href[7] -= 1.0                         # apply_numpy advances it itself
  rw, rm, rv = _apply_ref(opt, w0, m0, v0, g, lo, decay_end, ema_begin, href)
  gi = np.arange(lo, lo + n)
  tail, tr = gi >= ema_begin, gi < ema_begin
  # the tail: w -= g in fp32, bit for bit; its state untouched
  wt = (w0[tail].astype(np.float32) - g[tail].astype(np.float32)).astype(np.float64)
  assert np.array_equal(w1[tail], wt), "{}: tail elements {} not w - g".format(
      what, (lo + np.nonzero(w1[tail] != wt)[0][:5]).tolist() if tail.any() else [])
  assert np.array_equal(m1[tail], m0[tail]) and np.array_equal(v1[tail], v0[tail]), \
      what + ": tail state changed"
  if opt == "sgd":
    assert np.array_equal(m1, m0) and np.array_equal(v1, v0), what + ": SGD state changed"
  if opt == "momentum":
    assert np.array_equal(v1, v0), what + ": momentum touched state2"
  if not tr.any():
    return
  if opt in ("sgd", "momentum"):
    bw, bd = _sgd_bounds(opt, w0[tr], m0[tr], g[tr], lo, decay_end, h)
    err = np.abs(w1[tr] - rw[tr])
    assert (err <= bw).all(), "{}: master off by {} > bound {} at {}".format(
        what, err.max(), bw[np.argmax(err - bw)], lo + np.nonzero(tr)[0][np.argmax(err - bw)])
    if opt == "momentum":
      assert (np.abs(m1[tr] - rm[tr]) <= bd).all(), what + ": momentum state"
  else:
    for name, got, ref in (("master", w1, rw), ("m", m1, rm), ("v", v1, rv)):
      rel = np.linalg.norm(got[tr] - ref[tr]) / max(np.linalg.norm(ref[tr]), 1e-30)
      assert rel <= 1e-5, "{}: Adam {} relative error {}".format(what, name, rel)


class _ApplySlice(object):
  """One server's buffers for direct ps_apply launches, each between guard bands."""

  def __init__(self, n, seed, opt):
    g = _gen(seed)
    self.n = n
    self.master, self.mr, self.mb = _guarded(torch.randn(n, generator=g))
    s1 = torch.randn(n, generator=g) * 0.1 if opt != "sgd" else torch.zeros(n)
    s2 = torch.rand(n, generator=g) * 0.01 if opt == "adam" else torch.zeros(n)
    self.state1, self.s1r, self.s1b = _guarded(s1)
    self.state2, self.s2r, self.s2b = _guarded(s2)
    self.flags = torch.zeros(8, dtype=torch.int32, device="cuda")   # applied words + counter

  def launch(self, slot, h, lo, decay_end, ema_begin, opt, k, seq):
    self.wbf16, self.wr, self.wb = _unwritten(self.n, torch.bfloat16)
    _K().ps_apply({
        "master": self.master.data_ptr(), "state1": self.state1.data_ptr(),
        "state2": self.state2.data_ptr(), "wbf16": self.wbf16.data_ptr(),
        "slot": slot.data_ptr(), "hyper": h.data_ptr(), "n": self.n, "lo": lo,
        "decay_end": decay_end, "ema_begin": ema_begin,
        "applied_flag": self.flags.data_ptr() + 4 * k, "seq": seq,
        "block_counter": self.flags.data_ptr() + 4 * 7, "opt": OPTS[opt]})

  def state(self):
    return tuple(t.cpu().double().numpy() for t in (self.master, self.state1, self.state2))

  def intact(self):
    for r, b in ((self.mr, self.mb), (self.s1r, self.s1b), (self.s2r, self.s2b), (self.wr, self.wb)):
      _intact(r, b)


APPLY_CASES = [
    # (lo, n, decay_end, ema_begin): global indices, the slice is [lo, lo + n)
    (0, 64, 0, 0),
    (0, 64, 64, 64),
    (0, 64, 0, 64),
    (0, 64, 64, 0),
    (0, 64, 24, 48),
    (0, 48, 24, 42),            # the tail starts inside a group of four
    (0, 64, 41, 42),
    (0, 64, 42, 41),
    (0, 64, 43, 45),
    (64, 64, 100, 107),         # a second server's slice
    (64, 64, 30, 70),           # decay ends before the slice
    (64, 64, 200, 300),         # the slice is wholly trainable and decayed
    (64, 64, 0, 10),            # the slice is wholly tail
    (128, 0, 128, 128),         # an empty slice
    (8, BIG + 8, (BIG >> 1) + 3, BIG - 5),
]


@pytest.mark.parametrize("opt", ["sgd", "momentum", "adam"])
@pytest.mark.parametrize("lo,n,decay_end,ema_begin", APPLY_CASES)
def test_apply_against_float64(opt, lo, n, decay_end, ema_begin):
  sl = _ApplySlice(n, lo + n + decay_end, opt)
  h = _hyper(lr=0.01 if opt == "adam" else 0.05, momentum=0.9, wd=0.03, scale=0.5)
  for step in range(3):
    slot0 = torch.randn(n, generator=_gen(step * 31 + n))
    slot, slr, slb = _guarded(slot0)
    before = sl.state()
    if opt == "adam":
      h[7:8].add_(1.0)                       # as PSServer does before each apply
    hb = h.clone()
    sl.launch(slot, h, lo, decay_end, ema_begin, opt, k=step % 2, seq=step + 1)
    torch.cuda.synchronize()
    what = "{} lo={} n={} decay_end={} ema_begin={} step {}".format(
        opt, lo, n, decay_end, ema_begin, step)
    after = sl.state()
    _check_apply(opt, before, after, slot0.double().numpy(), lo, decay_end, ema_begin,
                 hb.cpu().double().numpy(), what)
    assert torch.equal(_bits(sl.wbf16), _bits(sl.master.cpu().to(torch.bfloat16))), \
        what + ": wbf16 is not bf16_rne(master)"
    assert torch.equal(h, hb), what + ": the kernel changed the hyper-parameters"
    flags = sl.flags.cpu().tolist()
    assert flags[step % 2] == step + 1, what + ": applied flag"
    assert flags[7] == 0, what + ": block counter not reset"
    assert torch.equal(_bits(slot), _bits(slot0)), what + ": the slot changed"
    sl.intact()
    _intact(slr, slb)
  if opt == "adam":
    assert float(h[7]) == 3.0


def test_apply_refusals():
  """Null state for an optimizer that needs it, and unaligned slices, are refused."""
  K = _K()
  sl = _ApplySlice(64, 5, "adam")
  slot, _, _ = _guarded(torch.zeros(64))
  h = _hyper()
  base = {"master": sl.master.data_ptr(), "state1": sl.state1.data_ptr(),
          "state2": sl.state2.data_ptr(), "wbf16": sl.master.data_ptr(), "slot": slot.data_ptr(),
          "hyper": h.data_ptr(), "n": 64, "lo": 0, "decay_end": 64, "ema_begin": 64,
          "applied_flag": sl.flags.data_ptr(), "seq": 9, "block_counter": sl.flags.data_ptr() + 28}
  before = sl.state()
  for what, kw in [("adam without v", dict(state2=0, opt=2)),
                   ("momentum without m", dict(state1=0, opt=1)),
                   ("no slot", dict(slot=0, opt=0)),
                   ("no counter", dict(block_counter=0, opt=0)),
                   ("n not a multiple of 8", dict(n=60, opt=0)),
                   ("lo not a multiple of 8", dict(lo=4, opt=0)),
                   ("unknown optimizer", dict(opt=3))]:
    with pytest.raises((ValueError, RuntimeError)):
      K.ps_apply(dict(base, **kw))
  torch.cuda.synchronize()
  assert all(np.array_equal(a, b) for a, b in zip(sl.state(), before))
  assert sl.flags.cpu().tolist() == [0] * 8


# -------------------------------------------------------------------------------- ps_push_slot
class _SlotWorker(object):
  """Worker-side sources (gradients [total], running statistics [R] and their pulled snapshot)."""

  def __init__(self, total, R, seed):
    g = _gen(seed)
    self.total, self.R = total, R
    self.g0 = torch.randn(total, generator=g)
    self.r0 = torch.randn(max(R, 1), generator=g)[:R]
    self.p0 = torch.randn(max(R, 1), generator=g)[:R]
    self.grads, self.gr, self.gb = _guarded(self.g0)
    self.running, self.rr, self.rb = _guarded(self.r0)
    self.pulled, self.pr, self.pb = _guarded(self.p0)

  def want(self, lo, n):
    """The slot contents: grads for the head, fl32(pulled - running) for the tail."""
    out = torch.empty(n)
    h = max(0, min(lo + n, self.total) - lo)
    out[:h] = self.g0[lo:lo + h]
    t0 = max(lo, self.total) - self.total
    out[h:] = self.p0[t0:t0 + n - h] - self.r0[t0:t0 + n - h]
    return out


def _push_slot(w, slot_buf, flags, lo, n, total, seq, need, grid=64, **over):
  """flags: int32 [8] on the device: [0] applied, [1] ready, [7] block counter.  The applied word
  already holds ``need`` (written on this stream before the launch)."""
  d = {"slot": slot_buf.data_ptr(), "grads": w.grads.data_ptr(), "running": w.running.data_ptr(),
       "running_pulled": w.pulled.data_ptr(), "n": n, "lo": lo, "total": total,
       "applied_flag": flags.data_ptr(), "need_applied": need,
       "ready_flag": flags.data_ptr() + 4, "seq": seq, "block_counter": flags.data_ptr() + 28,
       "grid": grid}
  d.update(over)
  _K().ps_push_slot(d)


SLOT_CASES = [   # (lo, n) with total 4096, 96 running statistics
    (0, 4096), (0, 4192), (4088, 40), (4096, 96), (4104, 16), (1024, 8), (2048, 0),
]


@pytest.mark.parametrize("lo,n", SLOT_CASES)
@pytest.mark.parametrize("grid", [1, 64])
def test_push_slot_is_bitwise(lo, n, grid):
  total, R = 4096, 96
  w = _SlotWorker(total, R, lo + n)
  slot, sr, sb = _unwritten(n)
  flags = torch.zeros(8, dtype=torch.int32, device="cuda")
  flags[0] = 5                                       # applied: need_applied 5 is met
  _push_slot(w, slot, flags, lo, n, total, seq=7, need=5, grid=grid)
  torch.cuda.synchronize()
  assert torch.equal(_bits(slot), _bits(w.want(lo, n))), "slot contents"
  assert flags.cpu().tolist() == [5, 7, 0, 0, 0, 0, 0, 0], "ready flag / counter"
  _intact(sr, sb)
  for r, b in ((w.gr, w.gb), (w.rr, w.rb), (w.pr, w.pb)):
    _intact(r, b)
  assert torch.equal(w.grads.cpu(), w.g0) and torch.equal(w.running.cpu(), w.r0)


def test_push_slot_refusals():
  """A slice reaching past total needs both running buffers; one below it needs the gradients.
  Each call would be allowed to run (need_applied is met), but none may launch."""
  total, R = 64, 16
  w = _SlotWorker(total, R, 3)
  slot, _, _ = _unwritten(80)
  flags = torch.zeros(8, dtype=torch.int32, device="cuda")
  for what, lo, n, over in [("no running", 0, 80, dict(running=0)),
                            ("no running snapshot", 64, 16, dict(running_pulled=0)),
                            ("no gradients", 0, 16, dict(grads=0)),
                            ("no slot", 0, 16, dict(slot=0)),
                            ("no ready flag", 0, 16, dict(ready_flag=0)),
                            ("no counter", 0, 16, dict(block_counter=0)),
                            ("unaligned slice", 4, 16, {})]:
    with pytest.raises((ValueError, RuntimeError)):
      _push_slot(w, slot, flags, lo, n, total, seq=1, need=0, **over)
  torch.cuda.synchronize()
  assert bool(pc.unwritten(slot).all()) and flags.cpu().tolist() == [0] * 8


# ------------------------------------------------------------------------------- ps_pull_model
def _pull_model(src_b16, src_f32, out, lo, n, total, decay_end, **over):
  d = {"wbf16": src_b16.data_ptr(), "master": src_f32.data_ptr(),
       "weights": out["weights"].data_ptr(), "aux32": out["aux32"].data_ptr(),
       "running": out["running"].data_ptr(), "running_pulled": out["pulled"].data_ptr(),
       "n": n, "lo": lo, "total": total, "decay_end": decay_end, "grid": 64}
  d.update(over)
  _K().ps_pull_model(d)


PULL_MODEL_CASES = [   # (lo, n, decay_end) with total 4096, 96 running statistics
    (1024, 1024, 1024),    # decay ends at the slice's start
    (1024, 1024, 1536),    # inside the slice
    (1024, 1024, 4096),    # at total
    (1024, 1024, 3000),    # past the slice
    (0, 4192, 2048),       # one server holds everything
    (3584, 608, 3584),     # the last slice, reaching into the running statistics
    (3584, 608, 4096),
    (4096, 96, 2048),      # a slice wholly in the tail
    (4104, 88, 4096),
    (2048, 0, 2048),
]


@pytest.mark.parametrize("lo,n,decay_end", PULL_MODEL_CASES)
def test_pull_model_is_bitwise(lo, n, decay_end):
  total, R = 4096, 96
  g = _gen(lo + n + decay_end)
  m0 = torch.randn(n, generator=g)
  b0 = (torch.randn(n, generator=g) * 2).to(torch.bfloat16)   # the serving copy, independent
  src_f32, fr, fb = _guarded(m0)
  src_b16, br, bb = _guarded(b0, dtype=torch.bfloat16)
  out, regions = {}, []
  for name, size, dt in (("weights", total, torch.bfloat16), ("aux32", total - decay_end, None),
                         ("running", R, None), ("pulled", R, None)):
    v, r, b = _unwritten(max(size, 1), dt or torch.float32)
    out[name] = v
    regions.append((r, b))
  _pull_model(src_b16, src_f32, out, lo, n, total, decay_end)
  torch.cuda.synchronize()
  hi = lo + n
  # bf16 weights: the slice's head, bitwise from the serving copy; the rest untouched
  a, b = lo, min(hi, total)
  wb = out["weights"].cpu()
  if b > a:
    assert torch.equal(_bits(wb[a:b]), _bits(b0[:b - a])), "weights"
  keep = torch.ones(total, dtype=torch.bool)
  keep[a:max(a, b)] = False
  assert bool(pc.unwritten(wb[keep]).all()), "weights outside the slice written"
  # fp32 copy of [decay_end, total) within the slice
  aux = out["aux32"].cpu()[:total - decay_end]
  a2, b2 = max(lo, decay_end), min(hi, total)
  keep = torch.ones(total - decay_end, dtype=torch.bool)
  if b2 > a2:
    assert torch.equal(_bits(aux[a2 - decay_end:b2 - decay_end]), _bits(m0[a2 - lo:b2 - lo]))
    keep[a2 - decay_end:b2 - decay_end] = False
  assert bool(pc.unwritten(aux[keep]).all()), "aux32 outside the slice written"
  # running statistics and their snapshot
  a3, b3 = max(lo, total), max(hi, total)
  for name in ("running", "pulled"):
    r = out[name].cpu()
    keep = torch.ones(R, dtype=torch.bool)
    if b3 > a3:
      assert torch.equal(_bits(r[a3 - total:b3 - total]), _bits(m0[a3 - lo:b3 - lo])), name
      keep[a3 - total:b3 - total] = False
    assert bool(pc.unwritten(r[keep]).all()), name + " outside the slice written"
  for r, bk in regions + [(fr, fb), (br, bb)]:
    _intact(r, bk)


def test_pull_model_refusals():
  total, R = 64, 16
  m0 = torch.randn(80, generator=_gen(9))
  src_f32, _, _ = _guarded(m0)
  src_b16, _, _ = _guarded(m0.bfloat16(), dtype=torch.bfloat16)
  out = {"weights": _unwritten(total, torch.bfloat16)[0], "aux32": _unwritten(total)[0],
         "running": _unwritten(R)[0], "pulled": _unwritten(R)[0]}
  for what, lo, n, de, over in [("no running", 0, 80, 64, dict(running=0)),
                                ("no running snapshot", 64, 16, 64, dict(running_pulled=0)),
                                ("no aux32", 0, 64, 32, dict(aux32=0)),
                                ("no aux32, decay ends inside", 32, 32, 48, dict(aux32=0)),
                                ("no weights", 0, 16, 64, dict(weights=0)),
                                ("decay_end past total", 0, 80, 72, {}),
                                ("unaligned decay_end", 0, 64, 36, {})]:
    with pytest.raises((ValueError, RuntimeError)):
      _pull_model(src_b16, src_f32, out, lo, n, total, de, **over)
  torch.cuda.synchronize()
  assert all(bool(pc.unwritten(v).all()) for v in out.values()), "a refused pull wrote"


# ---------------------------------------------------------------- through PSServer / PSClient
@pytest.fixture(scope="module")
def board():
  from tensorflowonspark_b200 import reservation
  srv = reservation.Server(1)
  addr = srv.start()
  yield addr
  srv.stop()


def _ctx_class(addr, num_ps, clients):
  class Ctx(object):
    def __init__(self, job, i, cid):
      self.job_name, self.task_index = job, i
      spec = {"ps": ["p:%d" % j for j in range(num_ps)]}
      for job_, count in clients:
        spec[job_] = ["%s:%d" % (job_, j) for j in range(count)]
      self.cluster_spec = spec
      self.cluster_id, self.server_addr, self.gpus = cid, addr, [0]
  return Ctx


def _numpy_push(w, lr, scale, g, lo, hi):
  """The shared-memory path of PSClient.push on one slice (float32 numpy arithmetic)."""
  w[lo:hi] -= (lr * scale) * g[lo:hi]


def _numpy_push_sparse(w, rows, idx, width, base, lr, scale, slices):
  """The shared-memory path of PSClient.push_sparse (float32 numpy arithmetic)."""
  for lo, hi in slices:
    for row, r in zip(rows, idx):
      s = base + int(r) * width
      b0, b1 = max(s, lo), min(s + width, hi)
      if b0 < b1:
        w[b0:b1] -= (lr * scale) * row[b0 - s:b1 - s]


E2E = [(1, 1003), (2, 1003), (3, 1003), (3, 8), (4, 96)]


@pytest.mark.parametrize("num_ps,numel", E2E)
def test_hogwild_pushes_through_the_client_match_the_numpy_path(board, num_ps, numel):
  """Dense and row-sparse pushes through PSClient on 1..4 servers (uneven last slices, empty
  servers, rows wider than a slice): single pushes bit for bit the shared-memory path's result
  (lr and scale are powers of two, so both round the same products), duplicate rows within
  gamma(d + 1) of the float64 sum."""
  from tensorflowonspark_b200.parallel import ps
  Ctx = _ctx_class(board, num_ps, [("worker", 1)])
  cid = "hog-%d-%d" % (num_ps, numel)
  w0 = torch.randn(numel, generator=_gen(numel))
  servers = [ps.PSServer(Ctx("ps", i, cid), numel, w0.cuda()) for i in range(num_ps)]
  client = ps.PSClient(Ctx("worker", 0, cid), local_servers=servers)
  slices = [(s.lo, s.hi) for s in servers]
  try:
    ref = w0.numpy().copy()
    out, orr, ob = _unwritten(numel)
    outb, brr, bb = _unwritten(numel, torch.bfloat16)
    client.pull(out_fp32=out, out_bf16=outb)
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(w0)) and torch.equal(_bits(outb), _bits(w0.bfloat16()))
    g = torch.randn(numel, generator=_gen(numel + 1))
    client.push(g.cuda(), lr=0.25, scale=0.5)
    _numpy_push(ref, 0.25, 0.5, g.numpy(), 0, numel)
    client.pull(out_fp32=out, out_bf16=outb)
    torch.cuda.synchronize()
    _assert_same(out, torch.from_numpy(ref), "dense push")
    _assert_same(outb, torch.from_numpy(ref).bfloat16(), "dense push, bf16 pull")
    # single sparse pushes (a wide row first: it holds whole slices)
    sparse = [(min(700, numel - 3), 3, [0]), (5, 1, [1, 0, 3]), (3, 2, [2])]
    if numel == 96:
      sparse = [(40, 3, [0, 1])]
    for width, base, idx in sparse:
      idx = [r for r in idx if base + (r + 1) * width <= numel]    # rows inside the vector
      if not idx:
        continue
      rows = torch.randn(len(idx), width, generator=_gen(width))
      client.push_sparse(rows.cuda(), torch.tensor(idx).cuda(), width, base=base, lr=0.5,
                         scale=1.0)
      _numpy_push_sparse(ref, rows.numpy(), idx, width, base, 0.5, 1.0, slices)
      client.pull(out_fp32=out)
      torch.cuda.synchronize()
      _assert_same(out, torch.from_numpy(ref), "sparse width {} base {}".format(width, base))
    # duplicates
    width, base = 5, 1
    nrows = (numel - base) // width
    idx = torch.randint(0, max(nrows, 1), (40,), generator=_gen(7))
    rows = torch.randn(40, width, generator=_gen(8))
    r64 = torch.from_numpy(ref).double()
    mag = r64.abs()
    before = r64.clone()
    for row, r in zip(rows.double(), idx.tolist()):
      r64[base + r * width:base + (r + 1) * width] -= 0.5 * row
      mag[base + r * width:base + (r + 1) * width] += (0.5 * row).abs()
    d = torch.zeros(numel, dtype=torch.float64)
    for r in idx.tolist():
      d[base + r * width:base + (r + 1) * width] += 1
    client.push_sparse(rows.cuda(), idx.cuda(), width, base=base, lr=0.5)
    client.pull(out_fp32=out)
    torch.cuda.synchronize()
    bound = torch.tensor([pc.gamma(int(c) + 1, U) for c in d.tolist()], dtype=torch.float64) * mag
    err = (out.cpu().double() - r64).abs()
    assert bool((err <= bound).all()), "duplicate sparse pushes"
    assert torch.equal(out.cpu().double()[d == 0], before[d == 0])
    for r, b in ((orr, ob), (brr, bb)):
      _intact(r, b)
  finally:
    client.close()
    for s in servers:
      s.close()


SLOT_E2E = [(1, 1000, 48, 600), (2, 1000, 48, 600), (3, 1000, 48, 600), (3, 8, 0, 8)]


@pytest.mark.parametrize("opt", ["sgd", "momentum", "adam"])
@pytest.mark.parametrize("num_ps,total,R,decay_end", SLOT_E2E)
def test_slot_mode_rounds_match_apply_numpy(board, opt, num_ps, total, R, decay_end):
  """Three clients, three rounds each, through PSServer / PSClient: every pull is bitwise the
  servers' state and every apply is apply_numpy in float64 from the state before it, within the
  per-apply bounds of test_apply_against_float64."""
  from tensorflowonspark_b200.parallel import ps
  numel = total + R
  Ctx = _ctx_class(board, num_ps, [("chief", 1), ("worker", 2)])
  cid = "slot-%s-%d-%d" % (opt, num_ps, numel)
  init = torch.randn(numel, generator=_gen(numel))
  servers = [ps.PSServer(Ctx("ps", i, cid), numel, init.cuda(), optimizer=opt,
                         lr=0.01 if opt == "adam" else 0.05, momentum=0.9, weight_decay=0.03,
                         decay_end=decay_end, ema_begin=total, grad_scale=0.5)
             for i in range(num_ps)]
  clients = [ps.PSClient(Ctx(j, i, cid), local_servers=servers)
             for j, i in (("chief", 0), ("worker", 0), ("worker", 1))]
  try:
    for rnd in range(3):
      for ci, c in enumerate(clients):
        weights, wr, wb = _unwritten(total, torch.bfloat16)
        aux, ar, ab = _unwritten(max(total - decay_end, 1))
        running, rr, rb = _unwritten(max(R, 1))
        running = running[:R]
        c.pull_model(weights, aux if total > decay_end else None, running if R else None,
                     decay_end=decay_end, total=total)
        torch.cuda.synchronize()
        master = torch.cat([s.master.cpu() for s in servers])
        wbf = torch.cat([s.wbf16.cpu() for s in servers])
        assert torch.equal(_bits(wbf), _bits(master.bfloat16())), "serving copy"
        assert torch.equal(_bits(weights), _bits(wbf[:total])), "pulled weights"
        if total > decay_end:
          assert torch.equal(_bits(aux[:total - decay_end]), _bits(master[decay_end:total]))
        if R:
          assert torch.equal(_bits(running), _bits(master[total:]))
        for r, b in ((wr, wb), (ar, ab), (rr, rb)):
          _intact(r, b)
        pulled = running.cpu().clone()
        if R:
          running.add_(0.1 * torch.randn(R, generator=_gen(rnd * 10 + ci)).cuda())
        grads = torch.randn(total, generator=_gen(rnd * 100 + ci)).cuda()
        before = [tuple(t.cpu().double().numpy() for t in (s.master, s.state1, s.state2))
                  for s in servers]
        c.push_grads(grads, running if R else None, total=total)
        torch.cuda.synchronize()
        assert [s.poll_once() for s in servers] == [1] * num_ps
        torch.cuda.synchronize()
        slot = torch.cat([grads.cpu(), pulled - running.cpu()]).double().numpy()
        for s, b in zip(servers, before):
          after = tuple(t.cpu().double().numpy() for t in (s.master, s.state1, s.state2))
          h = s.hyper.cpu().double().numpy()
          _check_apply(opt, b, after, slot[s.lo:s.hi], s.lo, decay_end, total, h,
                       "{} servers, client {} round {}, slice [{}, {})".format(
                           num_ps, ci, rnd, s.lo, s.hi))
          assert torch.equal(_bits(s.wbf16), _bits(s.master.cpu().bfloat16()))
          assert torch.equal(s.applied.cpu(), s.ready.cpu()), "applied flags"
          if opt == "adam":
            assert float(h[7]) == s.applies, "one Adam step per apply"
  finally:
    for c in clients:
      c.close()
    for s in servers:
      s.close()


def test_client_refuses_missing_buffers_before_any_launch(board):
  """PSClient.pull_model / push_grads against servers that hold running statistics."""
  from tensorflowonspark_b200.parallel import ps
  total, R, decay_end = 64, 16, 32
  Ctx = _ctx_class(board, 2, [("worker", 1)])
  server_list = [ps.PSServer(Ctx("ps", i, "refuse"), total + R, None, optimizer="sgd",
                             decay_end=decay_end, ema_begin=total) for i in range(2)]
  c = ps.PSClient(Ctx("worker", 0, "refuse"), local_servers=server_list)
  try:
    weights, _, _ = _unwritten(total, torch.bfloat16)
    aux, _, _ = _unwritten(total - decay_end)
    running, _, _ = _unwritten(R)
    for kw in (dict(running=None), dict(aux32=None), dict(weights=weights[:8])):
      args = dict(weights=weights, aux32=aux, running=running)
      args.update(kw)
      with pytest.raises(ValueError):
        c.pull_model(decay_end=decay_end, total=total, **args)
    grads = torch.zeros(total, device="cuda")
    with pytest.raises(ValueError):
      c.push_grads(grads, None, total=total)
    with pytest.raises(ValueError):          # running given, but never pulled
      c.push_grads(grads, torch.zeros(R, device="cuda"), total=total)
    torch.cuda.synchronize()
    assert c.pushes == 0
    assert all(bool(pc.unwritten(t).all()) for t in (weights, aux, running))
    assert all(int(s.ready.abs().sum()) == 0 for s in server_list)
  finally:
    c.close()
    for s in server_list:
      s.close()

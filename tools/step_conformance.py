"""Layer-by-layer float64 check of one real training step: the values a trainer's kernels pass to
one another, not only each kernel on fresh tensors.

Shared by tests/test_gpu_step_conformance.py (records and checks real steps, and shows that wiring
faults are caught) and tests/test_step_conformance_host.py (checks the references against torch
autograd and the checkers against planted faults on the CPU).

Recording (``record_step``)
---------------------------
While one ``train_step`` runs, ``igemm.Plan.run``, every ``ops.K`` entry point and the two
host-side clears (``StatsArena.zero``, ``FusedOptimizer.zero_grads``) are wrapped; each call is a
launch with an index.  Device writes the step makes with torch itself (``loss_sum.zero_()`` and
``correct.zero_()`` before the loss, the optimizer's hyper-parameter fills) are not launches of
their own: a write shows up at the next wrapped launch, which must own it.  After each launch
every registered buffer of the trainer is compared with
its last snapshot, on the device and bit for bit, and cloned when it changed.  So a value that a
later launch overwrites in place (an identity stage's gradient buffer holds block k's g_out, then
its g_x, then block k-1's g_x) stays available: ``Snapshots.before(name, L)`` is buffer ``name``
as launch L read it, ``after(name, L)`` as launch L left it.  Buffers are named after the network
definition (``layer2.1.r1``, ``layer2.1.u1.bn.mask``, ``stem.conv.w`` of the store...); names
that share storage (a block's input and the previous block's output) resolve to the same history.

Checking (``check_resnet_step``)
--------------------------------
The checker walks the network definition in the order the step runs it.  Each layer claims its
launches in sequence (``Claims``): a launch of another kind, or one left over at the end, fails.
Each launch may write only the buffers its layer owns (``_Ctx.owns``): a launch that clobbers an
activation between the layer that produced it and the layer that reads it fails, although the
reader's reference - which takes the buffer as the reader found it - would agree with the reader.
Each layer's outputs are compared with a float64 reference evaluated on the stored values of its
inputs, looked up by the NAME of the layer that feeds it in the network definition - never from
the consuming launch's own pointer arguments, so a launch that reads the wrong buffer disagrees
with its reference.  Because every reference is linearised at the trainer's own stored inputs,
errors do not compound from layer to layer and the per-element bounds are those of the kernel
suites (tools/plan_conformance.py); a wiring fault shows up as an O(1) miss.

A distilling trainer's step also holds its frozen teacher's folded forward pass, right after the
decode, and ``distill_xent`` in place of ``softmax_xent``.  ``teacher_buffers`` names the teacher's
buffers ``teacher.*``; every teacher launch is claimed by a ``teacher.*`` layer check, its
reference reads the student's decoded ``xp`` by name, and it may write only teacher buffers, so a
teacher launch that writes a student buffer fails.

The optimizer is checked from the snapshot before its launch: master, momentum and bf16 weights
against float64 momentum SGD with the weight-decay partition of the network definition (convolution
and dense weights decayed; batch-norm parameters and biases not, as ``torch.optim.SGD`` parameter
groups would set it), not the store's own flag.
"""
import importlib.util
import math
import os

import torch
import torch.nn.functional as F

_HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name):
  spec = importlib.util.spec_from_file_location(name, os.path.join(_HERE, name + ".py"))
  m = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(m)
  return m


pc = _load("plan_conformance")
kc = _load("kernel_conformance")

U = pc.U_FP32
_INT = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float16: torch.int16}


def f64(t):
  return t.to(torch.float64)


# ----------------------------------------------------------------------------- snapshots
class Launch(object):
  """One launch of the recorded step: ``kind`` is "plan", "k" (an ops.K entry point) or "host"."""

  def __init__(self, index, kind, name, plan=None):
    self.index, self.kind, self.name, self.plan = index, kind, name, plan
    self.wrote = []

  def __repr__(self):
    return "#{} {} {}".format(self.index, self.kind, self.name)


class Snapshots(object):
  """Histories of named buffers.  ``buffers``: (name, tensor) pairs; a tensor that lies inside an
  earlier registered one (a parameter inside the flat store, a statistics slot inside the arena)
  is a view of that base, otherwise it is a base of its own."""

  def __init__(self, buffers):
    self.bases = []      # [tensor]
    self.hist = []       # per base: [(launch index, clone)], index -1 = before the step
    self.where = {}      # name -> (base index, element offset, shape)
    for name, t in buffers:
      self.add(name, t)

  def add(self, name, t):
    es = t.element_size()
    p0, p1 = t.data_ptr(), t.data_ptr() + t.numel() * es
    for bi, b in enumerate(self.bases):
      q0 = b.data_ptr()
      if b.dtype == t.dtype and q0 <= p0 and p1 <= q0 + b.numel() * es:
        self.where[name] = (bi, (p0 - q0) // es, tuple(t.shape))
        return
    self.bases.append(t)
    self.hist.append([(-1, t.detach().clone())])
    self.where[name] = (len(self.bases) - 1, 0, tuple(t.shape))

  def update(self, index):
    """After launch ``index``: clone every base whose bits changed.  Returns their indices."""
    if not self.bases:
      return []
    diff = torch.stack([_differs(b, h[-1][1]) for b, h in zip(self.bases, self.hist)]).tolist()
    out = []
    for bi, d in enumerate(diff):
      if d:
        self.hist[bi].append((index, self.bases[bi].detach().clone()))
        out.append(bi)
    return out

  def _value(self, name, L, inclusive):
    bi, off, shape = self.where[name]
    val = None
    for i, v in self.hist[bi]:
      if i < L or (inclusive and i == L):
        val = v
      else:
        break
    n = math.prod(shape)
    return val.reshape(-1)[off:off + n].view(shape)

  def before(self, name, L):
    """Buffer ``name`` as launch L read it."""
    return self._value(name, L, False)

  def after(self, name, L):
    """Buffer ``name`` as launch L left it."""
    return self._value(name, L, True)

  def base_name(self, bi):
    return next(n for n, w in self.where.items() if w[0] == bi)

  def writers(self, name):
    bi = self.where[name][0]
    return [i for i, _ in self.hist[bi][1:]]

  def nbytes(self):
    return sum(v.numel() * v.element_size() for h in self.hist for _, v in h)


def _differs(a, b):
  it = _INT.get(a.dtype)
  if it is not None:
    return (a.reshape(-1).view(it) != b.reshape(-1).view(it)).any()
  return (a != b).any()


def record_step(net, batch, buffers):
  """Stage ``batch`` (images, labels), snapshot ``buffers`` and run one ``net.train_step()`` with
  every launch wrapped.  Returns (launches, Snapshots)."""
  from tensorflowonspark_b200 import _build, ops
  from tensorflowonspark_b200.models import engine
  from tensorflowonspark_b200.ops import igemm
  from tensorflowonspark_b200.parallel import fused_optim
  mod = _build.load(required=True)
  net.set_input(*batch)
  snaps = Snapshots(buffers)
  launches = []
  depth = [0]

  def wrapped(kind, name, fn, plan=None):
    def call(*a, **k):
      depth[0] += 1
      try:
        r = fn(*a, **k)
      finally:
        depth[0] -= 1
      if depth[0] == 0:
        la = Launch(len(launches), kind, name, plan)
        launches.append(la)
        la.wrote = snaps.update(la.index)
      return r
    return call

  patches = []

  def patch(obj, name, new):
    patches.append((obj, name, obj.__dict__.get(name, _MISSING)))
    setattr(obj, name, new)

  orig_run = igemm.Plan.run
  patch(igemm.Plan, "run", lambda self: wrapped("plan", "igemm_run", lambda: orig_run(self),
                                                self)())
  for name in dir(mod):
    fn = getattr(mod, name)
    if name.startswith("_") or isinstance(fn, type) or not callable(fn) \
        or name == "bn_set_row_reverse":
      continue
    patch(ops.K, name, wrapped("k", name, getattr(ops.K, name)))
  orig_zero = engine.StatsArena.zero
  patch(engine.StatsArena, "zero",
        lambda self: wrapped("host", "StatsArena.zero", lambda: orig_zero(self))())
  orig_zg = fused_optim.FusedOptimizer.zero_grads
  patch(fused_optim.FusedOptimizer, "zero_grads",
        lambda self: wrapped("host", "FusedOptimizer.zero_grads", lambda: orig_zg(self))())
  try:
    net.train_step()
    torch.cuda.synchronize()
  finally:
    for obj, name, old in reversed(patches):
      if old is _MISSING:
        delattr(obj, name)
      else:
        setattr(obj, name, old)
  return launches, snaps


_MISSING = object()


# ----------------------------------------------------------------------------- claims and report
class Claims(object):
  """Hands out the recorded launches in order: each layer check takes the launches it verifies,
  and every launch must be taken exactly once."""

  def __init__(self, launches):
    self.launches = list(launches)
    self.pos = 0
    self.owner = {}

  def take(self, layer, kind, name=None, plan=None):
    if self.pos >= len(self.launches):
      raise AssertionError("{}: expected a {} launch ({}), but the step ended".format(
          layer, kind, name or "plan"))
    la = self.launches[self.pos]
    ok = la.kind == kind and (name is None or la.name == name) and \
        (plan is None or la.plan is plan)
    if not ok:
      raise AssertionError("{}: expected a {} launch ({}) at {}, got {}".format(
          layer, kind, name or "its plan", self.pos, la))
    self.owner[la.index] = layer
    self.pos += 1
    return la.index

  def finish(self):
    left = self.launches[self.pos:]
    if left:
      raise AssertionError("{} launch(es) claimed by no layer check, first {}".format(
          len(left), left[0]))
    return len(self.owner)


class Report(object):
  """Collects every comparison: per layer the worst |err| / bound and the launch that produced
  it, per layer class the worst, and the failures."""

  def __init__(self):
    self.layers = {}     # layer -> [worst ratio, launch index, class]
    self.classes = {}    # class -> [worst ratio, layer]
    self.failures = []   # (launch index, layer, message)

  def _note(self, layer, cls, idx, ratio):
    w = self.layers.setdefault(layer, [0.0, idx, cls])
    if not ratio <= w[0]:
      w[0], w[1] = ratio, idx
    c = self.classes.setdefault(cls, [0.0, layer])
    if not ratio <= c[0]:
      c[0], c[1] = ratio, layer

  def close(self, layer, cls, idx, got, ref, bound, what=""):
    got = f64(got).reshape(ref.shape)
    err = (got - ref).abs()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=ref.device).expand_as(ref)
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300),
                        torch.where(err > 0, torch.full_like(err, float("inf")),
                                    torch.zeros_like(err)))
    ratio = torch.nan_to_num(ratio, nan=float("inf"))
    flat = ratio.reshape(-1)
    i = int(flat.argmax()) if flat.numel() else 0
    worst = float(flat[i]) if flat.numel() else 0.0
    self._note(layer, cls, idx, worst)
    if not worst <= 1.0:
      bad = int((flat > 1.0).sum())
      self.failures.append((idx, layer, "{} {} (launch #{}): {} of {} elements out of bound, worst "
                            "|err|/bound {:.3g} at flat index {}: got {!r} ref {!r} bound {!r}"
                            .format(layer, what or cls, idx, bad, flat.numel(), worst, i,
                                    float(got.reshape(-1)[i]), float(ref.reshape(-1)[i]),
                                    float(bound.reshape(-1)[i]))))
    return worst

  def exact(self, layer, cls, idx, wrong, what=""):
    """``wrong``: boolean tensor of elements that differ where they must be equal."""
    n = int(wrong.sum())
    self._note(layer, cls, idx, float("inf") if n else 0.0)
    if n:
      self.failures.append((idx, layer, "{} {} (launch #{}): {} of {} elements wrong".format(
          layer, what or cls, idx, n, wrong.numel())))

  def fail(self, idx, layer, msg):
    self.failures.append((idx, layer, "{} (launch #{}): {}".format(layer, idx, msg)))

  def failing_layers(self):
    return [layer for _, layer, _ in sorted(self.failures, key=lambda f: f[0])]

  def layer_table(self):
    """Every layer's worst |err| / bound and the launch that produced it, in launch order."""
    rows = ["{:<24} {:>8} {:>12}  {}".format("layer", "launch", "worst e/b", "class")]
    for layer, (r, idx, cls) in sorted(self.layers.items(), key=lambda kv: kv[1][1]):
      rows.append("{:<24} {:>8} {:>12.4f}  {}".format(layer, "#{}".format(idx), r, cls))
    return "\n".join(rows)

  def table(self):
    rows = ["{:<24} {:>12}  {}".format("layer class", "worst e/b", "at layer")]
    for cls in sorted(self.classes):
      r, layer = self.classes[cls]
      rows.append("{:<24} {:>12.4f}  {}".format(cls, r, layer))
    return "\n".join(rows)


# ----------------------------------------------------------------------------- float64 references
def nchw(t):
  return t.permute(0, 3, 1, 2)


def nhwc(t):
  return t.permute(0, 2, 3, 1)


def conv_ref(x, w, stride, pad):
  """(y, sum of magnitudes) of the convolution of x [N, H, W, Ci] with w [Co, k, k, Ci], NHWC."""
  xx, ww = nchw(x), w.permute(0, 3, 1, 2)
  y = F.conv2d(xx, ww, stride=stride, padding=pad)
  m = F.conv2d(xx.abs(), ww.abs(), stride=stride, padding=pad)
  return nhwc(y), nhwc(m)


def dgrad_ref(dy, w, xshape, stride, pad):
  """(dx, sum of magnitudes) of the data gradient of that convolution, dx of shape ``xshape``."""
  N, H, W, C = xshape
  ww = w.permute(0, 3, 1, 2)
  g = torch.nn.grad.conv2d_input((N, C, H, W), ww, nchw(dy), stride=stride, padding=pad)
  m = torch.nn.grad.conv2d_input((N, C, H, W), ww.abs(), nchw(dy).abs(), stride=stride,
                                 padding=pad)
  return nhwc(g), nhwc(m)


def wgrad_ref(dy, x, wshape, stride, pad):
  """(dw, sum of magnitudes) [Co, k, k, Ci] of that convolution."""
  Co, k, _, Ci = wshape
  g = torch.nn.grad.conv2d_weight(nchw(x), (Co, Ci, k, k), nchw(dy), stride=stride, padding=pad)
  m = torch.nn.grad.conv2d_weight(nchw(x).abs(), (Co, Ci, k, k), nchw(dy).abs(), stride=stride,
                                  padding=pad)
  return g.permute(0, 2, 3, 1), m.permute(0, 2, 3, 1)


def _stem_w(w):
  """The packed stem filter [Co, 7, 64] (7 rows x 8 columns x 8 channels) as an NCHW filter."""
  return w.reshape(w.shape[0], 7, 8, 8).permute(0, 3, 1, 2)


def stem_ref(xp, w, OW):
  """(y, magnitudes) of the stem over the packed input xp [N, H, Wp, 8] (image at column 3):
  output (n, oh, ow) = sum over rows r, columns j, channels c of xp[n, 2 oh - 3 + r, 2 ow + j, c]
  w[:, r, 8 j + c], rows outside the image 0."""
  ww = _stem_w(w)
  y = F.conv2d(nchw(xp), ww, stride=2, padding=(3, 0))[..., :OW]
  m = F.conv2d(nchw(xp).abs(), ww.abs(), stride=2, padding=(3, 0))[..., :OW]
  return nhwc(y), nhwc(m)


def stem_wgrad_ref(dy, xp):
  """(dw [Co, 7, 64], magnitudes) of the stem."""
  N, OH, OW, Co = dy.shape
  full = (xp.shape[2] - 8) // 2 + 1
  g = torch.zeros(N, Co, OH, full, dtype=dy.dtype, device=dy.device)
  g[..., :OW] = nchw(dy)
  shape = (Co, 8, 7, 8)
  dw = torch.nn.grad.conv2d_weight(nchw(xp), shape, g, stride=2, padding=(3, 0))
  m = torch.nn.grad.conv2d_weight(nchw(xp).abs(), shape, g.abs(), stride=2, padding=(3, 0))
  return (dw.permute(0, 2, 3, 1).reshape(Co, 7, 64), m.permute(0, 2, 3, 1).reshape(Co, 7, 64))


def mask_bits(mask, shape):
  """Bit e & 7 of byte e >> 3 for every flat element e of a tensor of ``shape``, as bool."""
  n = math.prod(shape)
  e = torch.arange(n, device=mask.device)
  return (((mask.reshape(-1)[e >> 3].to(torch.int64) >> (e & 7)) & 1) == 1).reshape(shape)


def col(t):
  """[P, C] view of an NHWC (or [P, C]) tensor."""
  return t.reshape(-1, t.shape[-1])


def xent_ref(logits, labels, V, scale):
  """(summed loss, dlogits [B, V], top-1 hits, logits of rows whose arg-max is a near tie) of the
  softmax cross-entropy, float64."""
  lg = logits[:, :V]
  lp = torch.log_softmax(lg, 1)
  y = labels.long()
  loss = -lp.gather(1, y[:, None])[:, 0]
  d = lp.exp()
  d[torch.arange(lg.shape[0], device=lg.device), y] -= 1.0
  top2 = lg.topk(min(2, V), 1).values
  tie = (top2[:, 0] - top2[:, -1]) <= 1e-6 * top2[:, 0].abs() if V > 1 else \
      torch.zeros(lg.shape[0], dtype=torch.bool, device=lg.device)
  hits = (lg.argmax(1) == y)
  return loss.sum() * scale, d * scale, hits, tie


def momentum_ref(w, s1, g, decay, lr, mom, wd):
  """(state, master, bounds) of fused_optim's momentum SGD on one fp32 vector (grad scale 1):
  g' = g + wd w (decayed elements), s = mom s + g', w = w - lr s; a few fp32 roundings each."""
  gg = g + torch.where(decay, wd * w, torch.zeros_like(w))
  s = mom * s1 + gg
  w1 = w - lr * s
  es = pc.gamma(3, U) * (mom * s1.abs() + g.abs() + torch.where(decay, wd * w.abs(),
                                                                 torch.zeros_like(w)))
  ew = lr * es + pc.gamma(2, U) * (w.abs() + lr * s.abs())
  return s, w1, es, ew


# ----------------------------------------------------------------------------- ResNet-50
def resnet_buffers(net):
  """(name, tensor) of every buffer a ResNetTrainer's training step reads or writes, named after
  the network definition; the flat store, optimizer state and arenas first."""
  st = net.store
  out = [("master", st.master), ("weights", st.weights), ("grads", st.grads), ("aux32", st.aux32),
         ("stats_arena", net.stats_arena.buf), ("running", net.running.buf)]
  if net.optim.state1 is not None:
    out.append(("state1", net.optim.state1))
  for s in st.order:
    for buf in ("master", "weights", "grads"):
      out.append(("{}:{}".format(buf, s["name"]), st._view(getattr(st, buf), s)))
  for name in ("in_u8", "labels", "xp", "stem_raw", "pool", "pool_idx", "g_stem_raw", "g_pool",
               "avg", "logits", "dlogits", "g_avg", "loss_sum", "correct"):
    out.append((name, getattr(net, name)))
  bns = [("stem.bn", net.stem_bn)]
  for b in net.blocks:
    for a in ("x", "r1", "a1", "r2", "a2", "r3", "out", "g_r1", "g_a1", "g_r2", "g_a2", "g_r3",
              "g_out", "g_x"):
      out.append(("{}.{}".format(b.name, a), getattr(b, a)))
    if b.ds is not None:
      for a in ("rd", "idn", "g_rd"):
        out.append(("{}.{}".format(b.name, a), getattr(b, a)))
    for u in ("u1", "u2", "u3", "ds"):
      if getattr(b, u) is not None:
        bns.append(("{}.{}.bn".format(b.name, u), getattr(b, u).bn))
  for name, bn in bns:
    for a in ("sum", "sumsq", "red_g", "red_gx", "mean", "invstd", "scale", "shift",
              "running_mean", "running_var"):
      t = getattr(bn, a, None)
      if t is not None:
        out.append(("{}.{}".format(name, a), t))
    m = getattr(bn, "_mask_buf", None)
    if m is not None:
      out.append(("{}.mask".format(name), m))
  return out


class _Ctx(object):
  """What a layer check needs: snapshots, claims, report, trainer options."""

  def __init__(self, net, launches, snaps, lr=0.1, momentum=0.9, weight_decay=1e-4):
    self.net, self.S, self.claims, self.rep = net, snaps, Claims(launches), Report()
    self.launches = launches
    self.lr, self.mom, self.wd = lr, momentum, weight_decay

  def owns(self, L, layer, *names):
    """Launch L may write only the buffers of ``names`` (their whole base buffers): a write
    anywhere else - a clobbered activation another layer still has to read - fails here."""
    mine = {self.S.where[n][0] for n in names if n in self.S.where}
    extra = [b for b in self.launches[L].wrote if b not in mine]
    if extra:
      self.rep.fail(L, layer, "wrote {} it does not own".format(
          ", ".join(self.S.base_name(b) for b in extra)))

  def b(self, name, L):
    return f64(self.S.before(name, L))

  def a(self, name, L):
    return self.S.after(name, L)

  def w(self, spec, L):
    return f64(self.S.before("weights:" + spec["name"], L))


def _stat_depth(plan, out):
  infos = plan.info()
  staged = out.shape[-1] % infos[0]["bn"] == 0 and out.shape[-1] % 8 == 0
  return pc.fwd_stat_depth(infos, staged)


def _conv_fwd(c, layer, conv, xname, yname, bnname):
  """A convolution's forward plan: the raw output and its fused statistics."""
  L = c.claims.take(layer, "plan", plan=conv.fwd)
  x = c.b(xname, L)
  ref, M = conv_ref(x, c.w(conv.sw, L), conv.stride, conv.pad)
  y = c.a(yname, L)
  n = conv.k * conv.k * conv.cin + 1
  c.rep.close(layer, "conv fwd", L, y, ref, pc.elem_bound(ref, M, n), "y")
  _stats(c, layer, L, conv.fwd, y, bnname)
  c.owns(L, layer, yname, "stats_arena")


def _stats(c, layer, L, plan, y, bnname):
  st = col(f64(y))
  gp = pc.gamma_prob(_stat_depth(plan, y))
  c.rep.close(layer, "conv fwd stats", L, c.a(bnname + ".sum", L), st.sum(0),
              gp * st.abs().sum(0), "col_sum")
  sq = st * st
  c.rep.close(layer, "conv fwd stats", L, c.a(bnname + ".sumsq", L), sq.sum(0), gp * sq.sum(0),
              "col_sumsq")


def _bn_fwd(c, layer, bn, xname, yname, resname, act, sample_scale=None):
  """bn_apply_finalize: statistics from the producing convolution's sums, y and the mask bits
  (``layer`` is also the batch norm's buffer prefix).  ``sample_scale``: the stochastic-depth
  factor of each row (float64 [P, 1]) from the host's draw."""
  L = c.claims.take(layer, "k", "bn_apply_finalize")
  x = col(c.b(xname, L))
  P = x.shape[0]
  refs = pc.bn_finalize_refs(c.b(layer + ".sum", L), c.b(layer + ".sumsq", L),
                             c.b("master:" + bn.sg["name"], L), c.b("master:" + bn.sb["name"], L),
                             c.b(layer + ".running_mean", L),
                             c.b(layer + ".running_var", L), float(P), bn.eps, bn.momentum)
  for name in ("mean", "invstd", "scale", "shift", "running_mean", "running_var"):
    c.rep.close(layer, "bn fwd stats", L, c.a(layer + "." + name, L), *refs[name], what=name)
  res = col(c.b(resname, L)) if resname else None
  ref, bound, pre, amb = pc.bn_apply_ref(x, f64(c.a(layer + ".scale", L)),
                                         f64(c.a(layer + ".shift", L)), res, act,
                                         sample_scale=sample_scale)
  c.rep.close(layer, "bn fwd y" if sample_scale is None else "bn fwd y (drop path)", L,
              col(c.a(yname, L)), ref, bound, "y")
  if getattr(bn, "mask", None) is not None:   # the bits the forward kept this step
    bits = col(mask_bits(c.a(layer + ".mask", L), (P, x.shape[1])))
    c.rep.exact(layer, "bn fwd mask", L, (bits != (pre > 0)) & ~amb, "mask bits")
  c.owns(L, layer, yname, layer + ".mask", layer + ".mean", layer + ".invstd", layer + ".scale",
         layer + ".shift", "running")


def _bn_bwd(c, layer, bn, bname, dyname, xname, maskname, dxname, producer,
            sample_scale=None):
  """A batch norm's backward: dgamma / dbeta from a fused reduction (``producer``: the data
  gradient plan that wrote dy and accumulated the sums) or an unfused bn_bwd_reduce, and dx.
  Under gradient accumulation (``bn.acc``) this micro-batch's dgamma / dbeta v go to scratch (or
  stay in registers on the fused path) and the apply adds them to the parameter gradient: that
  must be fl(gradient before + v).  ``sample_scale``: stochastic depth, the rows' factors s; the
  batch norm then sees s times the masked gradient."""
  acc = bn.acc is not None
  gname, bname_ = "grads:" + bn.sg["name"], "grads:" + bn.sb["name"]
  if not bn.fused_reduce:
    Lr = c.claims.take(layer, "k", "bn_bwd_reduce")
  L = c.claims.take(layer, "k", "bn_bwd_apply")
  L0 = L if bn.fused_reduce else Lr
  dy = col(c.b(dyname, L0))
  x = col(c.b(xname, L0))
  mean, invstd = c.b(bname + ".mean", L0), c.b(bname + ".invstd", L0)
  amb = None
  if maskname == bname + ".mask" and getattr(bn, "mask", None) is None:
    # the forward kept no bits: the backward recomputes relu(x scale + shift) > 0
    keep, amb = kc.relu_mask(x, c.b(bname + ".scale", L0), c.b(bname + ".shift", L0))
  else:
    keep = col(mask_bits(c.S.before(maskname, L0), tuple(c.S.before(xname, L0).shape)))
  g = dy * keep
  if sample_scale is not None:
    g = g * sample_scale        # one more fp32 product: a rounding deeper in every sum
  xm = x - mean
  P, C = x.shape
  cls = "bn bwd dgamma/dbeta" if sample_scale is None else "bn bwd dgamma/dbeta (drop path)"
  if bn.fused_reduce:
    # the sums of the data gradient's epilogue, then invstd (sum_gx - mean sum_g) in the apply
    gp = pc.gamma_prob(_stat_depth(producer, c.S.before(dyname, L)))
    sgx = (g * x).sum(0)
    e_gx = gp * (g * x).abs().sum(0)
    e_g = gp * g.abs().sum(0)
    ref_dg = invstd * (sgx - mean * g.sum(0))
    _, bnd3 = pc.bn_bwd_fused_dgamma_ref(g.sum(0), sgx, mean, invstd)
    bnd_dg = invstd * (e_gx + mean.abs() * e_g) + bnd3 * (1 + gp)
    dg, db = f64(c.a(gname, L)), f64(c.a(bname_, L))
    dd = (torch.zeros_like(dg), torch.zeros_like(db))
    if acc:
      # v never leaves the kernel: the gradient grew by v, up to the rounding of that addition
      dd = (U * dg.abs(), U * db.abs())
      dg, db = dg - c.b(gname, L), db - c.b(bname_, L)
    c.rep.close(layer, cls, L, dg, ref_dg, bnd_dg + dd[0], "dgamma")
    c.rep.close(layer, cls, L, db, g.sum(0), e_g + dd[1], "dbeta")
  else:
    tg, tb = (bname + ".red_gx", bname + ".red_g") if acc else (gname, bname_)
    depth = pc.red_grid_depth(P, C, 2) + (1 if sample_scale is not None else 0)
    (rg, bg), (rb, bb) = pc.bn_bwd_reduce_refs(g, xm, invstd, depth, c.b(tg, Lr), c.b(tb, Lr),
                                               None if amb is None else dy.abs() * amb)
    c.rep.close(layer, cls, Lr, c.a(tg, Lr), rg, bg, "dgamma")
    c.rep.close(layer, cls, Lr, c.a(tb, Lr), rb, bb, "dbeta")
    c.owns(Lr, layer, tg, tb)
    dg, db = c.b(tg, L), c.b(tb, L)
    dd = None
    if acc:
      _check_accumulated(c, layer, L, gname, tg)
      _check_accumulated(c, layer, L, bname_, tb)
  gam = c.b("master:" + bn.sg["name"], L)
  ref, bound = pc.bn_bwd_dx_ref(g, x, gam, mean, invstd, dg, db, amb,
                                roundings=10 if sample_scale is None else 11)
  if dd is not None:
    A = (gam * invstd).abs()
    bound = bound + A * invstd * xm.abs() * dd[0] / P + A * dd[1] / P
  c.rep.close(layer, "bn bwd dx" if sample_scale is None else "bn bwd dx (drop path)", L,
              col(c.a(dxname, L)), ref, bound, "dx")
  c.owns(L, layer, dxname, "grads")


def _check_accumulated(c, layer, L, accname, vname):
  """Launch L added this micro-batch's value (``vname`` as L read it) to ``accname``: exactly one
  fp32 round-to-nearest addition."""
  want = (c.S.before(accname, L).float() + c.S.before(vname, L).float()).view(torch.int32)
  got = c.S.after(accname, L).float().contiguous().view(torch.int32)
  c.rep.exact(layer, "bn bwd accumulate", L, got != want, accname + " += v")


def _wgrad(c, layer, conv, dyname, xname):
  L = c.claims.take(layer, "plan", plan=conv.wgrad)
  dw0 = c.b("grads:" + conv.sw["name"], L)
  ref, M = wgrad_ref(c.b(dyname, L), c.b(xname, L), conv.sw["shape"], conv.stride, conv.pad)
  c.rep.close(layer, "conv wgrad", L, c.a("grads:" + conv.sw["name"], L), dw0 + ref,
              pc.wgrad_bound(M, dw0.abs(), conv.wgrad.info()[0]), "dw")
  c.owns(L, layer, "grads")


def _dgrad(c, layer, conv, dyname, dxname, xshape, accumulate=False, maskname=None):
  L = c.claims.take(layer, "plan", plan=conv.dgrad)
  ref, M = dgrad_ref(c.b(dyname, L), c.w(conv.sw, L), xshape, conv.stride, conv.pad)
  n = conv.k * conv.k * conv.cout + 1
  if accumulate:
    prev = c.b(dxname, L)
    if maskname is not None:
      prev = prev * mask_bits(c.S.before(maskname, L), xshape)
    bound = pc.elem_bound(ref + prev, M, n, partial=ref, prev=prev)
    ref = ref + prev
  else:
    bound = pc.elem_bound(ref, M, n)
  c.rep.close(layer, "conv dgrad", L, c.a(dxname, L), ref, bound, "dx")
  c.owns(L, layer, dxname, "stats_arena")


def check_resnet_step(net, launches, snaps, lr=0.1, momentum=0.9, weight_decay=1e-4,
                      phase=(True, True)):
  """Check one recorded ResNetTrainer step (momentum SGD; with or without stochastic depth and
  gradient accumulation).  ``phase``: (zero the gradients first, update last) of the recorded
  micro-step, as ``net.accum.phase()`` gave it before the step.  Returns (Report, launches
  claimed); the claiming errors raise AssertionError naming the layer."""
  from tensorflowonspark_b200.ops import igemm
  c = _Ctx(net, launches, snaps, lr, momentum, weight_decay)
  rep, st = c.rep, net.store
  zero, update = phase
  dev = net.stem_raw.device

  def drop(bi, shape):
    """Block bi's stochastic-depth factor per row of a [N, H, W, C] tensor, from the host draw."""
    if net.dropper is None or not net.drop_path_rates[bi]:
      return None
    s = torch.as_tensor(net.last_drop_path[bi], dtype=torch.float64, device=dev)
    return s.repeat_interleave(shape[1] * shape[2])[:, None]

  # ---- forward
  L = c.claims.take("stats_arena", "host", "StatsArena.zero")
  rep.exact("stats_arena", "arena zero", L, c.a("stats_arena", L) != 0)
  c.owns(L, "stats_arena", "stats_arena")
  L = c.claims.take("decode", "k", "decode_normalize")
  ref, mag = kc.decode_ref(c.S.before("in_u8", L), c.S.before("xp", L).shape[2], 8,
                           igemm.STEM_PAD, net.mean, net.std)
  rep.close("decode", "decode", L, c.a("xp", L), ref,
            pc.U_BF16 * ref.abs() + (1 + pc.U_BF16) * pc.gamma(6, U) * mag, "xp")
  c.owns(L, "decode", "xp")
  if getattr(net, "teacher", None) is not None:
    _teacher_forward(c, net.teacher)
  L = c.claims.take("stem.conv", "plan", plan=net.p_stem)
  ref, M = stem_ref(c.b("xp", L), c.w(net.stem_w, L), net.stem_raw.shape[2])
  y = c.a("stem_raw", L)
  rep.close("stem.conv", "conv fwd", L, y, ref, pc.elem_bound(ref, M, 7 * 64 + 1), "y")
  _stats(c, "stem.conv", L, net.p_stem, y, "stem.bn")
  c.owns(L, "stem.conv", "stem_raw", "stats_arena")
  bn = net.stem_bn
  L = c.claims.take("stem.bn", "k", "stem_bn_relu_pool_fwd")
  x = c.b("stem_raw", L)
  refs = pc.bn_finalize_refs(c.b("stem.bn.sum", L), c.b("stem.bn.sumsq", L),
                             c.b("master:" + bn.sg["name"], L), c.b("master:" + bn.sb["name"], L),
                             c.b("stem.bn.running_mean", L), c.b("stem.bn.running_var", L),
                             float(x.numel() // bn.C), bn.eps, bn.momentum)
  for name in ("mean", "invstd", "scale", "shift", "running_mean", "running_var"):
    rep.close("stem.bn", "bn fwd stats", L, c.a("stem.bn." + name, L), *refs[name], what=name)
  lo, hi = kc.stem_act_bounds(x, f64(c.a("stem.bn.scale", L)), f64(c.a("stem.bn.shift", L)))
  ry, ridx, amb = kc.stem_pool_ref(lo, hi)
  rep.exact("stem.bn", "stem pool", L, ((f64(c.a("pool", L)) != ry) |
                                        (c.a("pool_idx", L).long() != ridx)) & ~amb, "pool / idx")
  c.owns(L, "stem.bn", "pool", "pool_idx", "stem.bn.mean", "stem.bn.invstd", "stem.bn.scale",
         "stem.bn.shift", "running")
  del lo, hi, ry, ridx, amb
  for bi, b in enumerate(net.blocks):
    n = b.name
    _conv_fwd(c, n + ".u1.conv", b.u1.conv, n + ".x", n + ".r1", n + ".u1.bn")
    _bn_fwd(c, n + ".u1.bn", b.u1.bn, n + ".r1", n + ".a1", None, 1)
    _conv_fwd(c, n + ".u2.conv", b.u2.conv, n + ".a1", n + ".r2", n + ".u2.bn")
    _bn_fwd(c, n + ".u2.bn", b.u2.bn, n + ".r2", n + ".a2", None, 1)
    _conv_fwd(c, n + ".u3.conv", b.u3.conv, n + ".a2", n + ".r3", n + ".u3.bn")
    if b.ds is not None:
      _conv_fwd(c, n + ".ds.conv", b.ds.conv, n + ".x", n + ".rd", n + ".ds.bn")
      _bn_fwd(c, n + ".ds.bn", b.ds.bn, n + ".rd", n + ".idn", None, 0)
      res = n + ".idn"
    else:
      res = n + ".x"
    _bn_fwd(c, n + ".u3.bn", b.u3.bn, n + ".r3", n + ".out", res, 1, drop(bi, b.r3.shape))
  last = net.blocks[-1].name + ".out"
  L = c.claims.take("avgpool", "k", "avgpool_fwd")
  ref, mag = kc.avgpool_ref(c.b(last, L))
  HW = math.prod(net.last.shape[1:3])
  rep.close("avgpool", "avgpool", L, c.a("avg", L), ref,
            pc.U_BF16 * ref.abs() + (1 + pc.U_BF16) * pc.gamma(HW + 3, U) * mag, "avg")
  c.owns(L, "avgpool", "avg")
  fc = net.fc
  L = c.claims.take("fc", "plan", plan=fc.fwd)
  a = c.b("avg", L)
  w = c.w(fc.sw, L)
  bias = c.b("master:" + fc.sbias["name"], L)
  ref = a @ w.t() + bias
  M = a.abs() @ w.abs().t() + bias.abs()
  rep.close("fc", "head fwd", L, c.a("logits", L), ref, pc.elem_bound(ref, M, fc.cin + 1, U),
            "logits")
  c.owns(L, "fc", "logits")
  if getattr(net, "teacher", None) is not None:
    _distill_loss(c, net)
  else:
    _xent_loss(c, net)
  _backward_and_update(c, net, zero, update, HW, fc, drop)
  return rep, c.claims.finish()


def _xent_loss(c, net):
  rep = c.rep
  V, B = net.num_classes, net.B
  L = c.claims.take("loss", "k", "softmax_xent")
  loss, dl, hits, tie = xent_ref(c.b("logits", L), c.S.before("labels", L), V, 1.0 / B)
  rep.close("loss", "loss", L, c.a("loss_sum", L).reshape(()), loss,
            2e-5 * abs(float(loss)) + 1e-6, "loss_sum")
  got = c.a("dlogits", L)
  rep.close("loss", "loss", L, got[:, :V], dl, pc.U_BF16 * dl.abs() + 1e-5 / B, "dlogits")
  if net.VP > V:
    rep.exact("loss", "loss", L, got[:, V:] != 0, "dlogits padding")
  nh = float(c.a("correct", L))
  if not int(hits[~tie].sum()) <= nh <= int(hits[~tie].sum()) + int(tie.sum()):
    rep.fail(L, "loss", "correct {} against {} top-1 hits".format(nh, int(hits.sum())))
  # (loss_sum and correct are cleared by torch just before the launch: charged to it)
  c.owns(L, "loss", "dlogits", "loss_sum", "correct")


def _backward_and_update(c, net, zero, update, HW, fc, drop):
  rep, B = c.rep, net.B
  # ---- backward
  if zero:   # the first micro-step of an accumulation window (every step without accumulation)
    L = c.claims.take("grads", "host", "FusedOptimizer.zero_grads")
    rep.exact("grads", "grads zero", L, c.a("grads", L) != 0)
    c.owns(L, "grads", "grads")
  L = c.claims.take("fc", "plan", plan=fc.wgrad)
  dl, a = c.b("dlogits", L), c.b("avg", L)
  dw0 = c.b("grads:" + fc.sw["name"], L)
  rep.close("fc", "head wgrad", L, c.a("grads:" + fc.sw["name"], L), dw0 + dl.t() @ a,
            pc.wgrad_bound(dl.abs().t() @ a.abs(), dw0.abs(), fc.wgrad.info()[0]), "dw")
  c.owns(L, "fc", "grads")
  L = c.claims.take("fc", "k", "colsum")
  dl = c.b("dlogits", L)
  b0 = c.b("grads:" + fc.sbias["name"], L)
  rep.close("fc", "head wgrad", L, c.a("grads:" + fc.sbias["name"], L), b0 + dl.sum(0),
            pc.gamma(dl.shape[0] + 1, U) * (b0.abs() + dl.abs().sum(0)), "dbias")
  c.owns(L, "fc", "grads")
  L = c.claims.take("fc", "plan", plan=fc.dgrad)
  dl, w = c.b("dlogits", L), c.w(fc.sw, L)
  rep.close("fc", "head dgrad", L, c.a("g_avg", L), dl @ w,
            pc.elem_bound(dl @ w, dl.abs() @ w.abs(), net.VP + 1), "g_avg")
  c.owns(L, "fc", "g_avg")
  L = c.claims.take("avgpool", "k", "avgpool_bwd")
  ga = c.b("g_avg", L)
  gl = net.blocks[-1].name + ".g_out"
  ref = (ga / HW).reshape(B, 1, 1, -1).expand(tuple(net.g_last.shape))
  rep.close("avgpool", "avgpool bwd", L, c.a(gl, L), ref,
            pc.U_BF16 * ref.abs() + (1 + pc.U_BF16) * pc.gamma(2, U) * ref.abs(), "g_last")
  c.owns(L, "avgpool", gl)
  for bi in reversed(range(len(net.blocks))):
    b = net.blocks[bi]
    n = b.name
    nxt = net.blocks[bi + 1] if bi + 1 < len(net.blocks) else None
    _bn_bwd(c, n + ".u3.bn", b.u3.bn, n + ".u3.bn", n + ".g_out", n + ".r3", n + ".u3.bn.mask",
            n + ".g_r3", nxt.u1.conv.dgrad if nxt is not None else None, drop(bi, b.r3.shape))
    _wgrad(c, n + ".u3.conv", b.u3.conv, n + ".g_r3", n + ".a2")
    _dgrad(c, n + ".u3.conv", b.u3.conv, n + ".g_r3", n + ".g_a2", tuple(b.a2.shape))
    _bn_bwd(c, n + ".u2.bn", b.u2.bn, n + ".u2.bn", n + ".g_a2", n + ".r2", n + ".u2.bn.mask",
            n + ".g_r2", b.u3.conv.dgrad)
    _wgrad(c, n + ".u2.conv", b.u2.conv, n + ".g_r2", n + ".a1")
    _dgrad(c, n + ".u2.conv", b.u2.conv, n + ".g_r2", n + ".g_a1", tuple(b.a1.shape))
    _bn_bwd(c, n + ".u1.bn", b.u1.bn, n + ".u1.bn", n + ".g_a1", n + ".r1", n + ".u1.bn.mask",
            n + ".g_r1", b.u2.conv.dgrad)
    _wgrad(c, n + ".u1.conv", b.u1.conv, n + ".g_r1", n + ".x")
    ident = b.ds is None
    # identity: g_x = mask(out) * g_out + dgrad(g_r1), in place over g_out
    _dgrad(c, n + ".u1.conv", b.u1.conv, n + ".g_r1", n + ".g_x", tuple(b.x.shape),
           accumulate=ident, maskname=n + ".u3.bn.mask" if ident else None)
    if b.ds is not None:
      _bn_bwd(c, n + ".ds.bn", b.ds.bn, n + ".ds.bn", n + ".g_out", n + ".rd", n + ".u3.bn.mask",
              n + ".g_rd", None)
      _wgrad(c, n + ".ds.conv", b.ds.conv, n + ".g_rd", n + ".x")
      _dgrad(c, n + ".ds.conv", b.ds.conv, n + ".g_rd", n + ".g_x", tuple(b.x.shape),
             accumulate=True)
  _stem_bwd(c, net)
  L = c.claims.take("stem.conv", "plan", plan=net.p_stem_wgrad)
  dw0 = c.b("grads:" + net.stem_w["name"], L)
  ref, M = stem_wgrad_ref(c.b("g_stem_raw", L), c.b("xp", L))
  rep.close("stem.conv", "conv wgrad", L, c.a("grads:" + net.stem_w["name"], L), dw0 + ref,
            pc.wgrad_bound(M, dw0.abs(), net.p_stem_wgrad.info()[0]), "dw")
  c.owns(L, "stem.conv", "grads")
  if update:
    _optimizer(c, 1.0 / net.accum.k)


def _stem_bwd(c, net):
  bn = net.stem_bn
  L = c.claims.take("stem.bn", "k", "stem_pool_bn_bwd")
  x = c.b("stem_raw", L)
  N, H, W, C = x.shape
  gsum, gmag, _ = kc.maxpool_bwd_ref(c.b("g_pool", L), c.S.before("pool_idx", L).long(), H, W,
                                     3, 2, 1)
  keep, amb = kc.relu_mask(x, c.b("stem.bn.scale", L), c.b("stem.bn.shift", L))
  g, gm = gsum * keep, gmag * keep
  mean, invstd = c.b("stem.bn.mean", L), c.b("stem.bn.invstd", L)
  xm = x - mean
  gp = pc.gamma_prob(kc.stem_bwd_depth(N, H, W, C))
  dg_ref = (g * xm).reshape(-1, C).sum(0) * invstd
  dg_bnd = gp * (gm * xm.abs()).reshape(-1, C).sum(0) * invstd + \
      (gmag * amb * xm.abs()).reshape(-1, C).sum(0) * invstd
  db_ref = g.reshape(-1, C).sum(0)
  db_bnd = gp * gm.reshape(-1, C).sum(0) + (gmag * amb).reshape(-1, C).sum(0)
  gname, bname = "grads:" + bn.sg["name"], "grads:" + bn.sb["name"]
  # under accumulation this micro-batch's sums go to scratch, and the kernel adds them to the
  # parameter gradient
  tg, tb = ("stem.bn.red_gx", "stem.bn.red_g") if bn.acc is not None else (gname, bname)
  c.rep.close("stem.bn", "bn bwd dgamma/dbeta", L, c.a(tg, L), c.b(tg, L) + dg_ref, dg_bnd,
              "dgamma")
  c.rep.close("stem.bn", "bn bwd dgamma/dbeta", L, c.a(tb, L), c.b(tb, L) + db_ref, db_bnd,
              "dbeta")
  if bn.acc is not None:
    for acc, v in ((gname, tg), (bname, tb)):
      want = (c.S.before(acc, L).float() + c.S.after(v, L).float()).view(torch.int32)
      c.rep.exact("stem.bn", "bn bwd accumulate", L,
                  c.S.after(acc, L).float().contiguous().view(torch.int32) != want, acc + " += v")
  dg, db = f64(c.a(tg, L)), f64(c.a(tb, L))
  ref, bound = pc.bn_bwd_dx_ref(col(g), col(x), c.b("master:" + bn.sg["name"], L), mean, invstd,
                                dg, db, col(amb), col(gmag))
  c.rep.close("stem.bn", "bn bwd dx", L, col(c.a("g_stem_raw", L)), ref, bound, "dx")
  c.owns(L, "stem.bn", "g_stem_raw", "grads", "stats_arena")


def _optimizer(c, gscale=1.0):
  """The fused update from the snapshot before its launch (single rank: one bucket).
  ``gscale``: 1 / k, the mean of the k micro-batches' summed gradients."""
  st = c.net.store
  L = c.claims.take("optimizer", "k", "allreduce_opt")
  decay = torch.zeros(st.total, dtype=torch.bool, device=st.master.device)
  for s in st.order:   # by the network definition: convolution and dense weights decay
    if s["name"].endswith(".w"):
      decay[s["offset"]:s["offset"] + s["numel"]] = True
  w, s1, g = c.b("master", L), c.b("state1", L), c.b("grads", L) * gscale
  s, w1, es, ew = momentum_ref(w, s1, g, decay, c.lr, c.mom, c.wd)
  c.rep.close("optimizer", "optimizer", L, c.a("state1", L), s, es, "momentum")
  c.rep.close("optimizer", "optimizer", L, c.a("master", L), w1, ew, "master")
  m = c.a("master", L)
  c.rep.exact("optimizer", "optimizer", L, f64(c.a("weights", L)) != pc.bf16_rne(f64(m)),
              "bf16 weights")
  tail = st.total - st.decay_end
  c.rep.exact("optimizer", "optimizer", L, c.a("aux32", L)[:tail] != m[st.decay_end:], "aux32")
  c.owns(L, "optimizer", "master", "state1", "weights", "aux32")


# ----------------------------------------------------------------------------- distillation
def teacher_buffers(teacher):
  """(name, tensor) of every buffer of a ResNetTrainer's distillation teacher (models/resnet.py
  _ResNetTeacher), named ``teacher.*`` after its network definition: the folded filters
  (``teacher.wf:<filter>``) and biases (``teacher.bf:<batch norm>``), the head's bf16 weight and
  fp32 bias, its own (never decoded) input buffer and its activations."""
  t = teacher.net
  st = t.store
  out = [("teacher.wf", t.wf), ("teacher.bf", t.bf), ("teacher.weights", st.weights),
         ("teacher.aux32", st.aux32), ("teacher.in_u8", t.in_u8), ("teacher.xp", t.xp)]
  off = 0
  for spec, bn in t._fold_units():
    out.append(("teacher.wf:" + spec["name"], st._view(t.wf, spec)))
    out.append(("teacher.bf:" + bn.name, t.bf[off:off + bn.C]))
    off += (bn.C + 7) // 8 * 8
  out.append(("teacher.weights:" + t.fc.sw["name"], st.w(t.fc.sw)))
  out.append(("teacher.aux32:" + t.fc.sbias["name"], st.f32(t.fc.sbias)))
  for name in ("stem_act", "pool", "pool_idx", "avg", "logits"):
    out.append(("teacher." + name, getattr(t, name)))
  for b in t.blocks:
    for a in ("a1", "a2", "out"):
      out.append(("teacher.{}.{}".format(b.name, a), getattr(b, a)))
  return out


def _folded_conv(c, layer, plan, xname, wname, bname, yname, stride, pad, relu, accumulate=False):
  """One folded convolution of the teacher: y = act(conv(x, w') + b' (+ y before, accumulate))."""
  L = c.claims.take(layer, "plan", plan=plan)
  x, w, bias = c.b(xname, L), c.b(wname, L), c.b(bname, L)
  ref, M = conv_ref(x, w, stride, pad)
  ref, M = ref + bias, M + bias.abs()
  n = w.shape[1] * w.shape[2] * w.shape[3] + 1
  # the accumulate epilogue rounds twice, RN(act(RN(conv + bias) + prev)) (plan_conformance)
  partial, prev = ref, None
  if accumulate:
    prev = c.b(yname, L)
    ref = ref + prev
  if relu:
    ref = ref.clamp_min(0.0)
  bound = pc.elem_bound(ref, M, n, partial=partial if accumulate else None, prev=prev)
  c.rep.close(layer, "teacher conv", L, c.a(yname, L), ref, bound, "y")
  c.owns(L, layer, yname)


def _teacher_forward(c, teacher):
  """The teacher's folded forward pass on the student's decoded ``xp``: stem (bias + ReLU), max
  pool, per block conv1 / conv2 (bias + ReLU), the projection (bias) and conv3 accumulating the
  shortcut (bias + ReLU), the average pool and the head."""
  t = teacher.net
  plans = list(t._f_plans)
  rep = c.rep
  L = c.claims.take("teacher.stem.conv", "plan", plan=plans.pop(0))
  w, bias = c.b("teacher.wf:" + t.stem_w["name"], L), c.b("teacher.bf:" + t.stem_bn.name, L)
  ref, M = stem_ref(c.b("xp", L), w, t.stem_act.shape[2])
  ref, M = (ref + bias).clamp_min(0.0), M + bias.abs()
  rep.close("teacher.stem.conv", "teacher conv", L, c.a("teacher.stem_act", L), ref,
            pc.elem_bound(ref, M, 7 * 64 + 2), "y")
  c.owns(L, "teacher.stem.conv", "teacher.stem_act")
  L = c.claims.take("teacher.maxpool", "k", "maxpool_fwd")
  ry, ridx = kc.maxpool_ref(c.b("teacher.stem_act", L), 3, 2, 1)
  rep.exact("teacher.maxpool", "teacher pool", L, (f64(c.a("teacher.pool", L)) != ry) |
            (c.a("teacher.pool_idx", L).long() != ridx), "pool / idx")
  c.owns(L, "teacher.maxpool", "teacher.pool", "teacher.pool_idx")
  cur = "teacher.pool"
  for b in t.blocks:
    n = "teacher." + b.name
    wf = lambda u: "teacher.wf:" + u.conv.sw["name"]   # noqa: E731
    bf = lambda u: "teacher.bf:" + u.bn.name            # noqa: E731
    _folded_conv(c, n + ".u1.conv", plans.pop(0), cur, wf(b.u1), bf(b.u1), n + ".a1", 1, 0, True)
    _folded_conv(c, n + ".u2.conv", plans.pop(0), n + ".a1", wf(b.u2), bf(b.u2), n + ".a2",
                 b.stride, 1, True)
    if b.ds is not None:
      _folded_conv(c, n + ".ds.conv", plans.pop(0), cur, wf(b.ds), bf(b.ds), n + ".out", b.stride,
                   0, False)
      cur = n + ".out"
    # identity blocks accumulate in place into the block input
    _folded_conv(c, n + ".u3.conv", plans.pop(0), n + ".a2", wf(b.u3), bf(b.u3), cur, 1, 0, True,
                 accumulate=True)
  assert not plans, "teacher plans left unclaimed"
  L = c.claims.take("teacher.avgpool", "k", "avgpool_fwd")
  ref, mag = kc.avgpool_ref(c.b(cur, L))
  HW = math.prod(t._f_last.shape[1:3])
  rep.close("teacher.avgpool", "teacher pool", L, c.a("teacher.avg", L), ref,
            pc.U_BF16 * ref.abs() + (1 + pc.U_BF16) * pc.gamma(HW + 3, U) * mag, "avg")
  c.owns(L, "teacher.avgpool", "teacher.avg")
  fc = t.fc
  L = c.claims.take("teacher.fc", "plan", plan=fc.fwd)
  a = c.b("teacher.avg", L)
  w = c.b("teacher.weights:" + fc.sw["name"], L)
  bias = c.b("teacher.aux32:" + fc.sbias["name"], L)
  ref = a @ w.t() + bias
  M = a.abs() @ w.abs().t() + bias.abs()
  rep.close("teacher.fc", "teacher head", L, c.a("teacher.logits", L), ref,
            pc.elem_bound(ref, M, fc.cin + 1, U), "logits")
  c.owns(L, "teacher.fc", "teacher.logits")


def distill_ref(s, z, labels, V, eps, alpha, T, scale):
  """(summed loss, dlogits [B, V]) of the distillation loss without a mix, float64:
  (1 - alpha) CE(s, smoothed one-hot) + alpha T^2 KL(softmax(z / T) || softmax(s / T))."""
  s, z = s[:, :V], z[:, :V]
  t = F.one_hot(labels.long(), V).to(s.dtype) * (1.0 - eps) + eps / V
  ls, lsT, lq = torch.log_softmax(s, 1), torch.log_softmax(s / T, 1), torch.log_softmax(z / T, 1)
  q = lq.exp()
  loss = ((1 - alpha) * -(t * ls).sum(1) + alpha * T * T * (q * (lq - lsT)).sum(1)).sum() * scale
  d = ((1 - alpha) * (ls.exp() - t) + alpha * T * (lsT.exp() - q)) * scale
  return loss, d


def _distill_loss(c, net):
  """distill_xent on the student's logits and the teacher's, as the two layers left them."""
  rep = c.rep
  V, B = net.num_classes, net.B
  L = c.claims.take("loss", "k", "distill_xent")
  if net.mix is not None:
    rep.fail(L, "loss", "the step check covers distillation without Mixup / CutMix")
    return
  T, alpha = net.distill_temperature, net.distill_alpha
  s, z = c.b("logits", L), c.b("teacher.logits", L)
  loss, dl = distill_ref(s, z, c.S.before("labels", L), V, net.label_smoothing, alpha, T, 1.0 / B)
  rep.close("loss", "distill loss", L, c.a("loss_sum", L).reshape(()), loss,
            4e-5 * abs(float(loss)) + 1e-6, "loss_sum")
  got = c.a("dlogits", L)
  rep.close("loss", "distill loss", L, got[:, :V], dl,
            pc.U_BF16 * dl.abs() + 1e-5 * (1 + T) / B, "dlogits")
  if net.VP > V:
    rep.exact("loss", "distill loss", L, got[:, V:] != 0, "dlogits padding")
  _, _, hits, tie = xent_ref(s, c.S.before("labels", L), V, 1.0 / B)
  nh = float(c.a("correct", L))
  if not int(hits[~tie].sum()) <= nh <= int(hits[~tie].sum()) + int(tie.sum()):
    rep.fail(L, "loss", "correct {} against {} top-1 hits".format(nh, int(hits.sum())))
  c.owns(L, "loss", "dlogits", "loss_sum", "correct")

"""Explicit-graph training engine on the native kernels.

There is no autograd and no tracing compiler here: a model is a list of layer
objects with static device buffers, ``forward()``/``backward()`` enqueue native
kernels on the current CUDA stream in a fixed order, and the whole step can be
captured once into a CUDA graph.  Parameters live in three flat buffers
(fp32 master, bf16 compute copy, fp32 gradients) so that the data-parallel
all-reduce and the optimizer are one fused kernel over contiguous ranges
(parallel/fused_optim.py).

This is the Hopper-native stand-in for what the reference delegates to Keras /
tf.distribute in its example programs (e.g. examples/mnist/keras/mnist_spark.py:
11-66, examples/resnet/resnet_cifar_dist.py:196-257).
"""
import math
import numbers

import numpy as np
import torch

from .. import ops
from ..ops import igemm


def _pad8(n):
  return (n + 7) // 8 * 8


class ParamStore(object):
  """Flat parameter storage.  Decayed parameters (conv / dense weights) come first,
  then the non-decayed ones (batch-norm scale/offset, biases)."""

  def __init__(self):
    self._specs = []  # (name, shape, decay, init_fn)
    self.finalized = False

  def register(self, name, shape, decay, init):
    assert not self.finalized
    spec = {"name": name, "shape": tuple(shape), "decay": bool(decay), "init": init}
    self._specs.append(spec)
    return spec

  def finalize(self, device, alloc=None, seed=1234, grads=True):
    """alloc(nbytes_name, numel, dtype) -> tensor lets the caller place the buffers in
    symmetric (peer-mapped) memory; default is ordinary device memory.  ``grads=False`` (an
    inference-only model) allocates no gradient buffer: ``g()`` then returns None."""
    order = [s for s in self._specs if s["decay"]] + [s for s in self._specs if not s["decay"]]
    off = 0
    for s in order:
      s["offset"] = off
      s["numel"] = int(math.prod(s["shape"]))
      off += _pad8(s["numel"])
    self.decay_end = sum(_pad8(s["numel"]) for s in order if s["decay"])
    self.total = _pad8(off)
    self.order = order
    if alloc is None:
      alloc = lambda name, n, dt: torch.zeros(n, dtype=dt, device=device)  # noqa: E731
    self.master = alloc("master", self.total, torch.float32)  # symmetric too: broadcastable
    self.weights = alloc("weights", self.total, torch.bfloat16)
    self.grads = alloc("grads", self.total, torch.float32) if grads else None
    # fp32 replica of the non-decayed tail (BN scale/offset are consumed in fp32)
    self.aux32 = alloc("aux32", max(8, self.total - self.decay_end), torch.float32)
    gen = torch.Generator(device="cpu")
    gen.manual_seed(seed)
    for s in order:
      v = s["init"](s["shape"], gen).to(torch.float32).reshape(-1)
      self.master[s["offset"]:s["offset"] + s["numel"]].copy_(v)
    self.weights.copy_(self.master)
    self.aux32[:self.total - self.decay_end].copy_(self.master[self.decay_end:])
    self.finalized = True
    self.by_name = {s["name"]: s for s in order}

  def _view(self, buf, s, base=0):
    return buf[s["offset"] - base:s["offset"] - base + s["numel"]].view(s["shape"])

  def w(self, s):
    return self._view(self.weights, s)

  def g(self, s):
    return None if self.grads is None else self._view(self.grads, s)

  def m(self, s):
    return self._view(self.master, s)

  def f32(self, s):
    """fp32 value of a non-decayed parameter as seen by every rank."""
    assert not s["decay"]
    return self._view(self.aux32, s, self.decay_end)

  def state_dict(self):
    # with world > 1 the fused all-reduce + optimizer kernel keeps the fp32 master current only
    # for this rank's own shard of every bucket: FusedOptimizer registers assemble(), which pulls
    # the peers' shards over NVLink before anything is saved or exported
    assemble = getattr(self, "_assemble", None)
    if assemble is not None:
      assemble()
    return {s["name"]: self.m(s).detach().cpu().clone() for s in self.order}

  def load_state_dict(self, sd):
    for s in self.order:
      if s["name"] in sd:
        self.m(s).copy_(sd[s["name"]].to(self.master.device, torch.float32).view(s["shape"]))
    self.weights.copy_(self.master)
    self.aux32[:self.total - self.decay_end].copy_(self.master[self.decay_end:])


class AveragedModel(object):
  """Exportable snapshot of a trainer's weight average (``trainer.averaged()``): ``state_dict()``
  is in the trainer's own format with every parameter replaced by its average, and the trainer's
  export attributes come along, so ``checkpoint.export_model(view, dir)`` writes an artefact the
  trainer's serving class loads and ``load_state_dict`` accepts."""

  def __init__(self, state, trainer):
    self._state = state
    # (the CIFAR trainer has no serving class: like the trainer, its view exports bare state)
    self.export_builder = getattr(trainer, "export_builder", None)
    self.export_builder_args = dict(getattr(trainer, "export_builder_args", {}))
    self.export_signatures = getattr(trainer, "export_signatures", None)

  def state_dict(self):
    return dict(self._state)


def averaged_params(store, optim):
  """({name: fp32 host tensor}, fp32 device vector) of the store's parameters taken from
  ``optim``'s complete weight average (the current parameters before the first update after a
  reset).  RuntimeError when there is no average."""
  if optim is None or getattr(optim, "ema", None) is None:
    raise RuntimeError("this trainer keeps no weight average: build it with ema_decay=d")
  avg = optim.average_master()
  return {s["name"]: store._view(avg, s).detach().cpu().clone() for s in store.order}, avg


def check_ema_decay(d, training=True):
  """Validated ``ema_decay`` of a trainer: None, or a float in [0, 1) (ValueError otherwise, and
  for any value with ``training=False``: an inference-only trainer has no optimizer)."""
  from ..parallel.fused_optim import check_ema_decay as check
  d = check(d)
  if d is not None and not training:
    raise ValueError("ema_decay needs training=True (an inference-only trainer has no optimizer)")
  return d


def check_clip_norm(c, training=True):
  """Validated ``clip_norm`` of a trainer: None, or a float > 0, inf allowed (ValueError
  otherwise, and for any value with ``training=False``: an inference-only trainer has no
  optimizer)."""
  from ..parallel.fused_optim import check_clip_norm as check
  c = check(c)
  if c is not None and not training:
    raise ValueError("clip_norm needs training=True (an inference-only trainer has no optimizer)")
  return c


def check_adam_args(beta1, beta2, epsilon):
  """Validated ``(beta1, beta2, epsilon)`` of a trainer (fused_optim.check_adam_args: ValueError
  before anything is allocated)."""
  from ..parallel.fused_optim import check_adam_args as check
  return check(beta1, beta2, epsilon)


def check_gradient_accumulation_steps(k, training=True):
  """Validated ``gradient_accumulation_steps`` of a trainer: an int k >= 1 (ValueError for bools,
  other types and k < 1, and for k != 1 with ``training=False``: an inference-only trainer takes
  no gradients)."""
  if isinstance(k, bool) or not isinstance(k, numbers.Integral):
    raise ValueError("gradient_accumulation_steps must be an int >= 1, not {!r}".format(k))
  if k < 1:
    raise ValueError("gradient_accumulation_steps must be >= 1, got {}".format(k))
  if k != 1 and not training:
    raise ValueError("gradient_accumulation_steps needs training=True (an inference-only trainer "
                     "takes no gradients)")
  return int(k)


def check_mix_args(mixup_alpha=0.0, cutmix_alpha=0.0, mix_prob=1.0, mix_switch_prob=0.5,
                   training=True):
  """Validated ``(mixup_alpha, cutmix_alpha, mix_prob, mix_switch_prob)`` of a trainer as floats:
  the alphas finite and >= 0, the probabilities in [0, 1] (ValueError otherwise, and for any value
  other than the default with ``training=False``: an inference-only trainer has no training
  batch to mix)."""
  vals = {}
  for name, v, lo, hi in (("mixup_alpha", mixup_alpha, 0.0, math.inf),
                          ("cutmix_alpha", cutmix_alpha, 0.0, math.inf),
                          ("mix_prob", mix_prob, 0.0, 1.0),
                          ("mix_switch_prob", mix_switch_prob, 0.0, 1.0)):
    if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(float(v)) \
        or not lo <= float(v) <= hi:
      rng = "finite and >= 0" if hi == math.inf else "in [0, 1]"
      raise ValueError("{} must be a real number {}, got {!r}".format(name, rng, v))
    vals[name] = float(v)
  if not training and (vals["mixup_alpha"] or vals["cutmix_alpha"] or vals["mix_prob"] != 1.0 or
                       vals["mix_switch_prob"] != 0.5):
    raise ValueError("mixup_alpha, cutmix_alpha, mix_prob and mix_switch_prob need training=True "
                     "(an inference-only trainer has no training batch to mix)")
  return (vals["mixup_alpha"], vals["cutmix_alpha"], vals["mix_prob"], vals["mix_switch_prob"])


MIX_MODES = ("none", "mixup", "cutmix")   # index = the mode code of the staged vector (kMix*)
MIX_SLOTS = 8                             # csrc/ops.h kMixSlots


class MixDraws(object):
  """The per-step Mixup / CutMix draw of a trainer: timm's ``Mixup`` in "batch" mode with
  ``correct_lam=True``, from a ``numpy.random.Generator`` seeded with ``(seed, rank)``.

  ``draw(H, W)`` returns ``(mode, lam, box)``: with probability ``1 - mix_prob`` the step does not
  mix (``("none", 1.0, (0, 0, 0, 0))``); otherwise the mode is cutmix with probability
  ``mix_switch_prob`` when both alphas are > 0 (else the one whose alpha is > 0) and
  lam ~ Beta(alpha, alpha) of that mode.  A CutMix box ``(y0, y1, x0, x1)`` (rows [y0, y1), columns
  [x0, x1) of the H x W image) is centred on a uniform pixel with sides int(H r), int(W r),
  r = sqrt(1 - lam), clipped to the image, and lam becomes 1 - box area / (H W)."""

  def __init__(self, mixup_alpha, cutmix_alpha, mix_prob=1.0, mix_switch_prob=0.5, seed=0, rank=0):
    self.mixup_alpha, self.cutmix_alpha = float(mixup_alpha), float(cutmix_alpha)
    self.mix_prob, self.mix_switch_prob = float(mix_prob), float(mix_switch_prob)
    self.rng = np.random.default_rng([int(seed), int(rank)])

  def draw(self, H, W):
    rng = self.rng
    if not rng.random() < self.mix_prob:
      return "none", 1.0, (0, 0, 0, 0)
    if self.mixup_alpha > 0 and self.cutmix_alpha > 0:
      cut = bool(rng.random() < self.mix_switch_prob)
    else:
      cut = self.cutmix_alpha > 0
    a = self.cutmix_alpha if cut else self.mixup_alpha
    lam = float(rng.beta(a, a))
    if not cut:
      return "mixup", lam, (0, 0, 0, 0)
    r = math.sqrt(1.0 - lam)
    ch, cw = int(H * r), int(W * r)
    cy, cx = int(rng.integers(0, H)), int(rng.integers(0, W))
    y0, y1 = min(max(cy - ch // 2, 0), H), min(max(cy + ch // 2, 0), H)
    x0, x1 = min(max(cx - cw // 2, 0), W), min(max(cx + cw // 2, 0), W)
    return "cutmix", 1.0 - (y1 - y0) * (x1 - x0) / float(H * W), (y0, y1, x0, x1)

  @staticmethod
  def vector(draw):
    """The draw as the kernels read it: [mode, lam, y0, y1, x0, x1, 0, 0] (fp32 on the device)."""
    mode, lam, box = draw
    return [float(MIX_MODES.index(mode)), float(lam)] + [float(v) for v in box] + [0.0, 0.0]


def check_drop_path_rate(r=0.0, training=True):
  """Validated ``drop_path_rate`` of a trainer as a float: a real, finite r with 0 <= r < 1
  (ValueError otherwise, for bools, and for r != 0 with ``training=False``: an inference-only
  trainer never drops)."""
  if isinstance(r, bool) or not isinstance(r, numbers.Real) or not math.isfinite(float(r)) \
      or not 0.0 <= float(r) < 1.0:
    raise ValueError("drop_path_rate must be a real number in [0, 1), got {!r}".format(r))
  if float(r) and not training:
    raise ValueError("drop_path_rate needs training=True (an inference-only trainer never drops)")
  return float(r)


def check_distill_args(teacher=None, teacher_depth=None, distill_alpha=0.5,
                       distill_temperature=1.0, training=True, multi_label=False):
  """Validated ``(teacher_depth, distill_alpha, distill_temperature)`` of a trainer, the last two
  as floats: ``teacher`` None or a mapping (a ``state_dict()``), ``teacher_depth`` None or an int,
  alpha a real in (0, 1], T a finite real > 0.  ValueError otherwise, for a non-default alpha, T or
  ``teacher_depth`` without a teacher, for any of the four with ``training=False`` (an
  inference-only trainer has no loss to distil into) and for a teacher with ``multi_label``
  (distillation is of softmax classifiers).  The teacher's tensors are checked by the trainer."""
  a, t = distill_alpha, distill_temperature
  if isinstance(a, bool) or not isinstance(a, numbers.Real) or not 0.0 < float(a) <= 1.0:
    raise ValueError("distill_alpha must be a real number in (0, 1], got {!r}".format(a))
  # the kernels take T in fp32: it must stay finite and nonzero there (1 / T finite too)
  ok = not isinstance(t, bool) and isinstance(t, numbers.Real) and math.isfinite(float(t)) \
      and float(t) > 0.0
  if ok:
    with np.errstate(over="ignore"):
      t32 = np.float32(t)
    ok = bool(np.isfinite(t32)) and t32 >= np.finfo(np.float32).tiny
  if not ok:
    raise ValueError("distill_temperature must be a finite real number > 0 that fp32 holds "
                     "(>= {:.3g}), got {!r}".format(float(np.finfo(np.float32).tiny), t))
  if teacher_depth is not None and (isinstance(teacher_depth, bool) or
                                    not isinstance(teacher_depth, numbers.Integral)):
    raise ValueError("teacher_depth must be an int, got {!r}".format(teacher_depth))
  given = teacher is not None or teacher_depth is not None or float(a) != 0.5 or float(t) != 1.0
  if given and not training:
    raise ValueError("teacher, teacher_depth, distill_alpha and distill_temperature need "
                     "training=True (an inference-only trainer has no loss to distil into)")
  if teacher is None:
    if given:
      raise ValueError("teacher_depth, distill_alpha and distill_temperature configure "
                       "distillation: they need a teacher")
  else:
    if not hasattr(teacher, "keys") or not hasattr(teacher, "__getitem__"):
      raise ValueError("teacher must be a state_dict() (a mapping of tensors), got {}".format(
          type(teacher).__name__))
    if multi_label:
      raise ValueError("a teacher distils a softmax classifier: not with multi_label=True")
  return (None if teacher_depth is None else int(teacher_depth)), float(a), float(t)


def drop_path_rates(r, n_blocks):
  """timm's linear decay of the stochastic-depth rate over the residual blocks of a network:
  block i of N (0-based) drops with p_i = r * i / (N - 1), so block 0 never drops and the last one
  drops at r.  (Huang et al. use p_l = r * l / L with l from 1, which drops the first block too.)"""
  if n_blocks < 2:
    return (0.0,) * n_blocks
  return tuple(r * i / (n_blocks - 1) for i in range(n_blocks))


class DropPathDraws(object):
  """The per-step stochastic-depth draw of a trainer (timm's ``DropPath(scale_by_keep=True)``),
  from its own ``numpy.random.Generator`` seeded with ``(seed, rank, 1)``: a stream apart from
  MixDraws' ``(seed, rank)``, so that turning drop path on leaves a mixing trainer's mix draws as
  they were.

  ``draw()`` returns float32 [n_blocks, B]: row i holds each sample's factor s_b for block i,
  ``keep_b / (1 - p_i)`` with keep_b ~ Bernoulli(1 - p_i) (0, or 1 / (1 - p_i) rounded to fp32).
  Rows of blocks with p_i = 0 are all ones and draw nothing."""

  def __init__(self, rates, B, seed=0, rank=0):
    self.rates, self.B = tuple(float(p) for p in rates), int(B)
    self.rng = np.random.default_rng([int(seed), int(rank), 1])

  def draw(self):
    out = np.ones((len(self.rates), self.B), dtype=np.float32)
    for i, p in enumerate(self.rates):
      if p > 0:
        keep = self.rng.random(self.B) < 1.0 - p
        out[i] = np.where(keep, np.float32(1.0 / (1.0 - p)), np.float32(0.0))
    return out


class GradAccumulation(object):
  """The update window of a trainer with ``gradient_accumulation_steps`` k (Keras's
  ``gradient_accumulation_steps``): ``train_step`` call i of a window is micro-step
  ``micro_step = i`` (0 .. k-1).  Micro-step 0 zeroes the fp32 gradients, every micro-step's
  backward adds into them, and only micro-step k-1 runs the fused all-reduce + update, with the
  optimizer's gradient scale ``hyper[3] = 1 / (world k)``: the update sees the mean of the k
  micro-batches' gradients over all ranks.  With k = 1 every step is both first and last, which is
  the step the trainers always ran."""

  def __init__(self, k):
    self.k = k
    self.micro_step = 0

  def phase(self, micro_step=None):
    """(zero the gradients first, run the all-reduce + update last) of a micro-step."""
    i = self.micro_step if micro_step is None else micro_step
    return i == 0, i == self.k - 1

  def advance(self):
    self.micro_step = (self.micro_step + 1) % self.k

  def restart(self, optim):
    """Start a new window: the partial sums are dropped (``optim`` zeroes the gradients), the next
    call is micro-step 0.  No-op with k = 1, whose every step zeroes the gradients itself."""
    if self.k > 1:
      self.micro_step = 0
      optim.zero_grads()

  def capture(self, device, step_kernels, mode, before_step=None):
    """CUDA graphs of the micro-steps, one per distinct phase ({phase: graph}): warm-up runs
    max(2, k) micro-steps eagerly on a side stream (two steps with k = 1, as before accumulation;
    with k > 1 every position of the window once), then each phase is captured.
    ``before_step``: called on the side stream before each warm-up step, as ``train_step`` does
    before a step (the Mixup / CutMix and drop-path draws and their staging); never inside a
    capture."""
    s = torch.cuda.Stream(device=device)
    s.wait_stream(torch.cuda.current_stream(device))
    with torch.cuda.stream(s):
      for _ in range(max(2, self.k)):
        if before_step is not None:
          before_step()
        step_kernels()
        self.advance()
    torch.cuda.current_stream(device).wait_stream(s)
    torch.cuda.synchronize(device)
    graphs, at = {}, self.micro_step
    for i in range(self.k):
      ph = self.phase(i)
      if ph in graphs:
        continue
      self.micro_step = i
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g, capture_error_mode=mode):
        step_kernels()
      graphs[ph] = g
    self.micro_step = at
    return graphs

  def run(self, graphs, step_kernels, optim):
    """One ``train_step``: replay this micro-step's graph (``optim.after_replay()`` after the
    final one: a cross-host communicator's all-reduce + update run outside the graph) or run it
    eagerly."""
    ph = self.phase()
    if graphs:
      graphs[ph].replay()
      if ph[1]:
        optim.after_replay()
    else:
      step_kernels()
    self.advance()


def he_normal(fan_in):
  std = math.sqrt(2.0 / fan_in)
  return lambda shape, gen: torch.randn(shape, generator=gen) * std


def constant(v):
  return lambda shape, gen: torch.full(shape, float(v))


def normal(std):
  return lambda shape, gen: torch.randn(shape, generator=gen) * std


def _run_wgrad(layer):
  """wgrad (+ bias gradient) of a Conv / Dense layer."""
  layer.wgrad.run()
  if layer.sbias is not None:
    ops.K.colsum(layer.dy, layer.store.g(layer.sbias))


class StatsArena(object):
  """One flat fp32 buffer holding the (sum, sumsq) accumulators of every batch norm of a trainer:
  a single memset per step replaces a clearing pass per layer."""

  def __init__(self, device, capacity=1 << 17):
    self.buf = torch.zeros(capacity, dtype=torch.float32, device=device)
    self.used = 0

  def take(self, n):
    n8 = (n + 7) // 8 * 8
    if self.used + n8 > self.buf.numel():
      raise RuntimeError("StatsArena capacity exceeded")
    out = self.buf[self.used:self.used + n]
    self.used += n8
    return out

  def zero(self):
    self.buf[:self.used].zero_()
    ops.count()


class RunningArena(object):
  """The running mean / variance of every batch norm of a trainer in ONE flat fp32 buffer
  ([mean_0 | var_0 | mean_1 | var_1 ...], each padded to 8 elements): the non-trainable model
  state is then a single tensor that checkpoints save, exports serve and the parameter server
  hosts as the tail of its vector (parallel/ps.py)."""

  def __init__(self, device, capacity=1 << 17):
    self.buf = torch.zeros(capacity, dtype=torch.float32, device=device)
    self.used = 0

  def take(self, C):
    C8 = (C + 7) // 8 * 8
    if self.used + 2 * C8 > self.buf.numel():
      raise RuntimeError("RunningArena capacity exceeded")
    mean = self.buf[self.used:self.used + C]
    var = self.buf[self.used + C8:self.used + C8 + C]
    var.fill_(1.0)
    self.used += 2 * C8
    return mean, var

  def tensor(self):
    return self.buf[:self.used]


class BatchNorm(object):
  """Training-mode batch norm over NHWC bf16 with statistics fused into the producer conv."""

  def __init__(self, store, name, C, eps=1e-5, momentum=0.1, zero_gamma=False):
    self.C, self.eps, self.momentum, self.name = C, eps, momentum, name
    self.sg = store.register(name + ".gamma", (C,), False, constant(0.0 if zero_gamma else 1.0))
    self.sb = store.register(name + ".beta", (C,), False, constant(0.0))
    self.store = store

  def build(self, device, arena=None, running=None):
    """``arena`` (StatsArena): take the (sum, sumsq) accumulators from a per-trainer arena that
    the trainer zeroes once per step; the statistics are then finalised inside the apply kernel
    (one launch less per batch norm and no clearing pass).  ``running`` (RunningArena): place
    the running statistics in the trainer's flat non-trainable-state buffer."""
    z = lambda: torch.zeros(self.C, dtype=torch.float32, device=device)  # noqa: E731
    self.arena = arena
    if arena is not None:
      self.sum, self.sumsq = arena.take(self.C), arena.take(self.C)
    else:
      self.sum, self.sumsq = z(), z()
    self.mean, self.invstd, self.scale, self.shift = z(), z(), z(), z()
    # accumulators of the backward reduction when it is fused into the epilogue of the data
    # gradient that produces this unit's dy (enable_fused_reduce): zeroed with the same memset
    self.red_g = self.red_gx = None
    self.fused_reduce = False
    if arena is not None:
      self.red_g, self.red_gx = arena.take(self.C), arena.take(self.C)
    if running is not None:
      self.running_mean, self.running_var = running.take(self.C)
    else:
      self.running_mean = z()
      self.running_var = torch.ones(self.C, dtype=torch.float32, device=device)
    self.gamma, self.beta = self.store.f32(self.sg), self.store.f32(self.sb)
    self.dgamma, self.dbeta = self.store.g(self.sg), self.store.g(self.sb)
    self.acc = None

  def accumulate_grads(self, scratch):
    """Gradient accumulation: from now on the backward ADDS this micro-batch's dgamma / dbeta to
    the parameter gradient.  The apply kernel forms dx from this micro-batch's values, so they are
    kept apart: in ``red_gx`` / ``red_g`` (arena slots zeroed every step, unused when the
    reduction is not fused) or in 2C floats of ``scratch``, a StatsArena the trainer zeroes every
    step.  A fused reduction needs no scratch: the apply kernel finishes the sums in registers.
    Call after the convolutions are built (``fused_reduce`` is final then)."""
    if self.fused_reduce:
      self.acc = (self.dgamma, self.dbeta)   # not read: the apply kernel works from red_g / red_gx
    elif self.red_g is not None:
      self.acc = (self.red_gx, self.red_g)
    else:
      self.acc = (scratch.take(self.C), scratch.take(self.C))

  @property
  def stats(self):
    return (self.sum, self.sumsq)

  def forward(self, x_raw, y, residual=None, act=1, training=True, rev=False, sample_scale=None):
    """``rev``: walk the rows last-to-first.  The convolution that produced ``x_raw`` wrote its
    tiles first-to-last, so the END of the tensor is what the 50 MB L2 still holds; the apply
    kernel then finishes at the START of ``y``, which is where the next convolution begins.
    ``sample_scale`` (stochastic depth; fp32 [N] on the device): y = act(s[n] bn(x) (+ residual)),
    with the batch and running statistics of bn(x) over the whole batch."""
    ss = {} if sample_scale is None else {"sample_scale": sample_scale}
    count = x_raw.numel() // self.C
    ops.C().bn_set_row_reverse(bool(rev))
    # a residual unit's ReLU mask depends on the sum, not on x alone: keep it as one bit per
    # element so that the backward pass does not have to re-read the whole bf16 output
    # (the buffer is never released: a captured CUDA graph may hold its address)
    if training and act == 1 and (residual is not None or getattr(self, "fused_reduce", False)):
      # (a unit whose backward reduction is fused into a dgrad epilogue always keeps the bits:
      # the epilogue and the apply kernel then read 1/16 of a byte per element for the mask)
      self.mask = self.ensure_mask(x_raw.numel(), x_raw.device)
    else:
      self.mask = None
    if training and getattr(self, "arena", None) is not None:
      ops.K.bn_apply_finalize(x_raw, residual, y, act, self.mask, self.sum, self.sumsq, self.gamma,
                              self.beta, self.running_mean, self.running_var, self.mean,
                              self.invstd, self.scale, self.shift, float(count), self.eps,
                              self.momentum, **ss)
      return
    if training:
      ops.K.bn_finalize(self.sum, self.sumsq, self.gamma, self.beta, self.running_mean,
                        self.running_var, self.mean, self.invstd, self.scale, self.shift,
                        float(count), self.eps, self.momentum)
    else:
      ops.K.bn_inference_coeffs(self.gamma, self.beta, self.running_mean, self.running_var,
                                self.scale, self.shift, self.eps)
    ops.K.bn_apply(x_raw, residual, self.scale, self.shift, y, act, self.mask, **ss)

  def ensure_mask(self, numel, device):
    """The unit's ReLU bit mask buffer (numel / 8 bytes), allocated once."""
    buf = getattr(self, "_mask_buf", None)
    if buf is None or buf.numel() * 8 != numel:
      buf = self._mask_buf = torch.empty(numel // 8, dtype=torch.uint8, device=device)
    return buf

  def backward(self, dy, x_raw, y, dx, dres=None, relu=True, residual=False, mask=None,
               rev=(False, False), sample_scale=None):
    """relu mask: recomputed from x_raw with the forward scale/shift when the unit has no
    residual input (saves reading y: 2 of 6-8 bytes per element); from the stored y otherwise;
    ``mask``: another unit's bit mask (a projection shortcut's BN sees the gradient of the block
    output, i.e. the ReLU that followed the *sum*).  ``sample_scale``: the forward's stochastic-depth
    factors; the batch norm's output gradient is then s[n] * the masked dy (``dres`` still gets
    the unscaled one), and the reduction runs as its own pass - it cannot be fused into a data
    gradient's epilogue."""
    ss = {} if sample_scale is None else {"sample_scale": sample_scale}
    mode = 0 if not relu else (1 if (residual or dres is not None) else 2)
    ysrc = y if mode == 1 else None
    if mask is not None and relu:
      mode, ysrc = 3, mask
    elif relu and getattr(self, "mask", None) is not None:
      mode, ysrc = 3, self.mask   # bit mask written by forward(): 1/16 of y's bytes
    # accumulation (accumulate_grads): dgamma / dbeta of this micro-batch go to scratch, the
    # apply kernel adds them to the parameter gradient
    dg, db = self.acc if self.acc is not None else (self.dgamma, self.dbeta)
    acc = {} if self.acc is None else {"acc_dgamma": self.dgamma, "acc_dbeta": self.dbeta}
    if getattr(self, "fused_reduce", False):
      if ss:
        raise ValueError("{}: sample_scale needs the unfused backward reduction (build the data "
                         "gradient that writes dy without dx_bn_reduce)".format(self.name))
      # sum(g), sum(g x) were accumulated by the epilogue of the data gradient that wrote dy
      # (ops/igemm.conv_dgrad(bn_reduce=...)): no reduction pass, the apply kernel finishes them
      ops.C().bn_set_row_reverse(bool(rev[1]))
      ops.K.bn_bwd_apply(dy, x_raw, ysrc, self.gamma, self.mean, self.invstd, dg, db, dx, dres,
                         mode, self.scale, self.shift, self.red_g, self.red_gx, **acc)
      ops.C().bn_set_row_reverse(False)
      return
    # rev = (reduce, apply) row order: each kernel starts at the end where the previous one
    # stopped, so that what it reads first is still in L2 (ResNetTrainer assigns the directions)
    ops.C().bn_set_row_reverse(bool(rev[0]))
    ops.K.bn_bwd_reduce(dy, x_raw, ysrc, self.mean, self.invstd, dg, db, mode, self.scale,
                        self.shift, **ss)
    ops.C().bn_set_row_reverse(bool(rev[1]))
    ops.K.bn_bwd_apply(dy, x_raw, ysrc, self.gamma, self.mean, self.invstd, dg, db, dx, dres,
                       mode, self.scale, self.shift, **acc, **ss)
    ops.C().bn_set_row_reverse(False)


class Conv(object):
  """Convolution parameters + its three igemm plans (fprop / dgrad / wgrad)."""

  def __init__(self, store, name, cin, cout, k, stride=1, pad=None, bias=False):
    self.cin, self.cout, self.k, self.stride = cin, cout, k, stride
    self.pad = (k // 2) if pad is None else pad
    self.name = name
    self.store = store
    self.sw = store.register(name + ".w", (cout, k, k, cin), True, he_normal(k * k * cin))
    self.sbias = store.register(name + ".b", (cout,), False, constant(0.0)) if bias else None

  def out_hw(self, H, W):
    return ((H + 2 * self.pad - self.k) // self.stride + 1,
            (W + 2 * self.pad - self.k) // self.stride + 1)

  def build(self, x, y, dy=None, dx=None, stats=None, relu=False, dx_accumulate=False,
            need_dgrad=True, training=True, dx_acc_mask=None, dx_bn_reduce=None):
    """``dx_bn_reduce``: the BatchNorm whose dy this layer's data gradient produces (its input
    has the shape of ``dx``): fuse that batch norm's backward reduction into the dgrad epilogue
    when the plan allows it (every pixel of dx written by this launch)."""
    st = self.store
    self.x, self.y = x, y
    if not training:
      stats = None  # inference: running statistics are used, nothing to accumulate
    bias = st.f32(self.sbias) if self.sbias is not None else None
    self.fwd = igemm.conv_fprop(x, st.w(self.sw), y, self.stride, self.pad, bias=bias, relu=relu,
                                stats=stats)
    self._fwd_args = (x, y, bias, relu, stats)
    self.fwd_remote = None
    self.wgrad = self.dgrad = None
    if training and dy is not None:
      self.wgrad = igemm.conv_wgrad(dy, x, st.g(self.sw), self.stride, self.pad)
      if need_dgrad and dx is not None:
        red = None
        if dx_bn_reduce is not None and dx_bn_reduce[0].red_g is not None:
          bn_below, x_below, mask_below = dx_bn_reduce
          red = (x_below, mask_below, bn_below.red_g, bn_below.red_gx)
        try:
          self.dgrad = igemm.conv_dgrad(dy, st.w(self.sw), dx, self.stride, self.pad,
                                        accumulate=dx_accumulate, acc_mask=dx_acc_mask,
                                        bn_reduce=red)
          if red is not None:
            dx_bn_reduce[0].fused_reduce = True
        except (ValueError, RuntimeError) as e:
          if red is None:
            raise
          # (a strided 1x1 does not write every pixel, odd channel counts leave ragged tiles)
          self.dgrad = igemm.conv_dgrad(dy, st.w(self.sw), dx, self.stride, self.pad,
                                        accumulate=dx_accumulate, acc_mask=dx_acc_mask)
    self.dy = dy

  def forward(self):
    self.fwd.run()

  def bind_remote_weights(self, flat_weights):
    """Second forward plan whose B operand (the filter) is fetched by TMA from ``flat_weights`` -
    a peer-mapped view of ANOTHER rank's bf16 weight buffer - instead of local memory: the
    startup broadcast fused with the first convolution that consumes the weights."""
    x, y, bias, relu, stats = self._fwd_args
    w = self.store._view(flat_weights, self.sw)
    self.fwd_remote = igemm.conv_fprop(x, w, y, self.stride, self.pad, bias=bias, relu=relu,
                                       stats=stats)

  def forward_remote(self):
    self.fwd_remote.run()

  def backward(self):
    _run_wgrad(self)
    if self.dgrad is not None:
      self.dgrad.run()


class Dense(object):
  """Fully connected layer on [B, K] activations (GEMM + bias (+ReLU) epilogue)."""

  def __init__(self, store, name, cin, cout, bias=True, init=None):
    self.cin, self.cout, self.name, self.store = cin, cout, name, store
    self.sw = store.register(name + ".w", (cout, cin), True, init or he_normal(cin))
    self.sbias = store.register(name + ".b", (cout,), False, constant(0.0)) if bias else None

  def build(self, x, y, dy=None, dx=None, relu=False, training=True):
    st = self.store
    bias = st.f32(self.sbias) if self.sbias is not None else None
    self.fwd = igemm.gemm(x, st.w(self.sw), y, "nk", bias=bias, relu=relu)
    self._fwd_args = (x, y, bias, relu)
    self.fwd_remote = None
    self.wgrad = self.dgrad = None
    self.dy = dy
    if training and dy is not None:
      self.wgrad = igemm.gemm_wgrad(dy, x, st.g(self.sw))
      if dx is not None:
        self.dgrad = igemm.gemm(dy, st.w(self.sw), dx, "kn")

  def forward(self):
    self.fwd.run()

  def bind_remote_weights(self, flat_weights):
    x, y, bias, relu = self._fwd_args
    self.fwd_remote = igemm.gemm(x, self.store._view(flat_weights, self.sw), y, "nk", bias=bias,
                                 relu=relu)

  def forward_remote(self):
    self.fwd_remote.run()

  def backward(self):
    _run_wgrad(self)
    if self.dgrad is not None:
      self.dgrad.run()

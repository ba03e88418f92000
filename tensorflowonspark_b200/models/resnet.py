"""ResNet (v1.5 bottleneck: 50/101/152; basic-block CIFAR variants 20/32/56) on the
native engine: NHWC bf16 activations, wgmma implicit-GEMM convolutions with
batch-norm statistics fused into their epilogues, fused BN+ReLU(+residual)
apply/backward kernels, fused all-reduce + momentum-SGD optimizer.

Workload parity: the reference trains ResNet-56/CIFAR-10 through an external
Keras model (examples/resnet/resnet_cifar_dist.py:208, momentum SGD with a
piecewise schedule :35-66); BASELINE.json names ResNet-50/ImageNet-shaped data
as the headline config.  Both are provided here.
"""
import math
import numbers
import os

import torch

from .. import ops
from ..ops import igemm
from . import engine, evaluation, serving
from .engine import BatchNorm, Conv, Dense, ParamStore, normal


class _Unit(object):
  """conv -> BN (-> +residual) -> ReLU with its forward and gradient buffers."""

  def __init__(self, store, name, cin, cout, k, stride, zero_gamma=False):
    self.conv = Conv(store, name + ".conv", cin, cout, k, stride)
    self.bn = BatchNorm(store, name + ".bn", cout, zero_gamma=zero_gamma)
    self.cout = cout


class _Block(object):
  pass


def _buf(shape, device, dtype=torch.bfloat16):
  return torch.zeros(shape, dtype=dtype, device=device)


def _check_head_args(num_classes, label_smoothing):
  """(num_classes, label_smoothing) as (int, float); ValueError unless num_classes is an int >= 1
  and label_smoothing a real number in [0, 1].  The trainers call it before they allocate."""
  if isinstance(num_classes, bool) or not isinstance(num_classes, numbers.Integral) \
      or num_classes < 1:
    raise ValueError("num_classes must be an int >= 1, got {!r}".format(num_classes))
  if isinstance(label_smoothing, bool) or not isinstance(label_smoothing, numbers.Real) \
      or not 0.0 <= float(label_smoothing) <= 1.0:     # NaN fails the comparison too
    raise ValueError("label_smoothing must be a real number in [0, 1], got {!r}".format(
        label_smoothing))
  return int(num_classes), float(label_smoothing)


def _check_multilabel_args(multi_label, pos_weight, num_classes, training=True):
  """(multi_label, pos_weight as a tuple of floats or None); ValueError unless multi_label is a
  bool and pos_weight is None or, on a multi-label training trainer, ``num_classes`` finite
  numbers >= 0.  The trainers call it before they allocate."""
  if not isinstance(multi_label, bool):
    raise ValueError("multi_label must be a bool, got {!r}".format(multi_label))
  if pos_weight is None:
    return multi_label, None
  if not multi_label:
    raise ValueError("pos_weight weighs the positives of the multi-label loss: it needs "
                     "multi_label=True")
  if not training:
    raise ValueError("pos_weight is a training loss option: not on a training=False trainer")
  try:
    w = tuple(float(v) for v in pos_weight)
  except (TypeError, ValueError):
    raise ValueError("pos_weight must be a sequence of {} numbers, got {!r}".format(
        num_classes, pos_weight))
  if len(w) != num_classes:
    raise ValueError("pos_weight must hold one value per class ({}), got {}".format(
        num_classes, len(w)))
  bad = [v for v in w if not (math.isfinite(v) and v >= 0.0)]
  if bad:
    raise ValueError("pos_weight values must be finite and >= 0, got {!r}".format(bad[0]))
  return multi_label, w


def _labels_buffer(B, V, multi_label, device):
  """Training labels: int32 class indices [B], or uint8 multi-hot targets [B, V]."""
  if multi_label:
    return torch.zeros((B, V), dtype=torch.uint8, device=device)
  return torch.zeros(B, dtype=torch.int32, device=device)


def _padded_head_init(V, std=0.01):
  """Initialiser of a classifier weight padded to ceil(V / 8) * 8 rows: the V real rows are drawn
  as ``normal(std)`` draws an unpadded [V, K] weight, the padding rows are zero.  Their logits are
  then 0 and their gradient, momentum and share of LARS's ||w|| stay exactly zero."""
  def init(shape, gen):
    w = torch.zeros(shape)
    w[:V] = torch.randn((V,) + tuple(shape[1:]), generator=gen) * std
    return w
  return init


_HEAD = ("fc.w", "fc.b")   # the classifier: what load_backbone leaves out


def _state_shapes(cls, depth, num_classes):
  """{name: shape} of the ``state_dict()`` of a ``cls`` trainer of ``depth`` with ``num_classes``
  classes, ``__running__`` included, from the parameter registration alone (nothing on a
  device)."""
  st = engine.ParamStore()
  cls._register(st, depth, num_classes)
  shapes = {s["name"]: s["shape"] for s in st._specs}
  # RunningArena: mean and var of every batch norm, each padded to 8
  shapes["__running__"] = (sum(2 * ((s["shape"][0] + 7) // 8 * 8) for s in st._specs
                               if s["name"].endswith(".gamma")),)
  return shapes


def _check_state_shapes(state, want, what):
  """ValueError naming the first tensor of ``state`` that is not in ``want`` ({name: shape}), is
  missing from it or has another shape; nothing is copied."""
  extra = sorted(set(state) - set(want))
  if extra:
    raise ValueError("{}: {} is not a tensor of this model (another depth or family?)".format(
        what, extra[0]))
  for name, shape in want.items():
    if name not in state:
      raise ValueError("{}: {} {} is missing from the state{}".format(
          what, name, shape, " (it must include the running statistics)"
          if name == "__running__" else " (another depth or family?)"))
    got = tuple(getattr(state[name], "shape", ()))
    if got != tuple(shape):
      raise ValueError("{}: {} has shape {} in the state, {} in this model{}".format(
          what, name, got, tuple(shape), " (a head for another class count?)"
          if name in _HEAD else ""))


def _check_teacher(cls, teacher, teacher_depth, alpha, temperature, depth, num_classes, training,
                   multi_label):
  """The distillation options of a ``cls`` trainer (engine.check_distill_args) and its teacher's
  tensors, checked before anything is allocated.  Returns (the teacher's depth, or None without a
  teacher; alpha; T)."""
  td, a, t = engine.check_distill_args(teacher, teacher_depth, alpha, temperature, training,
                                       multi_label)
  if teacher is None:
    return None, a, t
  td = depth if td is None else td
  if not cls._valid_depth(td):
    raise ValueError("teacher_depth {} is not a depth of {}".format(td, cls.__name__))
  _check_state_shapes(teacher, _state_shapes(cls, td, num_classes), "teacher")
  return td, a, t


# columns of the bn_fold table (csrc/ops.h kFold*)
FOLD_WEIGHT, FOLD_COUT, FOLD_PER_CHANNEL, FOLD_GAMMA, FOLD_BETA, FOLD_MEAN, FOLD_VAR, FOLD_BIAS = \
    range(8)


def fold_table(store, units, running):
  """Host table that drives the ``bn_fold`` kernel: one int64 row per (filter spec, BatchNorm) of
  ``units`` with the filter's offset in ``store.weights``, Cout, the elements per output channel,
  gamma / beta offsets in ``store.aux32``, running mean / var offsets in ``running``'s buffer
  (engine.RunningArena) and the unit's slot in the fp32 bias vector (each padded to 8).
  Returns (table [U, 8] int64, eps [U] fp32, row0 [U + 1] int64: prefix sums of Cout, bias length)."""
  rows, eps, row0, boff = [], [], [0], 0
  base = running.buf.data_ptr()
  for spec, bn in units:
    cout = spec["shape"][0]
    per = spec["numel"] // cout
    if bn.C != cout or per % 8 or spec["offset"] % 8:
      raise ValueError("bn_fold: {} does not fold into {}".format(bn.name, spec["name"]))
    rows.append([spec["offset"], cout, per, bn.sg["offset"] - store.decay_end,
                 bn.sb["offset"] - store.decay_end,
                 (bn.running_mean.data_ptr() - base) // 4, (bn.running_var.data_ptr() - base) // 4,
                 boff])
    eps.append(bn.eps)
    row0.append(row0[-1] + cout)
    boff += (cout + 7) // 8 * 8
  return (torch.tensor(rows, dtype=torch.int64), torch.tensor(eps, dtype=torch.float32),
          torch.tensor(row0, dtype=torch.int64), boff)


def multilabel_totals(h, V):
  """``eval_end()`` of a multi-label trainer from the summed multilabel_eval_metrics accumulator
  ``h`` (8 + 3 V values: rows scored, invalid rows, BCE sum, correct elements, exact-match rows,
  3 unused, then per-class TP [V], FP [V], FN [V]).  Precision, recall and F1 are micro averages of
  the summed counts, F1 = 2 TP / (2 TP + FP + FN); a ratio whose denominator is 0 is NaN.  A class
  with TP + FP + FN = 0 has F1 NaN and is left out of ``macro_f1`` (Keras's ``F1Score`` counts it
  as 0).  Raises ValueError when any row held a label byte other than 0 or 1."""
  if h[1] > 0:
    raise ValueError("evaluation saw {} row(s) with a label byte other than 0 or 1".format(
        int(h[1])))
  ratio = lambda a, b: a / b if b else float("nan")   # noqa: E731
  count = int(h[0])
  tp, fp, fn = h[8:8 + V], h[8 + V:8 + 2 * V], h[8 + 2 * V:8 + 3 * V]
  TP, FP, FN = sum(tp), sum(fp), sum(fn)
  per_class = [ratio(2 * a, 2 * a + b + c) for a, b, c in zip(tp, fp, fn)]
  present = [f for f in per_class if f == f]
  return {"count": count, "loss": ratio(h[2], count * V), "binary_accuracy": ratio(h[3], count * V),
          "exact_match": ratio(h[4], count), "precision": ratio(TP, TP + FP),
          "recall": ratio(TP, TP + FN), "f1": ratio(2 * TP, 2 * TP + FP + FN),
          "macro_f1": ratio(sum(present), len(present)), "f1_per_class": per_class}


class _Evaluator(object):
  """Held-out evaluation on a trainer's own buffers (``eval_begin`` / ``eval_step`` /
  ``eval_end`` of both ResNet trainers).

  The forward pass is the folded network of ``build_folded_inference`` (bias, ReLU and the
  residual add in the convolution epilogues) run on the trainer's activation buffers: the next
  training forward rewrites all of them, and backward reads only what its own forward wrote.  The
  filters are folded from the bf16 ``weights`` and ``aux32``, which are complete and identical on
  every rank (the fp32 masters are only current for a rank's own shard), with rank 0's running
  statistics - the ones its checkpoint and exports carry - so every rank scores the same model.
  Only the uint8 input batch, labels, folded filters and biases are extra memory, allocated on the
  first ``eval_begin``."""

  def __init__(self, net):
    st, dev, comm = net.store, net.device, net.comm
    self.net, self.comm = net, comm
    units = net._fold_units()
    tab, eps, row0, nbias = fold_table(st, units, net.running)
    self.tab, self.eps, self.row0 = tab.to(dev), eps.to(dev), row0.to(dev)
    self.rows = int(row0[-1])
    self.wf = torch.zeros_like(st.weights)
    self.bf = torch.zeros(nbias, dtype=torch.float32, device=dev)
    bias = {id(bn): self.bf[int(tab[i, FOLD_BIAS]):int(tab[i, FOLD_BIAS]) + bn.C]
            for i, (_, bn) in enumerate(units)}
    self.u8 = torch.zeros_like(net.in_u8)         # never in_u8: drivers stage a batch and replay
    self.labels = torch.zeros_like(net.labels)
    self.n_valid = torch.zeros(1, dtype=torch.int32, device=dev)
    self.V = net.num_classes
    self.multi_label = net.multi_label
    # multilabel_eval_metrics: 8 totals, then per-class TP / FP / FN (csrc/ops.h kMlEval*)
    slots = ops.C().multilabel_eval_slots(self.V) if self.multi_label else 8
    self.acc = torch.zeros(slots, dtype=torch.float64, device=dev)
    if comm is None:
      self.running = net.running.tensor()
    else:
      self.running = comm.alloc("eval_running", net.running.used, torch.float32)
    self.rank_sum = evaluation.RankSum(comm, "eval_totals", slots)
    self._wv, self._bias = (lambda spec: st._view(self.wf, spec)), bias
    # one forward (and graph) per model: "live" reads the head from the store, "averaged" (built
    # on the first averaged evaluation) from a copy of the averaged head in wf / head_b
    self._modes = {False: {"forward": net._eval_forward(self._wv, bias, self.u8), "graph": None,
                           "calls": 0}}
    self.averaged = False
    self.staging = evaluation.HostStaging(dev, net.B, self.u8.shape[1:], self.labels.shape[1:])

  @property
  def graph(self):
    """The captured evaluation of the live model (None before its second batch)."""
    return self._modes[False]["graph"]

  def _averaged_mode(self):
    net, st, fc = self.net, self.net.store, self.net.fc
    if True not in self._modes:
      self.head_b = torch.zeros(fc.cout, dtype=torch.float32, device=net.device)
      head = igemm.gemm(net.avg, st._view(self.wf, fc.sw), net.logits, "nk", bias=self.head_b)
      self._modes[True] = {"forward": net._eval_forward(self._wv, self._bias, self.u8, head.run),
                           "graph": None, "calls": 0}
    return fc

  def begin(self, averaged=False):
    """``averaged``: fold from the weight average (FusedOptimizer.averaged_weights(): complete
    and identical on every rank) instead of the live weights, with the same running statistics;
    the classifier then also runs on the averaged head."""
    net, comm = self.net, self.comm
    st = net.store
    weights, aux32 = net.optim.averaged_weights() if averaged else (st.weights, st.aux32)
    self.averaged = bool(averaged)
    self.acc.zero_()
    if comm is not None:
      self.running.copy_(net.running.tensor())
      comm.broadcast("eval_running", 0)
    ops.K.bn_fold(self.tab, self.eps, self.row0, self.rows, weights, aux32, self.running,
                  self.wf, self.bf)
    if averaged:   # (bn_fold writes only the convolution filters of wf: the head's rows are free)
      fc = self._averaged_mode()
      st._view(self.wf, fc.sw).copy_(st._view(weights, fc.sw))
      self.head_b.copy_(st._view(aux32, fc.sbias, st.decay_end))

  def _run(self):
    self._modes[self.averaged]["forward"]()
    if self.multi_label:
      ops.K.multilabel_eval_metrics(self.net.logits, self.labels, self.n_valid, self.acc, self.V)
    else:
      ops.K.eval_metrics(self.net.logits, self.labels, self.n_valid, self.acc, self.V)

  def step(self, images_u8, labels):
    n = len(images_u8)
    if n > self.net.B:
      raise ValueError("batch of {} rows exceeds the trainer's batch size {}".format(n, self.net.B))
    if n:
      x = torch.as_tensor(images_u8)
      self.u8[:n].copy_(x.reshape((n,) + tuple(self.u8.shape[1:])), non_blocking=True)
      self.labels[:n].copy_(torch.as_tensor(labels).reshape((n,) + tuple(self.labels.shape[1:])),
                            non_blocking=True)
    self.n_valid.fill_(n)
    m = self._modes[self.averaged]
    if m["graph"] is None and m["calls"] >= 1:
      m["graph"] = self._capture()
    if m["graph"] is not None:
      m["graph"].replay()
    else:
      self._run()
    m["calls"] += 1

  def _capture(self):
    """The evaluation forward + metric as one CUDA graph (after one eager call, like
    ServedResNet._capture); thread-local capture under a cross-host communicator, as in
    ResNetTrainer.capture."""
    g = torch.cuda.CUDAGraph()
    mode = "thread_local" if getattr(self.net.optim, "group_mode", False) else "global"
    with torch.cuda.graph(g, capture_error_mode=mode):
      self._run()
    return g

  def run(self, batches):
    """eval_step over (images, labels) pairs; host batches are staged in page-locked memory one
    batch ahead of the forward pass."""
    if self.multi_label:   # bool or uint8 host targets are staged as uint8 bytes
      self.staging.run(self.step, batches, label_dtype=lambda y: torch.uint8)
    else:
      self.staging.run(self.step, batches)

  def end(self):
    h = self.rank_sum(self.acc)
    if self.multi_label:
      return multilabel_totals(h, self.V)
    if h[3] > 0:
      raise ValueError("evaluation saw {} label(s) outside [0, {})".format(int(h[3]), self.V))
    count = int(h[0])
    mean = (lambda v: v / count) if count else (lambda v: float("nan"))
    return {"count": count, "loss": mean(h[4]), "top1": mean(h[1]), "top5": mean(h[2])}


class ResNetTrainer(object):
  """Static-buffer ResNet.  ``train_step(images_u8 | normalized, labels)`` runs
  forward, backward and the fused optimizer; ``forward_only`` serves inference."""

  CFG = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3), 152: (3, 8, 36, 3)}

  def __init__(self, depth=50, batch=256, image=224, num_classes=1000, device="cuda:0",
               lr=0.1, momentum=0.9, weight_decay=1e-4, comm=None, training=True, seed=1234,
               optimizer="momentum", trust_coefficient=0.001, label_smoothing=0.0,
               ema_decay=None, clip_norm=None, beta1=0.9, beta2=0.999, epsilon=1e-7,
               gradient_accumulation_steps=1, multi_label=False, pos_weight=None,
               mixup_alpha=0.0, cutmix_alpha=0.0, mix_prob=1.0, mix_switch_prob=0.5,
               drop_path_rate=0.0, teacher=None, teacher_depth=None, distill_alpha=0.5,
               distill_temperature=1.0):
    """``optimizer``: sgd | momentum | adam | adamw | lars | lamb (``trust_coefficient`` is LARS's
    eta; see parallel/fused_optim.py).  adam folds ``weight_decay`` into the gradient (L2), adamw
    decouples it (``torch.optim.AdamW``), lamb is layer-wise adaptive Adam (apex ``FusedLAMB``).
    ``beta1``, ``beta2`` in [0, 1) and ``epsilon`` > 0 are the Adam family's (Keras's defaults).

    ``clip_norm``: None, or c > 0 (inf allowed): the averaged gradient is clipped to global norm
    c before the update, as ``torch.nn.utils.clip_grad_norm_`` (Keras's ``global_clipnorm``),
    inside the fused optimizer kernels; ``grad_norm`` holds the norm of each step, and
    ``clip_norm=float("inf")`` only measures it.

    ``ema_decay``: None, or d in [0, 1): the optimizer also keeps an exponential moving average
    of the weights (Keras's ``use_ema``), fused into its update kernels; training is unchanged.
    ``averaged()`` exports it and ``evaluate(..., averaged=True)`` scores it.

    ``num_classes``: any int >= 1.  The head has ``VP = ceil(num_classes / 8) * 8`` rows; the
    padding rows start at zero and stay zero, and the loss, evaluation and serving read only the
    first ``num_classes`` logits.  ``label_smoothing`` (eps in [0, 1]): the training loss is the
    cross-entropy against (1 - eps) * onehot + eps / num_classes, as
    ``F.cross_entropy(label_smoothing=eps)``; evaluation reports the plain cross-entropy.

    ``gradient_accumulation_steps`` (k, an int >= 1; training only): the parameters are updated
    every k ``train_step`` calls with the mean of the gradients since the last update (Keras's
    ``gradient_accumulation_steps``).  Calls 1 .. k-1 of a window run forward, loss and backward
    and add into the gradient buffer, with no optimizer kernel and no communication; call k also
    runs the fused all-reduce + update.  Each micro-batch's loss is its own mean (``loss_sum`` is
    the micro-batch's), label smoothing applies per micro-batch, and the batch-norm batch and
    running statistics are per micro-batch, as in Keras and PyTorch.  Clipping, the LARS / LAMB
    norms, weight decay, the weight average and Adam's step advance once per update.
    ``micro_step`` is the position of the next call in its window (0 .. k-1).

    ``multi_label`` (bool): each image has a multi-hot target of ``num_classes`` entries, and the
    labels are uint8 (or bool) [n, num_classes], 0 = negative, 1 = positive (training counts any
    nonzero byte as positive).  The training loss is the mean over the B x V elements of the binary
    cross-entropy with logits (``torch.nn.BCEWithLogitsLoss``, Keras's
    ``BinaryCrossentropy(from_logits=True)``); ``label_smoothing`` eps then smooths the targets to
    y (1 - eps) + eps / 2, as Keras does.  ``pos_weight`` (training only): None or num_classes
    finite numbers >= 0, torch's ``pos_weight``: element (i, j) costs
    -[p_j t log sigmoid(l) + (1 - t) log(1 - sigmoid(l))].  ``train_step`` returns the mean loss
    and ``correct`` counts the rows whose prediction (logit > 0 per class) equals the target
    exactly; ``eval_end`` reports binary accuracy, exact match and micro / macro F1
    (``multilabel_totals``); serving returns a multi-hot ``prediction``.

    ``mixup_alpha``, ``cutmix_alpha`` (finite, >= 0; training only): Mixup and CutMix as timm's
    ``Mixup`` in "batch" mode with ``correct_lam=True``.  Each ``train_step`` call (each
    micro-step, each warm-up step of ``capture()``) draws one (mode, lam, box) on the host
    (engine.MixDraws, seeded with (``seed``, rank)); ``last_mix`` holds the last draw.  Row i of the
    local batch of B rows is paired with row B - 1 - i: Mixup trains on lam x_i + (1 - lam) x_p,
    CutMix pastes row p's pixels into a box of row i, and the target is lam s(y_i) + (1 - lam)
    s(y_p) with s the smoothed target above (one-hot or multi-hot).  ``mix_prob`` (in [0, 1]): the
    probability that a step mixes at all; ``mix_switch_prob`` (in [0, 1]): with both alphas > 0,
    the probability that a mixing step is CutMix.  ``correct`` then counts hits against the
    dominant sample (the row's own label when lam >= 0.5, its partner's otherwise).  Evaluation,
    serving and exports never mix.

    ``drop_path_rate`` (r in [0, 1); training only): stochastic depth as timm's
    ``DropPath(scale_by_keep=True)`` in its ``Bottleneck``: block i of the N residual blocks
    drops with p_i = r * i / (N - 1) (timm's linear decay; ``drop_path_rates`` holds them), and
    each sample's residual branch output is multiplied by s_b = keep_b / (1 - p_i),
    keep_b ~ Bernoulli(1 - p_i), before the shortcut is added: out = relu(s_b bn3(conv3(..)) +
    shortcut).  bn3's batch and running statistics are those of the whole batch, the shortcut
    (identity or projection) is never dropped, and the branch's gradient is s_b times the block
    output's.  Each ``train_step`` call (each micro-step, each warm-up step of ``capture()``)
    draws the factors of every block on the host (engine.DropPathDraws, seeded with (``seed``,
    rank, 1)); ``last_drop_path`` holds the last draw.  Evaluation, serving, ``averaged()`` and
    exports never drop.

    ``teacher`` (training only): None, or the ``state_dict()`` of a trained ResNetTrainer of depth
    ``teacher_depth`` (50, 101 or 152; default: this trainer's depth) with the same
    ``num_classes``, ``__running__`` included (``net.averaged().state_dict()`` too): knowledge
    distillation.  Every tensor is checked as ``load_backbone`` checks it, before anything is
    allocated.  The teacher is a frozen ``training=False`` replica with every batch norm folded
    into its convolutions (``build_folded_inference``, with its running statistics; it never drops
    a path and is never updated).  It runs inside every training step, right after the decode, on
    the student's decoded input (the mixed one under Mixup / CutMix), and the training loss of row
    i with student logits s, teacher logits z and the hard target t above becomes
    (1 - a) CE(s, t) + a T^2 KL(softmax(z / T) || softmax(s / T)), a = ``distill_alpha`` in (0, 1],
    T = ``distill_temperature`` (finite, > 0): ``(1-a) F.cross_entropy(s, y, label_smoothing=eps)
    + a T^2 F.kl_div(F.log_softmax(s/T), F.log_softmax(z/T), log_target=True,
    reduction="batchmean")``.  ``correct`` still counts the student's arg-max against the dominant
    label.  The teacher is not part of ``state_dict()``, checkpoints, the optimizer state,
    ``averaged()``, exports, evaluation or serving: a resumed run passes it again.  Not with
    ``multi_label``."""
    num_classes, self.label_smoothing = _check_head_args(num_classes, label_smoothing)
    self.multi_label, pos_weight = _check_multilabel_args(multi_label, pos_weight, num_classes,
                                                          training)
    mix_args = engine.check_mix_args(mixup_alpha, cutmix_alpha, mix_prob, mix_switch_prob,
                                     training)
    self.drop_path_rate = engine.check_drop_path_rate(drop_path_rate, training)
    self.teacher_depth, self.distill_alpha, self.distill_temperature = _check_teacher(
        type(self), teacher, teacher_depth, distill_alpha, distill_temperature, depth, num_classes,
        training, self.multi_label)
    k_acc = engine.check_gradient_accumulation_steps(gradient_accumulation_steps, training)
    self.ema_decay = engine.check_ema_decay(ema_decay, training)
    self.clip_norm = engine.check_clip_norm(clip_norm, training)
    beta1, beta2, epsilon = engine.check_adam_args(beta1, beta2, epsilon)
    assert depth in self.CFG, "bottleneck depths: 50/101/152"
    self.device = torch.device(device)
    self.B, self.image, self.num_classes, self.depth = batch, image, num_classes, depth
    self.training = training
    self.comm = comm
    dev = self.device
    st = self.store = ParamStore()
    B = batch

    # ---- parameters -----------------------------------------------------
    self.stem_w, self.stem_bn, self.blocks, self.fc, self.feat = self._register(st, depth,
                                                                                num_classes)
    VP = self.VP = (num_classes + 7) // 8 * 8
    self.drop_path_rates = engine.drop_path_rates(self.drop_path_rate, len(self.blocks))

    alloc = comm.alloc if comm is not None else None
    st.finalize(dev, alloc=alloc, seed=seed)

    # ---- buffers and plans -----------------------------------------------
    OH, OW, Wp = igemm.stem_geometry(image, image)
    self.in_u8 = _buf((B, image, image, 3), dev, torch.uint8)
    self.xp = _buf((B, image, Wp, 8), dev)
    self.labels = _labels_buffer(B, num_classes, self.multi_label, dev)
    self.pos_weight = None if pos_weight is None else torch.tensor(pos_weight, dtype=torch.float32,
                                                                   device=dev)
    self.stem_raw = _buf((B, OH, OW, 64), dev)
    PH, PW = (OH + 2 - 3) // 2 + 1, (OW + 2 - 3) // 2 + 1
    self.pool = _buf((B, PH, PW, 64), dev)
    self.pool_idx = _buf((B, PH, PW, 64), dev, torch.uint8)
    tr = training
    # all batch-norm statistics accumulators live in one arena that is zeroed once per step;
    # finalisation is folded into the apply kernels (engine.BatchNorm.build)
    # (sized from the model: ResNet-101 / 152 need more than the arenas' default capacity)
    c8 = sum((bn.C + 7) // 8 * 8 for bn in self._batch_norms())
    self.stats_arena = engine.StatsArena(dev, capacity=max(4 * c8, 1 << 17)) if tr else None
    # all BN running statistics, one flat buffer
    self.running = engine.RunningArena(dev, capacity=max(2 * c8, 1 << 17))
    self.stem_bn.build(dev, self.stats_arena, self.running)
    # training fuses the stem's BN + ReLU + max pool (_forward): the activation is never stored
    self.stem_act = None if tr else _buf((B, OH, OW, 64), dev)
    self.p_stem = igemm.stem_fprop(self.xp, st.w(self.stem_w), self.stem_raw,
                                   stats=self.stem_bn.stats if tr else None)
    if tr:
      self.g_stem_raw = _buf((B, OH, OW, 64), dev)
      self.p_stem_wgrad = igemm.stem_wgrad(self.g_stem_raw, self.xp, st.g(self.stem_w))

    x, H, W = self.pool, PH, PW
    prev_block = None
    gx = _buf(x.shape, dev) if tr else None  # gradient wrt the block input
    self.g_pool = gx
    for b, p in zip(self.blocks, self.drop_path_rates):
      b.drop_path = p
      s = b.stride
      H2, W2 = (H - 1) // s + 1, (W - 1) // s + 1
      w, c4 = b.width, b.width * 4
      b.x = x
      b.r1, b.a1 = _buf((B, H, W, w), dev), _buf((B, H, W, w), dev)
      b.r2, b.a2 = _buf((B, H2, W2, w), dev), _buf((B, H2, W2, w), dev)
      b.r3, b.out = _buf((B, H2, W2, c4), dev), _buf((B, H2, W2, c4), dev)
      if tr:
        b.g_r1, b.g_a1 = _buf(b.r1.shape, dev), _buf(b.a1.shape, dev)
        b.g_r2, b.g_a2 = _buf(b.r2.shape, dev), _buf(b.a2.shape, dev)
        b.g_r3 = _buf(b.r3.shape, dev)
        # identity blocks share the stage gradient buffer: g_out is rewritten in place
        # into g_x (masked residual gradient + conv1 dgrad accumulated on top)
        b.g_out = _buf(b.out.shape, dev) if b.ds is not None else gx
        b.g_x = gx
      else:
        b.g_r1 = b.g_a1 = b.g_r2 = b.g_a2 = b.g_r3 = b.g_out = b.g_x = None
      for u in (b.u1, b.u2, b.u3) + ((b.ds,) if b.ds else ()):
        u.bn.build(dev, self.stats_arena, self.running)
      ident = b.ds is None
      # the block output's ReLU mask (one bit per element, written by bn3's forward): identity
      # blocks fold "mask * dY" into conv1's accumulating dgrad instead of materialising it
      omask = b.u3.bn.ensure_mask(b.out.numel(), dev) if tr else None
      # Fused batch-norm backward reductions: the data gradient that WRITES a batch norm's dy
      # also accumulates that batch norm's sum(g), sum(g x):
      #   conv3.dgrad -> g_a2 = dy of bn2        conv2.dgrad -> g_a1 = dy of bn1
      #   identity block: conv1.dgrad (accumulating) completes g_x = dy of the PREVIOUS block's bn3
      red1 = (b.u1.bn, b.r1, b.u1.bn.ensure_mask(b.a1.numel(), dev)) if tr else None
      red2 = (b.u2.bn, b.r2, b.u2.bn.ensure_mask(b.a2.numel(), dev)) if tr else None
      redp = None
      # (a block that drops scales its bn3's gradient per sample: that reduction stays unfused)
      if tr and ident and prev_block is not None and not prev_block.drop_path:
        redp = (prev_block.u3.bn, prev_block.r3, prev_block.u3.bn.ensure_mask(
            prev_block.out.numel(), dev))
      b.u1.conv.build(x, b.r1, b.g_r1, b.g_x, stats=b.u1.bn.stats, dx_accumulate=ident,
                      training=tr, dx_acc_mask=omask if ident else None, dx_bn_reduce=redp)
      b.u2.conv.build(b.a1, b.r2, b.g_r2, b.g_a1, stats=b.u2.bn.stats, training=tr,
                      dx_bn_reduce=red1)
      b.u3.conv.build(b.a2, b.r3, b.g_r3, b.g_a2, stats=b.u3.bn.stats, training=tr,
                      dx_bn_reduce=red2)
      if b.ds is not None:
        b.rd, b.idn = _buf(b.r3.shape, dev), _buf(b.r3.shape, dev)
        b.g_rd = _buf(b.r3.shape, dev) if tr else None
        b.ds.conv.build(x, b.rd, b.g_rd, b.g_x, stats=b.ds.bn.stats, dx_accumulate=True,
                        training=tr)
      prev_block = b
      x, H, W = b.out, H2, W2
      if tr:
        gx = b.g_out
    self.last = x
    self.g_last = gx
    self.avg = _buf((B, self.feat), dev)
    self.logits = _buf((B, VP), dev, torch.float32)
    self.ldd = VP
    self.dlogits = _buf((B, VP), dev) if tr else None
    self.g_avg = _buf((B, self.feat), dev) if tr else None
    self.loss_sum = torch.zeros(1, dtype=torch.float32, device=dev)
    self.correct = torch.zeros(1, dtype=torch.float32, device=dev)
    self.fc.build(self.avg, self.logits, self.dlogits, self.g_avg, training=tr)

    self.optim = None
    if tr:
      from ..parallel.fused_optim import FusedOptimizer
      buckets = self._comm_buckets() if (comm is not None and comm.world > 1) else None
      self.optim = FusedOptimizer(st, comm=comm, opt=optimizer, lr=lr, momentum=momentum,
                                  weight_decay=weight_decay, buckets=buckets,
                                  trust_coefficient=trust_coefficient, ema_decay=self.ema_decay,
                                  clip_norm=self.clip_norm, beta1=beta1, beta2=beta2, eps=epsilon)
      if k_acc > 1:
        self.optim.set_accumulation(k_acc)
        for bn in self._batch_norms():
          bn.accumulate_grads(None)   # every one has its arena slots or a fused reduction
    self.accum = engine.GradAccumulation(k_acc)
    self._build_mix(mix_args, seed)
    self._build_drop_path(seed)
    self.graph = None
    self.graphs = None
    self.mean = [0.485, 0.456, 0.406]
    self.std = [0.229, 0.224, 0.225]
    self._assign_directions()
    self.teacher = None if teacher is None else _ResNetTeacher(self, teacher, self.teacher_depth)

  @classmethod
  def _register(cls, st, depth, num_classes):
    """Register the parameters of a ResNet-``depth`` with ``num_classes`` classes in ``st`` (host
    only).  Returns (stem filter spec, stem batch norm, blocks, head, feature width)."""
    stem_w = st.register("stem.conv.w", (64, 7, 64), True, cls._stem_init)
    stem_bn = BatchNorm(st, "stem.bn", 64)
    blocks = []
    cin = 64
    for si, nblocks in enumerate(cls.CFG[depth]):
      width = 64 * (2 ** si)
      for bi in range(nblocks):
        stride = 2 if (bi == 0 and si > 0) else 1
        b = _Block()
        name = "layer{}.{}".format(si + 1, bi)
        b.u1 = _Unit(st, name + ".u1", cin, width, 1, 1)
        b.u2 = _Unit(st, name + ".u2", width, width, 3, stride)
        b.u3 = _Unit(st, name + ".u3", width, width * 4, 1, 1, zero_gamma=True)
        b.ds = _Unit(st, name + ".ds", cin, width * 4, 1, stride) if bi == 0 else None
        b.stride, b.cin, b.width, b.name = stride, cin, width, name
        blocks.append(b)
        cin = width * 4
    VP = (num_classes + 7) // 8 * 8
    fc = Dense(st, "fc", cin, VP, bias=True,
               init=normal(0.01) if VP == num_classes else _padded_head_init(num_classes))
    return stem_w, stem_bn, blocks, fc, cin

  @classmethod
  def _valid_depth(cls, depth):
    return depth in cls.CFG

  def _build_mix(self, mix_args, seed):
    """Mixup / CutMix state: the host draws (engine.MixDraws) and the device vector each step's
    draw is staged into; neither exists when both alphas are 0."""
    (self.mixup_alpha, self.cutmix_alpha, self.mix_prob, self.mix_switch_prob) = mix_args
    self.mixer = self.mix = self.last_mix = None
    if self.mixup_alpha > 0 or self.cutmix_alpha > 0:
      rank = self.comm.rank if self.comm is not None else 0
      self.mixer = engine.MixDraws(self.mixup_alpha, self.cutmix_alpha, self.mix_prob,
                                   self.mix_switch_prob, seed=seed, rank=rank)
      self.mix = torch.zeros(engine.MIX_SLOTS, dtype=torch.float32, device=self.device)

  def _stage_mix(self):
    """Draw this step's mix on the host and copy it into ``mix`` on the current stream, ahead of
    the step's kernels (never inside a graph capture).  The source is a fresh pageable tensor: the
    copy takes the values before it returns, so the host never waits and never overwrites what a
    queued copy still reads."""
    if self.mixer is None:
      return
    self.last_mix = self.mixer.draw(self.image, self.image)
    self.mix.copy_(torch.tensor(engine.MixDraws.vector(self.last_mix), dtype=torch.float32),
                   non_blocking=True)

  def _mix_arg(self):
    """The ``mix`` keyword of the training decode and loss: none when the trainer does not mix,
    so such a trainer launches exactly what it did before mixing existed."""
    return {} if self.mix is None else {"mix": self.mix}

  def _build_drop_path(self, seed):
    """Stochastic-depth state: the host draws (engine.DropPathDraws) and the device tensor
    ``drop_scale`` [n_blocks, B] each step's factors are staged into; neither exists when
    ``drop_path_rate`` is 0."""
    self.dropper = self.drop_scale = self.last_drop_path = None
    if self.drop_path_rate > 0:
      rank = self.comm.rank if self.comm is not None else 0
      self.dropper = engine.DropPathDraws(self.drop_path_rates, self.B, seed=seed, rank=rank)
      self.drop_scale = torch.ones((len(self.blocks), self.B), dtype=torch.float32,
                                   device=self.device)

  def _stage_draws(self):
    """Draw this step's mix and drop-path factors on the host and copy them into ``mix`` and
    ``drop_scale`` on the current stream, ahead of the step's kernels (never inside a graph
    capture).  Each source is a fresh pageable tensor: the copy takes the values before it
    returns, so the host never waits and never overwrites what a queued copy still reads."""
    self._stage_mix()
    if self.dropper is not None:
      self.last_drop_path = self.dropper.draw()
      self.drop_scale.copy_(torch.from_numpy(self.last_drop_path.copy()), non_blocking=True)

  def _drop_arg(self, i):
    """The ``sample_scale`` keyword of block i's last batch norm: none when the block never
    drops, so a trainer without drop path launches exactly what it did before."""
    if self.drop_scale is None or not self.drop_path_rates[i]:
      return {}
    return {"sample_scale": self.drop_scale[i]}

  def _batch_norms(self):
    return [self.stem_bn] + [u.bn for b in self.blocks
                             for u in (b.u1, b.u2, b.u3) + ((b.ds,) if b.ds is not None else ())]

  @property
  def gradient_accumulation_steps(self):
    return self.accum.k

  @property
  def micro_step(self):
    """Position (0 .. k-1) of the next ``train_step`` in its accumulation window: the next call
    updates the parameters when ``micro_step == gradient_accumulation_steps - 1``."""
    return self.accum.micro_step

  def _assign_directions(self):
    """L2 hand-over ("serpentine") schedule.

    Activations are 13 - 411 MB per tensor at batch 256, the L2 holds 50 MB: a kernel that walks
    a tensor front to back leaves its TAIL in L2.  Every memory-bound kernel of the chain
    therefore starts at the end where its predecessor stopped:
      forward   conv (tiles ascending) -> BN apply (rows descending) -> next conv (ascending) ...
      backward  BN reduce (d) -> BN apply (not d) -> the unit's dgrad (d) -> next unit (not d) ...
    Only the ORDER in which tiles / rows are visited changes; results are identical."""
    d = False
    for b in reversed(self.blocks):
      for u in (b.u3, b.u2, b.u1):
        u.rev = (d, not d)
        if u.conv.dgrad is not None:
          u.conv.dgrad.set_reverse(d)
        d = not d
      if b.ds is not None:
        b.ds.rev = (False, True)

  def _comm_buckets(self):
    """Gradient buckets for overlapping the fused all-reduce with backward: (begin, end, tag)
    where tag is the index of the block after whose backward the range is final ('stem' = end
    of backward).  layer4+fc hold 2/3 of the parameters and are final a third into backward;
    what is left for the un-overlappable tail after the stem's weight gradient is only stem +
    layer1 (0.23 M of 25.6 M parameters) and the batch-norm parameters of stem..layer2."""
    st = self.store

    def first_offset(prefix, decay=True):
      return min(s["offset"] for s in st.order if s["decay"] == decay and s["name"].startswith(prefix))

    def first_block(prefix):
      return next(i for i, b in enumerate(self.blocks) if b.name.startswith(prefix))

    b2, b3, b4 = first_offset("layer2."), first_offset("layer3."), first_offset("layer4.")
    nd3 = first_offset("layer3.", decay=False)   # non-decayed tail: BN scale/offset in layer order
    return [(b4, st.decay_end, first_block("layer4.")), (b3, b4, first_block("layer3.")),
            (nd3, st.total, first_block("layer3.")), (b2, b3, first_block("layer2.")),
            (0, b2, "stem"), (st.decay_end, nd3, "stem")]

  @staticmethod
  def _stem_init(shape, gen):
    import math
    w = torch.randn((shape[0], 7, 7, 3), generator=gen) * math.sqrt(2.0 / (7 * 7 * 3))
    return igemm.pack_stem_weight(w)

  # ------------------------------------------------------------------ data
  def synthetic_batch(self, seed=0):
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    x = torch.randint(0, 256, (self.B, self.image, self.image, 3), dtype=torch.uint8, generator=g)
    if self.multi_label:   # each class present with probability 1/2
      y = torch.randint(0, 2, (self.B, self.num_classes), dtype=torch.uint8, generator=g)
    else:
      y = torch.randint(0, self.num_classes, (self.B,), dtype=torch.int32, generator=g)
    return x.to(self.device), y.to(self.device)

  def set_input(self, images_u8, labels=None):
    """Stage a uint8 NHWC batch (device or pinned host) into the static input buffers."""
    self.in_u8.copy_(images_u8, non_blocking=True)
    if labels is not None:
      self.labels.copy_(labels, non_blocking=True)

  # ------------------------------------------------- broadcast fused with use
  def bind_broadcast_root(self, root=0):
    """Prepare the fused startup broadcast: forward plans whose filters are read by TMA
    straight out of the ROOT rank's weight buffer over NVLink (tile by tile, as the wgmma
    main loop consumes them), while `bcast_pull` fills the local copy on a side stream."""
    comm = self.comm
    flat = ops.C().tensor_from_ptr(comm.peer_ptrs("weights")[root], [self.store.total], "bf16")
    self._root_weights = flat
    self._root = root
    w_stem = self.store._view(flat, self.stem_w)
    self.p_stem_remote = igemm.stem_fprop(self.xp, w_stem, self.stem_raw, stats=self.stem_bn.stats)
    for b in self.blocks:
      for u in (b.u1, b.u2, b.u3) + ((b.ds,) if b.ds is not None else ()):
        u.conv.bind_remote_weights(flat)
    self.fc.bind_remote_weights(flat)
    self._side = torch.cuda.Stream(device=self.device)

  def first_step_fused_broadcast(self):
    """First training step after start-up: the root's variables win (reference semantics of
    entering strategy.scope(), examples/mnist/keras/mnist_spark.py:55-56) without a separate
    broadcast phase in front of the first forward pass.  It is a ``train_step``: with
    ``gradient_accumulation_steps`` > 1 it is the first micro-step of a window (broadcast and
    accumulate, no update)."""
    comm = self.comm
    self._stage_draws()
    comm.broadcast("aux32", self._root)  # BN scale/offset + biases: tiny, consumed in fp32
    comm.barrier()                        # root's weights are final and visible
    main = torch.cuda.current_stream(self.device)
    self._side.wait_stream(main)
    with torch.cuda.stream(self._side):
      comm.broadcast("weights", self._root)     # local copy for the backward pass / later steps
      comm.broadcast("master", self._root, slot=60)  # fp32 masters restart from the root's values
    self._forward(True, remote=True)            # forward consumes the root's tiles over NVLink
    main.wait_stream(self._side)
    self._loss(True)
    zero, update = self.accum.phase()
    self._backward(zero, update)
    if update:
      self.optim.finish()
    self.accum.advance()
    return self.loss_sum

  # --------------------------------------------------------------- forward
  def _forward(self, training, remote=False):
    K = ops.K
    run = (lambda c: c.forward_remote()) if remote else (lambda c: c.forward())
    if self.stats_arena is not None:
      self.stats_arena.zero()   # the fused conv epilogues accumulate from zero every pass
    K.decode_normalize(self.in_u8, self.xp, igemm.STEM_PAD, self.mean, self.std,
                       **(self._mix_arg() if training else {}))
    if training and self.teacher is not None:
      self.teacher.run()      # its stem reads xp: the (mixed) input the student trains on
    (self.p_stem_remote if remote else self.p_stem).run()
    if training:
      # BN + ReLU + max pool in one pass over the raw conv output (csrc/stem_fused.cu): the
      # 411 MB stem activation is never written
      bn = self.stem_bn
      K.stem_bn_relu_pool_fwd(self.stem_raw, self.pool, self.pool_idx, bn.sum, bn.sumsq, bn.gamma,
                              bn.beta, bn.running_mean, bn.running_var, bn.mean, bn.invstd,
                              bn.scale, bn.shift, float(self.stem_raw.numel() // bn.C), bn.eps,
                              bn.momentum)
    else:
      self.stem_bn.forward(self.stem_raw, self.stem_act, None, 1, training)
      K.maxpool_fwd(self.stem_act, self.pool, self.pool_idx, 3, 2, 1)
    for bi, b in enumerate(self.blocks):
      for u, raw, act in ((b.u1, b.r1, b.a1), (b.u2, b.r2, b.a2)):
        run(u.conv)
        u.bn.forward(raw, act, None, 1, training, rev=True)
      run(b.u3.conv)
      if b.ds is not None:
        run(b.ds.conv)
        b.ds.bn.forward(b.rd, b.idn, None, 0, training, rev=True)
        idn = b.idn
      else:
        idn = b.x
      b.u3.bn.forward(b.r3, b.out, idn, 1, training, rev=True,
                      **(self._drop_arg(bi) if training else {}))
    K.avgpool_fwd(self.last, self.avg)
    run(self.fc)

  def _loss(self, with_grad):
    self.loss_sum.zero_()
    self.correct.zero_()
    mix = self._mix_arg() if with_grad else {}
    if self.multi_label:
      ops.K.sigmoid_bce(self.logits, self.labels, self.dlogits if with_grad else None,
                        self.loss_sum, self.correct, self.num_classes,
                        1.0 / (self.B * self.num_classes), label_smoothing=self.label_smoothing,
                        pos_weight=self.pos_weight, **mix)
      return
    if with_grad and self.teacher is not None:
      ops.K.distill_xent(self.logits, self.teacher.logits, self.labels, self.dlogits,
                         self.loss_sum, self.correct, self.num_classes, 1.0 / self.B,
                         label_smoothing=self.label_smoothing, alpha=self.distill_alpha,
                         temperature=self.distill_temperature, **mix)
      return
    ops.K.softmax_xent(self.logits, self.labels, self.dlogits if with_grad else None,
                       self.loss_sum, self.correct, self.num_classes, 1.0 / self.B,
                       label_smoothing=self.label_smoothing, **mix)

  # -------------------------------------------------------------- backward
  def _backward(self, zero=True, update=True):
    """``zero``: zero the gradients first; ``update``: start each bucket's all-reduce + update as
    soon as its gradients are final (gradient accumulation: only the window's last micro-step)."""
    K = ops.K
    if zero:
      self.optim.zero_grads()
    self.fc.backward()
    K.avgpool_bwd(self.g_avg, self.g_last)
    for bi in reversed(range(len(self.blocks))):
      b = self.blocks[bi]
      # out = relu(bn3(r3) + idn): the masked gradient goes to both branches; the mask is applied
      # where g_out is consumed (here, in conv1's accumulate epilogue, in the shortcut's BN)
      # stochastic depth: bn3 sees s_b * the masked gradient, the shortcut the unscaled one
      b.u3.bn.backward(b.g_out, b.r3, b.out, b.g_r3, relu=True, residual=True, rev=b.u3.rev,
                       **self._drop_arg(bi))
      b.u3.conv.backward()
      b.u2.bn.backward(b.g_a2, b.r2, b.a2, b.g_r2, relu=True, rev=b.u2.rev)
      b.u2.conv.backward()
      b.u1.bn.backward(b.g_a1, b.r1, b.a1, b.g_r1, relu=True, rev=b.u1.rev)
      b.u1.conv.backward()  # writes (ds) or accumulates (identity) into g_x
      if b.ds is not None:
        b.ds.bn.backward(b.g_out, b.rd, None, b.g_rd, relu=True, mask=b.u3.bn.mask, rev=b.ds.rev)
        b.ds.conv.backward()  # accumulates into g_x
      if update:
        self.optim.launch(bi)   # buckets that became final start their all-reduce now
    # max-pool backward recomputed inside the BN reduction and the BN apply: the gradient of the
    # stem activation (411 MB) is never written or read
    bn = self.stem_bn
    if bn.acc is None:
      K.stem_pool_bn_bwd(self.g_pool, self.pool_idx, self.stem_raw, bn.gamma, bn.mean, bn.invstd,
                         bn.scale, bn.shift, bn.dgamma, bn.dbeta, self.g_stem_raw)
    else:   # this micro-batch's dgamma / dbeta in scratch, added to the gradient by the apply
      K.stem_pool_bn_bwd(self.g_pool, self.pool_idx, self.stem_raw, bn.gamma, bn.mean, bn.invstd,
                         bn.scale, bn.shift, bn.acc[0], bn.acc[1], self.g_stem_raw,
                         acc_dgamma=bn.dgamma, acc_dbeta=bn.dbeta)
    ops.count()   # two launches
    self.p_stem_wgrad.run()

  # ------------------------------------------------------------------ API
  def step_kernels(self):
    """Forward + loss + backward + optimizer on the static buffers (capturable): the micro-step
    ``micro_step`` of the accumulation window, which it does not advance (``train_step`` does)."""
    zero, update = self.accum.phase()
    self._forward(True)
    self._loss(True)
    self._backward(zero, update)
    if update:
      self.optim.finish()

  def capture(self):
    """Capture the training step into CUDA graphs (launch-bound inner loop -> one launch): one
    graph without accumulation; with ``gradient_accumulation_steps`` k > 1 one per kind of
    micro-step (first, middle when k > 2, last), each replayed by ``train_step`` at its position.
    The warm-up trains eagerly: two steps without accumulation, k micro-steps with it.  Returns
    the graph of the updating step."""
    # cross-host communicator: its collectives stay outside the graph (FusedOptimizer.finish()
    # defers them), but the process group's watchdog thread may still poll events of the warm-up
    # collectives - thread-local capture keeps that from invalidating the capture
    mode = "thread_local" if getattr(self.optim, "group_mode", False) else "global"
    # the warm-up steps draw and stage their mix and drop-path factors as train_step does; the
    # graphs read ``mix`` and ``drop_scale``
    draws = self.mixer is not None or self.dropper is not None
    self.graphs = self.accum.capture(self.device, self.step_kernels, mode,
                                     before_step=self._stage_draws if draws else None)
    self.graph = self.graphs[(self.accum.k == 1, True)]
    return self.graph

  def train_step(self, images_u8=None, labels=None):
    if images_u8 is not None:
      self.set_input(images_u8, labels)
    self._stage_draws()
    # a captured step replays its graph; after the updating one a cross-host communicator runs
    # its all-reduce + update outside the graph (after_replay)
    self.accum.run(self.graphs if self.graph is not None else None, self.step_kernels, self.optim)
    return self.loss_sum  # device scalar: mean loss of the step (micro-batch)

  def forward_only(self, images_u8=None):
    if images_u8 is not None:
      self.set_input(images_u8)
    self._forward(False)
    return self.logits

  # ------------------------------------------ inference with folded batch norm
  def build_folded_inference(self, x=None):
    """``x``: the decoded input the stem reads (default ``xp``; a distilling student's ``xp`` for
    its teacher).  Serving path: every batch norm is folded into the convolution in front of it
    (w' = w * gamma / sqrt(var + eps) per output channel, bias = beta - mean * that scale, from
    the fp32 masters and the running statistics), ReLU and the residual add run in the conv
    epilogues (bias / ReLU / accumulate), identity blocks accumulate IN PLACE into their input.
    The forward pass is then 53 wgmma convolutions + 2 pools + the dense head: none of the 53
    batch-norm passes (2/3 of the inference-time HBM traffic) remains.  Call again after the
    parameters or running statistics change (``fold_batch_norms``)."""
    assert not self.training, "folded inference is built on a training=False trainer"
    st, dev = self.store, self.device
    units = self._fold_units()
    self.wf = torch.zeros_like(st.weights)        # folded bf16 filters, same layout as weights
    self.bf = torch.zeros(sum((bn.C + 7) // 8 * 8 for _, bn in units), dtype=torch.float32,
                          device=dev)
    bias, off = {}, 0
    for _, bn in units:
      bias[id(bn)] = self.bf[off:off + bn.C]
      off += (bn.C + 7) // 8 * 8
    self._f_plans, self._f_last = self._folded_plans(lambda spec: st._view(self.wf, spec), bias,
                                                     self.stem_act, x)
    self.fold_batch_norms()

  def _fold_units(self):
    """(filter spec, batch norm) of every convolution followed by a batch norm, stem first."""
    units = [(self.stem_w, self.stem_bn)]
    for b in self.blocks:
      for u in (b.u1, b.u2, b.u3) + ((b.ds,) if b.ds is not None else ()):
        units.append((u.conv.sw, u.bn))
    return units

  def _folded_plans(self, wv, bias, stem_out, x=None):
    """The folded network's convolutions: ``wv(spec)`` is a folded filter, ``bias[id(bn)]`` the
    folded batch norm's bias; the stem reads ``x`` (default ``xp``) and writes ``stem_out``.
    Returns (plans, last activation)."""
    x = self.xp if x is None else x
    plans = [igemm.stem_fprop(x, wv(self.stem_w), stem_out, bias=bias[id(self.stem_bn)],
                              relu=True)]
    cur = self.pool
    for b in self.blocks:
      s_ = b.stride
      plans.append(igemm.conv_fprop(cur, wv(b.u1.conv.sw), b.a1, 1, 0, bias=bias[id(b.u1.bn)],
                                    relu=True))
      plans.append(igemm.conv_fprop(b.a1, wv(b.u2.conv.sw), b.a2, s_, 1, bias=bias[id(b.u2.bn)],
                                    relu=True))
      if b.ds is not None:
        plans.append(igemm.conv_fprop(cur, wv(b.ds.conv.sw), b.out, s_, 0,
                                      bias=bias[id(b.ds.bn)]))
        target = b.out
      else:
        target = cur          # out = relu(conv3 + x): accumulate into x itself
      plans.append(igemm.conv_fprop(b.a2, wv(b.u3.conv.sw), target, 1, 0, bias=bias[id(b.u3.bn)],
                                    relu=True, accumulate=True))
      cur = target
    return plans, cur

  def _eval_forward(self, wv, bias, u8, head=None):
    """Evaluation forward pass on this trainer's activation buffers (see _Evaluator): the stem
    writes ``stem_raw``, which a training trainer has too.  ``head``: what runs the classifier
    (default ``fc.forward``, on the store's head)."""
    plans, last = self._folded_plans(wv, bias, self.stem_raw)
    K = ops.K

    def run():
      K.decode_normalize(u8, self.xp, igemm.STEM_PAD, self.mean, self.std)
      plans[0].run()
      K.maxpool_fwd(self.stem_raw, self.pool, self.pool_idx, 3, 2, 1)
      for p in plans[1:]:
        p.run()
      K.avgpool_fwd(last, self.avg)
      (head or self.fc.forward)()
    return run

  def fold_batch_norms(self):
    st = self.store
    off = 0
    for spec, bn in self._fold_units():
      scale = st.m(bn.sg) * torch.rsqrt(bn.running_var + bn.eps)
      w = st.m(spec).float()
      st._view(self.wf, spec).copy_(w * scale.view(-1, *([1] * (w.dim() - 1))))
      self.bf[off:off + bn.C].copy_(st.m(bn.sb) - bn.running_mean * scale)
      off += (bn.C + 7) // 8 * 8

  def forward_folded(self):
    """logits of the staged batch through the folded network (capturable)."""
    ops.K.decode_normalize(self.in_u8, self.xp, igemm.STEM_PAD, self.mean, self.std)
    return self.run_folded()

  def run_folded(self):
    """``forward_folded`` without the decode: the folded network on the input its stem was built
    to read (``build_folded_inference(x)``); returns ``logits`` (capturable)."""
    K = ops.K
    self._f_plans[0].run()
    K.maxpool_fwd(self.stem_act, self.pool, self.pool_idx, 3, 2, 1)
    for p in self._f_plans[1:]:
      p.run()
    K.avgpool_fwd(self._f_last, self.avg)
    self.fc.forward()
    return self.logits

  # ------------------------------------------------------- held-out evaluation
  def eval_begin(self, averaged=False):
    """Start an evaluation pass: zero the totals, take rank 0's running statistics and fold every
    batch norm into a copy of the current bf16 filters (one launch).  Stream-ordered after the
    last ``train_step``; the first call allocates the evaluation buffers and plans.
    ``averaged=True`` folds the weight average instead (``ema_decay``; RuntimeError without it):
    the model ``averaged()`` exports, with the live running statistics."""
    if averaged:
      self._check_average()
    if getattr(self, "_evaluator", None) is None:
      self._evaluator = _Evaluator(self)
    self._evaluator.begin(averaged)

  def eval_step(self, images_u8, labels):
    """Add the top-1 / top-5 / loss totals of n <= B images (host or device, uint8 NHWC) and their
    labels (``multi_label``: bool or uint8 [n, V] targets and the multi-label totals).  Runs the
    folded network on the training buffers, leaving ``in_u8`` / ``labels`` and the training state
    untouched; ``logits`` then holds the batch's logits.  No host sync."""
    self._eval_state().step(images_u8, labels)

  def eval_end(self):
    """Totals summed over all ranks (identical on every rank): {"count", "loss", "top1", "top5"};
    the last three are means over ``count`` (NaN when it is 0).  ``loss`` is the plain
    cross-entropy whatever the trainer's ``label_smoothing``, so that scores of runs with different
    smoothing compare.  Raises ValueError on every rank when any rank saw a label outside
    [0, num_classes).  With ``multi_label``: {"count", "loss", "binary_accuracy", "exact_match",
    "precision", "recall", "f1", "macro_f1", "f1_per_class"} (``multilabel_totals``; the loss is
    the plain BCE, a mean over count * V), and the ValueError is for a label byte other than 0 / 1."""
    return self._eval_state().end()

  def evaluate(self, batches, averaged=False):
    """eval_begin(averaged) + eval_step over ``(images, labels)`` pairs + eval_end.  Host batches
    go through page-locked staging: the copy of batch i + 1 overlaps the forward pass of batch i."""
    self.eval_begin(averaged)
    self._evaluator.run(batches)
    return self.eval_end()

  def _check_average(self):
    if getattr(self.optim, "ema", None) is None:
      raise RuntimeError("this trainer keeps no weight average: build it with ema_decay=d")

  @property
  def grad_norm(self):
    """Device fp32 [1]: the global norm N of the last step's averaged gradient, before clipping
    (updated by every replay of the captured step); None without ``clip_norm``."""
    return self.optim.grad_norm if self.optim is not None else None

  def averaged(self):
    """Snapshot of the weight average as an exportable model (engine.AveragedModel): its
    ``state_dict()`` is this trainer's with every parameter replaced by its average and the live
    running statistics, so ``checkpoint.export_model(net.averaged(), dir)`` exports the average as
    Keras does after ``finalize_variable_values()``.  RuntimeError without ``ema_decay``."""
    self._check_average()
    sd, _ = engine.averaged_params(self.store, self.optim)
    sd["__running__"] = self.running.tensor().detach().cpu().clone()
    return engine.AveragedModel(sd, self)

  def _eval_state(self):
    if getattr(self, "_evaluator", None) is None:
      raise RuntimeError("eval_begin() has not been called")
    return self._evaluator

  def set_lr(self, lr):
    self.optim.set_lr(lr)

  # ------------------------------------------------- checkpoints / serving
  export_builder = "tensorflowonspark_b200.models.resnet:build_served"

  @property
  def export_signatures(self):
    """logits [n, V] fp32 and prediction: the arg-max class (int64 [n]), or with ``multi_label``
    the multi-hot uint8 [n, V] of logit > 0, one bytes cell of V values per row (as the U-Net's
    mask)."""
    sig = {"inputs": {"image": "image"}, "outputs": {"logits": "logits", "prediction": "prediction"},
           "input_dtypes": {"image": "uint8"}}
    if self.multi_label:
      sig["output_dtypes"] = {"prediction": "uint8"}
      sig["output_shapes"] = {"logits": [-1, self.num_classes],
                              "prediction": [-1, self.num_classes]}
    return {"serving_default": sig}

  @property
  def export_builder_args(self):
    args = {"depth": self.depth, "image": self.image, "num_classes": self.num_classes}
    if self.multi_label:   # an export without the key serves as softmax
      args["multi_label"] = True
    return args

  def state_dict(self):
    """Parameters (fp32 masters, assembled across ranks when sharded) + the batch-norm running
    statistics: everything inference or a resumed run needs."""
    sd = dict(self.store.state_dict())
    sd["__running__"] = self.running.tensor().detach().cpu().clone()
    return sd

  def load_state_dict(self, sd):
    """Parameters and running statistics of ``state_dict()``; resets the weight average (the
    optimizer's ``load_state_dict`` restores a saved one) and restarts the accumulation window
    (partial sums dropped, ``micro_step = 0``).  ``state_dict()`` may be taken mid-window; it
    holds no partial sums."""
    sd = dict(sd)
    running = sd.pop("__running__", None)
    self.store.load_state_dict(sd)
    if running is not None:
      self.running.tensor().copy_(running.to(self.device))
    if self.optim is not None:
      self.optim.reset_average()
      self.accum.restart(self.optim)

  def load_backbone(self, state):
    """Start from a trained backbone: ``state`` is the ``state_dict()`` of a trainer of the same
    depth with any class count.  Loads every parameter except the classifier (``fc.w``, ``fc.b``)
    and the batch-norm running statistics (``__running__``), like ``load_state_dict``; the head
    keeps its seeded initialisation and the optimizer state is untouched.  Every tensor is checked
    before anything is copied: a missing, unexpected or wrongly shaped one raises ValueError and
    leaves the trainer as it was.  Resets the weight average."""
    want = {s["name"]: s["shape"] for s in self.store.order if s["name"] not in _HEAD}
    want["__running__"] = tuple(self.running.tensor().shape)
    extra = sorted(set(state) - set(want) - set(_HEAD))
    if extra:
      raise ValueError("load_backbone: {} is not a tensor of this trainer (another depth?)".format(
          extra[0]))
    for name, shape in want.items():
      if name not in state:
        raise ValueError("load_backbone: {} {} is missing from the state (another depth?)".format(
            name, shape))
      got = tuple(state[name].shape)
      if got != shape:
        raise ValueError("load_backbone: {} has shape {} in the state, {} in this trainer".format(
            name, got, shape))
    self.load_state_dict({k: v for k, v in state.items() if k not in _HEAD})


class ServedResNet(serving.Replica):
  """Inference callable behind ``pipeline.TFModel`` / ``TFParallel``: one bf16 replica on the
  executor's GPU.  ``submit(inputs)`` stages a uint8 NHWC batch in page-locked memory, copies it
  on the copy stream and enqueues the forward pass (~165 launches) + arg-max and an async
  read-back of ``logits`` and ``prediction``; ``collect()`` returns the oldest submitted batch
  (models/serving.Replica).  ``multi_label``: ``prediction`` is the multi-hot uint8 [n, V] of
  logit > 0 instead of the arg-max."""

  def __init__(self, state, depth=50, image=224, num_classes=1000, batch=256, device="cuda:0",
               multi_label=False):
    torch.cuda.set_device(torch.device(device))
    self.net = ResNetTrainer(depth=depth, batch=batch, image=image, num_classes=num_classes,
                             device=device, training=False, multi_label=multi_label)
    self.net.load_state_dict(state)
    self.folded = os.environ.get("TFOS_SERVE_FOLD_BN", "1") == "1"
    if self.folded:
      self.net.build_folded_inference()
    self._fwd = self.net.forward_folded if self.folded else (lambda: self.net._forward(False))
    self.image, self.V, self.multi_label = image, num_classes, multi_label
    if multi_label:
      self.pred_dev = torch.zeros((batch, num_classes), dtype=torch.uint8, device=self.net.device)
    else:
      self.pred_dev = torch.zeros(batch, dtype=torch.int64, device=self.net.device)
    super(ServedResNet, self).__init__(
        self.net.device, batch, (image, image, 3),
        {"logits": self.net.logits[:, :num_classes], "prediction": self.pred_dev},
        self.net.set_input)

  def _run(self):
    self._fwd()
    if self.multi_label:
      self.pred_dev.copy_(self.net.logits[:, :self.V] > 0)
    else:
      self.pred_dev.copy_(self.net.logits[:, :self.V].argmax(1))


def build_served(state, depth=50, image=224, num_classes=1000, batch=None, multi_label=False, **_):
  """Export builder (utils/checkpoint.py): rebuilds the replica on the executor's GPU.  An export
  written before multi-label heads existed has no ``multi_label`` and serves as softmax."""
  return ServedResNet(state, depth=depth, image=image, num_classes=num_classes,
                      batch=serving.serve_batch(batch), multi_label=bool(multi_label))


class _ResNetTeacher(object):
  """Frozen distillation teacher of a ResNetTrainer: a ``training=False`` replica of ``depth``
  on the student's device and batch, loaded from ``state`` and folded once
  (``build_folded_inference``), whose stem reads the student's decoded input ``xp``.  ``run()``
  launches its folded forward pass (convolutions, pools, head); it writes only the replica's own
  buffers and leaves the teacher's logits in ``logits``."""

  def __init__(self, student, state, depth):
    self.net = ResNetTrainer(depth=depth, batch=student.B, image=student.image,
                             num_classes=student.num_classes, device=student.device,
                             training=False)
    self.net.load_state_dict(state)
    self.net.build_folded_inference(x=student.xp)
    self.logits = self.net.logits

  def run(self):
    self.net.run_folded()


class _CifarTeacher(object):
  """Frozen distillation teacher of a CifarResNetTrainer: a CifarResNetTrainer of ``depth`` on the
  student's device and batch, loaded from ``state``, with every batch norm folded once on the host
  (``ResNetTrainer.fold_batch_norms``: fp32 masters and running statistics) into a copy of its
  filters.  Its folded plans (``_folded_plans``) read the student's decoded input ``x8``; ``run()``
  launches them, the average pool and the head, writing only the teacher's own buffers, and
  leaves the teacher's logits in ``logits``.  Its optimizer is never stepped."""

  def __init__(self, student, state, depth):
    net = self.net = CifarResNetTrainer(depth=depth, batch=student.B,
                                        num_classes=student.num_classes, device=student.device)
    net.load_state_dict(state)
    st = net.store
    units = net._fold_units()
    net.wf = torch.zeros_like(st.weights)
    net.bf = torch.zeros(sum((bn.C + 7) // 8 * 8 for _, bn in units), dtype=torch.float32,
                         device=net.device)
    bias, off = {}, 0
    for _, bn in units:
      bias[id(bn)] = net.bf[off:off + bn.C]
      off += (bn.C + 7) // 8 * 8
    ResNetTrainer.fold_batch_norms(net)
    self.plans, self.last = net._folded_plans(lambda spec: st._view(net.wf, spec), bias,
                                              student.x8)
    self.logits = net.logits

  def run(self):
    for p in self.plans:
      p.run()
    ops.K.avgpool_fwd(self.last, self.net.avg)
    self.net.fc.forward()


class CifarResNetTrainer(object):
  """ResNet-20/32/56 for 32x32 inputs (basic blocks, 16/32/64 channels) - the network the
  reference example actually trains (examples/resnet/resnet_cifar_dist.py:208, ``resnet56``,
  momentum SGD, batch 128, weight decay 2e-4).  ``optimizer``, ``num_classes``,
  ``label_smoothing``, ``ema_decay``, ``clip_norm``, ``beta1``, ``beta2``, ``epsilon``,
  ``gradient_accumulation_steps``, ``multi_label``, ``pos_weight``, ``mixup_alpha``,
  ``cutmix_alpha``, ``mix_prob``, ``mix_switch_prob``, ``drop_path_rate``, ``teacher``,
  ``teacher_depth``, ``distill_alpha`` and ``distill_temperature`` as in ResNetTrainer (the CutMix
  box is drawn on the 32 x 32 image; stochastic depth scales the output of each basic block's
  second batch norm, as in timm's ``BasicBlock``; the teacher is the ``state_dict()`` of a
  CifarResNetTrainer of any valid depth, folded once on the host, whose folded convolutions read
  the student's decoded ``x8``)."""

  def __init__(self, depth=56, batch=128, num_classes=10, device="cuda:0", lr=0.1, momentum=0.9,
               weight_decay=2e-4, comm=None, seed=1234, optimizer="momentum",
               trust_coefficient=0.001, label_smoothing=0.0, ema_decay=None, clip_norm=None,
               beta1=0.9, beta2=0.999, epsilon=1e-7, gradient_accumulation_steps=1,
               multi_label=False, pos_weight=None, mixup_alpha=0.0, cutmix_alpha=0.0, mix_prob=1.0,
               mix_switch_prob=0.5, drop_path_rate=0.0, teacher=None, teacher_depth=None,
               distill_alpha=0.5, distill_temperature=1.0):
    num_classes, self.label_smoothing = _check_head_args(num_classes, label_smoothing)
    self.multi_label, pos_weight = _check_multilabel_args(multi_label, pos_weight, num_classes)
    mix_args = engine.check_mix_args(mixup_alpha, cutmix_alpha, mix_prob, mix_switch_prob)
    self.drop_path_rate = engine.check_drop_path_rate(drop_path_rate)
    self.teacher_depth, self.distill_alpha, self.distill_temperature = _check_teacher(
        type(self), teacher, teacher_depth, distill_alpha, distill_temperature, depth, num_classes,
        True, self.multi_label)
    k_acc = engine.check_gradient_accumulation_steps(gradient_accumulation_steps)
    self.ema_decay = engine.check_ema_decay(ema_decay)
    self.clip_norm = engine.check_clip_norm(clip_norm)
    beta1, beta2, epsilon = engine.check_adam_args(beta1, beta2, epsilon)
    assert (depth - 2) % 6 == 0
    self.device = dev = torch.device(device)
    self.B, self.image, self.num_classes = batch, 32, num_classes
    self.comm = comm
    self.VP = (num_classes + 7) // 8 * 8
    B = batch
    st = self.store = ParamStore()
    self.stem, self.blocks, self.fc = self._register(st, depth, num_classes)
    self.drop_path_rates = engine.drop_path_rates(self.drop_path_rate, len(self.blocks))
    st.finalize(dev, alloc=comm.alloc if comm is not None else None, seed=seed)

    self.in_u8 = _buf((B, 32, 32, 3), dev, torch.uint8)
    self.x8 = _buf((B, 32, 32, 8), dev)
    self.labels = _labels_buffer(B, num_classes, self.multi_label, dev)
    self.pos_weight = None if pos_weight is None else torch.tensor(pos_weight, dtype=torch.float32,
                                                                   device=dev)
    self.stem_raw, self.stem_act = _buf((B, 32, 32, 16), dev), _buf((B, 32, 32, 16), dev)
    self.g_stem_raw = _buf((B, 32, 32, 16), dev)
    self.running = engine.RunningArena(dev)
    self.stem.bn.build(dev, None, self.running)
    gx = _buf((B, 32, 32, 16), dev)
    self.g_stem_act = gx
    self.stem.conv.build(self.x8, self.stem_raw, self.g_stem_raw, None, stats=self.stem.bn.stats,
                         need_dgrad=False)
    x, H = self.stem_act, 32
    for b in self.blocks:
      H2, w = (H - 1) // b.stride + 1, b.width
      b.x = x
      b.r1, b.a1 = _buf((B, H2, H2, w), dev), _buf((B, H2, H2, w), dev)
      b.r2, b.out = _buf((B, H2, H2, w), dev), _buf((B, H2, H2, w), dev)
      b.g_r1, b.g_a1, b.g_r2 = _buf(b.r1.shape, dev), _buf(b.a1.shape, dev), _buf(b.r2.shape, dev)
      b.g_out = _buf(b.out.shape, dev) if b.ds is not None else gx
      b.g_x = gx
      for u in (b.u1, b.u2) + ((b.ds,) if b.ds else ()):
        u.bn.build(dev, None, self.running)
      ident = b.ds is None
      b.u1.conv.build(x, b.r1, b.g_r1, b.g_x, stats=b.u1.bn.stats, dx_accumulate=ident)
      b.u2.conv.build(b.a1, b.r2, b.g_r2, b.g_a1, stats=b.u2.bn.stats)
      if b.ds is not None:
        b.rd, b.idn, b.g_rd = _buf(b.r2.shape, dev), _buf(b.r2.shape, dev), _buf(b.r2.shape, dev)
        b.ds.conv.build(x, b.rd, b.g_rd, b.g_x, stats=b.ds.bn.stats, dx_accumulate=True)
      x, H, gx = b.out, H2, b.g_out
    self.last, self.g_last = x, gx
    self.avg, self.g_avg = _buf((B, 64), dev), _buf((B, 64), dev)
    self.logits = _buf((B, self.VP), dev, torch.float32)
    self.dlogits = _buf((B, self.VP), dev)
    self.loss_sum = torch.zeros(1, dtype=torch.float32, device=dev)
    self.correct = torch.zeros(1, dtype=torch.float32, device=dev)
    self.fc.build(self.avg, self.logits, self.dlogits, self.g_avg)
    from ..parallel.fused_optim import FusedOptimizer
    self.optim = FusedOptimizer(st, comm=comm, opt=optimizer, lr=lr, momentum=momentum,
                                weight_decay=weight_decay, trust_coefficient=trust_coefficient,
                                ema_decay=self.ema_decay, clip_norm=self.clip_norm, beta1=beta1,
                                beta2=beta2, eps=epsilon)
    # accumulation: the batch norms have no statistics arena; their per-micro-batch dgamma /
    # dbeta live in one of their own, zeroed once per micro-step
    self.grad_scratch = None
    if k_acc > 1:
      self.optim.set_accumulation(k_acc)
      self.grad_scratch = engine.StatsArena(dev)
      for _, bn in self._fold_units():
        bn.accumulate_grads(self.grad_scratch)
    self.accum = engine.GradAccumulation(k_acc)
    self._build_mix(mix_args, seed)
    self._build_drop_path(seed)
    self.graph = None
    self.graphs = None
    self.mean, self.std = [0.4914, 0.4822, 0.4465], [0.2470, 0.2435, 0.2616]
    self.teacher = None if teacher is None else _CifarTeacher(self, teacher, self.teacher_depth)

  @staticmethod
  def _register(st, depth, num_classes):
    """Register the parameters of a CIFAR ResNet-``depth`` in ``st`` (host only).  Returns (stem
    unit, blocks, head)."""
    n = (depth - 2) // 6
    stem = _Unit(st, "stem", 8, 16, 3, 1)
    blocks = []
    cin = 16
    for si, width in enumerate((16, 32, 64)):
      for bi in range(n):
        stride = 2 if (bi == 0 and si > 0) else 1
        b = _Block()
        name = "stage{}.{}".format(si + 1, bi)
        b.u1 = _Unit(st, name + ".u1", cin, width, 3, stride)
        b.u2 = _Unit(st, name + ".u2", width, width, 3, 1, zero_gamma=True)
        b.ds = _Unit(st, name + ".ds", cin, width, 1, stride) if stride != 1 else None
        b.stride, b.width = stride, width
        blocks.append(b)
        cin = width
    fc = Dense(st, "fc", 64, (num_classes + 7) // 8 * 8, bias=True, init=normal(0.01))
    return stem, blocks, fc

  @staticmethod
  def _valid_depth(depth):
    return (isinstance(depth, numbers.Integral) and not isinstance(depth, bool) and depth >= 8 and
            (depth - 2) % 6 == 0)

  synthetic_batch = ResNetTrainer.synthetic_batch
  state_dict = ResNetTrainer.state_dict
  load_state_dict = ResNetTrainer.load_state_dict
  load_backbone = ResNetTrainer.load_backbone
  set_input = ResNetTrainer.set_input
  _loss = ResNetTrainer._loss
  capture = ResNetTrainer.capture
  train_step = ResNetTrainer.train_step
  set_lr = ResNetTrainer.set_lr
  eval_begin = ResNetTrainer.eval_begin
  eval_step = ResNetTrainer.eval_step
  eval_end = ResNetTrainer.eval_end
  evaluate = ResNetTrainer.evaluate
  _eval_state = ResNetTrainer._eval_state
  _check_average = ResNetTrainer._check_average
  averaged = ResNetTrainer.averaged
  grad_norm = ResNetTrainer.grad_norm
  gradient_accumulation_steps = ResNetTrainer.gradient_accumulation_steps
  micro_step = ResNetTrainer.micro_step
  _build_mix = ResNetTrainer._build_mix
  _stage_mix = ResNetTrainer._stage_mix
  _mix_arg = ResNetTrainer._mix_arg
  _build_drop_path = ResNetTrainer._build_drop_path
  _stage_draws = ResNetTrainer._stage_draws
  _drop_arg = ResNetTrainer._drop_arg

  def _fold_units(self):
    """(filter spec, batch norm) of every convolution followed by a batch norm, stem first."""
    units = [(self.stem.conv.sw, self.stem.bn)]
    for b in self.blocks:
      for u in (b.u1, b.u2) + ((b.ds,) if b.ds is not None else ()):
        units.append((u.conv.sw, u.bn))
    return units

  def _folded_plans(self, wv, bias, x=None):
    """The folded basic-block network on the training buffers: bias + ReLU in every epilogue, the
    shortcut into ``out``, conv2 accumulating the residual into ``out`` (projection blocks) or in
    place into the block input (identity blocks).  The stem reads ``x`` (default ``x8``).
    Returns (plans, last activation)."""
    conv = lambda x, u, y, **kw: igemm.conv_fprop(  # noqa: E731
        x, wv(u.conv.sw), y, u.conv.stride, u.conv.pad, bias=bias[id(u.bn)], **kw)
    cur = self.stem_act
    plans = [conv(self.x8 if x is None else x, self.stem, cur, relu=True)]
    for b in self.blocks:
      plans.append(conv(cur, b.u1, b.a1, relu=True))
      if b.ds is not None:
        plans.append(conv(cur, b.ds, b.out))
        cur = b.out
      plans.append(conv(b.a1, b.u2, cur, relu=True, accumulate=True))
    return plans, cur

  def _eval_forward(self, wv, bias, u8, head=None):
    """Folded basic-block network (``_folded_plans``) on the training buffers (see _Evaluator).
    ``head`` as in ResNetTrainer."""
    plans, last = self._folded_plans(wv, bias)
    K = ops.K

    def run():
      K.decode_normalize(u8, self.x8, 0, self.mean, self.std)
      for p in plans:
        p.run()
      K.avgpool_fwd(last, self.avg)
      (head or self.fc.forward)()
    return run

  def step_kernels(self):
    K = ops.K
    zero, update = self.accum.phase()
    K.decode_normalize(self.in_u8, self.x8, 0, self.mean, self.std, **self._mix_arg())
    if self.teacher is not None:
      self.teacher.run()      # its stem reads x8: the (mixed) input the student trains on
    self.stem.conv.forward()
    self.stem.bn.forward(self.stem_raw, self.stem_act, None, 1, True)
    for bi, b in enumerate(self.blocks):
      b.u1.conv.forward()
      b.u1.bn.forward(b.r1, b.a1, None, 1, True)
      b.u2.conv.forward()
      if b.ds is not None:
        b.ds.conv.forward()
        b.ds.bn.forward(b.rd, b.idn, None, 0, True)
      b.u2.bn.forward(b.r2, b.out, b.idn if b.ds is not None else b.x, 1, True,
                      **self._drop_arg(bi))
    K.avgpool_fwd(self.last, self.avg)
    self.fc.forward()
    self._loss(True)
    if zero:
      self.optim.zero_grads()
    if self.grad_scratch is not None:
      self.grad_scratch.zero()
    self.fc.backward()
    K.avgpool_bwd(self.g_avg, self.g_last)
    for bi in reversed(range(len(self.blocks))):
      b = self.blocks[bi]
      # stochastic depth: u2's dx is formed from s_b * the masked gradient; dres (the shortcut's,
      # written in place into g_out) stays unscaled
      b.u2.bn.backward(b.g_out, b.r2, b.out, b.g_r2, dres=b.g_out, relu=True, **self._drop_arg(bi))
      b.u2.conv.backward()
      b.u1.bn.backward(b.g_a1, b.r1, b.a1, b.g_r1, relu=True)
      b.u1.conv.backward()
      if b.ds is not None:
        b.ds.bn.backward(b.g_out, b.rd, None, b.g_rd, relu=False)
        b.ds.conv.backward()
    self.stem.bn.backward(self.g_stem_act, self.stem_raw, self.stem_act, self.g_stem_raw, relu=True)
    self.stem.conv.backward()
    if update:
      self.optim.step()


def piecewise_lr(epoch, batch_size, base=0.1, boundaries=(91, 136, 182), factors=(0.1, 0.01, 0.001)):
  """LR schedule of the reference ResNet example (resnet_cifar_dist.py:35-66):
  0.1 * bs/128, multiplied by 0.1 / 0.01 / 0.001 from epochs 91 / 136 / 182."""
  lr = base * batch_size / 128.0
  for b, f in zip(boundaries, factors):
    if epoch >= b:
      lr = base * batch_size / 128.0 * f
  return lr


def poly_warmup_lr(step, total_steps, base_lr, warmup_steps, end_lr=0.0, power=2.0):
  """Large-batch (LARS) schedule: linear warm-up from 0 to ``base_lr`` over ``warmup_steps``
  steps (``step`` 0 .. ``warmup_steps - 1`` take ``base_lr * (step + 1) / warmup_steps``), then
  polynomial decay ``end_lr + (base_lr - end_lr) * (1 - p) ** power``, where p runs from 0 at
  ``step = warmup_steps`` to 1 at ``step = total_steps``."""
  if step < warmup_steps:
    return base_lr * (step + 1) / float(warmup_steps)
  decay_steps = max(1, total_steps - warmup_steps)
  p = min(1.0, float(step - warmup_steps) / decay_steps)
  return end_lr + (base_lr - end_lr) * (1.0 - p) ** power

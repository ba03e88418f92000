"""Fused gradient all-reduce + optimizer step (csrc/optim_comm.cu).

Replaces the collective the reference gets from
``tf.distribute.experimental.MultiWorkerMirroredStrategy`` (reference user code:
examples/mnist/keras/mnist_spark.py:11,55-66; TFoS itself only provides the
cluster spec, tensorflowonspark/TFSparkNode.py:373-384) *and* the Keras
optimizer update that follows it: one kernel per gradient bucket pulls the peer
shards over NVLink, averages, applies SGD / momentum / Adam to the fp32 master
shard and stores the new bf16 weights into every rank's weight buffer (also AdamW, LARS and
LAMB, below).

Buckets are contiguous ranges of the flat parameter vector.  A model may pass
``buckets=[(begin, end, tag), ...]`` and call ``launch(tag)`` from inside its
backward pass as soon as the gradients of that range are final; the kernels then
run on a dedicated communication stream, overlapped with the rest of backward,
and ``finish()`` joins the streams (``exposed_ms()`` reports how long that join
actually waited).  ``step()`` = everything at once on the current stream.

Across hosts (``comm`` is a parallel/group_comm.GroupComm) the peer loads are replaced by a
``torch.distributed`` all-reduce of each bucket, followed by the same kernel in its single-rank
form with scale 1 / world, replicated on every rank.  The collective is not recorded into a
CUDA graph: while a trainer captures its step, ``finish()`` only notes that the update is due,
and ``after_replay()`` - called by the trainers after every graph replay - runs it eagerly.

LARS (``opt="lars"``) gives every adapted tensor - the decayed head: conv and dense weights -
its own trust ratio ``eta * |w| / (|g| + wd * |w|)`` from the norms of its fp32 master and of
its AVERAGED gradient, and runs momentum with lr * trust applied inside the velocity:
``v = m v + lr trust (g + wd w); w = w - v``.  The non-decayed tail takes ``v = m v + lr g``.
``state1`` holds that velocity (momentum's ``state1`` does not carry lr, so a momentum checkpoint
does not continue under LARS).  The norms need the whole reduced tensor, so every bucket runs a
separate, deterministic norm pass (csrc/optim_comm.cu ``lars_norms``) between the reduce-scatter
and the update: ``[PHASE 1 ->] norms (+ exchange of per-tensor partials among the local peers)
-> update [+ all-gather]``.  A bucket bound must not cut an adapted tensor.

AdamW (``opt="adamw"``) is ``torch.optim.AdamW`` / Keras's ``AdamW``: decoupled weight decay on the
decayed head, ``w = w (1 - lr wd)``, then Adam's step ``w = w - lr (m / c1) / (sqrt(v / c2) + eps)``
(``opt="adam"`` folds ``wd w`` into the gradient instead).  With ``wd = 0`` it is bitwise Adam.

LAMB (``opt="lamb"``, the LAMB paper's Algorithm 2 as in apex ``FusedLAMB`` / TF Addons ``LAMB``)
is to Adam what LARS is to momentum: ``r = (m / c1) / (sqrt(v / c2) + eps) + wd w`` and, for each
adapted tensor, ``w = w - lr ratio r`` with ``ratio = |w| / |r|`` (1 if a norm is 0) from the fp32
master before the step and the step's new moments; the tail takes ``w = w - lr r`` without decay.
``trust_coefficient`` is not used.  It runs in LARS's shape: the same tables and bucket rules, and
a norm pass between the reduce-scatter and the update that recomputes m', v' and r in registers
(it writes no state, so the update alone advances it, once per step).  adam, adamw and lamb share
their state (``state1 = m``, ``state2 = v``, ``hyper[7] = t``) and hyper layout, so a checkpoint of
one continues under the others.

Weight average (``ema_decay=d``): the update kernels also keep an exponential moving average of
every parameter, ``ema``, placed and sharded like ``state1``.  The first update after a reset
(construction, ``reset_average()``, loading a state without it) copies the new master, each later
one applies ``avg = d avg + (1 - d) w`` in fp32 to the master just written - the rule of Keras's
``use_ema`` optimizers.  d and the update count n live in ``hyper[8]`` / ``hyper[9]`` and n
advances on the device like Adam's step, so a replayed CUDA graph keeps averaging.  Training is
unchanged bit for bit; ``averaged_weights()`` rounds the average into the layout of the store's
bf16 weights and fp32 tail for evaluation and export.

Gradient clipping by global norm (``clip_norm=c``): ``torch.nn.utils.clip_grad_norm_(max_norm=c)``
applied to the averaged gradient ``g = hyper[3] * sum_r g_r`` before the update.  The averaged
gradient only exists inside the fused kernels, so they compute its norm N over the whole vector
(every bucket, decayed head and fp32 tail) in a fixed order, without float atomics:
``N = |hyper[3]| sqrt(sum of per-rank, per-bucket sums of squares)``.  ``coef = c / (N + 1e-6)``
clamped to at most 1 (a NaN norm gives NaN, an infinite one 0, as in torch) is folded into the
scale: the update kernels read a per-step copy of ``hyper``, ``hyper_step``, whose slot 3 is
``fl(hyper[3] * coef)``, so every optimizer (and LARS's trust ratio) sees the clipped gradient and
weight decay is added after clipping.  LAMB's ratio is not linear in the gradient, so its norm pass
must see the clipped one: with clipping it runs after ``clip_finalize``, reading ``hyper_step``.
When ``c / (N + 1e-6) >= 1`` (``c = inf`` included) the step is bitwise the unclipped one.  No
bucket may update before every bucket is reduced, so a bucket's ``launch(tag)`` runs only its
reduction and sum of squares; ``finish()`` (or ``after_replay()``)
finalises N into ``grad_norm`` and runs every bucket's update:

  no peers / GroupComm : [NCCL all-reduce ->] grad_sumsq of the bucket
  one host, P2P / NVLS : PHASE 3 (reduce-scatter + sum of squares of the shard, published to
                         every peer's table before the exit barrier)
  HierComm             : [PHASE 1 ->] NCCL all-reduce of the shard -> grad_sumsq of the shard
                         (+ exchange among the local peers)
  LARS                 : any of the above, then the bucket's lars_norms
  then, once           : clip_finalize -> every bucket's [LAMB norm pass ->] update (PHASE 0 or 2),
                         both reading hyper_step
"""
import bisect
import math
import numbers

import torch

from .. import ops

# kernel codes (csrc/ops.h kOpt*).  OPTS keeps the four it has always had (code that enumerates it
# sees the same set); OPTIMIZERS is every optimizer FusedOptimizer runs.
OPTS = {"sgd": 0, "momentum": 1, "adam": 2, "lars": 3}
OPTIMIZERS = dict(OPTS, adamw=4, lamb=5)
# the optimizers with Adam's state: state1 = m, state2 = v, hyper[7] = step
ADAM_STATE = (OPTIMIZERS["adam"], OPTIMIZERS["adamw"], OPTIMIZERS["lamb"])
# csrc/ops.h kLarsMaxTensors: adapted tensors one shard of a bucket may intersect
LARS_MAX_TENSORS = 256
# elements per work item of the LARS norm pass (one CTA reduces one segment at a time)
LARS_SEGMENT = 16384


# hyper-parameter slots: lr, momentum, wd, grad scale, beta1 | eta, beta2, eps, Adam step; with a
# weight average also its decay and update count (csrc/ops.h kHyper / kHyperEma)
HYPER, HYPER_EMA = 8, 10


def check_ema_decay(d):
  """Validated ``ema_decay``: None, or a real number in [0, 1) as a float (ValueError otherwise)."""
  if d is None:
    return None
  if isinstance(d, bool) or not isinstance(d, numbers.Real) or not 0.0 <= float(d) < 1.0:
    raise ValueError("ema_decay must be None or a real number in [0, 1), got {!r}".format(d))
  return float(d)


def check_clip_norm(c):
  """Validated ``clip_norm``: None, or a real number > 0 (inf allowed) as a float (ValueError
  otherwise: bools, NaN, zero, negative numbers and non-numbers)."""
  if c is None:
    return None
  if isinstance(c, bool) or not isinstance(c, numbers.Real) or not float(c) > 0.0:
    raise ValueError("clip_norm must be None or a real number > 0 (inf allowed), got {!r}".format(c))
  return float(c)


def check_adam_args(beta1, beta2, epsilon):
  """Validated ``(beta1, beta2, epsilon)`` of the Adam family as floats: each beta a real number in
  [0, 1), epsilon a finite real number > 0 (ValueError otherwise, bools included)."""
  for name, b in (("beta1", beta1), ("beta2", beta2)):
    if isinstance(b, bool) or not isinstance(b, numbers.Real) or not 0.0 <= float(b) < 1.0:
      raise ValueError("{} must be a real number in [0, 1), got {!r}".format(name, b))
  if (isinstance(epsilon, bool) or not isinstance(epsilon, numbers.Real)
      or not (math.isfinite(float(epsilon)) and float(epsilon) > 0.0)):
    raise ValueError("epsilon must be a finite real number > 0, got {!r}".format(epsilon))
  return float(beta1), float(beta2), float(epsilon)


def check_weight_decay(wd):
  """Validated ``weight_decay``: a finite real number >= 0 as a float (ValueError otherwise)."""
  if (isinstance(wd, bool) or not isinstance(wd, numbers.Real)
      or not (math.isfinite(float(wd)) and float(wd) >= 0.0)):
    raise ValueError("weight_decay must be a finite real number >= 0, got {!r}".format(wd))
  return float(wd)


def _shard(b, e, world, rank):
  """[lo, hi) of ``rank``'s shard of bucket [b, e) - the arithmetic of allreduce_opt_kernel."""
  n = e - b
  chunk = ((n + world - 1) // world + 7) // 8 * 8
  return b + min(n, chunk * rank), b + min(n, chunk * (rank + 1))


def lars_tables(bounds, buckets, world, seg_len=LARS_SEGMENT):
  """Work tables of the LARS norm pass.

  ``bounds``: the adapted tensors tile ``[0, bounds[-1])`` (= ``decay_end``), tensor ``t`` being
  ``[bounds[t], bounds[t + 1])``.  ``buckets``: ``(begin, end, ...)`` element ranges.  Returns,
  per bucket and per rank, ``{"t0", "nt", "seg", "tseg"}``: the shard intersects tensors
  ``t0 .. t0 + nt - 1``; ``seg`` lists ``(lo, hi)`` segments of at most ``seg_len`` elements, each
  inside one tensor and the shard, tensor after tensor; ``tseg[j] .. tseg[j + 1]`` are local
  tensor ``j``'s segments.  Raises ValueError when a bucket bound falls inside an adapted tensor
  or a shard intersects more than LARS_MAX_TENSORS of them."""
  assert seg_len % 8 == 0 and seg_len > 0
  decay_end = bounds[-1]
  starts = set(bounds)
  out = []
  for bi, bk in enumerate(buckets):
    b, e = bk[0], bk[1]
    for x in (b, e):
      if 0 < x < decay_end and x not in starts:
        raise ValueError("LARS: bucket {} bound {} falls inside an adapted tensor (each tensor's "
                         "norm must come from one bucket)".format(bi, x))
    per_rank = []
    for r in range(world):
      lo, hi = _shard(b, e, world, r)
      ahi = min(hi, decay_end)
      tab = {"t0": 0, "nt": 0, "seg": [], "tseg": [0]}
      if lo < ahi:
        t0 = bisect.bisect_right(bounds, lo) - 1
        t1 = bisect.bisect_left(bounds, ahi)
        if t1 - t0 > LARS_MAX_TENSORS:
          raise ValueError("LARS: rank {}'s shard of bucket {} intersects {} adapted tensors; the "
                           "update kernel holds at most {} (split the bucket)".format(
                               r, bi, t1 - t0, LARS_MAX_TENSORS))
        tab["t0"], tab["nt"] = t0, t1 - t0
        for t in range(t0, t1):
          s, stop = max(bounds[t], lo), min(bounds[t + 1], ahi)
          while s < stop:
            tab["seg"].append((s, min(stop, s + seg_len)))
            s += seg_len
          tab["tseg"].append(len(tab["seg"]))
      per_rank.append(tab)
    out.append(per_rank)
  return out


class FusedOptimizer(object):

  def __init__(self, store, comm=None, opt="momentum", lr=0.1, momentum=0.9, weight_decay=0.0,
               beta1=0.9, beta2=0.999, eps=1e-7, buckets=None, trust_coefficient=0.001,
               ema_decay=None, clip_norm=None):
    """``trust_coefficient``: LARS eta (``opt="lars"``; it takes the slot of Adam's beta1 in
    the hyper-parameter vector, which LARS does not use).  ``ema_decay``: None (no average) or
    the decay d in [0, 1) of the weight average.  ``clip_norm``: None or the global-norm
    threshold c > 0 (inf: measure only); ``grad_norm`` then holds N of the last step (see the
    module docstring)."""
    self.ema_decay = check_ema_decay(ema_decay)
    self.clip_norm = check_clip_norm(clip_norm)
    self.store, self.comm = store, comm
    self.opt = OPTIMIZERS[opt]
    self.lars = self.opt == OPTIMIZERS["lars"]
    self.lamb = self.opt == OPTIMIZERS["lamb"]
    if self.lars:
      beta1 = trust_coefficient
    dev = store.master.device
    self.device = dev
    # group mode: gradients travel through torch.distributed, the kernel sees a world of one
    # hierarchical mode (group_comm.HierComm): the kernel's world is the host; the shards are
    # summed across hosts through torch.distributed between its two halves (PHASE 1 / PHASE 2)
    self.group_mode = bool(getattr(comm, "cross_host", False))
    self.hier_mode = bool(getattr(comm, "hierarchical", False))
    self.gworld = comm.world if comm is not None else 1
    if comm is None or self.group_mode:
      self.world, self.rank = 1, 0
    elif self.hier_mode:
      self.world, self.rank = comm.local_world, comm.local_rank
    else:
      self.world, self.rank = comm.world, comm.rank
    self.deferred = False
    hyper = [lr, momentum, weight_decay, 1.0 / self.gworld, beta1, beta2, eps, 0.0]
    if self.ema_decay is not None:
      hyper += [self.ema_decay, 0.0]
    self.hyper = torch.tensor(hyper, dtype=torch.float32, device=dev)
    # with peers, the optimizer state lives in symmetric memory like the master copy: a rank only
    # ever updates its own shard of each bucket, so whoever saves a checkpoint pulls the other
    # shards over NVLink (assemble())
    def _state(name):
      if comm is not None and self.world > 1:    # (never in group mode: the state is replicated)
        t = comm.alloc(name, store.total, torch.float32)
        t.zero_()
        return t
      return torch.zeros_like(store.master)
    self.state1 = _state("state1") if self.opt != 0 else None
    self.state2 = _state("state2") if self.opt in ADAM_STATE else None
    self.ema = _state("ema") if self.ema_decay is not None else None
    self._avg = None   # averaged_weights()'s buffers, allocated on first use
    self.step_count = 0
    # CTAs of the fused kernel: one per SM alone, 64 peer-to-peer, 48 with NVLS (below)
    self.grid = 132 if self.world == 1 else 64
    n = store.total
    if not buckets:
      buckets = [(0, n, None)]
    for b, e, _ in buckets:
      assert b % 8 == 0 and b < e <= n, "bucket bounds must be multiples of 8 inside the vector"
    self.buckets = list(buckets)
    if self.lars or self.lamb:   # (validates the buckets before anything is allocated)
      self._lars_bounds = [s["offset"] for s in store.order if s["decay"]] + [store.decay_end]
      self._lars_tab = lars_tables(self._lars_bounds, self.buckets, self.world)
    self._args = []
    for slot, (b, e, tag) in enumerate(self.buckets):
      d = {
          "master": store.master.data_ptr(),
          "state1": self.state1.data_ptr() if self.state1 is not None else 0,
          "state2": self.state2.data_ptr() if self.state2 is not None else 0,
          "hyper": self.hyper.data_ptr(),
          "begin": b, "end": e, "decay_end": store.decay_end,
          "world": self.world, "rank": self.rank, "slot": slot, "opt": self.opt,
          "grid": self.grid, "zero_grads": 0,
          "aux_begin": store.decay_end,
      }
      if self.ema is not None:
        d["ema"] = self.ema.data_ptr()
      if comm is None or self.group_mode or (self.hier_mode and self.world == 1):
        d["grads"] = [store.grads.data_ptr()]
        d["weights"] = [store.weights.data_ptr()]
        d["aux32"] = [store.aux32.data_ptr()]
      else:
        d["grads"] = comm.peer_ptrs("grads")
        d["weights"] = comm.peer_ptrs("weights")
        d["aux32"] = comm.peer_ptrs("aux32")
        d["flags"] = comm.flag_ptrs()
        d["epoch"] = comm.epoch_ptr(slot)
        d["block_counter"] = comm.counter_ptr(slot)
        # NVLS: one multimem.ld_reduce through the switch replaces the world peer loads, one
        # multimem.st the world peer stores (selected when the buffers have multicast addresses)
        mc = getattr(comm, "mc_ptr", None)
        if mc is not None and comm.mc_ptr("grads") and comm.mc_ptr("weights"):
          d["grads_mc"] = comm.mc_ptr("grads")
          d["weights_mc"] = comm.mc_ptr("weights")
          d["aux32_mc"] = comm.mc_ptr("aux32")
          d["grid"] = 48
      self._args.append(d)
    self.nvls = bool(self._args and self._args[0].get("grads_mc"))
    if self.lars or self.lamb:
      self._build_lars(store, comm)
    self.grad_norm = None
    if self.clip_norm is not None:
      self._build_clip(store, comm)
    self._by_tag = {}
    for i, (_, _, tag) in enumerate(self.buckets):
      self._by_tag.setdefault(tag, []).append(i)
    self._launched = set()
    store._assemble = self.assemble   # ParamStore.state_dict() must see every rank's shards
    self.overlap = len(self.buckets) > 1 and dev.type == "cuda"
    if self.overlap:
      self.comm_stream = torch.cuda.Stream(device=dev)
      self._ev_ready = [torch.cuda.Event() for _ in self.buckets]
      self._ev_wait0 = torch.cuda.Event(enable_timing=True)
      self._ev_wait1 = torch.cuda.Event(enable_timing=True)

  def _build_lars(self, store, comm):
    """Device tables of the norm pass and the norms table: ``world`` rows of ``T`` entries
    {sum g^2 (LAMB: sum r^2), sum w^2, 0, 0}, row r written by rank r (symmetric with peers,
    multicast on NVLS).  Entries of tensors outside a rank's shards stay 0, so every rank may sum
    all rows."""
    dev = self.device
    T = len(self._lars_bounds) - 1
    n_norms = self.world * max(1, T) * 4
    if comm is not None and self.world > 1:
      self.lars_norms = comm.alloc("lars_norms", n_norms, torch.float32, multicast=self.nvls)
      self.lars_norms.zero_()
      norms = comm.peer_ptrs("lars_norms")
      norms_mc = comm.mc_ptr("lars_norms") if self.nvls else 0
    else:
      self.lars_norms = torch.zeros(n_norms, dtype=torch.float32, device=dev)
      norms, norms_mc = [self.lars_norms.data_ptr()], 0
    self._lars_off = torch.tensor(self._lars_bounds, dtype=torch.int64, device=dev)
    self._lars_bufs, self._lars_args, self._lars_phase = [], [], []
    for i, d in enumerate(self._args):
      tab = self._lars_tab[i][self.rank]
      seg = torch.tensor([x for s in tab["seg"] for x in s] or [0, 0], dtype=torch.int64, device=dev)
      tseg = torch.tensor(tab["tseg"], dtype=torch.int32, device=dev)
      partial = torch.zeros(max(2, 2 * len(tab["seg"])), dtype=torch.float32, device=dev)
      counter = torch.zeros(1, dtype=torch.int32, device=dev)
      self._lars_bufs.append((seg, tseg, partial, counter))
      d.update(lars_off=self._lars_off.data_ptr(), lars_norms=self.lars_norms.data_ptr(),
               lars_t0=tab["t0"], lars_nt=tab["nt"], lars_T=T)
      nd = {"grads": d["grads"][self.rank if self.world > 1 else 0], "master": store.master.data_ptr(),
            "seg": seg.data_ptr(), "tseg": tseg.data_ptr(), "partial": partial.data_ptr(),
            "nseg": len(tab["seg"]), "t0": tab["t0"], "nt": tab["nt"], "T": T,
            "world": self.world, "rank": self.rank, "slot": i, "norms": norms,
            "norms_mc": norms_mc, "block_counter": counter.data_ptr()}
      if self.world > 1:
        nd.update(flags=d["flags"], epoch=d["epoch"])
      if self.lamb:
        nd.update(lamb=1, hyper=d["hyper"], state1=d["state1"], state2=d["state2"])
      self._lars_args.append(nd)
      self._lars_phase.append((dict(d, phase=1), dict(d, phase=2)))

  def _build_clip(self, store, comm):
    """Gradient clipping's buffers and launch arguments.  ``clip_sq``: ``world`` rows of one
    {sum g^2, 0, 0, 0} entry per bucket, row r written by rank r (symmetric with peers)."""
    dev, nb = self.device, len(self.buckets)
    if comm is not None and self.world > 1:
      self.clip_sq = comm.alloc("clip_sq", self.world * nb * 4, torch.float32)
      self.clip_sq.zero_()
      table = comm.peer_ptrs("clip_sq")
    else:
      self.clip_sq = torch.zeros(self.world * nb * 4, dtype=torch.float32, device=dev)
      table = [self.clip_sq.data_ptr()]
    self.grad_norm = torch.zeros(1, dtype=torch.float32, device=dev)
    self.hyper_step = torch.zeros_like(self.hyper)
    grid = 132   # >= every grid of the sum-of-squares passes (csrc/ptx.cuh kSmCount)
    self._clip_partial = torch.zeros(nb * grid, dtype=torch.float32, device=dev)
    self._clip_counter = torch.zeros(nb, dtype=torch.int32, device=dev)
    self._clip_phase1, self._clip_reduce, self._clip_update = [], [], []
    hs = self.hyper_step.data_ptr()
    for i, d in enumerate(self._args):
      if self.lars or self.lamb:
        phase1, phase2 = self._lars_phase[i]
        one = self._args[i]
      else:
        phase1, phase2, one = dict(d, phase=1), dict(d, phase=2), d
      partial = self._clip_partial.data_ptr() + 4 * grid * i
      if self.world > 1 and not self.hier_mode:
        red = dict(phase1, phase=3, clip_sq=table, clip_partial=partial, clip_nb=nb, clip_index=i)
      else:
        lo, hi = self.shard_bounds(i, self.rank)
        red = {"grads": store.grads.data_ptr(), "lo": lo, "hi": hi, "partial": partial,
               "block_counter": self._clip_counter.data_ptr() + 4 * i, "table": table, "nb": nb,
               "index": i, "world": self.world, "rank": self.rank, "slot": i}
        if self.world > 1:
          red.update(flags=d["flags"], epoch=d["epoch"])
      self._clip_phase1.append(phase1)
      self._clip_reduce.append(red)
      self._clip_update.append(dict(phase2 if (self.world > 1 or self.hier_mode) else one,
                                    hyper=hs))
    # LAMB: the norm pass of the clipped step, run by _update_all() after clip_finalize
    self._clip_lamb_norms = [dict(nd, hyper=hs) for nd in self._lars_args] if self.lamb else None
    self._clip_pending = False

  def set_lr(self, lr):
    self.hyper[0:1].fill_(float(lr))

  def set_accumulation(self, k):
    """Gradient accumulation over k micro-batches (the trainers' ``gradient_accumulation_steps``):
    the gradient buffer holds the sum of k micro-batches, so the grad scale ``hyper[3]`` becomes
    fp32(1 / (world k)).  state_dict() still saves the k-free 1 / world, and load_state_dict()
    keeps this optimizer's own k, so a checkpoint loads under any k."""
    self.accumulation = int(k)
    self.hyper[3:4].fill_(1.0 / (self.gworld * self.accumulation))

  def zero_grads(self):
    self.store.grads.zero_()
    ops.count()
    self._launched = set()

  def _bump_step(self):
    if self.opt in ADAM_STATE:
      self.step_count += 1
      self.hyper[7:8].add_(1.0)
    if self.ema is not None:
      self.hyper[9:10].add_(1.0)     # n: the kernels copy the master at n = 1, decay after

  # ------------------------------------------------------------ weight average
  def reset_average(self):
    """Restart the average: until the next update it is the current parameters, after that
    update it equals the new master (n = 0).  No-op without an average."""
    if self.ema is not None:
      self.hyper[9:10].zero_()

  def average_count(self):
    """n, the updates folded into the average since it was last reset (host sync)."""
    return int(self.hyper[9].item()) if self.ema is not None else 0

  def averaged_weights(self):
    """The complete weight average on this rank: ``(weights, aux32)``, a bf16 buffer in the
    layout of ``store.weights`` and an fp32 one in that of ``store.aux32`` - what ``bn_fold``
    and the U-Net forward read.  bf16 is rounded to nearest even by the ps_pull kernel
    (``pack_bf16x2``, as the update kernel rounds masters), so these are exactly the weights a
    trainer loading the exported average derives.  Before the first update after a reset they
    are the current parameters.  Pulls the peers' shards first (assemble()); stream-ordered
    between two steps like assemble().  Returns buffers owned by the optimizer, rewritten by the
    next call."""
    if self.ema is None:
      raise RuntimeError("this optimizer keeps no weight average (ema_decay=None)")
    st = self.store
    src = self.average_master()
    if self._avg is None:
      self._avg = (torch.empty_like(st.weights), torch.zeros_like(st.aux32))
    w, aux = self._avg
    ops.K.ps_pull(src.data_ptr(), None, w, st.total)
    aux[:st.total - st.decay_end].copy_(src[st.decay_end:])
    return w, aux

  def average_master(self):
    """fp32 [total] vector of the complete average (the masters themselves while n = 0), after
    pulling the peers' shards; a view of ``ema`` or ``store.master``, not a copy."""
    if self.ema is None:
      raise RuntimeError("this optimizer keeps no weight average (ema_decay=None)")
    if self.average_count() == 0:
      self.assemble()
      return self.store.master
    self.assemble(("ema",))
    return self.ema

  # ---------------------------------------------------------------- overlap
  def launch(self, tag):
    """Gradients of every bucket tagged ``tag`` are final on the current stream: run their
    fused all-reduce + update on the communication stream now."""
    if not self.overlap or self._capturing_group():
      return
    if not self._launched:
      self._bump_step()
    main = torch.cuda.current_stream(self.device)
    for i in self._by_tag.get(tag, []):
      if i in self._launched:
        continue
      self._ev_ready[i].record(main)
      self.comm_stream.wait_event(self._ev_ready[i])
      with torch.cuda.stream(self.comm_stream):
        if self.clip_norm is not None:
          self._reduce_bucket(i)     # the update waits for every bucket's norm: _launch_all()
        else:
          self._run_bucket(i)
      self._launched.add(i)

  def _launch_all(self):
    """launch() every tag, then (clipping) the norm and every bucket's update on the
    communication stream."""
    for tag in list(self._by_tag):
      self.launch(tag)
    if self.clip_norm is not None:
      with torch.cuda.stream(self.comm_stream):
        self._update_all()

  def finish(self):
    """Launch whatever has not been launched and make the current stream wait for all of it."""
    if self._capturing_group():
      self.deferred = True      # the collective stays outside the graph: after_replay() runs it
      return
    if not self.overlap:
      return self.step()
    self._launch_all()
    main = torch.cuda.current_stream(self.device)
    timing = not torch.cuda.is_current_stream_capturing()  # timed events cannot be captured
    if timing:
      self._ev_wait0.record(main)
    main.wait_stream(self.comm_stream)
    if timing:
      self._ev_wait1.record(main)
    self._timed = timing

  def exposed_ms(self):
    """Device time the compute stream spent waiting for the communication stream in the last
    ``finish()`` - the non-overlapped part of the all-reduce (0 when fully hidden)."""
    if not self.overlap or not getattr(self, "_timed", False):
      return None
    self._ev_wait1.synchronize()
    return self._ev_wait0.elapsed_time(self._ev_wait1)

  # ------------------------------------------------------------ everything
  def step(self, bucket=None):
    """Launch the fused kernel for one bucket (or all) on the current stream.  Stream order
    guarantees this rank's gradients are complete; the kernel's flag barrier covers the peers."""
    if self._capturing_group():
      self.deferred = True      # see finish()
      return
    if self.clip_norm is not None and bucket is not None and len(self.buckets) > 1:
      raise ValueError("clip_norm: the norm covers every bucket, step() them all at once")
    self._bump_step()
    todo = range(len(self.buckets)) if bucket is None else [bucket]
    if self.clip_norm is not None:
      for i in todo:
        self._reduce_bucket(i)
      self._update_all()
      return
    for i in todo:
      self._run_bucket(i)

  def _run_bucket(self, i):
    if self.lars or self.lamb:
      return self._run_bucket_lars(i)
    if self.hier_mode:
      d = self._args[i]
      if self.world > 1:
        ops.K.allreduce_opt(dict(d, phase=1))          # NVLink reduce-scatter inside the host
      lo, hi = self.shard_bounds(i, self.rank)
      if hi > lo:
        self.comm.all_reduce_inter(self.store.grads[lo:hi])   # this rank's shard, across hosts
      ops.K.allreduce_opt(dict(d, phase=2))            # update + all-gather inside the host
      return
    if self.group_mode:
      b, e, _ = self.buckets[i]
      self.comm.all_reduce(self.store.grads[b:e])     # SUM; the kernel scales by 1 / world
    ops.K.allreduce_opt(self._args[i])

  def _run_bucket_lars(self, i):
    """reduce-scatter -> per-tensor norms (+ exchange among the local peers) -> update +
    all-gather, all on the bucket's flag slot.  Without peers: norms -> one-pass update.  LARS and
    LAMB (its norm pass reads the hyper vector and the moments, see _build_lars)."""
    phase1, phase2 = self._lars_phase[i]
    if self.hier_mode:
      if self.world > 1:
        ops.K.allreduce_opt(phase1)
      lo, hi = self.shard_bounds(i, self.rank)
      if hi > lo:
        self.comm.all_reduce_inter(self.store.grads[lo:hi])
      ops.K.lars_norms(self._lars_args[i])
      ops.K.allreduce_opt(phase2)
      return
    if self.group_mode:
      b, e, _ = self.buckets[i]
      self.comm.all_reduce(self.store.grads[b:e])
    if self.world > 1:
      ops.K.allreduce_opt(phase1)
      ops.K.lars_norms(self._lars_args[i])
      ops.K.allreduce_opt(phase2)
    else:
      ops.K.lars_norms(self._lars_args[i])
      ops.K.allreduce_opt(self._args[i])

  def _reduce_bucket(self, i):
    """Clipping, first half of bucket i: its gradient fully reduced and the sum of squares of
    this rank's share of it in the norm table (+ LARS norms; LAMB's wait for the clipped scale,
    _update_all()); no update."""
    if self.hier_mode:
      if self.world > 1:
        ops.K.allreduce_opt(self._clip_phase1[i])
      lo, hi = self.shard_bounds(i, self.rank)
      if hi > lo:
        self.comm.all_reduce_inter(self.store.grads[lo:hi])
      ops.K.grad_sumsq(self._clip_reduce[i])
    elif self.world > 1:
      ops.K.allreduce_opt(self._clip_reduce[i])      # PHASE 3
    else:
      if self.group_mode:
        b, e, _ = self.buckets[i]
        self.comm.all_reduce(self.store.grads[b:e])
      ops.K.grad_sumsq(self._clip_reduce[i])
    if self.lars:
      ops.K.lars_norms(self._lars_args[i])
    self._clip_pending = True

  def _update_all(self):
    """Clipping, second half: N into grad_norm, the clipped scale into hyper_step, then every
    bucket's update.  Runs once per set of reductions."""
    if not self._clip_pending:
      return
    ops.K.clip_finalize(self.clip_sq.data_ptr(), self.world, len(self.buckets),
                        self.hyper.data_ptr(), self.hyper.numel(), self.clip_norm,
                        self.hyper_step.data_ptr(), self.grad_norm.data_ptr())
    for i, d in enumerate(self._clip_update):
      if self.lamb:
        ops.K.lars_norms(self._clip_lamb_norms[i])
      ops.K.allreduce_opt(d)
    self._clip_pending = False

  def _capturing_group(self):
    return ((self.group_mode or self.hier_mode) and self.device.type == "cuda"
            and torch.cuda.is_current_stream_capturing())

  def after_replay(self):
    """Trainers call this after ``graph.replay()``: in group mode the captured step ends with the
    local gradients complete and this runs all-reduce + update eagerly; otherwise a no-op."""
    if self.deferred:
      self._launched = set()
      if self.overlap:
        self._launch_all()
        torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)
      else:
        self.step()

  # ------------------------------------------------------ sharded state
  def shard_bounds(self, bucket, rank):
    """[lo, hi) of ``rank``'s shard of bucket ``bucket`` - the same arithmetic as
    allreduce_opt_kernel (csrc/optim_comm.cu): ceil(n / world) rounded up to 8 elements."""
    b, e, _ = self.buckets[bucket]
    n = e - b
    chunk = ((n + self.world - 1) // self.world + 7) // 8 * 8
    return b + min(n, chunk * rank), b + min(n, chunk * (rank + 1))

  def assemble(self, names=None):
    """Make THIS rank's fp32 master and optimizer state complete.

    With world > 1 the fused kernel updates master/state only for the rank's own shard of every
    bucket; the rest of the local copy is stale.  This pulls every peer's shards out of the
    peers' symmetric buffers (plain device copies over NVLink on the current stream).  It is not
    a collective: only the saving rank needs to call it.  It is consistent as long as it is
    stream-ordered between two of this rank's steps - a peer cannot finish its next update
    before this rank has contributed its gradients (the kernel's entry barrier).  The weight
    average is pulled too; ``names`` restricts the pull to some of master / state1 / state2 /
    ema."""
    if self.world == 1 or self.comm is None:
      return
    C = ops.C()
    n = self.store.total
    bufs = [("master", self.store.master)]
    if self.state1 is not None:
      bufs.append(("state1", self.state1))
    if self.state2 is not None:
      bufs.append(("state2", self.state2))
    if self.ema is not None:
      bufs.append(("ema", self.ema))
    for name, local in bufs:
      if names is not None and name not in names:
        continue
      ptrs = self.comm.peer_ptrs(name)
      for r in range(self.world):
        if r == self.rank:
          continue
        remote = C.tensor_from_ptr(ptrs[r], [n], "f32")
        for i in range(len(self.buckets)):
          lo, hi = self.shard_bounds(i, r)
          if hi > lo:
            local[lo:hi].copy_(remote[lo:hi])

  def state_dict(self):
    self.assemble()
    sd = {"step": self.step_count}
    if self.state1 is not None:
      sd["state1"] = self.state1.detach().cpu()
    if self.state2 is not None:
      sd["state2"] = self.state2.detach().cpu()
    if self.ema is not None:
      sd["ema"] = self.ema.detach().cpu()
      sd["ema_count"] = self.average_count()
    sd["hyper"] = self.hyper.detach().cpu()
    if getattr(self, "accumulation", 1) != 1:
      sd["hyper"] = sd["hyper"].clone()
      sd["hyper"][3] = 1.0 / self.gworld
    return sd

  def load_state_dict(self, sd):
    """Inverse of state_dict().  ``hyper`` may come from an optimizer with or without an average
    (10 or 8 entries): its first 8 are loaded, the decay stays this optimizer's own.  The average
    and its count are loaded when ``sd`` has them; otherwise the average is reset."""
    self.step_count = int(sd.get("step", 0))
    if self.state1 is not None and "state1" in sd:
      self.state1.copy_(sd["state1"])
    if self.state2 is not None and "state2" in sd:
      self.state2.copy_(sd["state2"])
    if "hyper" in sd:
      self.hyper[:HYPER].copy_(torch.as_tensor(sd["hyper"])[:HYPER])
      if getattr(self, "accumulation", 1) != 1:
        self.set_accumulation(self.accumulation)
    if self.ema is not None:
      if "ema" in sd:
        self.ema.copy_(sd["ema"])
        self.hyper[9:10].fill_(float(sd.get("ema_count", 1)))
      else:
        self.reset_average()

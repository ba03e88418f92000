"""Fused gradient all-reduce + optimizer step (csrc/optim_comm.cu).

Replaces the collective the reference gets from
``tf.distribute.experimental.MultiWorkerMirroredStrategy`` (reference user code:
examples/mnist/keras/mnist_spark.py:11,55-66; TFoS itself only provides the
cluster spec, tensorflowonspark/TFSparkNode.py:373-384) *and* the Keras
optimizer update that follows it: one kernel per gradient bucket pulls the peer
shards over NVLink, averages, applies SGD / momentum / Adam to the fp32 master
shard and stores the new bf16 weights into every rank's weight buffer.

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
"""
import torch

from .. import ops

OPTS = {"sgd": 0, "momentum": 1, "adam": 2}


class FusedOptimizer(object):

  def __init__(self, store, comm=None, opt="momentum", lr=0.1, momentum=0.9, weight_decay=0.0,
               beta1=0.9, beta2=0.999, eps=1e-7, buckets=None, grid=None):
    self.store, self.comm = store, comm
    self.opt = OPTS[opt]
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
    self.hyper = torch.tensor([lr, momentum, weight_decay, 1.0 / self.gworld, beta1, beta2, eps, 0.0],
                              dtype=torch.float32, device=dev)
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
    self.state2 = _state("state2") if self.opt == 2 else None
    self.step_count = 0
    import os
    env_grid = int(os.environ.get("TFOS_AR_GRID", "0"))   # CTAs of the fused kernel (experiments)
    grid = grid or env_grid or None
    self.grid = grid or (132 if self.world == 1 else 64)
    n = store.total
    if not buckets:
      buckets = [(0, n, None)]
    for b, e, _ in buckets:
      assert b % 8 == 0 and b < e <= n, "bucket bounds must be multiples of 8 inside the vector"
    self.buckets = list(buckets)
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
          d["grid"] = grid or 48
      self._args.append(d)
    self.nvls = bool(self._args and self._args[0].get("grads_mc"))
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

  def set_lr(self, lr):
    self.hyper[0:1].fill_(float(lr))

  def zero_grads(self):
    self.store.grads.zero_()
    ops.count()
    self._launched = set()

  def _bump_step(self):
    if self.opt == 2:
      self.step_count += 1
      self.hyper[7:8].add_(1.0)

  # ---------------------------------------------------------------- overlap
  def add_producer_stream(self, stream):
    """Gradients are also written by kernels on ``stream`` (the weight-gradient side stream):
    every consumer of the gradient buffer waits for it."""
    if not hasattr(self, "_producers"):
      self._producers = []
    self._producers.append((stream, {}))

  def _join_producers(self, consumer, key):
    for stream, events in getattr(self, "_producers", []):
      ev = events.get(key)
      if ev is None:
        ev = events[key] = torch.cuda.Event()
      ev.record(stream)
      consumer.wait_event(ev)

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
      self._join_producers(self.comm_stream, i)
      with torch.cuda.stream(self.comm_stream):
        self._run_bucket(i)
      self._launched.add(i)

  def finish(self):
    """Launch whatever has not been launched and make the current stream wait for all of it."""
    if self._capturing_group():
      self.deferred = True      # the collective stays outside the graph: after_replay() runs it
      return
    if not self.overlap:
      if self.device.type == "cuda":
        self._join_producers(torch.cuda.current_stream(self.device), "finish")
      return self.step()
    for tag in list(self._by_tag):
      self.launch(tag)
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
    self._bump_step()
    todo = range(len(self.buckets)) if bucket is None else [bucket]
    for i in todo:
      self._run_bucket(i)

  def _run_bucket(self, i):
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

  def _capturing_group(self):
    return ((self.group_mode or self.hier_mode) and self.device.type == "cuda"
            and torch.cuda.is_current_stream_capturing())

  def after_replay(self):
    """Trainers call this after ``graph.replay()``: in group mode the captured step ends with the
    local gradients complete and this runs all-reduce + update eagerly; otherwise a no-op."""
    if self.deferred:
      self._launched = set()
      if self.overlap:
        for tag in list(self._by_tag):
          self.launch(tag)
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

  def assemble(self):
    """Make THIS rank's fp32 master and optimizer state complete.

    With world > 1 the fused kernel updates master/state only for the rank's own shard of every
    bucket; the rest of the local copy is stale.  This pulls every peer's shards out of the
    peers' symmetric buffers (plain device copies over NVLink on the current stream).  It is not
    a collective: only the saving rank needs to call it.  It is consistent as long as it is
    stream-ordered between two of this rank's steps - a peer cannot finish its next update
    before this rank has contributed its gradients (the kernel's entry barrier)."""
    if self.world == 1 or self.comm is None:
      return
    C = ops.C()
    n = self.store.total
    bufs = [("master", self.store.master)]
    if self.state1 is not None:
      bufs.append(("state1", self.state1))
    if self.state2 is not None:
      bufs.append(("state2", self.state2))
    for name, local in bufs:
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
    sd["hyper"] = self.hyper.detach().cpu()
    return sd

  def load_state_dict(self, sd):
    self.step_count = int(sd.get("step", 0))
    if self.state1 is not None and "state1" in sd:
      self.state1.copy_(sd["state1"])
    if self.state2 is not None and "state2" in sd:
      self.state2.copy_(sd["state2"])
    if "hyper" in sd:
      self.hyper.copy_(sd["hyper"])

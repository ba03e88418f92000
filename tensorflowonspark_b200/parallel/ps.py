"""Asynchronous parameter server on GPU (and a shared-memory twin for CPU executors).

The reference reaches this through TensorFlow: ``tf.train.Server`` between-graph replication in
TF1 (tensorflowonspark/TFNode.py:126-132) or ``ParameterServerStrategy`` in TF2 (examples/mnist/
estimator/mnist_spark_streaming.py:86); TFoS itself only reserves ``num_ps`` executors for the
'ps' role and parks them on a control queue (TFCluster.py:260-262, TFSparkNode.py:442-458).

Here a 'ps' node owns a slice of the flat fp32 parameter vector **resident on its GPU**,
publishes the CUDA IPC handle on the reservation board, and sleeps.  Workers map that memory
and, without any barrier (Hogwild-style asynchronous SGD):

  * ``pull()``  - ``ps_pull`` kernel: peer loads of the parameters over NVLink, writing the local
    fp32 copy and the bf16 compute copy in one pass;
  * ``push()``  - ``ps_push_dense`` kernel: ``w_ps += -lr * scale * g`` applied *in the PS GPU's
    memory* with remote ``red.add.f32`` - the gradient never lands in a staging buffer;
  * ``push_sparse()`` - row-indexed scatter-apply for embedding-style (IndexedSlices) gradients.

On CPU-only executors the same interface is backed by POSIX shared memory + numpy (used by the
CPU test-suite and BASELINE config #1 style runs).

**Slot mode** (``start_cluster_server(params=..., optimizer="momentum" | "adam" | "sgd", ...)``):
the reference's parameter server runs *any* optimizer, its slot variables living on the ps task
(examples/mnist/estimator/mnist_spark_streaming.py:86,139; tensorflowonspark/TFNode.py:70-154).
Here the PS GPU keeps the fp32 parameters, the optimizer state and a bf16 serving copy; every
worker owns two gradient *slots* in the PS GPU's memory:

  worker  ``push_grads``  ps_push_slot kernel: device-side bounded wait until its slot is free,
          one-way NVLink stores of the fp32 gradients (+ batch-norm running-statistics deltas
          for the non-trainable tail), ``st.release.sys`` of a sequence number;
  server  ``serve_forever``  polls the sequence numbers and runs ps_apply (SGD / momentum / Adam
          over the resident state at HBM speed, refreshes the serving copy, marks the slot
          applied);
  worker  ``pull_model``  ps_pull_model kernel: peer loads of the bf16 weights + the fp32 tail
          (BN scale/offset, biases, running statistics) - half the bytes of an fp32 pull.

Workers never wait for each other; a worker only waits for its *own* slot (back-pressure).
The shared-memory twin implements the same protocol with numpy so the life-cycle is testable on
CPU executors.
"""
import logging
import time

import numpy as np

logger = logging.getLogger(__name__)


def _use_cuda(ctx):
  try:
    import torch
    return bool(getattr(ctx, "gpus", None)) and torch.cuda.is_available()
  except Exception:
    return False


def _board(ctx):
  from .. import reservation
  return reservation.Client(ctx.server_addr)


def _ps_count(ctx):
  return len(ctx.cluster_spec.get("ps", []))


def _slices(numel, num_ps):
  per = ((numel + num_ps - 1) // num_ps + 7) // 8 * 8
  return [(min(numel, i * per), min(numel, (i + 1) * per)) for i in range(num_ps)]


def _sparse_plan(lo, hi, base, width):
  """How a server owning flat elements [lo, hi) applies a row-sparse push to a [rows, width] table
  at flat offset ``base``: ``(r0, r1, cuts)``.  Rows r0 <= r < r1 lie wholly inside the slice (the
  sparse kernel); ``cuts`` lists ``(r, a, b)`` for each row the slice cuts, whose owned elements
  are [a, b) (the dense kernel).  Every row appears at most once, in one of the two: a row wider
  than the slice can be cut at both of its edges."""
  if hi <= max(lo, base):
    return 0, 0, []
  first = max(lo - base, 0) // width        # rows overlapping the slice: first .. last
  last = (hi - 1 - base) // width
  r0 = first + int(base + first * width < lo)
  r1 = last + 1 - int(base + (last + 1) * width > hi)
  cuts = []
  for r in sorted({first, last}):
    s = base + r * width
    if s < lo or s + width > hi:
      cuts.append((r, max(s, lo), min(s + width, hi)))
  return r0, max(r0, r1), cuts


def _check_pull_model(numel, total, decay_end, weights, aux32, running):
  """Refuse, before any launch, a GPU ``pull_model`` whose destinations cannot hold what the
  servers send: the bf16 weights [total], the fp32 copy of [decay_end, total) and the running
  statistics [total, numel)."""
  if weights is None or weights.numel() < total:
    raise ValueError("pull_model needs bf16 weights of at least total = {} elements".format(total))
  if not 0 <= decay_end <= total:
    raise ValueError("pull_model needs 0 <= decay_end <= total, got {} and {}".format(
        decay_end, total))
  if decay_end < total and (aux32 is None or aux32.numel() < total - decay_end):
    raise ValueError("pull_model needs aux32 of at least total - decay_end = {} elements".format(
        total - decay_end))
  if total > numel:
    raise ValueError("total {} exceeds the {} parameters the servers hold".format(total, numel))
  if numel > total and (running is None or running.numel() != numel - total):
    raise ValueError("the servers hold {} running statistics past total: pull_model needs "
                     "running of that length".format(numel - total))


def _check_push_grads(numel, total, grads, running, running_pulled):
  """Refuse, before any launch, a GPU ``push_grads`` whose sources do not cover the servers'
  slices: the gradients [total] and, past total, the running statistics together with the
  snapshot ``pull_model`` took of them."""
  if total > numel:
    raise ValueError("total {} exceeds the {} parameters the servers hold".format(total, numel))
  if total > 0 and (grads is None or grads.numel() < total):
    raise ValueError("push_grads needs gradients of at least total = {} elements".format(total))
  if numel > total:
    if running is None or running.numel() != numel - total:
      raise ValueError("the servers hold {} running statistics past total: push_grads needs "
                       "running of that length".format(numel - total))
    if running_pulled is None or running_pulled.numel() != running.numel():
      raise ValueError("push_grads with running statistics needs a pull_model(..., running) "
                       "first: their deltas are taken against what it pulled")


OPTS = {"sgd": 0, "momentum": 1, "adam": 2}
NSLOTS = 2   # gradient slots per worker on each server (push i+1 overlaps the apply of push i)


def _clients(ctx):
  """(job, task) of every node that may push: everything that is not a ps, in a fixed order."""
  out = []
  for job in sorted(ctx.cluster_spec):
    if job != "ps":
      out.extend((job, i) for i in range(len(ctx.cluster_spec[job])))
  return out


def _pad8(n):
  return (int(n) + 7) // 8 * 8


def _slot_layout(n, num_clients, cuda):
  """Byte offsets inside one server's allocation (both sides compute it from the same inputs)."""
  off, lay = 0, {}
  def take(name, nbytes):
    nonlocal off
    lay[name] = off
    off += (nbytes + 255) // 256 * 256
  take("master", 4 * n)
  take("state1", 4 * n)
  take("state2", 4 * n)
  take("wbf16", 2 * n if cuda else 0)
  take("slots", 4 * n * num_clients * NSLOTS)
  take("ready", 4 * num_clients * NSLOTS)
  take("applied", 4 * num_clients * NSLOTS)
  take("hyper", 4 * 8)
  take("counter", 4 * 8)
  lay["bytes"] = off
  return lay


def apply_numpy(master, state1, state2, hyper, g, lo, decay_end, ema_begin, opt):
  """One server-side optimizer step on host arrays - the twin of ps_apply_kernel (csrc/
  optim_comm.cu): ``g`` is the received slice for global elements [lo, lo + len(g)); elements at or
  beyond ``ema_begin`` are the non-trainable tail (``w -= g``: running-statistics deltas), the
  rest get gradient scale hyper[3], L2 on the elements below ``decay_end``, then SGD / momentum /
  Adam (``opt`` 0 / 1 / 2; Adam advances its step count hyper[7])."""
  h = hyper
  idx = np.arange(lo, lo + g.size)
  tr, ema = idx < ema_begin, idx >= ema_begin
  w = master
  w[ema] -= g[ema]
  gg = g[tr] * h[3]
  gg = gg + h[2] * w[tr] * (idx[tr] < decay_end)
  if opt == 1:
    state1[tr] = h[1] * state1[tr] + gg
    gg = state1[tr]
  elif opt == 2:
    h[7] += 1.0
    state1[tr] = h[4] * state1[tr] + (1 - h[4]) * gg
    state2[tr] = h[5] * state2[tr] + (1 - h[5]) * gg * gg
    gg = (state1[tr] / (1 - h[4] ** h[7])) / (np.sqrt(state2[tr] / (1 - h[5] ** h[7])) + h[6])
  w[tr] -= h[0] * gg


class PSServer(object):
  """Runs inside a 'ps' node: hosts parameters [lo, hi) of the flat vector."""

  def __init__(self, ctx, numel, init=None, optimizer=None, lr=0.1, momentum=0.9,
               weight_decay=0.0, beta1=0.9, beta2=0.999, eps=1e-7, decay_end=None,
               ema_begin=None, grad_scale=1.0):
    self.ctx = ctx
    self.numel = int(numel)
    if optimizer is not None:
      return self._init_slot_mode(ctx, init, optimizer, [lr, momentum, weight_decay, grad_scale,
                                                          beta1, beta2, eps, 0.0],
                                  decay_end, ema_begin)
    self.slot_mode = False
    self.lo, self.hi = _slices(self.numel, _ps_count(ctx))[ctx.task_index]
    n = self.hi - self.lo
    key = "ps/{}/{}".format(ctx.cluster_id, ctx.task_index)
    board = _board(ctx)
    self.cuda = _use_cuda(ctx)
    if self.cuda:
      import torch
      from .. import ops
      torch.cuda.set_device(0)
      ptr, handle = ops.C().symm_alloc(max(256, n * 4))
      self.tensor = ops.C().tensor_from_ptr(ptr, [n], "f32")
      if init is not None:
        self.tensor.copy_(torch.as_tensor(init, dtype=torch.float32).reshape(-1)[self.lo:self.hi])
      torch.cuda.synchronize()
      board.put(key, {"kind": "cuda", "handle": handle, "lo": self.lo, "hi": self.hi,
                      "numel": self.numel})
    else:
      from multiprocessing import shared_memory
      self.shm = shared_memory.SharedMemory(create=True, size=max(8, n * 4))
      self.array = np.ndarray((n,), dtype=np.float32, buffer=self.shm.buf)
      self.array[:] = 0 if init is None else np.asarray(init, dtype=np.float32).reshape(-1)[
          self.lo:self.hi]
      board.put(key, {"kind": "shm", "name": self.shm.name, "lo": self.lo, "hi": self.hi,
                      "numel": self.numel})
    board.close()
    logger.info("ps:%d serving parameters [%d, %d) on %s", ctx.task_index, self.lo, self.hi,
                "GPU" if self.cuda else "shared memory")

  # ------------------------------------------------------------- slot mode
  def _init_slot_mode(self, ctx, init, optimizer, hyper, decay_end, ema_begin):
    self.slot_mode = True
    self.opt = OPTS[optimizer]
    if self.numel % 8:
      raise ValueError("slot mode needs a parameter count that is a multiple of 8")
    self.lo, self.hi = _slices(self.numel, _ps_count(ctx))[ctx.task_index]
    n = self.n = self.hi - self.lo
    self.decay_end = self.numel if decay_end is None else int(decay_end)
    self.ema_begin = self.numel if ema_begin is None else int(ema_begin)
    self.clients = _clients(ctx)
    W = len(self.clients)
    self.cuda = _use_cuda(ctx)
    lay = self.layout = _slot_layout(n, W, self.cuda)
    key = "ps/{}/{}".format(ctx.cluster_id, ctx.task_index)
    info = {"lo": self.lo, "hi": self.hi, "numel": self.numel, "slot_mode": True,
            "clients": [list(c) for c in self.clients], "decay_end": self.decay_end,
            "ema_begin": self.ema_begin, "opt": self.opt}
    if self.cuda:
      import torch
      from .. import ops
      torch.cuda.set_device(0)
      C = ops.C()
      self.base, handle = C.symm_alloc(lay["bytes"])
      view = lambda name, count, dt: C.tensor_from_ptr(self.base + lay[name], [count], dt)  # noqa: E731
      self.master = view("master", n, "f32")
      self.state1, self.state2 = view("state1", n, "f32"), view("state2", n, "f32")
      self.wbf16 = view("wbf16", n, "bf16")
      self.ready = view("ready", W * NSLOTS, "i32")
      self.applied = view("applied", W * NSLOTS, "i32")
      self.hyper = view("hyper", 8, "f32")
      if init is not None:
        self.master.copy_(torch.as_tensor(init, dtype=torch.float32).reshape(-1)[self.lo:self.hi])
      self.wbf16.copy_(self.master)
      self.hyper.copy_(torch.tensor(hyper, dtype=torch.float32))
      torch.cuda.synchronize()
      info.update(kind="cuda", handle=handle)
    else:
      from multiprocessing import shared_memory
      self.shm = shared_memory.SharedMemory(create=True, size=lay["bytes"])
      self.shm.buf[:lay["bytes"]] = bytes(lay["bytes"])
      view = lambda name, count, dt: np.ndarray((count,), dtype=dt, buffer=self.shm.buf,  # noqa: E731
                                                offset=lay[name])
      self.master = view("master", n, np.float32)
      self.state1, self.state2 = view("state1", n, np.float32), view("state2", n, np.float32)
      self.ready = view("ready", W * NSLOTS, np.int32)
      self.applied = view("applied", W * NSLOTS, np.int32)
      self.hyper = view("hyper", 8, np.float32)
      self.slots = view("slots", n * W * NSLOTS, np.float32)
      if init is not None:
        self.master[:] = np.asarray(init, dtype=np.float32).reshape(-1)[self.lo:self.hi]
      self.hyper[:] = hyper
      info.update(kind="shm", name=self.shm.name)
    self.array = self.master if not self.cuda else None
    self.tensor = self.master if self.cuda else None
    self._applied_host = [0] * (W * NSLOTS)
    self.applies = 0
    board = _board(ctx)
    board.put(key, info)
    board.close()
    logger.info("ps:%d slot mode (%s) serving [%d, %d) to %d clients on %s", ctx.task_index,
                optimizer, self.lo, self.hi, W, "GPU" if self.cuda else "shared memory")

  def _apply(self, k, seq):
    """Apply gradient slot ``k`` (= client * NSLOTS + slot) to the resident state."""
    n = self.n
    if self.cuda:
      from .. import ops
      if self.opt == 2:
        self.hyper[7:8].add_(1.0)
      ops.K.ps_apply({
          "master": self.master.data_ptr(), "state1": self.state1.data_ptr(),
          "state2": self.state2.data_ptr(), "wbf16": self.wbf16.data_ptr(),
          "slot": self.base + self.layout["slots"] + 4 * n * k, "hyper": self.hyper.data_ptr(),
          "n": n, "lo": self.lo, "decay_end": self.decay_end, "ema_begin": self.ema_begin,
          "applied_flag": self.applied.data_ptr() + 4 * k, "seq": int(seq),
          "block_counter": self.base + self.layout["counter"], "opt": self.opt})
    else:
      apply_numpy(self.master, self.state1, self.state2, self.hyper,
                  self.slots[k * n:(k + 1) * n].copy(), self.lo, self.decay_end, self.ema_begin, self.opt)
      self.applied[k] = seq
    self._applied_host[k] = int(seq)
    self.applies += 1

  def poll_once(self):
    """Apply every slot whose sequence number moved; returns how many were applied."""
    if self.cuda:
      ready = self.ready.cpu().tolist()
    else:
      ready = self.ready.tolist()
    done = 0
    for k, seq in enumerate(ready):
      if seq > self._applied_host[k]:
        self._apply(k, seq)
        done += 1
    return done

  def values(self):
    if self.cuda:
      return self.tensor.detach().cpu().numpy().copy()
    return self.array.copy()

  def serve_forever(self, poll=1.0):
    """Park until the driver stops this node (the node runtime kills the process); in slot mode
    this is the apply loop."""
    if not getattr(self, "slot_mode", False):
      while True:
        time.sleep(poll)
    idle = 0
    while True:
      if self.poll_once():
        idle = 0
      else:
        idle += 1
        time.sleep(0.00005 if idle < 2000 else 0.002)

  def close(self):
    if not self.cuda:
      try:
        self.shm.close()
        self.shm.unlink()
      except Exception:
        pass


class PSClient(object):
  """Worker-side handle on all parameter servers of the cluster."""

  def __new__(cls, ctx, timeout=600, local_servers=None):
    # servers that published a TCP endpoint (ps and workers on different hosts, parallel/ps_net.py)
    # are reached through the network client, which has the same surface
    if cls is PSClient and not local_servers:
      board = _board(ctx)
      first = board.get("ps/{}/0".format(ctx.cluster_id), timeout)
      board.close()
      if first.get("kind") == "tcp":
        from . import ps_net
        return ps_net.NetPSClient(ctx, timeout)
    return super(PSClient, cls).__new__(cls)

  def __init__(self, ctx, timeout=600, local_servers=None):
    """``local_servers``: PSServer objects living in THIS process (single-process use and the
    kernel checks) - their memory is addressed directly instead of through CUDA IPC, which
    cannot open a handle inside the process that exported it."""
    self.ctx = ctx
    board = _board(ctx)
    self.parts = []
    for i in range(_ps_count(ctx)):
      info = board.get("ps/{}/{}".format(ctx.cluster_id, i), timeout)
      self.parts.append(info)
    board.close()
    self.numel = self.parts[0]["numel"]
    self.cuda = self.parts[0]["kind"] == "cuda"
    self.slot_mode = bool(self.parts[0].get("slot_mode"))
    if self.slot_mode:
      me = [ctx.job_name, ctx.task_index]
      self.client_id = self.parts[0]["clients"].index(me)
      self.num_clients = len(self.parts[0]["clients"])
      self.pushes = 0
    if self.cuda:
      import torch
      from .. import ops
      torch.cuda.set_device(0)
      self._local_servers = local_servers
      if local_servers:
        self.ptrs = [getattr(sv, "base", None) or sv.tensor.data_ptr() for sv in local_servers]
      else:
        self.ptrs = [ops.C().symm_open(p["handle"]) for p in self.parts]
      self.hyper = torch.zeros(8, dtype=torch.float32, device="cuda")
      if self.slot_mode:
        self.layouts = [_slot_layout(p["hi"] - p["lo"], self.num_clients, True)
                        for p in self.parts]
        self._counter = torch.zeros(8, dtype=torch.int32, device="cuda")
        self._running_pulled = None
    else:
      from multiprocessing import shared_memory
      self.shms = [shared_memory.SharedMemory(name=p["name"]) for p in self.parts]
      if self.slot_mode:
        self.layouts = [_slot_layout(p["hi"] - p["lo"], self.num_clients, False)
                        for p in self.parts]
        self.arrays = [np.ndarray((p["hi"] - p["lo"],), dtype=np.float32, buffer=s.buf,
                                  offset=l["master"])
                       for p, s, l in zip(self.parts, self.shms, self.layouts)]
      else:
        self.arrays = [np.ndarray((p["hi"] - p["lo"],), dtype=np.float32, buffer=s.buf)
                       for p, s in zip(self.parts, self.shms)]

  # ------------------------------------------------------------- slot mode
  def set_lr(self, lr):
    """Change the learning rate the servers apply (hyper-parameters live with the state)."""
    for i, p in enumerate(self.parts):
      if self.cuda:
        from .. import ops
        h = ops.C().tensor_from_ptr(self.ptrs[i] + self.layouts[i]["hyper"], [8], "f32")
        h[0:1].fill_(float(lr))
      else:
        np.ndarray((8,), dtype=np.float32, buffer=self.shms[i].buf,
                   offset=self.layouts[i]["hyper"])[0] = lr

  def pull_model(self, weights=None, aux32=None, running=None, decay_end=None, total=None):
    """Slot mode: fetch the model the servers hold.  GPU: bf16 ``weights`` [total], fp32 ``aux32``
    (= elements [decay_end, total)) and the ``running`` statistics tail are filled by one kernel
    per server; CPU: returns the flat fp32 vector."""
    if not self.cuda:
      return np.concatenate([a for a in self.arrays]) if len(self.arrays) > 1 \
          else self.arrays[0].copy()
    if weights is None:
      raise ValueError("pull_model on a GPU needs the bf16 weights buffer")
    total = int(total if total is not None else weights.numel())
    decay_end = int(decay_end if decay_end is not None else total)
    _check_pull_model(self.numel, total, decay_end, weights, aux32, running)
    import torch
    from .. import ops
    if running is not None and (self._running_pulled is None
                                or self._running_pulled.numel() != running.numel()):
      self._running_pulled = torch.zeros_like(running)
    for p, ptr, lay in zip(self.parts, self.ptrs, self.layouts):
      ops.K.ps_pull_model({
          "wbf16": ptr + lay["wbf16"], "master": ptr + lay["master"],
          "weights": weights.data_ptr(), "aux32": aux32.data_ptr() if aux32 is not None else 0,
          "running": running.data_ptr() if running is not None else 0,
          "running_pulled": self._running_pulled.data_ptr() if running is not None else 0,
          "n": p["hi"] - p["lo"], "lo": p["lo"], "total": total, "decay_end": decay_end,
          "grid": 64})

  def push_grads(self, grads, running=None, total=None):
    """Slot mode: hand this step's gradients (flat fp32, length ``total``) to the servers.  The
    non-trainable tail, if any, is sent as (pulled - current) running statistics."""
    if self.cuda:
      total = int(total if total is not None else grads.numel())
      _check_push_grads(self.numel, total, grads, running, self._running_pulled)
    self.pushes += 1
    seq, slot = self.pushes, self.pushes % NSLOTS
    need = max(0, seq - NSLOTS)        # what must have been applied before the slot is reused
    k = self.client_id * NSLOTS + slot
    if self.cuda:
      from .. import ops
      for p, ptr, lay in zip(self.parts, self.ptrs, self.layouts):
        n = p["hi"] - p["lo"]
        ops.K.ps_push_slot({
            "slot": ptr + lay["slots"] + 4 * n * k, "grads": grads.data_ptr(),
            "running": running.data_ptr() if running is not None else 0,
            "running_pulled": self._running_pulled.data_ptr() if running is not None else 0,
            "n": n, "lo": p["lo"], "total": total,
            "applied_flag": ptr + lay["applied"] + 4 * k, "need_applied": need,
            "ready_flag": ptr + lay["ready"] + 4 * k, "seq": seq,
            "block_counter": self._counter.data_ptr(), "grid": 64})
      return
    g = grads.detach().cpu().numpy() if hasattr(grads, "detach") else np.asarray(grads)
    g = g.reshape(-1).astype(np.float32)
    for p, shm, lay in zip(self.parts, self.shms, self.layouts):
      n = p["hi"] - p["lo"]
      W = self.num_clients
      applied = np.ndarray((W * NSLOTS,), dtype=np.int32, buffer=shm.buf, offset=lay["applied"])
      ready = np.ndarray((W * NSLOTS,), dtype=np.int32, buffer=shm.buf, offset=lay["ready"])
      slots = np.ndarray((n * W * NSLOTS,), dtype=np.float32, buffer=shm.buf, offset=lay["slots"])
      t0 = time.time()
      while applied[k] < need:          # back-pressure: the server has not drained this slot yet
        time.sleep(0.0002)
        if time.time() - t0 > 120:
          raise RuntimeError("parameter server did not apply slot {} within 120 s".format(k))
      slots[k * n:(k + 1) * n] = g[p["lo"]:p["hi"]]
      ready[k] = seq

  # ------------------------------------------------------------------ pull
  def pull(self, out_fp32=None, out_bf16=None):
    """Fetch the current parameters.  GPU: fills the given device tensors (either may be None);
    CPU: returns a numpy copy (and fills ``out_fp32`` if it is a numpy array / torch tensor)."""
    if self.cuda:
      from .. import ops
      for p, ptr in zip(self.parts, self.ptrs):
        lo, hi = p["lo"], p["hi"]
        ops.K.ps_pull(ptr, out_fp32[lo:hi] if out_fp32 is not None else None,
                      out_bf16[lo:hi] if out_bf16 is not None else None, hi - lo)
      return out_fp32 if out_fp32 is not None else out_bf16
    flat = np.concatenate([a for a in self.arrays]) if len(self.arrays) > 1 else self.arrays[0].copy()
    if out_fp32 is not None:
      if hasattr(out_fp32, "numpy"):
        out_fp32.copy_(__import__("torch").from_numpy(flat))
      else:
        out_fp32[:] = flat
    return flat

  # ------------------------------------------------------------------ push
  def push(self, grad, lr, scale=1.0):
    """Apply ``w -= lr * scale * grad`` on the servers, asynchronously and without locking."""
    if self.cuda:
      from .. import ops
      self.hyper[0] = float(lr)
      self.hyper[3] = float(scale)
      for p, ptr in zip(self.parts, self.ptrs):
        ops.K.ps_push_dense(ptr, grad[p["lo"]:p["hi"]], self.hyper)
      return
    g = grad.detach().cpu().numpy() if hasattr(grad, "detach") else np.asarray(grad)
    g = g.reshape(-1).astype(np.float32)
    for p, a in zip(self.parts, self.arrays):
      a -= (lr * scale) * g[p["lo"]:p["hi"]]

  def push_sparse(self, grad_rows, indices, width, base=0, lr=1.0, scale=1.0):
    """Row-sparse update of a [rows, width] table stored at flat offset ``base``.  A row that
    straddles a server boundary is split: each server applies the elements it owns."""
    if self.cuda:
      import torch
      from .. import ops
      self.hyper[0] = float(lr)
      self.hyper[3] = float(scale)
      idx = indices.to(torch.int32)
      for p, ptr in zip(self.parts, self.ptrs):
        lo, hi = p["lo"], p["hi"]
        r0, r1, cuts = _sparse_plan(lo, hi, base, width)
        sel = (idx >= r0) & (idx < r1)
        if r1 > r0 and bool(sel.any()):
          rows = grad_rows[sel].contiguous()
          local = (idx[sel] - r0).contiguous()
          off = base + r0 * width - lo
          ops.K.ps_push_sparse(ptr + 4 * off, rows, local, self.hyper)
        # rows cut by this server's boundaries: the owned element range goes through the dense kernel
        for r, a, b in cuts:
          s0 = base + r * width
          for k in torch.nonzero(idx == r).flatten().tolist():
            seg = grad_rows[k].reshape(-1)[a - s0:b - s0].to(torch.float32).contiguous()
            ops.K.ps_push_dense(ptr + 4 * (a - lo), seg, self.hyper)
      return
    g = grad_rows.detach().cpu().numpy() if hasattr(grad_rows, "detach") else np.asarray(grad_rows)
    ix = indices.detach().cpu().numpy() if hasattr(indices, "detach") else np.asarray(indices)
    for p, a in zip(self.parts, self.arrays):
      for row, r in zip(g, ix):
        s = base + int(r) * width
        b0, b1 = max(s, p["lo"]), min(s + width, p["hi"])   # the part of the row this server owns
        if b0 < b1:
          a[b0 - p["lo"]:b1 - p["lo"]] -= (lr * scale) * row[b0 - s:b1 - s]

  def close(self):
    if self.cuda:
      from .. import ops
      for ptr in ([] if getattr(self, "_local_servers", None) else self.ptrs):
        try:
          ops.C().symm_close(ptr)
        except Exception:
          pass
    else:
      for s in self.shms:
        s.close()


class PSWorker(object):
  """Drives a native trainer (models/*: flat ParamStore + RunningArena) against slot-mode
  servers: ``step()`` = pull_model -> forward -> loss -> backward -> push_grads, all enqueued on
  the current stream, no host synchronisation and no barrier with the other workers."""

  def __init__(self, trainer, client):
    self.net, self.ps = trainer, client
    st = trainer.store
    assert client.numel == st.total + trainer.running.tensor().numel(), \
        "the servers were started for a different model"

  @staticmethod
  def server_args(trainer, optimizer="momentum", **hyper):
    """kwargs for ``ctx.start_cluster_server`` on the ps node: initial values = the trainer's
    parameters followed by its batch-norm running statistics (the non-trainable tail)."""
    import torch
    st = trainer.store
    flat = torch.cat([st.master.detach().float().reshape(-1), trainer.running.tensor().detach()])
    return dict(params=flat, optimizer=optimizer, decay_end=st.decay_end, ema_begin=st.total,
                **hyper)

  def pull(self):
    st = self.net.store
    self.ps.pull_model(st.weights, st.aux32, self.net.running.tensor(), decay_end=st.decay_end,
                       total=st.total)

  def step(self, images=None, labels=None):
    net, st = self.net, self.net.store
    self.pull()                                   # stale-tolerant read over NVLink
    if images is not None:
      net.set_input(images, labels)
    net._forward(True)
    net._loss(True)
    net._backward()
    self.ps.push_grads(st.grads, net.running.tensor(), total=st.total)
    return net.loss_sum


def attach(ctx, params=None, init=None, transport=None, **server_kwargs):
  """PSServer on a 'ps' node (``params`` = number of elements or an initial flat tensor;
  ``optimizer=...`` and its hyper-parameters select slot mode), PSClient everywhere else.
  ``transport``: 'ipc' | 'tcp' for the servers (default: by the hosts of the cluster spec, see
  :func:`transport`); clients follow what the servers published."""
  choose = globals()["transport"]
  if ctx.job_name == "ps":
    if params is None:
      raise ValueError("a ps node must be told the parameter count: start_cluster_server(params=N)")
    if hasattr(params, "numel") or isinstance(params, np.ndarray):
      init = params
      numel = int(params.numel() if hasattr(params, "numel") else params.size)
    else:
      numel = int(params)
    if (transport or choose(ctx)) == "tcp":
      from . import ps_net
      return ps_net.NetPSServer(ctx, numel, init, **server_kwargs)
    return PSServer(ctx, numel, init, **server_kwargs)
  return PSClient(ctx)


def transport(ctx):
  """'ipc' (CUDA IPC / shared memory: every node on one host) or 'tcp' (parallel/ps_net.py);
  ``TFOS_PS_TRANSPORT`` overrides the choice made from the hosts named in the cluster spec."""
  import os
  forced = os.environ.get("TFOS_PS_TRANSPORT", "auto")
  if forced in ("tcp", "ipc"):
    return forced
  hosts = set(a.rsplit(":", 1)[0] for nodes in ctx.cluster_spec.values() for a in nodes)
  return "tcp" if len(hosts) > 1 else "ipc"

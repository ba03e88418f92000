"""Pieces that every trainer's held-out evaluation shares (resnet._Evaluator, unet._SegEvaluator):
the sum of an fp64 accumulator over ranks and the host-batch staging loop."""
import numpy as np
import torch

from .. import ops


class RankSum(object):
  """Sum of an fp64 accumulator of ``slots`` values over all ranks, identical on every rank:
  in rank order through a symmetric buffer named ``name`` on one host (then ``all_reduce_inter``
  for HierComm), ``all_reduce`` for GroupComm, the accumulator itself without a communicator."""

  def __init__(self, comm, name, slots):
    self.comm, self.name, self.slots = comm, name, slots
    self.kind = None if comm is None else (
        "group" if getattr(comm, "cross_host", False) else
        "hier" if getattr(comm, "hierarchical", False) else "symm")
    self.totals = self.peers = None
    if self.kind in ("symm", "hier"):
      # fp64[slots] in a symmetric fp32 buffer: every rank sums all ranks' copies in rank order
      self.totals = comm.alloc(name, 2 * slots, torch.float32).view(torch.float64)

  def __call__(self, acc):
    """The summed ``acc`` as a host list of floats."""
    comm = self.comm
    if self.kind is None:
      tot = acc
    elif self.kind == "group":
      tot = acc.clone()
      comm.all_reduce(tot)
    else:
      if self.peers is None:
        C = ops.C()
        self.peers = [C.tensor_from_ptr(p, [2 * self.slots], "f32").view(torch.float64)
                      for p in comm.peer_ptrs(self.name)]
      self.totals.copy_(acc)
      comm.barrier()              # every rank's totals are written
      tot = self.peers[0].clone()
      for p in self.peers[1:]:
        tot += p
      comm.barrier()              # every rank has read them before the next pass rewrites them
      if self.kind == "hier":
        comm.all_reduce_inter(tot)
    return tot.cpu().tolist()


class HostStaging(object):
  """Runs ``step(images, labels)`` over (images, labels) pairs of at most ``batch`` rows.  Device
  batches go straight to ``step``; host batches are staged in page-locked memory and copied one
  batch ahead of the forward pass (DevicePrefetcher), so the copy of batch i + 1 overlaps the
  forward pass of batch i.  ``label_dtype(y)`` is the torch dtype host labels are staged in."""

  def __init__(self, device, batch, image_shape, label_shape):
    self.device, self.batch = device, batch
    self.image_shape, self.label_shape = tuple(image_shape), tuple(label_shape)
    self.feeders = {}

  def _feeder(self, dtype):
    if dtype not in self.feeders:
      from ..feed import DevicePrefetcher
      self.feeders[dtype] = DevicePrefetcher([((self.batch,) + self.image_shape, torch.uint8),
                                              ((self.batch,) + self.label_shape, dtype)],
                                             self.device, depth=2)
    return self.feeders[dtype]

  def run(self, step, batches, label_dtype=lambda y: torch.int32):
    pending = []

    def flush():
      n, feeder = pending.pop(0)
      dx, dy = feeder.pop()
      step(dx[:n], dy[:n])
      feeder.release()

    for images, labels in batches:
      if isinstance(images, torch.Tensor) and images.is_cuda:
        while pending:
          flush()
        step(images, labels)
        continue
      x = images.numpy() if isinstance(images, torch.Tensor) else np.asarray(images)
      y = labels.numpy() if isinstance(labels, torch.Tensor) else np.asarray(labels)
      n = len(x)
      if n > self.batch:
        raise ValueError("batch of {} rows exceeds the trainer's batch size {}".format(
            n, self.batch))
      feeder = self._feeder(label_dtype(y))
      hx, hy = feeder.acquire_host()
      hx.numpy()[:n] = x.reshape((n,) + self.image_shape)
      hy.numpy()[:n] = y.reshape((n,) + self.label_shape)
      feeder.push_host()
      pending.append((n, feeder))
      if len(pending) > 1:   # batch i + 1 is on its way: run batch i
        flush()
    while pending:
      flush()

"""What every served GPU replica behind ``pipeline.TFModel`` shares (models/resnet.ServedResNet,
models/unet.ServedUNet): uint8 image rows staged in page-locked memory and copied on a copy
stream, the network's device work captured as one CUDA graph after the first batch, and the
outputs read back into double-buffered page-locked memory behind an event.  ``submit`` enqueues
a batch and returns; ``collect`` returns the oldest one - pipeline._run_model drives a replica one
batch ahead, so the H2D copy of batch i+1 and the host's row handling overlap the kernels of
batch i.

Environment: ``TFOS_SERVE_BATCH`` (rows per batch, default 256), ``TFOS_SERVE_GRAPH`` (1: replay a
CUDA graph after the first batch), ``TFOS_SERVE_COPY_THREADS`` (threads filling the staging buffer
from row cells, default 4)."""
import os

import numpy as np
import torch


def serve_batch(batch=None):
  """Rows per served batch: ``batch`` when given, else ``TFOS_SERVE_BATCH`` (default 256)."""
  return int(batch or os.environ.get("TFOS_SERVE_BATCH", "256"))


class Replica(object):
  """Base of the served replicas.  A subclass builds its network, then calls ``__init__`` with
  the batch, the shape of one input image, its outputs as ``{name: device tensor [batch, ...]}``
  (views allowed; read back per batch in this order) and ``set_input(device_uint8_batch)``, and
  implements ``_run()``: the device work of one batch on the staged input (eager on the first
  batch, captured into a CUDA graph after it)."""

  def __init__(self, device, batch, image_shape, outputs, set_input):
    from ..feed import DevicePrefetcher
    self.B, self.image_shape = batch, tuple(image_shape)
    self.row_bytes = int(np.prod(self.image_shape))
    self._device = torch.device(device)
    self.feeder = DevicePrefetcher([((batch,) + self.image_shape, torch.uint8)], self._device,
                                   depth=2)
    self._outputs = dict(outputs)
    self.selected = tuple(self._outputs)
    self._host = {}          # name -> two page-locked buffers, allocated on first read-back
    self._set_input = set_input
    self.done = [torch.cuda.Event() for _ in range(2)]
    self._pending = []
    self._k = 0
    self.graph, self._batches = None, 0
    self.use_graph = os.environ.get("TFOS_SERVE_GRAPH", "1") == "1"
    self.copy_threads = max(1, int(os.environ.get("TFOS_SERVE_COPY_THREADS", "4")))
    if self.copy_threads > 1:
      from concurrent.futures import ThreadPoolExecutor
      self._pool = ThreadPoolExecutor(max_workers=self.copy_threads, thread_name_prefix="tfos-stage")

  def _run(self):
    raise NotImplementedError

  def _select_outputs(self, names):
    """Read back only the outputs ``names`` from the next submitted batch on; a selection that
    changes the device work (``_run`` may consult ``selected``) is captured anew."""
    names = tuple(dict.fromkeys(names))
    unknown = [n for n in names if n not in self._outputs]
    if unknown:
      raise ValueError("unknown output(s) {}: the model offers {}".format(unknown,
                                                                        list(self._outputs)))
    sel = tuple(n for n in self._outputs if n in names)
    if sel != self.selected:
      self.selected, self.graph, self._batches = sel, None, 0

  def _check_rows(self, n):
    if n > self.B:
      raise ValueError("batch of {} rows exceeds the served batch size {}".format(n, self.B))

  def submit(self, inputs):
    x = inputs["image"] if isinstance(inputs, dict) else inputs
    x = np.asarray(x)
    n = len(x)
    self._check_rows(n)
    x = x.reshape((n,) + self.image_shape)
    if n < self.B:   # ragged tail: pad (the padded rows' outputs are dropped)
      x = np.concatenate([x, np.zeros((self.B - n,) + x.shape[1:], dtype=x.dtype)])
    self.feeder.push_arrays([x])
    self._enqueue(n)

  def submit_rows(self, columns):
    """Same as :meth:`submit` for a column of raw row cells (bytes / memoryview / ndarray, one
    uint8 image each): every row is copied ONCE, straight into the page-locked staging buffer the
    H2D copy reads - no intermediate batch array (pipeline._run_model uses this when a served
    model offers it)."""
    rows = columns["image"] if isinstance(columns, dict) else columns
    n = len(rows)
    self._check_rows(n)
    (host,) = self.feeder.acquire_host()
    hv = host.numpy().reshape(self.B, -1)
    want = self.row_bytes

    def fill(lo, hi):
      for r in range(lo, hi):
        row = rows[r]
        a = np.frombuffer(row, dtype=np.uint8) if not isinstance(row, np.ndarray) \
            else row.reshape(-1)
        if a.size != want:
          raise ValueError("row {} holds {} values, the served image needs {} ({})".format(
              r, a.size, want, "x".join(str(d) for d in self.image_shape)))
        hv[r] = a

    # 38.5 MB per 256-image ResNet batch: one thread copies ~5 GB/s, which is slower than the GPU
    # consumes it (8.5 vs 6.5 ms per batch); numpy releases the GIL during the copies, so a few
    # threads fill disjoint row ranges of the staging buffer in parallel
    k = self.copy_threads
    if k > 1 and n >= 4 * k:
      step = (n + k - 1) // k
      list(self._pool.map(lambda i: fill(i * step, min(n, (i + 1) * step)), range(k)))
    else:
      fill(0, n)
    if n < self.B:
      hv[n:] = 0
    self.feeder.push_host()
    self._enqueue(n)

  def _capture(self):
    """The whole device work of one batch as ONE CUDA graph: the host thread that also fills the
    staging buffers spends microseconds, not a millisecond, per batch on launches."""
    dev = self._device
    cur = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(cur)
    with torch.cuda.stream(side):
      self._run()
    cur.wait_stream(side)
    torch.cuda.synchronize(dev)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      self._run()
    self.graph = g

  def _host_buffers(self, name):
    bufs = self._host.get(name)
    if bufs is None:
      t = self._outputs[name]
      bufs = self._host[name] = [torch.empty(t.shape, dtype=t.dtype).pin_memory()
                                 for _ in range(2)]
    return bufs

  def _enqueue(self, n):
    (dx,) = self.feeder.pop()
    self._set_input(dx)
    self.feeder.release()
    if self.graph is None and self.use_graph and self._batches >= 1:
      self._capture()
    if self.graph is not None:
      self.graph.replay()
    else:
      self._run()
    self._batches += 1
    k = self._k
    self._k ^= 1
    for name in self.selected:
      self._host_buffers(name)[k].copy_(self._outputs[name], non_blocking=True)
    self.done[k].record(torch.cuda.current_stream(self._device))
    self._pending.append((k, n, self.selected))

  def collect(self):
    k, n, names = self._pending.pop(0)
    self.done[k].synchronize()
    return {name: self._host[name][k][:n].numpy().copy() for name in names}

  def pending(self):
    return len(self._pending)

  def __call__(self, **inputs):
    self.submit(inputs)
    return self.collect()

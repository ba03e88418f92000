"""Segmentation U-Net of the reference (examples/segmentation/segmentation_spark.py:67-119) on the
native engine: frozen MobileNetV2 encoder (128x128x3 input, five skip taps) + four pix2pix
``upsample`` blocks (Conv2DTranspose 3x3 stride 2 -> BatchNorm -> ReLU; 512/256/128/64 filters)
+ a final Conv2DTranspose to the class logits; Adam, per-pixel sparse cross-entropy.

Kernel mapping:
  encoder   1x1 expand / project convs -> wgmma GEMM with folded inference-BN bias and fused
            ReLU6; 3x3 depthwise -> depthwise3x3 kernel (bias + ReLU6 fused); stem 3x3/s2 ->
            implicit GEMM.  Forward only (``layer.trainable = False`` in the reference, :83).
  decoder   Conv2DTranspose forward = the stride-2 *data-gradient* implicit GEMM (four output
            parity classes), with batch-norm statistics fused into its epilogue; its backward
            = stride-2 fprop (input gradient) + stride-2 wgrad.  Channel concatenation is a
            strided 16-byte copy into the concat buffer.
There is no pretrained checkpoint on this box (no network): the encoder is random-initialised,
which leaves shapes, FLOPs and memory traffic - everything the benchmarks measure - unchanged.
"""
import math

import numpy as np
import torch

from .. import ops
from ..ops import igemm
from . import evaluation, serving
from .engine import BatchNorm, ParamStore, RunningArena, constant, he_normal

# (expansion t, out channels c, repeats n, stride s) - MobileNetV2, width 1.0
MBV2 = [(1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2),
        (6, 320, 1, 1)]
#: blocks whose *expansion* output is a skip tap (Keras names block_{1,3,6,13}_expand_relu)
SKIP_BLOCKS = (1, 3, 6, 13)


def _buf(shape, dev, dtype=torch.bfloat16):
  return torch.zeros(shape, dtype=dtype, device=dev)


class _FrozenConv(object):
  """1x1 or 3x3 convolution + folded inference batch-norm (+ReLU6), forward only."""

  def __init__(self, gen, cin, cout, k, stride, act, dev):
    w = torch.randn(cout, k, k, cin, generator=gen) * math.sqrt(2.0 / (k * k * cin))
    gamma = 1.0 + 0.1 * torch.randn(cout, generator=gen)
    beta, mean = 0.1 * torch.randn(cout, generator=gen), 0.1 * torch.randn(cout, generator=gen)
    var = 1.0 + 0.1 * torch.rand(cout, generator=gen)
    scale = gamma / torch.sqrt(var + 1e-3)
    self.w = (w * scale.view(-1, 1, 1, 1)).to(dev, torch.bfloat16).contiguous()
    self.bias = (beta - mean * scale).to(dev, torch.float32).contiguous()
    self.k, self.stride, self.act = k, stride, act

  def build(self, x, y):
    self.x, self.y = x, y
    self.plan = igemm.conv_fprop(x, self.w, y, self.stride, self.k // 2, bias=self.bias,
                                 relu=self.act)

  def forward(self):
    self.plan.run()


class _FrozenDepthwise(object):

  def __init__(self, gen, c, stride, dev):
    w = torch.randn(9, c, generator=gen) * math.sqrt(2.0 / 9)
    scale = 1.0 + 0.1 * torch.randn(c, generator=gen)
    self.w = (w * scale.view(1, -1)).to(dev, torch.bfloat16).contiguous()
    self.bias = (0.1 * torch.randn(c, generator=gen)).to(dev, torch.float32).contiguous()
    self.stride = stride

  def build(self, x, y):
    self.x, self.y = x, y

  def forward(self):
    ops.K.depthwise3x3_fwd(self.x, self.w, self.bias, self.y, self.stride, 2)


class MobileNetV2Encoder(object):
  """Frozen feature extractor returning the five skip tensors."""

  def __init__(self, batch, image, dev, seed=7):
    gen = torch.Generator(device="cpu")
    gen.manual_seed(seed)
    B = batch
    self.x = _buf((B, image, image, 8), dev)  # 3 real + 5 zero channels (16-byte pixels)
    self.layers = []
    H = image // 2
    cur = _buf((B, H, H, 32), dev)
    stem = _FrozenConv(gen, 8, 32, 3, 2, 2, dev)
    stem.w[..., 3:] = 0
    stem.build(self.x, cur)
    self.layers.append(stem)
    self.skips = []
    cin, block = 32, 0
    for t, c, n, s in MBV2:
      for i in range(n):
        stride = s if i == 0 else 1
        inp = cur
        hidden = cin * t
        if t != 1:
          e = _FrozenConv(gen, cin, hidden, 1, 1, 2, dev)
          ebuf = _buf((B, H, H, hidden), dev)
          e.build(cur, ebuf)
          self.layers.append(e)
          cur = ebuf
          if block in SKIP_BLOCKS:
            self.skips.append(cur)
        H2 = (H - 1) // stride + 1
        d = _FrozenDepthwise(gen, hidden, stride, dev)
        dbuf = _buf((B, H2, H2, hidden), dev)
        d.build(cur, dbuf)
        self.layers.append(d)
        p = _FrozenConv(gen, hidden, c, 1, 1, 0, dev)
        pbuf = _buf((B, H2, H2, c), dev)
        p.build(dbuf, pbuf)
        self.layers.append(p)
        cur = pbuf
        if stride == 1 and cin == c:
          self.layers.append(_Residual(pbuf, inp))
        cin, H, block = c, H2, block + 1
    self.skips.append(cur)  # block_16_project, 4x4x320 at 128 input
    self.out_hw = H

  def forward(self):
    for layer in self.layers:
      layer.forward()
    return self.skips


class _Residual(object):

  def __init__(self, y, x):
    self.y, self.x = y, x

  def forward(self):
    ops.K.add_act(self.y, self.x, self.y, 0)


class _Upsample(object):
  """Conv2DTranspose(filters, 3, strides=2, padding='same', use_bias=False) -> BN -> ReLU."""

  def __init__(self, store, name, cin, cout):
    self.cin, self.cout, self.store = cin, cout, store
    # layout [Cin, 3, 3, Cout]: K-rows of the dgrad-style forward, KRSC of the backward fprop
    self.sw = store.register(name + ".w", (cin, 3, 3, cout), True, he_normal(9 * cin))
    self.bn = BatchNorm(store, name + ".bn", cout)

  def build(self, x, raw, act_out, g_act, g_raw, g_x, dev, running, training=True):
    """x [B,h,w,cin] -> raw/act_out [B,2h,2w,cout]; g_* are the matching gradient buffers;
    ``running`` (engine.RunningArena) holds the batch norm's running statistics.
    ``training=False``: only the inference convolution is planned (g_* are not used)."""
    st = self.store
    self.bn.build(dev, running=running)
    self.x, self.raw, self.act = x, raw, act_out
    self.g_act, self.g_raw = g_act, g_raw
    self.fwd = self.wgrad = self.dgrad = None
    if training:
      # BN statistics are fused into every parity-class launch of the transposed conv
      self.fwd = igemm.conv_dgrad(x, st.w(self.sw), raw, 2, 1, stats=self.bn.stats)
    # inference (predict, evaluation): the same convolution without the statistics, so that it
    # leaves nothing in the accumulators that the next training step's bn_finalize would read
    self.fwd_inference = igemm.conv_dgrad(x, st.w(self.sw), raw, 2, 1)
    if not training:
      return
    self.wgrad = igemm.conv_wgrad(x, g_raw, st.g(self.sw), 2, 1)
    self.dgrad = igemm.conv_fprop(g_raw, st.w(self.sw), g_x, 2, 1) if g_x is not None else None

  def forward(self, training=True):
    (self.fwd if training else self.fwd_inference).run()
    self.bn.forward(self.raw, self.act, None, 1, training)

  def forward_eval(self, mean, var, scale, shift):
    """Inference forward with the running statistics ``mean`` / ``var`` (rank 0's copy during an
    evaluation); the batch norm's coefficients go to ``scale`` / ``shift``, the evaluator's own."""
    self.fwd_inference.run()
    bn = self.bn
    ops.K.bn_inference_coeffs(bn.gamma, bn.beta, mean, var, scale, shift, bn.eps)
    ops.C().bn_set_row_reverse(False)
    ops.K.bn_apply(self.raw, None, scale, shift, self.act, 1, None)

  def backward(self):
    self.bn.backward(self.g_act, self.raw, self.act, self.g_raw, relu=True)
    self.wgrad.run()
    if self.dgrad is not None:
      self.dgrad.run()


class UNetTrainer(object):
  """Static-buffer U-Net for ``batch`` images of ``image`` x ``image`` x 3 and ``classes`` labels.
  ``training=False`` builds only what the forward pass needs (predict, evaluate, serving): no
  gradient buffers, no backward or statistics-fused plans and no optimizer (``optim`` is None)."""

  UP = (512, 256, 128, 64)

  def __init__(self, batch=64, image=128, classes=3, device="cuda:0", lr=1e-3, comm=None, seed=1234,
               training=True):
    assert classes <= 8
    self.device = dev = torch.device(device)
    self.B, self.image, self.classes = batch, image, classes
    self.comm = comm
    self.training = tr = training
    B = batch
    self.encoder = MobileNetV2Encoder(batch, image, dev)
    skips = self.encoder.skips  # [64x64x96, 32x32x144, 16x16x192, 8x8x576, 4x4x320]
    st = self.store = ParamStore()
    self.ups = []
    cin = skips[-1].shape[-1]
    for i, f in enumerate(self.UP):
      self.ups.append(_Upsample(st, "up{}".format(i), cin, f))
      cin = f + skips[-2 - i].shape[-1]
    self.s_last = st.register("last.w", (cin, 3, 3, 8), True, he_normal(9 * cin))
    self.s_last_b = st.register("last.b", (8,), False, constant(0.0))
    st.finalize(dev, alloc=comm.alloc if comm is not None else None, seed=seed, grads=tr)

    x, h = skips[-1], skips[-1].shape[1]
    g_x = None  # the encoder is frozen: no gradient flows into it
    # the decoder batch norms' running statistics, one flat buffer (checkpoints, evaluation)
    self.running = RunningArena(dev, capacity=2 * sum(self.UP))
    self.cats, self.g_cats = [], []
    for i, up in enumerate(self.ups):
      f, skip = self.UP[i], skips[-2 - i]
      h *= 2
      raw, act = _buf((B, h, h, f), dev), _buf((B, h, h, f), dev)
      g_act = g_raw = g_cat = None
      if tr:
        g_act, g_raw = _buf((B, h, h, f), dev), _buf((B, h, h, f), dev)
      up.build(x, raw, act, g_act, g_raw, g_x, dev, self.running, training=tr)
      cat = _buf((B, h, h, f + skip.shape[-1]), dev)
      if tr:
        g_cat = _buf(cat.shape, dev)
        self.g_cats.append((g_cat, g_act, f))
      self.cats.append((cat, act, skip, f))
      x, g_x = cat, g_cat
    h *= 2
    self.logits = _buf((B, h, h, 8), dev)
    self.dlogits = _buf((B, h, h, 8), dev) if tr else None
    self.labels = torch.zeros(B, h, h, dtype=torch.int32, device=dev)
    self.p_last = igemm.conv_dgrad(x, st.w(self.s_last), self.logits, 2, 1, bias=st.f32(self.s_last_b))
    self.p_last_wgrad = self.p_last_dgrad = self.optim = None
    if tr:
      self.p_last_wgrad = igemm.conv_wgrad(x, self.dlogits, st.g(self.s_last), 2, 1)
      self.p_last_dgrad = igemm.conv_fprop(self.dlogits, st.w(self.s_last), g_x, 2, 1)
    self.loss_sum = torch.zeros(1, dtype=torch.float32, device=dev)
    self.correct = torch.zeros(1, dtype=torch.float32, device=dev)
    self.in_u8 = _buf((B, image, image, 3), dev, torch.uint8)
    if tr:
      from ..parallel.fused_optim import FusedOptimizer
      self.optim = FusedOptimizer(st, comm=comm, opt="adam", lr=lr, weight_decay=0.0)
    self.graph = None

  # ------------------------------------------------------------------ data
  def synthetic_batch(self, seed=0):
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    x = torch.randint(0, 256, (self.B, self.image, self.image, 3), dtype=torch.uint8, generator=g)
    y = torch.randint(0, self.classes, (self.B, self.image, self.image), dtype=torch.int32,
                      generator=g)
    return x.to(self.device), y.to(self.device)

  def set_input(self, images_u8, labels=None):
    self.in_u8.copy_(images_u8, non_blocking=True)
    if labels is not None:
      self.labels.copy_(labels.reshape(self.labels.shape), non_blocking=True)

  # ------------------------------------------------------------------ step
  def _forward(self, training=True, u8=None, bn=None):
    """Forward pass of the image batch in ``u8`` (default ``in_u8``).  ``bn``: one
    (mean, var, scale, shift) per decoder block for an evaluation forward (_Upsample.forward_eval)."""
    K = ops.K
    # [0, 255] -> [-1, 1] (the reference normalises with x / 127.5 - 1... here (x/255 - .5)/.5)
    K.decode_normalize(self.in_u8 if u8 is None else u8, self.encoder.x, 0, [0.5, 0.5, 0.5],
                       [0.5, 0.5, 0.5])
    self.encoder.forward()
    for i, (up, (cat, act, skip, f)) in enumerate(zip(self.ups, self.cats)):
      if bn is None:
        up.forward(training)
      else:
        up.forward_eval(*bn[i])
      K.copy_channels(act, cat, f, 0, 0)
      K.copy_channels(skip, cat, skip.shape[-1], 0, f)
    self.p_last.run()

  def step_kernels(self):
    if not self.training:
      raise RuntimeError("this UNetTrainer was built with training=False: it cannot train")
    K = ops.K
    self._forward(True)
    self.loss_sum.zero_()
    self.correct.zero_()
    npix = self.labels.numel()
    K.pixel_xent(self.logits, self.labels, self.dlogits, self.loss_sum, self.correct, self.classes,
                 1.0 / npix)
    self.optim.zero_grads()
    self.p_last_wgrad.run()
    K.colsum(self.dlogits, self.store.g(self.s_last_b))
    self.p_last_dgrad.run()
    for up, (g_cat, g_act, f) in zip(reversed(self.ups), reversed(self.g_cats)):
      K.copy_channels(g_cat, g_act, f, 0, 0)  # gradient of the decoder half of the concat
      up.backward()
    self.optim.step()

  def capture(self):
    s = torch.cuda.Stream(device=self.device)
    s.wait_stream(torch.cuda.current_stream(self.device))
    with torch.cuda.stream(s):
      for _ in range(2):
        self.step_kernels()
    torch.cuda.current_stream(self.device).wait_stream(s)
    torch.cuda.synchronize(self.device)
    g = torch.cuda.CUDAGraph()
    # cross-host communicator: its collectives stay outside the graph (FusedOptimizer.finish()
    # defers them), but the process group's watchdog thread may still poll events of the warm-up
    # collectives - thread-local capture keeps that from invalidating the capture
    mode = "thread_local" if getattr(self.optim, "group_mode", False) else "global"
    with torch.cuda.graph(g, capture_error_mode=mode):
      self.step_kernels()
    self.graph = g

  def train_step(self, images_u8=None, labels=None):
    if images_u8 is not None:
      self.set_input(images_u8, labels)
    if self.graph is not None:
      self.graph.replay()
      self.optim.after_replay()   # cross-host communicator: all-reduce + update outside the graph
    else:
      self.step_kernels()
    return self.loss_sum

  def predict(self, images_u8=None):
    """Logits [B, H, W, classes] of ``images_u8`` (staged into ``in_u8``), with the decoder batch
    norms on their running statistics; accumulates no batch statistics."""
    if images_u8 is not None:
      self.set_input(images_u8)
    self._forward(False)
    return self.logits[..., :self.classes]

  # ------------------------------------------------------------------ state
  def state_dict(self):
    """Parameters (fp32 masters, assembled across ranks when sharded) + the decoder batch norms'
    running statistics (``__running__``) + the frozen encoder (``__encoder__``: one (bf16 filter,
    fp32 bias) pair per convolution of ``encoder.layers``, in that order, as the forward uses
    them): everything inference or a resumed run needs, independent of the loading host's RNG."""
    sd = dict(self.store.state_dict())
    sd["__running__"] = self.running.tensor().detach().cpu().clone()
    sd["__encoder__"] = [(c.w.detach().cpu().clone(), c.bias.detach().cpu().clone())
                         for c in self._encoder_convs()]
    return sd

  def load_state_dict(self, sd):
    """Inverse of state_dict(); a dict without ``__running__`` keeps the current running
    statistics, one without ``__encoder__`` (checkpoints written before the encoder was part of
    the state) keeps the seeded encoder."""
    sd = dict(sd)
    running = sd.pop("__running__", None)
    encoder = sd.pop("__encoder__", None)
    if encoder is not None:
      convs = self._encoder_convs()
      if len(encoder) != len(convs) or any(
          w.shape != c.w.shape or b.shape != c.bias.shape for c, (w, b) in zip(convs, encoder)):
        raise ValueError("__encoder__ does not match this U-Net's encoder ({} convolutions)".format(
            len(convs)))
      for c, (w, b) in zip(convs, encoder):
        c.w.copy_(w.to(self.device, torch.bfloat16))
        c.bias.copy_(b.to(self.device, torch.float32))
    self.store.load_state_dict(sd)
    if running is not None:
      self.running.tensor().copy_(running.to(self.device))

  def _encoder_convs(self):
    return [c for c in self.encoder.layers if not isinstance(c, _Residual)]

  # ------------------------------------------------------------------ serving
  export_builder = "tensorflowonspark_b200.models.unet:build_served"
  export_signatures = {"serving_default": {
      "inputs": {"image": "image"}, "outputs": {"mask": "mask", "logits": "logits"},
      "input_dtypes": {"image": "uint8"},
      "output_dtypes": {"mask": "uint8", "logits": "float32"}}}

  @property
  def export_builder_args(self):
    return {"image": self.image, "classes": self.classes}

  # ------------------------------------------------------- held-out evaluation
  def eval_begin(self):
    """Start an evaluation pass: zero the totals and take rank 0's running statistics.
    Stream-ordered after the last ``train_step``; the first call allocates the evaluation
    buffers."""
    if getattr(self, "_evaluator", None) is None:
      self._evaluator = _SegEvaluator(self)
    self._evaluator.begin()

  def eval_step(self, images_u8, masks):
    """Add the totals of n <= B images (uint8 [n, H, W, 3]) and their masks ([n, H, W], uint8 or
    int32, host or device; widened on the device, out-of-range values count as invalid).  Runs
    the forward pass on the training buffers with the running statistics, leaving ``in_u8`` /
    ``labels`` and the training state untouched; ``logits`` then holds the batch's logits.  No
    host sync."""
    self._eval_state().step(images_u8, masks)

  def eval_end(self):
    """Totals summed over all ranks (identical on every rank), see seg_eval_result.  Raises
    ValueError on every rank when any rank saw a mask value outside [0, classes)."""
    return self._eval_state().end()

  def evaluate(self, batches):
    """eval_begin + eval_step over ``(images, masks)`` pairs + eval_end.  Host batches go through
    page-locked staging: the copy of batch i + 1 overlaps the forward pass of batch i."""
    self.eval_begin()
    self._evaluator.run(batches)
    return self.eval_end()

  def _eval_state(self):
    if getattr(self, "_evaluator", None) is None:
      raise RuntimeError("eval_begin() has not been called")
    return self._evaluator


# accumulator slots of seg_eval_metrics (csrc/ops.h kSegEval*); slot SEG_IMAGES counts images
SEG_COUNT, SEG_CORRECT, SEG_INVALID, SEG_LOSS, SEG_CONFUSION, SEG_SLOTS = 0, 1, 2, 3, 4, 68
SEG_IMAGES, SEG_ACC = 68, 72


def seg_eval_result(totals, classes):
  """Host metrics from the summed accumulator ``totals`` (a sequence of SEG_ACC floats):
  {"count": scored pixels, "images", "loss", "accuracy", "mean_iou", "iou": [classes values]}.
  IoU of class c = cm[c, c] / (row_c + col_c - cm[c, c]) of the confusion matrix cm[label, pred];
  a class with an empty union has IoU NaN and is left out of mean_iou (NaN when every class is).
  loss and accuracy are means over the scored pixels (NaN when there are none).  Raises
  ValueError when any mask value was outside [0, classes)."""
  h = [float(v) for v in totals]
  if h[SEG_INVALID] > 0:
    raise ValueError("evaluation saw {} mask value(s) outside [0, {})".format(
        int(h[SEG_INVALID]), classes))
  count = int(h[SEG_COUNT])
  cm = [h[SEG_CONFUSION + 8 * y:SEG_CONFUSION + 8 * y + 8] for y in range(8)]
  iou = []
  for c in range(classes):
    inter = cm[c][c]
    union = sum(cm[c][:classes]) + sum(cm[y][c] for y in range(classes)) - inter
    iou.append(inter / union if union > 0 else float("nan"))
  seen = [v for v in iou if v == v]
  mean = (lambda v: v / count) if count else (lambda v: float("nan"))
  return {"count": count, "images": int(h[SEG_IMAGES]), "loss": mean(h[SEG_LOSS]),
          "accuracy": mean(h[SEG_CORRECT]),
          "mean_iou": sum(seen) / len(seen) if seen else float("nan"), "iou": iou}


def _widen(masks):
  """Mask values as int32 without narrowing any of them: values beyond the int32 range are
  clamped, which keeps them outside [0, classes) and so invalid."""
  m = torch.as_tensor(masks)
  if m.dtype in (torch.uint8, torch.int32):
    return m
  return m.long().clamp(-1, 2 ** 31 - 1)


class _SegEvaluator(object):
  """Held-out evaluation on a UNetTrainer's own buffers (eval_begin / eval_step / eval_end).

  The forward pass is the inference network (transposed convolutions without batch statistics,
  batch norms on running statistics) on the trainer's activation buffers: the next training
  forward rewrites all of them, and backward reads only what its own forward wrote.  The bf16
  filters and aux32 are identical on every rank; the running statistics are rank 0's - the ones
  its checkpoint carries - so every rank scores the same model.  Only the uint8 images, int32
  masks, per-block batch-norm coefficients and the metric accumulators are extra memory,
  allocated on the first eval_begin."""

  def __init__(self, net):
    dev, comm = net.device, net.comm
    self.net, self.comm, self.V = net, comm, net.classes
    self.u8 = torch.zeros_like(net.in_u8)         # never in_u8: drivers stage a batch and replay
    self.labels = torch.zeros_like(net.labels)
    self.n_valid = torch.zeros(1, dtype=torch.int32, device=dev)
    self.acc = torch.zeros(SEG_ACC, dtype=torch.float64, device=dev)
    self.partial = torch.zeros(ops.C().seg_eval_scratch(self.labels.numel()), dtype=torch.float64,
                               device=dev)
    self.counter = torch.zeros(1, dtype=torch.int32, device=dev)
    if comm is None:
      self.running = net.running.tensor()
    else:
      self.running = comm.alloc("seg_eval_running", net.running.used, torch.float32)
    base = net.running.buf.data_ptr()
    view = lambda t: self.running[(t.data_ptr() - base) // 4:][:t.numel()]  # noqa: E731
    self.bn = [(view(up.bn.running_mean), view(up.bn.running_var),
                torch.zeros(up.cout, dtype=torch.float32, device=dev),
                torch.zeros(up.cout, dtype=torch.float32, device=dev)) for up in net.ups]
    self.rank_sum = evaluation.RankSum(comm, "seg_eval_totals", SEG_ACC)
    self.staging = evaluation.HostStaging(dev, net.B, self.u8.shape[1:], self.labels.shape[1:])
    self.graph, self.calls, self.images = None, 0, 0

  def begin(self):
    net, comm = self.net, self.comm
    self.acc.zero_()
    self.images = 0
    if comm is not None:
      self.running.copy_(net.running.tensor())
      comm.broadcast("seg_eval_running", 0)

  def _run(self):
    self.net._forward(False, self.u8, self.bn)
    ops.K.seg_eval_metrics(self.net.logits, self.labels, self.n_valid, self.acc, self.partial,
                           self.counter, self.V)

  def step(self, images_u8, masks):
    n = len(images_u8)
    if n > self.net.B:
      raise ValueError("batch of {} images exceeds the trainer's batch size {}".format(
          n, self.net.B))
    if n:
      x = torch.as_tensor(images_u8)
      self.u8[:n].copy_(x.reshape((n,) + tuple(self.u8.shape[1:])), non_blocking=True)
      self.labels[:n].copy_(_widen(masks).reshape((n,) + tuple(self.labels.shape[1:])),
                            non_blocking=True)
    self.n_valid.fill_(n)
    if self.graph is None and self.calls >= 1:
      self._capture()
    if self.graph is not None:
      self.graph.replay()
    else:
      self._run()
    self.calls += 1
    self.images += n

  def _capture(self):
    """The evaluation forward + metric as one CUDA graph, after one eager call; thread-local
    capture under a cross-host communicator, as in UNetTrainer.capture."""
    g = torch.cuda.CUDAGraph()
    mode = "thread_local" if getattr(self.net.optim, "group_mode", False) else "global"
    with torch.cuda.graph(g, capture_error_mode=mode):
      self._run()
    self.graph = g

  def run(self, batches):
    """eval_step over (images, masks) pairs; host masks are staged as uint8 when they are uint8,
    as int32 otherwise."""
    def host(pairs):
      for x, y in pairs:
        if not (isinstance(x, torch.Tensor) and x.is_cuda):
          y = _widen(y.numpy() if isinstance(y, torch.Tensor) else np.asarray(y))
        yield x, y
    self.staging.run(self.step, host(batches),
                     lambda y: torch.uint8 if y.dtype == np.uint8 else torch.int32)

  def end(self):
    self.acc[SEG_IMAGES].fill_(self.images)
    return seg_eval_result(self.rank_sum(self.acc), self.V)


class ServedUNet(serving.Replica):
  """Inference callable behind ``pipeline.TFModel`` / the inference CLI: one bf16 U-Net replica
  (a ``training=False`` trainer) on the executor's GPU.  Input ``image``: uint8 [n, H, W, 3] (or
  one row cell of H*W*3 bytes per image).  Outputs ``mask``: uint8 [n, H, W], the class every
  pixel is predicted as - exactly the prediction evaluation scores (seg_predict); ``logits``:
  fp32 [n, H, W, classes].  The forward pass + seg_predict run as one CUDA graph after the first
  batch; ``select_outputs`` keeps the logits (12x the bytes of the mask at 3 classes) on the
  device unless they are asked for (models/serving.Replica)."""

  def __init__(self, state, image=128, classes=3, batch=256, device="cuda:0"):
    torch.cuda.set_device(torch.device(device))
    self.net = UNetTrainer(batch=batch, image=image, classes=classes, device=device,
                           training=False)
    self.net.load_state_dict(state)
    self.image, self.V = image, classes
    dev = self.net.device
    self.mask = torch.zeros(batch, image, image, dtype=torch.uint8, device=dev)
    self.logits = torch.zeros(batch, image, image, classes, dtype=torch.float32, device=dev)
    super(ServedUNet, self).__init__(dev, batch, (image, image, 3),
                                     {"mask": self.mask, "logits": self.logits},
                                     self.net.set_input)

  def select_outputs(self, names):
    """Compute and read back only the outputs ``names`` (``mask`` and / or ``logits``) from the
    next batch on; ValueError for a name the model does not offer."""
    self._select_outputs(names)

  def _run(self):
    self.net._forward(False)
    ops.K.seg_predict(self.net.logits, self.mask,
                      self.logits if "logits" in self.selected else None, self.V)


def build_served(state, image=128, classes=3, batch=None, **_):
  """Export builder (utils/checkpoint.py): rebuilds the replica on the executor's GPU with
  ``TFOS_SERVE_BATCH`` rows per batch unless ``batch`` is given."""
  return ServedUNet(state, image=image, classes=classes, batch=serving.serve_batch(batch))

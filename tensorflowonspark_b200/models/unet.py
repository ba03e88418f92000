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

import torch

from .. import ops
from ..ops import igemm
from .engine import BatchNorm, ParamStore, constant, he_normal

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

  def build(self, x, raw, act_out, g_act, g_raw, g_x, dev):
    """x [B,h,w,cin] -> raw/act_out [B,2h,2w,cout]; g_* are the matching gradient buffers."""
    st = self.store
    self.bn.build(dev)
    self.x, self.raw, self.act = x, raw, act_out
    self.g_act, self.g_raw = g_act, g_raw
    # BN statistics are fused into every parity-class launch of the transposed conv
    self.fwd = igemm.conv_dgrad(x, st.w(self.sw), raw, 2, 1, stats=self.bn.stats)
    self.wgrad = igemm.conv_wgrad(x, g_raw, st.g(self.sw), 2, 1)
    self.dgrad = igemm.conv_fprop(g_raw, st.w(self.sw), g_x, 2, 1) if g_x is not None else None

  def forward(self, training=True):
    self.fwd.run()
    self.bn.forward(self.raw, self.act, None, 1, training)

  def backward(self):
    self.bn.backward(self.g_act, self.raw, self.act, self.g_raw, relu=True)
    self.wgrad.run()
    if self.dgrad is not None:
      self.dgrad.run()


class UNetTrainer(object):
  """Static-buffer U-Net for ``batch`` images of ``image`` x ``image`` x 3 and ``classes`` labels."""

  UP = (512, 256, 128, 64)

  def __init__(self, batch=64, image=128, classes=3, device="cuda:0", lr=1e-3, comm=None, seed=1234):
    assert classes <= 8
    self.device = dev = torch.device(device)
    self.B, self.image, self.classes = batch, image, classes
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
    st.finalize(dev, alloc=comm.alloc if comm is not None else None, seed=seed)

    x, h = skips[-1], skips[-1].shape[1]
    g_x = None  # the encoder is frozen: no gradient flows into it
    self.cats, self.g_cats = [], []
    for i, up in enumerate(self.ups):
      f, skip = self.UP[i], skips[-2 - i]
      h *= 2
      raw, act = _buf((B, h, h, f), dev), _buf((B, h, h, f), dev)
      g_act, g_raw = _buf((B, h, h, f), dev), _buf((B, h, h, f), dev)
      up.build(x, raw, act, g_act, g_raw, g_x, dev)
      cat = _buf((B, h, h, f + skip.shape[-1]), dev)
      g_cat = _buf(cat.shape, dev)
      self.cats.append((cat, act, skip, f))
      self.g_cats.append((g_cat, g_act, f))
      x, g_x = cat, g_cat
    h *= 2
    self.logits = _buf((B, h, h, 8), dev)
    self.dlogits = _buf((B, h, h, 8), dev)
    self.labels = torch.zeros(B, h, h, dtype=torch.int32, device=dev)
    self.p_last = igemm.conv_dgrad(x, st.w(self.s_last), self.logits, 2, 1, bias=st.f32(self.s_last_b))
    self.p_last_wgrad = igemm.conv_wgrad(x, self.dlogits, st.g(self.s_last), 2, 1)
    self.p_last_dgrad = igemm.conv_fprop(self.dlogits, st.w(self.s_last), g_x, 2, 1)
    self.loss_sum = torch.zeros(1, dtype=torch.float32, device=dev)
    self.correct = torch.zeros(1, dtype=torch.float32, device=dev)
    self.in_u8 = _buf((B, image, image, 3), dev, torch.uint8)
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
  def _forward(self, training=True):
    K = ops.K
    # [0, 255] -> [-1, 1] (the reference normalises with x / 127.5 - 1... here (x/255 - .5)/.5)
    K.decode_normalize(self.in_u8, self.encoder.x, 0, [0.5, 0.5, 0.5], [0.5, 0.5, 0.5])
    self.encoder.forward()
    for up, (cat, act, skip, f) in zip(self.ups, self.cats):
      up.forward(training)
      K.copy_channels(act, cat, f, 0, 0)
      K.copy_channels(skip, cat, skip.shape[-1], 0, f)
    self.p_last.run()

  def step_kernels(self):
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
    if images_u8 is not None:
      self.set_input(images_u8)
    self._forward(False)
    return self.logits[..., :self.classes]

"""Segmentation U-Net of the reference (examples/segmentation/segmentation_spark.py:67-119) on the
native engine: frozen MobileNetV2 encoder (128x128x3 input, five skip taps) + four pix2pix
``upsample`` blocks (Conv2DTranspose 3x3 stride 2 -> BatchNorm -> ReLU; 512/256/128/64 filters)
+ a final Conv2DTranspose to the class logits; Adam, per-pixel sparse cross-entropy.

Kernel mapping:
  encoder   1x1 expand / project convs -> wgmma GEMM with folded inference-BN bias and fused
            ReLU6; 3x3 depthwise -> depthwise3x3 kernel (bias + ReLU6 fused); stem 3x3/s2 ->
            implicit GEMM.  Frozen by default (``layer.trainable = False`` in the reference, :83).
  fine-tune ``UNetTrainer(encoder_trainable_from=k)`` also trains the stem and blocks (k = 0) or
            blocks block_k..block_16: batch norm stays folded (frozen statistics), the folded
            filters and biases are the parameters.  1x1 wgrad / dgrad and the stem wgrad are
            implicit GEMMs; every ReLU6 sits at a depthwise conv's input or output, so one fused
            depthwise3x3_bwd launch applies both derivatives and produces dx, dw, the depthwise
            bias gradient and the producer's bias gradient (deterministic, no float atomics).
  decoder   Conv2DTranspose forward = the stride-2 *data-gradient* implicit GEMM (four output
            parity classes), with batch-norm statistics fused into its epilogue; its backward
            = stride-2 fprop (input gradient) + stride-2 wgrad.  Channel concatenation is a
            strided 16-byte copy into the concat buffer.
There are no pretrained ImageNet weights: the encoder is random-initialised from a fixed seed,
which leaves shapes, FLOPs and memory traffic - everything the benchmarks measure - unchanged, and
fine-tuning is how a user improves those features.
"""
import functools
import math
import numbers

import numpy as np
import torch

from .. import ops
from ..ops import igemm
from . import evaluation, serving
from . import engine
from .engine import BatchNorm, ParamStore, RunningArena, constant, he_normal

# (expansion t, out channels c, repeats n, stride s) - MobileNetV2, width 1.0
MBV2 = [(1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2),
        (6, 320, 1, 1)]
#: blocks whose *expansion* output is a skip tap (Keras names block_{1,3,6,13}_expand_relu)
SKIP_BLOCKS = (1, 3, 6, 13)
#: inverted-residual blocks block_0 .. block_16
NUM_BLOCKS = sum(n for _, _, n, _ in MBV2)


def encoder_depthwise_shapes(image=128):
  """(block, H, C, stride) of the 17 depthwise layers: input H x H x C, as the encoder builds them."""
  out, H, cin = [], image // 2, 32
  for t, c, n, s in MBV2:
    for i in range(n):
      stride = s if i == 0 else 1
      out.append((len(out), H, cin * t, stride))
      H, cin = (H - 1) // stride + 1, c
  return out


def _buf(shape, dev, dtype=torch.bfloat16):
  return torch.zeros(shape, dtype=dtype, device=dev)


class _EncoderUnit(object):
  """Folded filter ``w`` and bias ``bias`` of one encoder convolution.  Frozen: standalone bf16 /
  fp32 tensors.  Trainable (fine-tuning): register() makes the folded values parameters of the
  trainer's ParamStore (the filter decayed, the bias not, so kernels read it in fp32 from aux32)
  and bind() points ``w`` / ``bias`` at their store views once the store is finalized."""

  def _init_values(self, w, bias, dev, trainable):
    self.trainable = trainable
    if trainable:
      self.init, self.w, self.bias = (w, bias), None, None   # fp32 values the masters start from
    else:
      self.w = w.to(dev, torch.bfloat16).contiguous()
      self.bias = bias.to(dev, torch.float32).contiguous()

  def register(self, store, name):
    w, b = self.init
    self.sw = store.register(name + ".w", w.shape, True, lambda shape, gen, v=w: v.clone())
    self.sb = store.register(name + ".b", b.shape, False, lambda shape, gen, v=b: v.clone())

  def bind(self, store):
    self.w, self.bias, self.init = store.w(self.sw), store.f32(self.sb), None


class _FrozenConv(_EncoderUnit):
  """1x1 or 3x3 convolution + folded inference batch-norm (+ReLU6)."""

  def __init__(self, gen, cin, cout, k, stride, act, dev, trainable=False):
    w = torch.randn(cout, k, k, cin, generator=gen) * math.sqrt(2.0 / (k * k * cin))
    gamma = 1.0 + 0.1 * torch.randn(cout, generator=gen)
    beta, mean = 0.1 * torch.randn(cout, generator=gen), 0.1 * torch.randn(cout, generator=gen)
    var = 1.0 + 0.1 * torch.rand(cout, generator=gen)
    scale = gamma / torch.sqrt(var + 1e-3)
    self._init_values(w * scale.view(-1, 1, 1, 1), beta - mean * scale, dev, trainable)
    self.k, self.stride, self.act = k, stride, act

  def zero_input_channels(self, c0):
    """Zero the filter taps of input channels >= c0 (the stem's padding channels)."""
    (self.init[0] if self.trainable else self.w)[..., c0:] = 0

  def connect(self, x, y):
    self.x, self.y = x, y

  def build(self):
    self.plan = igemm.conv_fprop(self.x, self.w, self.y, self.stride, self.k // 2, bias=self.bias,
                                 relu=self.act)

  def forward(self):
    self.plan.run()


class _FrozenDepthwise(_EncoderUnit):

  def __init__(self, gen, c, stride, dev, trainable=False):
    w = torch.randn(9, c, generator=gen) * math.sqrt(2.0 / 9)
    scale = 1.0 + 0.1 * torch.randn(c, generator=gen)
    self._init_values(w * scale.view(1, -1), 0.1 * torch.randn(c, generator=gen), dev, trainable)
    self.stride = stride

  def connect(self, x, y):
    self.x, self.y = x, y

  def build(self):
    pass

  def forward(self):
    ops.K.depthwise3x3_fwd(self.x, self.w, self.bias, self.y, self.stride, 2)


class _Block(object):
  """One inverted-residual block: Keras index, units (expand is None for block 0), its input and
  output buffers, and whether the input is added to the output."""

  def __init__(self, index, expand, dw, project, inp, out, residual):
    self.index, self.expand, self.dw, self.project = index, expand, dw, project
    self.inp, self.out, self.residual = inp, out, residual


class MobileNetV2Encoder(object):
  """Feature extractor returning the five skip tensors.

  ``trainable_from`` None: every unit frozen, forward only.  k in 0..16: the units of blocks
  k..16 (and the stem for k = 0) register in ``store``; call bind() once the store is finalized
  (it builds the forward plans on the store views), then build_backward()."""

  def __init__(self, batch, image, dev, seed=7, trainable_from=None, store=None):
    gen = torch.Generator(device="cpu")
    gen.manual_seed(seed)
    B = batch
    self.dev, self.trainable_from = dev, trainable_from
    trains = lambda b: trainable_from is not None and b >= trainable_from  # noqa: E731
    self.x = _buf((B, image, image, 8), dev)  # 3 real + 5 zero channels (16-byte pixels)
    self.layers, self.blocks = [], []
    H = image // 2
    cur = _buf((B, H, H, 32), dev)
    stem = self.stem = _FrozenConv(gen, 8, 32, 3, 2, 2, dev, trainable=trains(0))
    stem.zero_input_channels(3)
    stem.connect(self.x, cur)
    self.layers.append(stem)
    units = [("encoder.stem", stem)]
    self.skips = []
    cin, block = 32, 0
    for t, c, n, s in MBV2:
      for i in range(n):
        stride = s if i == 0 else 1
        inp = cur
        hidden = cin * t
        e = None
        name = "encoder.block{}.".format(block)
        if t != 1:
          e = _FrozenConv(gen, cin, hidden, 1, 1, 2, dev, trainable=trains(block))
          ebuf = _buf((B, H, H, hidden), dev)
          e.connect(cur, ebuf)
          self.layers.append(e)
          units.append((name + "expand", e))
          cur = ebuf
          if block in SKIP_BLOCKS:
            self.skips.append(cur)
        H2 = (H - 1) // stride + 1
        d = _FrozenDepthwise(gen, hidden, stride, dev, trainable=trains(block))
        dbuf = _buf((B, H2, H2, hidden), dev)
        d.connect(cur, dbuf)
        self.layers.append(d)
        p = _FrozenConv(gen, hidden, c, 1, 1, 0, dev, trainable=trains(block))
        pbuf = _buf((B, H2, H2, c), dev)
        p.connect(dbuf, pbuf)
        self.layers.append(p)
        units += [(name + "dw", d), (name + "project", p)]
        cur = pbuf
        residual = stride == 1 and cin == c
        if residual:
          self.layers.append(_Residual(pbuf, inp))
        self.blocks.append(_Block(block, e, d, p, inp, pbuf, residual))
        cin, H, block = c, H2, block + 1
    self.skips.append(cur)  # block_16_project, 4x4x320 at 128 input
    self.out_hw = H
    self.trainable_units = [u for _, u in units if u.trainable]
    for name, u in units:
      if u.trainable:
        u.register(store, name)
    self.backward_ops = []
    if trainable_from is None:
      self._build_forward()

  def _build_forward(self):
    for layer in self.layers:
      if not isinstance(layer, _Residual):
        layer.build()

  def bind(self, store):
    """Point the trainable units at the finalized store's views and build the forward plans."""
    for u in self.trainable_units:
      u.bind(store)
    self._build_forward()

  def build_backward(self, store, g_top, skip_grads, accumulate=False):
    """Plan the backward of the trainable blocks, top down.  ``g_top``: gradient of block_16's
    project output (written by the decoder); ``skip_grads``: {block index: (tensor, channel
    offset)} - the slice of an up-block's concatenation gradient that belongs to that block's
    expand output.  Per block: project wgrad + bias colsum + dgrad, the fused depthwise backward
    (both ReLU6 derivatives, the skip gradient, the producer's bias gradient), expand wgrad and,
    above the lowest trainable block, expand dgrad into the block input's gradient - accumulated
    when the block is residual, whose input and output share one gradient buffer.
    ``accumulate`` (gradient accumulation): the depthwise backward adds its filter and bias
    gradients instead of storing them (every other producer here adds anyway)."""
    st, dev, K = store, self.dev, ops.K
    lowest = self.trainable_from
    run = self.backward_ops
    g_out = g_top
    for blk in reversed(self.blocks):
      if blk.index < lowest:
        break
      e, d, p = blk.expand, blk.dw, blk.project
      g_d = _buf(d.y.shape, dev)
      run += [igemm.conv_wgrad(g_out, d.y, st.g(p.sw)).run,
              functools.partial(K.colsum, g_out, st.g(p.sb)),
              igemm.conv_dgrad(g_out, p.w, g_d).run]
      g_x = _buf(d.x.shape, dev)   # gradient of the producer's pre-activation (expand or stem)
      producer = e if e is not None else self.stem
      add, add_off = skip_grads.get(blk.index, (None, 0))
      N, H, _, C = d.x.shape
      scratch = torch.zeros(ops.C().depthwise3x3_bwd_scratch(N, H, C, d.stride),
                            dtype=torch.float32, device=dev)
      run.append(functools.partial(K.depthwise3x3_bwd, d.x, d.w, d.y, g_d, add, add_off, g_x,
                                   st.g(d.sw), st.g(d.sb), st.g(producer.sb), scratch, d.stride,
                                   accumulate=accumulate))
      if e is None:   # block 0: its input is the stem's output
        run.append(igemm.conv_wgrad(g_x, self.x, st.g(self.stem.sw), 2, 1).run)
        continue
      run.append(igemm.conv_wgrad(g_x, blk.inp, st.g(e.sw)).run)
      if blk.index > lowest:
        g_in = g_out if blk.residual else _buf(blk.inp.shape, dev)
        run.append(igemm.conv_dgrad(g_x, e.w, g_in, accumulate=blk.residual).run)
        g_out = g_in

  def forward(self):
    for layer in self.layers:
      layer.forward()
    return self.skips

  def backward(self):
    for op in self.backward_ops:
      op()


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


def _trainable_from(k, training):
  """Validated ``encoder_trainable_from``: None, or a block index in 0..16 (training only)."""
  if k is None:
    return None
  if isinstance(k, bool) or not isinstance(k, numbers.Integral):
    raise ValueError("encoder_trainable_from must be None or an int in 0..16, not {!r}".format(k))
  if not 0 <= k < NUM_BLOCKS:
    raise ValueError("encoder_trainable_from must be in 0..16, got {}".format(k))
  if not training:
    raise ValueError("encoder_trainable_from needs training=True (an inference-only U-Net has no "
                     "gradients)")
  return int(k)


def _optimizer_args(optimizer, weight_decay, beta1, beta2, epsilon, training, defaults):
  """Validated ``(optimizer, weight_decay, beta1, beta2, epsilon)``: optimizer one of adam | adamw
  | lamb, weight_decay finite >= 0, the Adam family's betas and epsilon; any value other than the
  default needs training=True (ValueError otherwise)."""
  from ..parallel.fused_optim import check_weight_decay
  if optimizer not in ("adam", "adamw", "lamb"):
    raise ValueError("optimizer must be one of adam | adamw | lamb, got {!r}".format(optimizer))
  weight_decay = check_weight_decay(weight_decay)
  beta1, beta2, epsilon = engine.check_adam_args(beta1, beta2, epsilon)
  args = (optimizer, weight_decay, beta1, beta2, epsilon)
  if not training:
    for name, v, d in zip(("optimizer", "weight_decay", "beta1", "beta2", "epsilon"), args, defaults):
      if v != d:
        raise ValueError("{} needs training=True (an inference-only U-Net has no optimizer)"
                         .format(name))
  return args


#: the training losses of UNetTrainer(loss=...)
LOSSES = ("cross_entropy", "focal", "dice", "dice_ce")


def _loss_args(loss, focal_gamma, dice_smooth, training, defaults):
  """Validated ``(loss, focal_gamma, dice_smooth)``: loss one of LOSSES, focal_gamma a finite
  real >= 0, dice_smooth a finite real > 0.  A value other than its default needs training=True,
  a non-default focal_gamma the focal loss and a non-default dice_smooth a loss with Dice
  (ValueError otherwise)."""
  if not isinstance(loss, str) or loss not in LOSSES:
    raise ValueError("loss must be one of {}, got {!r}".format(" | ".join(LOSSES), loss))

  def real(name, v, ok, what):
    if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(v) or not ok(v):
      raise ValueError("{} must be a finite real {}, got {!r}".format(name, what, v))
    return float(v)
  focal_gamma = real("focal_gamma", focal_gamma, lambda v: v >= 0, ">= 0")
  dice_smooth = real("dice_smooth", dice_smooth, lambda v: v > 0, "> 0")
  args = (loss, focal_gamma, dice_smooth)
  names = ("loss", "focal_gamma", "dice_smooth")
  if not training:
    for name, v, d in zip(names, args, defaults):
      if v != d:
        raise ValueError("{} needs training=True (an inference-only U-Net has no loss)".format(name))
  if focal_gamma != defaults[1] and loss != "focal":
    raise ValueError("focal_gamma needs loss='focal', not {!r}".format(loss))
  if dice_smooth != defaults[2] and loss not in ("dice", "dice_ce"):
    raise ValueError("dice_smooth needs loss='dice' or 'dice_ce', not {!r}".format(loss))
  return args


#: most classes a U-Net can have: its masks (served output, DataFeed wire format) are uint8
MAX_CLASSES = 256


def _classes(v):
  """Validated class count: an int in 1..MAX_CLASSES."""
  if isinstance(v, bool) or not isinstance(v, numbers.Integral):
    raise ValueError("classes must be an int in 1..{}, not {!r}".format(MAX_CLASSES, v))
  if not 1 <= v <= MAX_CLASSES:
    raise ValueError("classes must be in 1..{}, got {}".format(MAX_CLASSES, v))
  return int(v)


def _ignore_index(v):
  """Validated ``ignore_index``: None, or an int in the int32 range (labels are int32)."""
  if v is None:
    return None
  if isinstance(v, bool) or not isinstance(v, numbers.Integral):
    raise ValueError("ignore_index must be None or an int, not {!r}".format(v))
  if not -2 ** 31 <= v < 2 ** 31:
    raise ValueError("ignore_index must fit in int32, got {}".format(v))
  return int(v)


def _class_weights(v, classes):
  """Validated ``class_weights``: None, or a tuple of ``classes`` finite, non-negative, not all
  zero weights, rounded to fp32 as the kernels read them."""
  if v is None:
    return None
  if isinstance(v, (torch.Tensor, np.ndarray)):
    v = v.tolist()
  if isinstance(v, (str, bytes, bool, numbers.Number)) or not hasattr(v, "__len__"):
    raise ValueError("class_weights must be None or a sequence of {} numbers, not {!r}".format(
        classes, v))
  if len(v) != classes:
    raise ValueError("class_weights needs one weight per class ({}), got {}".format(classes, len(v)))
  if any(isinstance(w, bool) or not isinstance(w, numbers.Real) for w in v):
    raise ValueError("class_weights must be real numbers, got {!r}".format(v))
  w = tuple(float(np.float32(x)) for x in v)
  if not all(math.isfinite(x) and x >= 0 for x in w):
    raise ValueError("class_weights must be finite and non-negative, got {!r}".format(v))
  if not any(w):
    raise ValueError("class_weights are all zero")
  return w


def padded_classes(classes):
  """Channels of the logits for ``classes`` labels: 8 up to 8 classes (one 16-byte load per
  pixel), else the next multiple of 8 (the wide kernels, csrc/seg_wide.cuh)."""
  return 8 if classes <= 8 else -(-classes // 8) * 8


def synthetic_labels(x, classes=3):
  """Learnable synthetic labels of uint8 images [..., 3] (no dataset needed): at 3 classes the
  trimap (red > 127) + (green > 200); at any other count the red channel quantised into
  ``classes`` equal bands, red * classes // 256, which reaches every class of [0, classes).
  A torch tensor gives int32 labels, a numpy array uint8 ones (the DataFeed wire format)."""
  if isinstance(x, torch.Tensor):
    if classes == 3:
      return (x[..., 0] > 127).int() + (x[..., 1] > 200).int()
    return x[..., 0].int() * classes // 256
  if classes == 3:
    return (x[..., 0] > 127).astype(np.uint8) + (x[..., 1] > 200).astype(np.uint8)
  return (x[..., 0].astype(np.int32) * classes // 256).astype(np.uint8)


class UNetTrainer(object):
  """Static-buffer U-Net for ``batch`` images of ``image`` x ``image`` x 3 and ``classes`` labels
  (1..256).  The head's logits have padded_classes(classes) channels.
  ``training=False`` builds only what the forward pass needs (predict, evaluate, serving): no
  gradient buffers, no backward or statistics-fused plans and no optimizer (``optim`` is None).

  ``encoder_trainable_from``: None (default) trains the decoder only, on a frozen encoder.  An int
  k fine-tunes the encoder too: 0 trains the stem and all 17 inverted-residual blocks, k in 1..16
  the Keras blocks block_k .. block_16.  Their folded (batch norm in the filter) filters and biases
  become parameters ``encoder.stem.{w,b}`` / ``encoder.block{b}.{expand,dw,project}.{w,b}`` of the
  store, starting from exactly the frozen network of the same seed; the optimizer and gradient
  all-reduce cover them like every other parameter.

  ``ignore_index`` and ``class_weights`` are the loss options of
  ``F.cross_entropy(logits, y, weight=class_weights, ignore_index=ignore_index)``, for training and
  evaluation (also of a ``training=False`` trainer's ``evaluate``).  ``ignore_index``: None or an
  int32 value; a pixel whose label equals it takes no part in the loss, the gradient, the hit
  count ``correct`` or any evaluation total (void pixels, 255 in PASCAL VOC, Cityscapes and
  COCO-Stuff).  It may lie inside [0, classes), as in PyTorch: that class is then never scored.
  uint8 masks only carry 0..255, so a larger or negative value never matches one.
  ``class_weights``: None or ``classes`` finite, non-negative weights, not all zero (rounded to
  fp32).  With S the non-ignored pixels of a step and w[y] the weight of label y (1 without
  weights, and for a label outside [0, classes) that is not ignored):
  loss = sum_S w[y] l_p / sum_S w[y] and dlogits_p = w[y] (softmax_p - onehot_p) / sum_S w[y],
  exactly 0 for ignored pixels.  When sum_S w[y] = 0 (every pixel ignored, or only zero-weight
  classes present) the loss and the gradient are 0, where PyTorch gives NaN.  The denominator is
  computed on the device each step (``loss_norm``), so a captured step uses its own batch's.
  Under data parallelism each rank normalises by its own denominator and the gradient all-reduce
  averages, as DDP does with a mean-reduced CrossEntropyLoss.  With neither option the step
  launches exactly the kernels it did without them.  ``loss_norm`` (fp64 [3], training only) holds
  the last step's [sum_S w[y], |S|, 1 / sum_S w[y]]: loss_sum is the mean loss and
  correct / loss_norm[1] the pixel accuracy, without a host sync.

  ``ema_decay``: None, or d in [0, 1) (training only): the Adam update kernels also keep an
  exponential moving average of every parameter, trainable encoder units included (Keras's
  ``use_ema``); training is unchanged.  ``averaged()`` exports it, ``evaluate(..., averaged=True)``
  scores it.

  ``clip_norm``: None, or c > 0, inf allowed (training only): the averaged gradient is clipped to
  global norm c before the Adam update, as ``torch.nn.utils.clip_grad_norm_``; ``grad_norm`` holds
  the norm of each step (``clip_norm=float("inf")`` only measures it).

  ``optimizer`` (training only): adam (default; L2 ``weight_decay`` folded into the gradient),
  adamw (decoupled decay, ``torch.optim.AdamW``) or lamb (layer-wise adaptive Adam, apex
  ``FusedLAMB``); see parallel/fused_optim.py.  ``weight_decay``: a finite real >= 0, applied to
  the filters (conv weights, trainable encoder filters included), never to biases.  ``beta1``,
  ``beta2`` in [0, 1) and ``epsilon`` > 0 as Keras's Adam.  With ``training=False`` each of these
  must keep its default.

  ``gradient_accumulation_steps`` (k, an int >= 1; k != 1 needs training=True): the parameters are
  updated every k ``train_step`` calls with the mean of the gradients since the last update
  (Keras's ``gradient_accumulation_steps``).  Calls 1 .. k-1 of a window add into the gradient
  buffer and launch no optimizer kernel and no communication; call k also runs the all-reduce +
  update.  Each micro-batch's loss is its own mean; ``ignore_index`` / ``class_weights``
  normalise each micro-batch by its own denominator (``loss_norm``), as each rank does under data
  parallelism; the decoder batch norms' batch and running statistics are per micro-batch, as in
  Keras and PyTorch.  Clipping, weight decay, the weight average and Adam's step advance once
  per update.  ``micro_step`` is the position of the next call in its window (0 .. k-1).

  ``loss`` (training only): ``"cross_entropy"`` (default), ``"focal"``, ``"dice"`` or
  ``"dice_ce"``.  With S the non-ignored pixels of the micro-batch, w the class weights (1
  without them) and p the softmax over the ``classes`` real channels:
    * focal (Lin et al.; Keras ``CategoricalFocalCrossentropy`` with ``alpha`` per class given by
      ``class_weights``), exponent ``focal_gamma`` (a finite real >= 0, default 2):
      FL_p = -(1 - p_y)^gamma log p_y, normalised as the cross-entropy is,
      loss = sum_S w[y] FL_p / sum_S w[y].  gamma = 0 is the cross-entropy: the same gradient, bit
      for bit.  A label outside [0, classes) that is not ignored keeps its cross-entropy terms.
    * dice (MONAI ``DiceLoss(softmax=True, to_onehot_y=True, batch=True)``), smoothing
      ``dice_smooth`` (a finite real > 0, default 1e-5) in numerator and denominator: per class c,
      I_c = sum_S p_c [y = c], P_c = sum_S p_c, Y_c = |{y = c}| and
      D_c = (2 I_c + smooth) / (P_c + Y_c + smooth); loss = sum_c w_c (1 - D_c) / sum_c w_c, so the
      class weights average the classes rather than weigh pixels.  A label outside [0, classes)
      adds to P_c only; an empty S gives loss 0 and a zero gradient.
    * dice_ce: the (optioned) cross-entropy plus the Dice loss, weight 1 each (MONAI
      ``DiceCELoss``).
  The Dice statistics are those of each micro-batch on each rank (like the batch-norm
  statistics): under gradient accumulation each micro-batch has its own Dice loss, and under data
  parallelism each rank its own, averaged by the gradient all-reduce.  The Dice losses launch one
  more kernel per step (the statistics pass, seg_dice_stats); focal launches as many as the
  cross-entropy.  Evaluation keeps reporting the (optioned) cross-entropy; the per-class Dice
  coefficient of the evaluation's masks is 2 IoU / (1 + IoU) of its ``iou``.  A non-default
  ``focal_gamma`` needs ``loss="focal"``, a non-default ``dice_smooth`` a Dice loss."""

  UP = (512, 256, 128, 64)
  # optimizer, weight_decay, beta1, beta2, epsilon: the defaults (the U-Net's Adam before they
  # were options)
  OPT_DEFAULTS = ("adam", 0.0, 0.9, 0.999, 1e-7)
  # loss, focal_gamma, dice_smooth
  LOSS_DEFAULTS = ("cross_entropy", 2.0, 1e-5)

  def __init__(self, batch=64, image=128, classes=3, device="cuda:0", lr=1e-3, comm=None, seed=1234,
               training=True, encoder_trainable_from=None, ignore_index=None, class_weights=None,
               ema_decay=None, clip_norm=None, optimizer="adam", weight_decay=0.0, beta1=0.9,
               beta2=0.999, epsilon=1e-7, gradient_accumulation_steps=1, loss="cross_entropy",
               focal_gamma=2.0, dice_smooth=1e-5):
    classes = _classes(classes)
    self.loss, self.focal_gamma, self.dice_smooth = _loss_args(
        loss, focal_gamma, dice_smooth, training, self.LOSS_DEFAULTS)
    k_acc = engine.check_gradient_accumulation_steps(gradient_accumulation_steps, training)
    self.ema_decay = engine.check_ema_decay(ema_decay, training)
    self.clip_norm = engine.check_clip_norm(clip_norm, training)
    opt_args = _optimizer_args(optimizer, weight_decay, beta1, beta2, epsilon, training,
                               self.OPT_DEFAULTS)
    k = self.encoder_trainable_from = _trainable_from(encoder_trainable_from, training)
    self.ignore_index = _ignore_index(ignore_index)
    self.class_weights = _class_weights(class_weights, classes)
    self.VP = VP = padded_classes(classes)
    self.device = dev = torch.device(device)
    self.B, self.image, self.classes = batch, image, classes
    self.comm = comm
    self.training = tr = training
    B = batch
    st = self.store = ParamStore()
    self.encoder = MobileNetV2Encoder(batch, image, dev, trainable_from=k, store=st)
    skips = self.encoder.skips  # [64x64x96, 32x32x144, 16x16x192, 8x8x576, 4x4x320]
    self.ups = []
    cin = skips[-1].shape[-1]
    for i, f in enumerate(self.UP):
      self.ups.append(_Upsample(st, "up{}".format(i), cin, f))
      cin = f + skips[-2 - i].shape[-1]
    self.s_last = st.register("last.w", (cin, 3, 3, VP), True, he_normal(9 * cin))
    self.s_last_b = st.register("last.b", (VP,), False, constant(0.0))
    st.finalize(dev, alloc=comm.alloc if comm is not None else None, seed=seed, grads=tr)
    if k is not None:
      self.encoder.bind(st)

    x, h = skips[-1], skips[-1].shape[1]
    # a frozen encoder takes no gradient; a fine-tuned one gets block_16's output gradient here
    g_x = self.g_top = _buf(x.shape, dev) if k is not None else None
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
    self.logits = _buf((B, h, h, VP), dev)
    self.dlogits = _buf((B, h, h, VP), dev) if tr else None
    self.labels = torch.zeros(B, h, h, dtype=torch.int32, device=dev)
    self.p_last = igemm.conv_dgrad(x, st.w(self.s_last), self.logits, 2, 1, bias=st.f32(self.s_last_b))
    self.p_last_wgrad = self.p_last_dgrad = self.optim = None
    if tr:
      self.p_last_wgrad = igemm.conv_wgrad(x, self.dlogits, st.g(self.s_last), 2, 1)
      self.p_last_dgrad = igemm.conv_fprop(self.dlogits, st.w(self.s_last), g_x, 2, 1)
    if k is not None:
      # up-block i concatenates skips[-2 - i], the expand output of SKIP_BLOCKS[-1 - i]
      skip_grads = {SKIP_BLOCKS[-1 - i]: (g_cat, f) for i, (g_cat, _, f) in enumerate(self.g_cats)}
      self.encoder.build_backward(st, self.g_top, skip_grads, accumulate=k_acc > 1)
    self.loss_sum = torch.zeros(1, dtype=torch.float32, device=dev)
    self.correct = torch.zeros(1, dtype=torch.float32, device=dev)
    # the loss options' device state: weights [VP] (zero in the padding channels), the
    # pre-pass's scratch and its result; without options loss_norm is the constant denominator
    self.weights = None
    if self.class_weights is not None:
      self.weights = torch.zeros(VP, dtype=torch.float32, device=dev)
      self.weights[:classes] = torch.tensor(self.class_weights, dtype=torch.float32)
    self.loss_opts = self.ignore_index is not None or self.class_weights is not None
    self.loss_norm = self._norm_scratch = None
    if tr:
      npix = self.labels.numel()
      self.loss_norm = torch.tensor([npix, npix, float(np.float32(1.0 / npix))],
                                    dtype=torch.float64, device=dev)
      if self.loss_opts:
        self._norm_scratch = torch.zeros(ops.C().seg_label_norm_scratch(classes),
                                         dtype=torch.int64, device=dev)
    # the Dice losses: seg_dice_stats' gradient coefficients [A; B] and scratch
    self.dice_coef = self._dice_scratch = None
    if self.loss in ("dice", "dice_ce"):
      self.dice_coef = torch.zeros(2, VP, dtype=torch.float32, device=dev)
      self._dice_scratch = torch.zeros(ops.C().seg_dice_scratch(VP), dtype=torch.float32,
                                       device=dev)
    self.in_u8 = _buf((B, image, image, 3), dev, torch.uint8)
    if tr:
      from ..parallel.fused_optim import FusedOptimizer
      optimizer, weight_decay, beta1, beta2, epsilon = opt_args
      self.optim = FusedOptimizer(st, comm=comm, opt=optimizer, lr=lr, weight_decay=weight_decay,
                                  ema_decay=self.ema_decay, clip_norm=self.clip_norm, beta1=beta1,
                                  beta2=beta2, eps=epsilon)
    # accumulation: the decoder batch norms' per-micro-batch dgamma / dbeta, zeroed every step
    self.grad_scratch = None
    if k_acc > 1:
      self.optim.set_accumulation(k_acc)
      self.grad_scratch = engine.StatsArena(dev, capacity=2 * sum(self.UP))
      for up in self.ups:
        up.bn.accumulate_grads(self.grad_scratch)
    self.accum = engine.GradAccumulation(k_acc)
    self.graph = None
    self.graphs = None
    self._live = None   # (weights, aux32) saved while an averaged evaluation has the average in

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

  @property
  def gradient_accumulation_steps(self):
    return self.accum.k

  @property
  def micro_step(self):
    """Position (0 .. k-1) of the next ``train_step`` in its accumulation window."""
    return self.accum.micro_step

  def step_kernels(self):
    """Micro-step ``micro_step`` of the accumulation window (not advanced: ``train_step`` does)."""
    if not self.training:
      raise RuntimeError("this UNetTrainer was built with training=False: it cannot train")
    K = ops.K
    zero, update = self.accum.phase()
    self._forward(True)
    self.loss_sum.zero_()
    self.correct.zero_()
    self._loss()
    if zero:
      self.optim.zero_grads()
    if self.grad_scratch is not None:
      self.grad_scratch.zero()
    self.p_last_wgrad.run()
    K.colsum(self.dlogits, self.store.g(self.s_last_b))
    self.p_last_dgrad.run()
    for up, (g_cat, g_act, f) in zip(reversed(self.ups), reversed(self.g_cats)):
      K.copy_channels(g_cat, g_act, f, 0, 0)  # gradient of the decoder half of the concat
      up.backward()
    self.encoder.backward()   # fine-tuning only: nothing to run on a frozen encoder
    if update:
      self.optim.step()

  def _loss(self):
    """The loss kernels of a step on ``logits`` and ``labels``: loss_sum and correct add this
    micro-batch's loss and hits (they are not zeroed here), dlogits is overwritten."""
    K = ops.K
    npix = self.labels.numel()
    if self.loss_opts:   # the denominator sum_S w[y] of this batch's labels, on the device
      K.seg_label_norm(self.labels, self.loss_norm, self._norm_scratch, self.classes,
                       self.ignore_index, self.weights)
    # without options ignore_index and weights are None and the scale is the host's 1 / npix
    norm = self.loss_norm if self.loss_opts else None
    if self.loss == "cross_entropy":
      K.pixel_xent(self.logits, self.labels, self.dlogits, self.loss_sum, self.correct,
                   self.classes, 1.0 / npix, self.ignore_index, self.weights, norm)
      return
    if self.dice_coef is not None:   # this micro-batch's Dice statistics, before the gradient
      K.seg_dice_stats(self.logits, self.labels, self.dice_coef, self.loss_sum, self._dice_scratch,
                       self.classes, self.dice_smooth, self.ignore_index, self.weights)
    K.seg_loss_grad(self.logits, self.labels, self.dlogits, self.loss_sum, self.correct,
                    self.classes, 1.0 / npix, self.ignore_index, self.weights, norm,
                    focal_gamma=self.focal_gamma if self.loss == "focal" else None,
                    cross_entropy=self.loss != "dice", dice_coef=self.dice_coef)

  def capture(self):
    """CUDA graphs of the training step: one, or with accumulation one per kind of micro-step
    (see ResNetTrainer.capture); the warm-up trains eagerly."""
    # cross-host communicator: its collectives stay outside the graph (FusedOptimizer.finish()
    # defers them), but the process group's watchdog thread may still poll events of the warm-up
    # collectives - thread-local capture keeps that from invalidating the capture
    mode = "thread_local" if getattr(self.optim, "group_mode", False) else "global"
    self.graphs = self.accum.capture(self.device, self.step_kernels, mode)
    self.graph = self.graphs[(self.accum.k == 1, True)]

  def train_step(self, images_u8=None, labels=None):
    if self._swapped_in():
      raise RuntimeError("an averaged evaluation holds the weight average in the weights: call "
                         "eval_end() before training")
    if images_u8 is not None:
      self.set_input(images_u8, labels)
    # after the updating graph a cross-host communicator runs all-reduce + update outside it
    self.accum.run(self.graphs if self.graph is not None else None, self.step_kernels, self.optim)
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
    running statistics (``__running__``) + the encoder (``__encoder__``: one (bf16 filter, fp32
    bias) pair per convolution of ``encoder.layers``, in that order, as the forward uses them,
    with their current values when the encoder is fine-tuned): everything inference or a resumed
    run needs, independent of the loading host's RNG.  A fine-tuning trainer's parameters include
    the fp32 masters ``encoder.*`` of its trainable units."""
    sd = dict(self.store.state_dict())
    sd["__running__"] = self.running.tensor().detach().cpu().clone()
    sd["__encoder__"] = [(c.w.detach().cpu().clone(), c.bias.detach().cpu().clone())
                         for c in self._encoder_convs()]
    return sd

  def load_state_dict(self, sd):
    """Inverse of state_dict(); a dict without ``__running__`` keeps the current running
    statistics, one without ``__encoder__`` (checkpoints written before the encoder was part of
    the state) keeps the seeded encoder.  ``__encoder__`` is applied first, then any ``encoder.*``
    fp32 masters: a frozen run's checkpoint starts fine-tuning from its encoder, a fine-tuning
    checkpoint resumes with exact masters, and a frozen trainer ignores ``encoder.*``.  Restarts
    the accumulation window (partial sums dropped, ``micro_step = 0``); ``state_dict()`` may be
    taken mid-window and holds no partial sums."""
    sd = dict(sd)
    running = sd.pop("__running__", None)
    encoder = sd.pop("__encoder__", None)
    if encoder is not None:
      convs = self._encoder_convs()
      if len(encoder) != len(convs) or any(
          w.shape != c.w.shape or b.shape != c.bias.shape for c, (w, b) in zip(convs, encoder)):
        raise ValueError("__encoder__ does not match this U-Net's encoder ({} convolutions)".format(
            len(convs)))
      st = self.store
      for c, (w, b) in zip(convs, encoder):
        if c.trainable:   # into the masters: store.load_state_dict rounds them to the bf16 copy
          st.m(c.sw).copy_(w.to(self.device, torch.bfloat16).float())
          st.m(c.sb).copy_(b.to(self.device, torch.float32))
        else:
          c.w.copy_(w.to(self.device, torch.bfloat16))
          c.bias.copy_(b.to(self.device, torch.float32))
    self.store.load_state_dict(sd)
    if running is not None:
      self.running.tensor().copy_(running.to(self.device))
    if self.optim is not None:    # (the optimizer's load_state_dict restores a saved average)
      self.optim.reset_average()
      self.accum.restart(self.optim)

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

  @property
  def grad_norm(self):
    """Device fp32 [1]: the global norm N of the last step's averaged gradient, before clipping
    (updated by every replay of the captured step); None without ``clip_norm``."""
    return self.optim.grad_norm if self.optim is not None else None

  def averaged(self):
    """Snapshot of the weight average as an exportable model (engine.AveragedModel): its
    ``state_dict()`` is this trainer's with every parameter replaced by its average, the live
    running statistics, and ``__encoder__`` with the averaged trainable units (the filter rounded
    to bf16 to nearest even, as the update kernel rounds masters).  ``checkpoint.export_model(
    net.averaged(), dir)`` exports the average for ServedUNet.  RuntimeError without
    ``ema_decay``."""
    sd, avg = engine.averaged_params(self.store, self.optim)
    st = self.store
    sd["__running__"] = self.running.tensor().detach().cpu().clone()
    sd["__encoder__"] = [
        (st._view(avg, c.sw).to(torch.bfloat16).cpu(), st._view(avg, c.sb).detach().cpu().clone())
        if c.trainable else (c.w.detach().cpu().clone(), c.bias.detach().cpu().clone())
        for c in self._encoder_convs()]
    return engine.AveragedModel(sd, self)

  def _swapped_in(self):
    return self._live is not None and self._live[2]

  def _swap_average(self, on):
    """Put the weight average into ``weights`` / ``aux32`` (the evaluation forward and the
    trainable encoder units read them), saving the live values; ``on=False`` puts those back,
    bit for bit.  The masters and optimizer state are never touched."""
    st = self.store
    if on:
      w, aux = self.optim.averaged_weights()    # RuntimeError without an average
      if not self._swapped_in():
        if self._live is None:
          self._live = [torch.empty_like(st.weights), torch.empty_like(st.aux32), False]
        self._live[0].copy_(st.weights)
        self._live[1].copy_(st.aux32)
        self._live[2] = True
      st.weights.copy_(w)
      st.aux32.copy_(aux)
    elif self._swapped_in():
      st.weights.copy_(self._live[0])
      st.aux32.copy_(self._live[1])
      self._live[2] = False

  # ------------------------------------------------------- held-out evaluation
  def eval_begin(self, averaged=False):
    """Start an evaluation pass: zero the totals and take rank 0's running statistics.
    Stream-ordered after the last ``train_step``; the first call allocates the evaluation
    buffers.  ``averaged=True`` scores the weight average (``ema_decay``; RuntimeError without
    it) with the live running statistics: the average is swapped into ``weights`` / ``aux32``
    until ``eval_end()``, which restores the live values; ``train_step`` raises RuntimeError in
    between."""
    if averaged and (self.optim is None or self.optim.ema is None):
      raise RuntimeError("this trainer keeps no weight average: build it with ema_decay=d")
    self._swap_average(averaged)
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
    ValueError on every rank when any rank saw a mask value outside [0, classes) that is not
    ``ignore_index``.  With ``ignore_index`` the result also has ``"ignored"``: the pixels left
    out.  With ``class_weights`` the loss is the weighted mean.  Ends an averaged evaluation:
    the live weights are back afterwards, also when the totals raise."""
    try:
      return self._eval_state().end()
    finally:
      self._swap_average(False)

  def evaluate(self, batches, averaged=False):
    """eval_begin(averaged) + eval_step over ``(images, masks)`` pairs + eval_end.  Host batches
    go through page-locked staging: the copy of batch i + 1 overlaps the forward pass of batch i.
    The live weights are restored even when a batch raises."""
    self.eval_begin(averaged)
    try:
      self._evaluator.run(batches)
    except BaseException:
      self._swap_average(False)
      raise
    return self.eval_end()

  def _eval_state(self):
    if getattr(self, "_evaluator", None) is None:
      raise RuntimeError("eval_begin() has not been called")
    return self._evaluator


# accumulator slots of seg_eval_metrics (csrc/ops.h kSegEval*); slot SEG_IMAGES counts images
SEG_COUNT, SEG_CORRECT, SEG_INVALID, SEG_LOSS, SEG_CONFUSION, SEG_SLOTS = 0, 1, 2, 3, 4, 68
SEG_IMAGES, SEG_ACC = 68, 72


def seg_eval_layout(classes):
  """(images slot, first confusion slot, confusion row stride, accumulator length) of the
  evaluation accumulator for ``classes`` labels.  Up to 8 classes: the SEG_* layout, an 8 x 8
  confusion matrix.  More: [count, correct, invalid, loss, images, confusion classes x classes]
  (csrc/ops.h kSegWide*; the binding's seg_eval_slots(classes) is its length)."""
  if classes <= 8:
    return SEG_IMAGES, SEG_CONFUSION, 8, SEG_ACC
  return 4, 5, classes, 5 + classes * classes


def seg_eval_result(totals, classes, class_weights=None):
  """Host metrics from the summed accumulator ``totals`` (seg_eval_layout(classes) floats):
  {"count": scored pixels, "images", "loss", "accuracy", "mean_iou", "iou": [classes values]}.
  IoU of class c = cm[c, c] / (row_c + col_c - cm[c, c]) of the confusion matrix cm[label, pred];
  a class with an empty union has IoU NaN and is left out of mean_iou (NaN when every class is).
  loss and accuracy are means over the scored pixels (NaN when there are none).  With
  ``class_weights`` (``classes`` values) the loss slot holds sum w[y] l_p and the loss is its
  weighted mean, divided by sum_c w_c row_c (NaN when that is 0); IoU and accuracy stay
  unweighted.  Raises ValueError when any mask value was outside [0, classes)."""
  images, conf, ld, _ = seg_eval_layout(classes)
  if classes <= 8:
    h = [float(v) for v in totals]
    cm = [h[conf + ld * y:conf + ld * y + ld] for y in range(ld)]
    iou = []
    for c in range(classes):
      inter = cm[c][c]
      union = sum(cm[c][:classes]) + sum(cm[y][c] for y in range(classes)) - inter
      iou.append(inter / union if union > 0 else float("nan"))
  else:   # V x V cells: numpy (the same sums, in float64, of integer-valued counts)
    t = np.asarray(totals, dtype=np.float64)
    h = [float(v) for v in t[:conf]]
    cm = t[conf:conf + classes * classes].reshape(classes, classes)
    inter = np.diagonal(cm)
    union = cm.sum(axis=1) + cm.sum(axis=0) - inter
    with np.errstate(invalid="ignore", divide="ignore"):
      iou = [float(v) for v in np.where(union > 0, inter / np.where(union > 0, union, 1), np.nan)]
  if h[SEG_INVALID] > 0:
    raise ValueError("evaluation saw {} mask value(s) outside [0, {})".format(
        int(h[SEG_INVALID]), classes))
  count = int(h[SEG_COUNT])
  seen = [v for v in iou if v == v]
  mean = (lambda v: v / count) if count else (lambda v: float("nan"))
  loss = mean(h[SEG_LOSS])
  if class_weights is not None:
    rows = np.asarray(totals, dtype=np.float64)[conf:conf + ld * classes].reshape(classes, ld)
    wsum = float(np.dot(np.asarray(class_weights, dtype=np.float64), rows[:, :classes].sum(axis=1)))
    loss = h[SEG_LOSS] / wsum if wsum > 0 else float("nan")
  return {"count": count, "images": int(h[images]), "loss": loss,
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
    self.images_slot, _, _, slots = seg_eval_layout(self.V)
    self.acc = torch.zeros(slots, dtype=torch.float64, device=dev)
    self.partial = torch.zeros(ops.C().seg_eval_scratch(self.labels.numel(), self.V),
                               dtype=torch.float64, device=dev)
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
    self.rank_sum = evaluation.RankSum(comm, "seg_eval_totals", slots)
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
    net = self.net
    net._forward(False, self.u8, self.bn)
    ops.K.seg_eval_metrics(net.logits, self.labels, self.n_valid, self.acc, self.partial,
                           self.counter, self.V, net.ignore_index, net.weights)

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
    self.acc[self.images_slot].fill_(self.images)
    net = self.net
    res = seg_eval_result(self.rank_sum(self.acc), self.V, net.class_weights)
    if net.ignore_index is not None:   # every pixel of the images is scored, invalid or ignored
      res["ignored"] = res["images"] * net.image * net.image - res["count"]
    return res


class ServedUNet(serving.Replica):
  """Inference callable behind ``pipeline.TFModel`` / the inference CLI: one bf16 U-Net replica
  (a ``training=False`` trainer) on the executor's GPU.  Input ``image``: uint8 [n, H, W, 3] (or
  one row cell of H*W*3 bytes per image).  Outputs ``mask``: uint8 [n, H, W], the class every
  pixel is predicted as - exactly the prediction evaluation scores (seg_predict); ``logits``:
  fp32 [n, H, W, classes].  The forward pass + seg_predict run as one CUDA graph after the first
  batch; ``select_outputs`` keeps the logits (12x the bytes of the mask at 3 classes) on the
  device unless they are asked for (models/serving.Replica).  Above 8 classes the logits'
  device buffer (2.5 GB at batch 256 and 150 classes) is only allocated once ``logits`` is
  selected."""

  def __init__(self, state, image=128, classes=3, batch=256, device="cuda:0"):
    torch.cuda.set_device(torch.device(device))
    self.net = UNetTrainer(batch=batch, image=image, classes=classes, device=device,
                           training=False)
    self.net.load_state_dict(state)
    self.image, self.V = image, classes
    dev = self.net.device
    self.mask = torch.zeros(batch, image, image, dtype=torch.uint8, device=dev)
    self._logits_shape = (batch, image, image, classes)
    self.logits = None if classes > 8 else torch.zeros(self._logits_shape, dtype=torch.float32,
                                                       device=dev)
    super(ServedUNet, self).__init__(dev, batch, (image, image, 3),
                                     {"mask": self.mask, "logits": self.logits},
                                     self.net.set_input)

  def select_outputs(self, names):
    """Compute and read back only the outputs ``names`` (``mask`` and / or ``logits``) from the
    next batch on; ValueError for a name the model does not offer."""
    self._select_outputs(names)

  def _run(self):
    want = "logits" in self.selected
    if want and self.logits is None:   # first eager batch with logits selected (never in capture)
      self.logits = torch.zeros(self._logits_shape, dtype=torch.float32, device=self.net.device)
      self._outputs["logits"] = self.logits
    self.net._forward(False)
    ops.K.seg_predict(self.net.logits, self.mask, self.logits if want else None, self.V)


def build_served(state, image=128, classes=3, batch=None, **_):
  """Export builder (utils/checkpoint.py): rebuilds the replica on the executor's GPU with
  ``TFOS_SERVE_BATCH`` rows per batch unless ``batch`` is given."""
  return ServedUNet(state, image=image, classes=classes, batch=serving.serve_batch(batch))

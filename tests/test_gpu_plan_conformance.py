"""Every implicit-GEMM plan and batch-norm / elementwise launch the models build, replayed on fresh
seeded tensors and checked element by element against float64 (tools/plan_conformance.py holds the
bounds and their derivation).

A module fixture builds each model once while the ``ops.igemm`` builders, ``Plan.set_reverse``,
the ``ops.K`` batch-norm / elementwise entry points and ``bn_set_row_reverse`` are wrapped, and
runs one eager training step (or one inference forward).  Each call becomes a signature - op,
argument shapes and dtypes, scalar flags, the row / tile order and, for GEMM plans, the kernel
instance ``Plan.info()`` reports.  The trainers are freed before anything is replayed.

Checks per replayed signature:
  * forward-like plans: two rows of every M box (rotating over the 128 row positions), all output
    columns, against the float64 im2col dot products and the documented epilogue; no systematic
    rounding bias; fused statistics and BN-backward sums against float64 sums of what was stored;
    the output with the opposite tile order bit for bit equal;
  * weight gradients: every (tap, 64-channel slice pair) sampled, from a non-zero dW;
  * batch norm: y / dx / dres per element, mask bits exact away from 0, dgamma / dbeta within the
    summation bound, results bit for bit equal under the opposite row order;
  * every output lives between guard bands that must stay intact, and non-accumulating outputs
    start as NaN so that an element no kernel wrote fails.
"""
import gc
import importlib.util
import inspect
import os
import zlib

import pytest

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location(
    "plan_conformance", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                     "tools", "plan_conformance.py"))
pc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(pc)
_spec = importlib.util.spec_from_file_location(
    "kernel_conformance", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                       "tools", "kernel_conformance.py"))
kc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(kc)

GEMM_BUILDERS = ("gemm", "gemm_wgrad", "conv_fprop", "conv_dgrad", "conv_wgrad", "stem_fprop",
                 "stem_wgrad")
DEV = "cuda"
K_OPS = ("bn_apply", "bn_apply_finalize", "bn_bwd_reduce", "bn_bwd_apply", "depthwise3x3_fwd",
         "add_act", "colsum", "bn_inference_coeffs")

# ----------------------------------------------------------------------------- recording


def _spec_of(v):
  """The signature of one argument: a tensor's shape and dtype (and the values of an int64 index
  table: they decide what a launch does), scalars as they are."""
  import torch
  if isinstance(v, torch.Tensor):
    if v.dtype == torch.int64 and v.numel() <= 4096:
      return ("T", tuple(v.shape), "int64", tuple(v.reshape(-1).tolist()))
    return ("T", tuple(v.shape), str(v.dtype).replace("torch.", ""))
  if isinstance(v, (tuple, list)):
    return tuple(_spec_of(x) for x in v)
  if isinstance(v, dict):
    return tuple(sorted((k, _spec_of(x)) for k, x in v.items()))
  if isinstance(v, float):
    return round(v, 6)
  return v


class _Recorder(object):

  def __init__(self):
    self.gemm = []    # [op, frozen args, infos (list of dicts, mutable for set_reverse)]
    # every ops.K launch: (op, positional spec, sorted keyword spec, row reverse, aliases); the
    # aliases index the positional arguments followed by the keyword arguments in sorted order
    self.k = []
    self.row_reverse = False
    self._depth = 0


def _free():
  """After the last reference to a trainer is gone."""
  import torch
  torch.cuda.synchronize()
  gc.collect()
  torch.cuda.empty_cache()


def _resnet50_train():
  from tensorflowonspark_b200.models import resnet
  net = resnet.ResNetTrainer(50, batch=256, image=224)
  net.train_step(*net.synthetic_batch())


def _resnet50_serving():
  # batch norms folded into the filters, residual accumulate + ReLU epilogues
  from tensorflowonspark_b200.models import resnet
  net = resnet.ResNetTrainer(50, batch=256, image=224, training=False)
  net.forward_only()
  net.build_folded_inference()
  net.forward_folded()


def _resnet50_small():
  from tensorflowonspark_b200.models import resnet
  net = resnet.ResNetTrainer(50, batch=8, image=64)
  net.train_step(*net.synthetic_batch())


def _cifar():
  from tensorflowonspark_b200.models import resnet
  resnet.CifarResNetTrainer(20, batch=128).step_kernels()


def _unet_train():
  from tensorflowonspark_b200.models import unet
  net = unet.UNetTrainer(batch=64, image=128, training=True)
  net.train_step(*net.synthetic_batch())


def _unet_predict():
  from tensorflowonspark_b200.models import unet
  net = unet.UNetTrainer(batch=64, image=128, training=False)
  net.predict(net.synthetic_batch()[0])


def _mnist():
  from tensorflowonspark_b200.models import mnist
  mnist.MnistTrainer(batch=64).train_step()


DEFAULT_MODELS = (_resnet50_train, _resnet50_serving, _resnet50_small, _cifar, _unet_train,
                  _unet_predict, _mnist)


def _alias_pairs(vals):
  import torch
  return tuple((j, i) for i in range(1, len(vals)) for j in range(i)
               if isinstance(vals[i], torch.Tensor) and isinstance(vals[j], torch.Tensor)
               and vals[i].data_ptr() == vals[j].data_ptr() and vals[i].dtype == vals[j].dtype)


def _record_models(rec, models=DEFAULT_MODELS):
  """Run each callable of ``models`` (it builds a trainer, runs it and drops it) while the igemm
  builders, ``Plan.set_reverse``, ``bn_set_row_reverse`` and every ``ops.K`` entry point are
  wrapped, freeing the GPU memory after each."""
  import torch
  from tensorflowonspark_b200 import _build, ops
  from tensorflowonspark_b200.ops import igemm
  mod = _build.load(required=True)
  with pytest.MonkeyPatch.context() as mp:
    for name in GEMM_BUILDERS:
      fn = getattr(igemm, name)
      sig = inspect.signature(fn)

      def wrap(*a, _fn=fn, _sig=sig, _name=name, **k):
        rec._depth += 1
        try:
          plan = _fn(*a, **k)
        finally:
          rec._depth -= 1
        if rec._depth == 0:
          b = _sig.bind(*a, **k)
          b.apply_defaults()
          args = pc.freeze({n: _spec_of(v) for n, v in b.arguments.items()})
          entry = [_name, args, plan.info()]
          rec.gemm.append(entry)
          plan._conformance = entry
        return plan
      mp.setattr(igemm, name, wrap)
    orig_rev = igemm.Plan.set_reverse

    def set_reverse(self, flag):
      orig_rev(self, flag)
      entry = getattr(self, "_conformance", None)
      if entry is not None:
        for i in entry[2]:
          if i["kind"] == 0:
            i["reverse"] = int(bool(flag))
    mp.setattr(igemm.Plan, "set_reverse", set_reverse)
    orig_rowrev = mod.bn_set_row_reverse

    def row_rev(flag):
      rec.row_reverse = bool(flag)
      orig_rowrev(flag)
    mp.setattr(mod, "bn_set_row_reverse", row_rev)
    for name in dir(mod):
      fn = getattr(mod, name)
      if name.startswith("_") or isinstance(fn, type) or not callable(fn):
        continue

      def wrapk(*a, _fn=fn, _name=name, **k):
        kw = sorted(k.items())
        rec.k.append((_name, _spec_of(tuple(a)), _spec_of(tuple(kw)), rec.row_reverse,
                      _alias_pairs(list(a) + [v for _, v in kw])))
        return _fn(*a, **k)
      mp.setattr(ops.K, name, wrapk, raising=False)
    for model in models:
      model()
      _free()
  _free()


@pytest.fixture(scope="module")
def recorded():
  import torch
  torch.cuda.set_device(0)
  torch.cuda.reset_peak_memory_stats()
  rec = _Recorder()
  _record_models(rec)
  return {"gemm": distinct_plans(rec), "k": pc.dedup(c for c in rec.k if c[0] in K_OPS)}


def distinct_plans(rec):
  """The recorded igemm plans without repeats: (op, args, infos)."""
  gemm = {}
  for op, args, infos in rec.gemm:
    gemm.setdefault((op, args, pc.freeze(infos)), (op, args, infos))
  return list(gemm.values())


# ----------------------------------------------------------------------------- synthetic cases
# (name, builder, kwargs of tensor shapes / flags).  Shapes: ("x", shape) bf16 input, ("w", shape)
# bf16 filter, ("o", shape, dtype) output, ("b", n) fp32 bias, ("s", n) statistics pair,
# ("m", n bytes) bit mask, ("r", shape) bn_reduce tuple.
def _fp(cin, cout, hw, n=2, k=3, s=1, **kw):
  oh = (hw + 2 * (k // 2) - k) // s + 1
  d = {"x": ("x", (n, hw, hw, cin)), "w": ("w", (cout, k, k, cin)),
       "y": ("o", (n, oh, oh, cout)), "stride": s, "pad": k // 2}
  d.update(kw)
  return ("conv_fprop", d)


def _dg(cin, cout, hw, n=2, k=3, s=1, **kw):
  oh = (hw + 2 * (k // 2) - k) // s + 1
  d = {"dy": ("x", (n, oh, oh, cout)), "w": ("w", (cout, k, k, cin)),
       "dx": ("o", (n, hw, hw, cin)), "stride": s, "pad": k // 2}
  d.update(kw)
  return ("conv_dgrad", d)


def _gm(m, k, n, ldo=None, layout="nk", fp32=False, **kw):
  d = {"a": ("x", (m, k)), "b": ("w", (n, k) if layout == "nk" else (k, n)),
       "out": ("o", (m, ldo or n), "float32" if fp32 else "bfloat16"), "b_layout": layout}
  d.update(kw)
  return ("gemm", d)


SYNTHETIC = {
    # the ReLU6 epilogue on the paths that apply it after the residual / into fp32
    "relu6_accumulate_staged": _fp(64, 128, 14, bias=("b", 128), relu=2, accumulate=True),
    "relu6_accumulate_direct": _fp(64, 24, 14, bias=("b", 24), relu=2, accumulate=True),
    "relu6_fp32_out": _gm(300, 64, 64, fp32=True, bias=("b", 64), relu=2),
    "relu6_fp32_accumulate": _gm(300, 64, 128, fp32=True, bias=("b", 128), relu=2,
                                 accumulate=True),
    "relu6_bf16_staged": _fp(96, 128, 16, bias=("b", 128), relu=2),
    # ragged columns: 24 channels and the 1000-class head
    "ragged_n24": _fp(32, 24, 9, bias=("b", 24), relu=1),
    "head_1000": _gm(256, 2048, 1000, bias=("b", 1000)),
    # an output pitch that is not a multiple of 8, and columns between n_valid and ldo
    "ldo10": _gm(200, 64, 10, bias=("b", 10)),
    "ldo32_n24": _gm(200, 64, 24, ldo=32, bias=("b", 24)),
    # several images per M box (box_n > 1), one tile in all
    "box_n_gt1": _fp(64, 64, 4, n=6, k=3),
    "single_tile": _gm(100, 64, 64),
    # more than 8 column tiles at many tiles: not weight-stationary
    "n_tiles_gt8": _gm(33000, 64, 2304),
    # weight-stationary and prefetch instances walked in reverse
    "resident_reverse": _fp(64, 256, 56, n=16, k=1, reverse=True),
    "prefetch_reverse": _dg(256, 64, 56, n=4, k=1, accumulate=True, acc_mask=("m",),
                            bn_reduce=("r",), reverse=True),
    # kn GEMM (dense-layer data gradient) with statistics
    "gemm_kn_stats": _gm(512, 128, 256, layout="kn", stats=("s", 256)),
}


def _dispatch_sweep():
  """One small case per (BN, b_mn, EPI) of launch_fwd, so that each instance is run even if no
  model plan reaches it."""
  out = {}
  for bn in (64, 128, 256):
    out["sweep_fprop_bn{}_plain".format(bn)] = _fp(64, bn, 12)
    out["sweep_fprop_bn{}_stats".format(bn)] = _fp(64, bn, 12, stats=("s", bn))
    out["sweep_fprop_bn{}_generic".format(bn)] = _fp(64, bn, 12, bias=("b", bn), relu=1)
    out["sweep_dgrad_bn{}_plain".format(bn)] = _dg(bn, 64, 12, epi_prefetch=False)
    out["sweep_dgrad_bn{}_acc".format(bn)] = _dg(bn, 64, 12, accumulate=True, acc_mask=("m",),
                                                 epi_prefetch=False)
    out["sweep_dgrad_bn{}_red".format(bn)] = _dg(bn, 64, 12, bn_reduce=("r",), epi_prefetch=False)
    out["sweep_dgrad_bn{}_accred".format(bn)] = _dg(bn, 64, 12, accumulate=True, acc_mask=("m",),
                                                    bn_reduce=("r",), epi_prefetch=False)
    out["sweep_dgrad_bn{}_generic".format(bn)] = _dg(bn, 64, 12, s=2, bias=("b", bn),
                                                     stats=("s", bn))
    if bn >= 128:
      out["sweep_dgrad_bn{}_acc_pf".format(bn)] = _dg(bn, 64, 12, accumulate=True)
      out["sweep_dgrad_bn{}_red_pf".format(bn)] = _dg(bn, 64, 12, bn_reduce=("r",))
      out["sweep_dgrad_bn{}_accred_pf".format(bn)] = _dg(bn, 64, 12, accumulate=True,
                                                         bn_reduce=("r",))
  return out


SYNTHETIC.update(_dispatch_sweep())

# ----------------------------------------------------------------------------- tensors


class _Gen(object):
  """Seeded inputs.  Filters are scaled so that outputs have a standard deviation near 3: ReLU6
  clamps a fair share of them."""

  def __init__(self, seed):
    import torch
    self.g = torch.Generator(device=DEV)
    self.g.manual_seed(seed)

  def randn(self, shape, dtype, scale=1.0, shift=0.0):
    import torch
    return (torch.randn(shape, generator=self.g, device=DEV) * scale + shift).to(dtype)

  def bits(self, n):
    import torch
    return torch.randint(0, 256, (n,), generator=self.g, device=DEV, dtype=torch.uint8)


def _make_gemm_inputs(op, args, gen):
  """Fresh tensors for a recorded / synthetic builder call.  Returns (kwargs, outputs) where
  outputs maps a name to (view, backing, initial copy or None)."""
  import torch
  a = dict(args)
  kw, outs = {}, {}
  fan = 1

  def shape_of(v):
    return v[1]
  # filter fan-in for the scaling
  for name in ("w", "b"):
    if name in a and isinstance(a[name], tuple) and a[name] and a[name][0] in ("T", "w"):
      s = shape_of(a[name])
      if op in ("conv_dgrad",):
        fan = s[0] * (s[1] * s[2] if len(s) == 4 else 1)
      elif op == "gemm" and a.get("b_layout") == "kn":
        fan = s[0]
      elif op == "stem_fprop":
        fan = s[1] * s[2]
      else:
        fan = int(torch.tensor(s[1:]).prod())
  acc = bool(a.get("accumulate"))
  # Plans without an activation get operands of mean 1 (sd 0.5): their outputs, weight gradients
  # and column sums are then about as large as the sums of magnitudes that bound their errors, so
  # a missing tap, M box or pixel split exceeds the bound even at millions of pixels, and the
  # rounding-bias statistic has elements to work on.  Plans with ReLU / ReLU6 keep zero-mean
  # operands with outputs of standard deviation ~3, so that both clamps are exercised.
  linear = _is_wgrad(op) or not a.get("relu")
  wscale = 3.0 / max(1, fan) ** 0.5

  def operand(shape, is_w):
    if linear:
      return gen.randn(shape, torch.bfloat16, 0.5 * (3.0 / fan if is_w else 1.0),
                       3.0 / fan if is_w else 1.0)
    return gen.randn(shape, torch.bfloat16, wscale if is_w else 1.0)
  out_name = {"gemm": "out", "conv_fprop": "y", "conv_dgrad": "dx", "stem_fprop": "y",
              "gemm_wgrad": "dw", "conv_wgrad": "dw", "stem_wgrad": "dw"}[op]
  out_shape = None
  for name, v in a.items():
    if not isinstance(v, tuple) or not v:
      kw[name] = v
      continue
    tag = v[0]
    if name == out_name:
      shape = v[1]
      out_shape = shape
      dtype = torch.float32 if (tag == "T" and v[2] == "float32") or \
          (tag == "o" and len(v) > 2 and v[2] == "float32") else torch.bfloat16
      if op in ("gemm_wgrad", "conv_wgrad", "stem_wgrad"):
        view, back = pc.guarded(shape, torch.float32, DEV)
        view.copy_(gen.randn(shape, torch.float32))
      elif acc:
        view, back = pc.guarded(shape, dtype, DEV)
        view.copy_(gen.randn(shape, dtype, 0.5, 1.0) if linear else gen.randn(shape, dtype, 2.0))
      else:
        view, back = pc.guarded(shape, dtype, DEV,
                                pc.UNWRITTEN_FP32 if dtype == torch.float32 else pc.UNWRITTEN_BF16)
      outs["out"] = (view, back, view.clone())
      kw[name] = view
    elif tag == "T" and v[2] == "bfloat16" or tag in ("x", "w"):
      is_w = name in ("w", "b") or tag == "w"
      kw[name] = operand(v[1], is_w)
    elif name == "bias" or tag == "b":
      n = v[1][0] if tag == "T" else v[1]
      kw[name] = gen.randn((n,), torch.float32)
    elif name == "stats" or tag == "s":
      n = v[0][1][0] if tag != "s" else v[1]
      s0, b0 = pc.guarded((n,), torch.float32, DEV)
      s1, b1 = pc.guarded((n,), torch.float32, DEV)
      s0.zero_()
      s1.zero_()
      outs["stats"] = ((s0, b0), (s1, b1))
      kw[name] = (s0, s1)
    elif name == "acc_mask" or tag == "m":
      kw[name] = None  # filled once the output shape is known
      outs["_acc_mask"] = v
    elif name == "bn_reduce" or tag == "r":
      kw[name] = None
      outs["_bn_reduce"] = v
    else:
      raise AssertionError("unhandled argument {} {}".format(name, v))
  if "_acc_mask" in outs:
    del outs["_acc_mask"]
    n = int(torch.tensor(out_shape).prod()) // 8
    kw["acc_mask"] = gen.bits(n)
  if "_bn_reduce" in outs:
    spec = outs.pop("_bn_reduce")
    C = out_shape[-1]
    rx = gen.randn(out_shape, torch.bfloat16, 0.5, 1.0)
    has_mask = spec[0] == "r" or spec[1] is not None
    rm = gen.bits(int(torch.tensor(out_shape).prod()) // 8) if has_mask else None
    s0, b0 = pc.guarded((C,), torch.float32, DEV)
    s1, b1 = pc.guarded((C,), torch.float32, DEV)
    s0.zero_()
    s1.zero_()
    outs["red"] = ((s0, b0), (s1, b1))
    kw["bn_reduce"] = (rx, rm, s0, s1)
  return kw, outs


# ----------------------------------------------------------------------------- references
def _pixels_nhw(flat, OH, OW):
  n = flat // (OH * OW)
  r = flat % (OH * OW)
  return n, r // OW, r % OW


def _gather_nhwc(t, n, h, w):
  """t[n, h, w, :] with zeros where (h, w) is outside the tensor; float64."""
  import torch
  H, W = t.shape[1], t.shape[2]
  ok = (h >= 0) & (h < H) & (w >= 0) & (w < W)
  v = t[n, h.clamp(0, H - 1), w.clamp(0, W - 1), :].to(torch.float64)
  return v * ok.unsqueeze(1)


def _im2col(op, kw, flat):
  """(A rows [P, K] float64, B [K, N] float64) of the sampled flat output pixels."""
  import torch
  if op == "gemm":
    a, b = kw["a"], kw["b"]
    A = a[flat].to(torch.float64)
    B = b.to(torch.float64).t() if kw.get("b_layout", "nk") == "nk" else b.to(torch.float64)
    return A, B
  if op == "conv_fprop":
    x, w, y = kw["x"], kw["w"], kw["y"]
    s, p = kw.get("stride", 1), kw.get("pad", 0)
    n, oh, ow = _pixels_nhw(flat, y.shape[1], y.shape[2])
    Cout, R, S, Cin = w.shape
    A = torch.cat([_gather_nhwc(x, n, oh * s - p + r, ow * s - p + q)
                   for r in range(R) for q in range(S)], 1)
    return A, w.reshape(Cout, -1).to(torch.float64).t()
  if op == "conv_dgrad":
    dy, w, dx = kw["dy"], kw["w"], kw["dx"]
    s, p = kw.get("stride", 1), kw.get("pad", 0)
    n, h, ww = _pixels_nhw(flat, dx.shape[1], dx.shape[2])
    Cout, R, S, Cin = w.shape
    cols = []
    for r in range(R):
      for q in range(S):
        th, tw = h + p - r, ww + p - q
        ok = (th % s == 0) & (tw % s == 0)
        v = _gather_nhwc(dy, n, torch.where(ok, th // s, -1), torch.where(ok, tw // s, -1))
        cols.append(v)
    A = torch.cat(cols, 1)
    return A, w.permute(1, 2, 0, 3).reshape(R * S * Cout, Cin).to(torch.float64)
  if op == "stem_fprop":
    xp, w, y = kw["xp"], kw["w"], kw["y"]
    n, oh, ow = _pixels_nhw(flat, y.shape[1], y.shape[2])
    H = xp.shape[1]
    cols = []
    for r in range(7):
      h = 2 * oh - 3 + r
      ok = (h >= 0) & (h < H)
      win = torch.stack([xp[n, h.clamp(0, H - 1), 2 * ow + j, :] for j in range(8)], 1)
      cols.append(win.reshape(len(flat), 64).to(torch.float64) * ok.unsqueeze(1))
    return torch.cat(cols, 1), w.reshape(w.shape[0], -1).to(torch.float64).t()
  raise AssertionError(op)


def _mask_bits(bits, flat, ldo, N):
  """Mask bits of elements (flat pixel, column < N) of a [pixels, ldo] tensor; float64 0 / 1."""
  import torch
  e = flat.unsqueeze(1) * ldo + torch.arange(N, device=flat.device).unsqueeze(0)
  return ((bits[e >> 3].to(torch.int64) >> (e & 7)) & 1).to(torch.float64)


def _act(v, relu):
  if relu == 0 or relu is False:
    return v
  v = v.clamp_min(0.0)
  return v.clamp_max(6.0) if int(relu) == 2 else v


def _check_fwd(op, kw, outs, infos, what):
  """Element-wise check of a forward-like plan after one run.  Returns whether the rounding-bias
  statistic had enough elements to be checked (None where it does not apply: accumulating or
  fp32 outputs)."""
  import torch
  view, back, init = outs["out"]
  fp32 = view.dtype == torch.float32
  u_out = pc.U_FP32 if fp32 else pc.U_BF16
  ldo = view.shape[-1]
  out2 = view.reshape(-1, ldo)
  N = {"gemm": lambda: kw["b"].shape[0] if kw.get("b_layout", "nk") == "nk" else kw["b"].shape[1],
       "conv_fprop": lambda: kw["w"].shape[0], "stem_fprop": lambda: kw["w"].shape[0],
       "conv_dgrad": lambda: kw["w"].shape[3]}[op]()
  # flat output pixel of each sample (the plans address out[(n OH + h) OW + w]; a GEMM is one
  # row of M pixels); plans of up to 64 K pixels are checked in full
  if out2.shape[0] <= 65536:
    n, h, w = pc.all_pixels(infos, DEV)
  else:
    n, h, w = pc.sample_pixels(infos, DEV)[:3]
  if op == "gemm":
    flat = w
  else:
    flat = (n * view.shape[1] + h) * view.shape[2] + w
  A, B = _im2col(op, kw, flat)
  conv = A @ B
  M = A.abs() @ B.abs()
  nchain = A.shape[1] + 1
  bias = kw.get("bias")
  if bias is not None:
    conv = conv + bias.to(torch.float64)[:N]
    M = M + bias.to(torch.float64).abs()[:N]
  relu = int(kw.get("relu", 0))
  partial = conv
  prevm = None
  if kw.get("accumulate"):
    prev = init.reshape(-1, ldo)[flat, :N].to(torch.float64)
    if kw.get("acc_mask") is not None:
      prev = prev * _mask_bits(kw["acc_mask"], flat, ldo, N)
    prevm = prev
    pre = partial + prev
  else:
    pre = partial
  ref = _act(pre, relu)
  got = out2[flat, :N]
  bound = pc.elem_bound(ref, M, nchain, u_out, partial=partial if prevm is not None else None,
                        prev=prevm)
  pc.check_close(got, ref, bound, what + " out")
  bias_checked = None
  if prevm is None and not fp32:
    # systematic rounding bias, over elements the activation did not change
    keep = pre == ref
    mean, _ = pc.check_no_bias(got[keep], ref[keep], M[keep], nchain, what, u_out)
    bias_checked = mean is not None
  # every non-accumulating element written, nothing past n_valid, guard bands intact
  assert pc.guard_intact(view, back), what + ": guard band overwritten"
  if not kw.get("accumulate"):
    un = pc.unwritten(out2)
    assert not bool(un[:, :N].any()), "{}: {} elements never written".format(what,
                                                                            int(un[:, :N].sum()))
    if ldo > N:
      assert bool(un[:, N:].all()), what + ": columns past n_valid written"
  stored = out2[:, :N].to(torch.float64)
  # the column sums: fp32 round-to-nearest along the epilogue's reduction tree
  staged = not fp32 and N % infos[0]["bn"] == 0 and ldo % 8 == 0
  g_sum = pc.gamma_prob(pc.fwd_stat_depth(infos, staged))
  if "stats" in outs:
    (s0, b0), (s1, b1) = outs["stats"]
    for t, bk in ((s0, b0), (s1, b1)):
      assert pc.guard_intact(t, bk), what + ": statistics guard band"
    pc.check_close(s0, stored.sum(0), g_sum * stored.abs().sum(0), what + " col_sum")
    sq = stored * stored
    pc.check_close(s1, sq.sum(0), g_sum * sq.sum(0), what + " col_sumsq")
  if "red" in outs:
    (s0, b0), (s1, b1) = outs["red"]
    rx, rm = kw["bn_reduce"][0], kw["bn_reduce"][1]
    P = stored.shape[0]
    g = stored
    if rm is not None:
      allp = torch.arange(P, device=DEV)
      g = g * _mask_bits(rm, allp, ldo, N)
    x = rx.reshape(-1, N).to(torch.float64)
    pc.check_close(s0, g.sum(0), g_sum * g.abs().sum(0), what + " sum_g")
    gx = g * x
    pc.check_close(s1, gx.sum(0), g_sum * gx.abs().sum(0), what + " sum_gx")
    for t, bk in outs["red"]:
      assert pc.guard_intact(t, bk), what + ": BN-backward sums guard band"
  return bias_checked


def _replay_fwd(op, args, infos, what, reverse=None):
  """Build the plan on fresh tensors, check it reaches the recorded instance, run, check, run again
  in the opposite tile order and require the same bits."""
  import torch
  from tensorflowonspark_b200.ops import igemm
  gen = _Gen(zlib.crc32(what.encode()))
  kw, outs = _make_gemm_inputs(op, args, gen)
  plan = getattr(igemm, op)(**kw)
  got_infos = plan.info()
  if infos is not None:
    strip = lambda L: [{k: v for k, v in i.items() if k != "reverse"} for i in L]  # noqa: E731
    assert strip(got_infos) == strip(infos), what + ": replay built another kernel instance"
    rev = bool(infos[0].get("reverse", 0))
  else:
    rev = bool(reverse)
  plan.set_reverse(rev)
  plan.run()
  torch.cuda.synchronize()
  bias_checked = _check_fwd(op, kw, outs, plan.info(), what)
  first = outs["out"][0].clone()
  view = outs["out"][0]
  view.copy_(outs["out"][2])
  for key in ("stats", "red"):
    if key in outs:
      for t, _ in outs[key]:
        t.zero_()
  plan.set_reverse(not rev)
  plan.run()
  torch.cuda.synchronize()
  ib = (lambda t: t.view(torch.int32)) if view.dtype == torch.float32 else \
      (lambda t: t.view(torch.int16))
  assert torch.equal(ib(first), ib(view)), "{}: tile order changes {} elements".format(
      what, int((ib(first) != ib(view)).sum()))
  return bias_checked


def _replay_wgrad(op, args, infos, what):
  import torch
  from tensorflowonspark_b200.ops import igemm
  gen = _Gen(zlib.crc32(what.encode()))
  kw, outs = _make_gemm_inputs(op, args, gen)
  plan = getattr(igemm, op)(**kw)
  got = plan.info()
  assert got == infos, what + ": replay built another kernel instance"
  plan.run()
  torch.cuda.synchronize()
  dw, back, dw0 = outs["out"]
  assert pc.guard_intact(dw, back), what + ": guard band overwritten"
  # (dy, x as [pixels, channels] per tap, dw as [Cout, taps, Cin])
  if op == "gemm_wgrad":
    dy, x = kw["dy"], kw["x"]
    taps = [lambda idx: x[:, idx].to(torch.float64)]
    Cout, Cin = dw.shape
    dy2 = dy
  elif op == "conv_wgrad":
    dy, x = kw["dy"], kw["x"]
    s, p = kw.get("stride", 1), kw.get("pad", 0)
    Cout, R, S, Cin = dw.shape
    N, OH, OW, _ = dy.shape
    dy2 = dy.reshape(-1, Cout)
    flat = torch.arange(N * OH * OW, device=DEV)
    n, oh, ow = _pixels_nhw(flat, OH, OW)
    taps = []
    for r in range(R):
      for q in range(S):
        taps.append(lambda idx, r=r, q=q: _gather_nhwc(x[..., idx], n, oh * s - p + r,
                                                       ow * s - p + q))
  else:   # stem_wgrad
    dy, xp = kw["dy"], kw["xp"]
    Cout = dw.shape[0]
    Cin = 64
    N, OH, OW, _ = dy.shape
    dy2 = dy.reshape(-1, Cout)
    flat = torch.arange(N * OH * OW, device=DEV)
    n, oh, ow = _pixels_nhw(flat, OH, OW)
    H = xp.shape[1]
    taps = []
    for r in range(7):
      def tap(idx, r=r):
        h = 2 * oh - 3 + r
        ok = (h >= 0) & (h < H)
        win = torch.stack([xp[n, h.clamp(0, H - 1), 2 * ow + j, :] for j in range(8)], 1)
        return win.reshape(-1, 64)[:, idx].to(torch.float64) * ok.unsqueeze(1)
      taps.append(tap)
  dy2 = dy2.reshape(-1, Cout) if op != "gemm_wgrad" else dy
  # two output channels per 64-channel slice of Cout and Cin, rotating with the slice
  cos = sorted({min(Cout - 1, 64 * i + (7 * i + d) % 64) for i in range(-(-Cout // 64))
                for d in (0, 37)})
  cis = sorted({min(Cin - 1, 64 * i + (11 * i + d) % 64) for i in range(-(-Cin // 64))
                for d in (3, 45)})
  ci_t = torch.tensor(cis, device=DEV)
  co_t = torch.tensor(cos, device=DEV)
  g = dy2[:, co_t].to(torch.float64)
  dwv = dw.reshape(Cout, len(taps), Cin)
  dw0v = dw0.reshape(Cout, len(taps), Cin)
  for t, fn in enumerate(taps):
    xt = fn(ci_t)
    ref = dw0v[co_t][:, t][:, ci_t].to(torch.float64) + g.t() @ xt
    M = dw0v[co_t][:, t][:, ci_t].to(torch.float64).abs() + g.abs().t() @ xt.abs()
    bound = pc.wgrad_bound(M - dw0v[co_t][:, t][:, ci_t].to(torch.float64).abs(),
                           dw0v[co_t][:, t][:, ci_t].to(torch.float64).abs(), infos[0])
    pc.check_close(dwv[co_t][:, t][:, ci_t], ref, bound, "{} tap {}".format(what, t))


# ----------------------------------------------------------------------------- coverage table
def dispatch_table():
  """The instances launch_fwd dispatches to (csrc/igemm.cu), plus the modes and wgrad kinds."""
  rows = []
  for bn in (64, 128, 256):
    for epi in (0, 1, 4):
      rows.append(("fwd", bn, 0, epi))
    for epi in (0, 2, 4, 8, 10):
      rows.append(("fwd", bn, 1, epi))
    if bn >= 128:
      for epi in (18, 24, 26):
        rows.append(("fwd", bn, 1, epi))
  rows += [("mode", "b_resident"), ("mode", "reverse"), ("mode", "stem"),
           ("mode", "reverse+b_resident"), ("mode", "reverse+prefetch")]
  rows += [("wgrad", "generic"), ("wgrad", "wide"), ("wgrad", "onepass_3x3"),
           ("wgrad", "stem")]
  return rows


def entries_of(infos):
  out = set()
  for i in infos:
    if i["kind"] == 0:
      out.add(("fwd", i["bn"], i["b_mn"], i["epi"]))
      if i["b_resident"]:
        out.add(("mode", "b_resident"))
      if i["reverse"]:
        out.add(("mode", "reverse"))
        if i["b_resident"]:
          out.add(("mode", "reverse+b_resident"))
        if i["epi"] & 16:
          out.add(("mode", "reverse+prefetch"))
      if i["stem"]:
        out.add(("mode", "stem"))
    else:
      kind = {0: "wide" if i["bn"] == 256 else "generic", 1: "stem", 2: "onepass_3x3"}[i["stem"]]
      out.add(("wgrad", kind))
  return out


# ----------------------------------------------------------------------------- tests
def _is_wgrad(op):
  return op in ("gemm_wgrad", "conv_wgrad", "stem_wgrad")


def test_gemm_plans_match_float64(recorded):
  """Every recorded igemm plan, replayed on fresh tensors."""
  import torch
  failures = []
  bias_runs = []   # bf16 plans without accumulate or activation: did the bias statistic apply?
  for idx, (op, args, infos) in enumerate(recorded["gemm"]):
    what = "{}#{} bn{} epi{} {}".format(op, idx, infos[0]["bn"], infos[0].get("epi", "-"),
                                       [v[1] for v in dict(args).values()
                                        if isinstance(v, tuple) and v and v[0] == "T"])
    try:
      if _is_wgrad(op):
        _replay_wgrad(op, args, infos, what)
      else:
        ran = _replay_fwd(op, args, infos, what)
        if ran is not None and not dict(args).get("relu"):
          bias_runs.append(ran)
    except AssertionError as e:
      failures.append(str(e))
    torch.cuda.empty_cache()
  print("replayed {} igemm signatures; peak allocated {:.1f} GB; rounding-bias check ran on {} "
        "of {} plans without accumulate or activation".format(
            len(recorded["gemm"]), torch.cuda.max_memory_allocated() / 1e9, sum(bias_runs),
            len(bias_runs)))
  assert not failures, "\n".join(failures[:20])
  # it needs gamma_K M far below u |ref|: every plan with K up to ~4096 on these operands
  assert sum(bias_runs) * 2 >= len(bias_runs), "rounding-bias check ran on too few plans"


@pytest.mark.parametrize("name", sorted(SYNTHETIC))
def test_synthetic_plan(name):
  op, args = SYNTHETIC[name]
  a = dict(args)
  reverse = a.pop("reverse", False)
  ran = _replay_fwd(op, pc.freeze(a), None, name, reverse)
  if ran is not None and not a.get("relu"):
    assert ran, name + ": too few elements for the rounding-bias check"


def test_dispatch_coverage(recorded):
  """Each launch_fwd instance, mode and weight-gradient kind is reached by a model plan or a
  named synthetic case."""
  import torch
  count = {e: 0 for e in dispatch_table()}
  for op, args, infos in recorded["gemm"]:
    for e in entries_of(infos):
      if e in count:
        count[e] += 1
  from tensorflowonspark_b200.ops import igemm
  for name in sorted(SYNTHETIC):
    op, args = SYNTHETIC[name]
    a = dict(args)
    reverse = a.pop("reverse", False)
    kw, _ = _make_gemm_inputs(op, pc.freeze(a), _Gen(1))
    plan = getattr(igemm, op)(**kw)
    plan.set_reverse(reverse)
    for e in entries_of(plan.info()):
      if e in count:
        count[e] += 1
    del plan, kw
  torch.cuda.empty_cache()
  print("\n{:<40} {:>6}".format("dispatch entry", "cases"))
  for e in dispatch_table():
    print("{:<40} {:>6}".format(" ".join(str(x) for x in e), count[e]))
  missing = [e for e, c in count.items() if c == 0]
  assert not missing, "unreached dispatch entries: {}".format(missing)


# --------------------------------------------------------------- batch norm and elementwise ops
def _bn_tensors(spec, gen, alias):
  """Fresh tensors for a recorded ops.K call (positional specs, then keyword specs)."""
  import torch
  out = []
  for i, s in enumerate(spec):
    if isinstance(s, tuple) and s and s[0] == "T":
      shape, dt = s[1], getattr(torch, s[2])
      if dt == torch.bfloat16:
        out.append(gen.randn(shape, dt, 1.5, 0.2))
      elif dt == torch.uint8:
        out.append(gen.bits(int(torch.tensor(shape).prod())).view(shape))
      else:
        # per-channel parameters and statistics: positive, around 1
        out.append(gen.randn(shape, dt, 0.5).abs() + 0.5)
    else:
      out.append(s)
  for j, i in alias:
    out[i] = out[j]
  return out


def _guard_out(t, unwritten=True):
  import torch
  fill = None
  if unwritten:
    fill = pc.UNWRITTEN_BF16 if t.dtype == torch.bfloat16 else (
        pc.UNWRITTEN_FP32 if t.dtype == torch.float32 else None)
  v, b = pc.guarded(tuple(t.shape), t.dtype, DEV, fill)
  if not unwritten or fill is None:
    v.copy_(t)
  return v, b


def _run_k(op, a, rev, kw=None):
  import torch
  from tensorflowonspark_b200 import _build
  C = _build.load(required=True)
  C.bn_set_row_reverse(rev)
  try:
    getattr(C, op)(*a, **(kw or {}))
  finally:
    C.bn_set_row_reverse(False)
  torch.cuda.synchronize()


def _f64(t):
  import torch
  return t.to(torch.float64)


def _bits_of(mask, P, Cn):
  import torch
  e = torch.arange(P * Cn, device=DEV)
  return ((mask.reshape(-1)[e >> 3].to(torch.int64) >> (e & 7)) & 1).reshape(P, Cn).bool()


def _check_k(op, spec, kwspec, rev, alias, what):
  """Replay one recorded ops.K call.  Keyword arguments: only the accumulating bn_bwd_apply
  (acc_dgamma / acc_dbeta) is checked here; any other keyword fails the replay."""
  import torch
  gen = _Gen(zlib.crc32(what.encode()))
  vals = _bn_tensors(tuple(spec) + tuple(v for _, v in kwspec), gen, alias)
  a, kwv = vals[:len(spec)], dict(zip((n for n, _ in kwspec), vals[len(spec):]))
  if kwv and not (op == "bn_bwd_apply" and sorted(kwv) == ["acc_dbeta", "acc_dgamma"]):
    raise AssertionError("{}: no float64 replay for keywords {}".format(what, sorted(kwv)))
  u = pc.U_FP32
  if op in ("bn_apply", "bn_apply_finalize"):
    if op == "bn_apply":
      x, res, scale, shift, y, act, mask = a
    else:
      (x, res, y, act, mask, s_sum, s_sq, gam, bet, rm, rv, mean, invstd, scale, shift, count,
       eps, mom) = a
      Cn = x.shape[-1]
      xx = _f64(x).reshape(-1, Cn)
      s_sum.copy_(xx.sum(0).float())
      s_sq.copy_((xx * xx).sum(0).float())
      count = float(xx.shape[0])
      a[15] = count
    yv, yb = _guard_out(y)
    a[4 if op == "bn_apply" else 2] = yv
    if mask is not None:
      mv, mb = _guard_out(mask, False)
      a[6 if op == "bn_apply" else 4] = mv
    saved = [t.clone() if isinstance(t, torch.Tensor) else t for t in a]
    _run_k(op, a, rev)
    if op == "bn_apply_finalize":
      refs = pc.bn_finalize_refs(_f64(s_sum), _f64(s_sq), _f64(gam), _f64(bet), _f64(saved[9]),
                                 _f64(saved[10]), count, eps, mom)
      for name, got in (("mean", mean), ("invstd", invstd), ("scale", scale), ("shift", shift),
                        ("running_mean", rm), ("running_var", rv)):
        pc.check_close(got, refs[name][0], refs[name][1], what + " " + name)
    Cn = x.shape[-1]
    ref, bound, pre, amb = pc.bn_apply_ref(_f64(x).reshape(-1, Cn), _f64(scale), _f64(shift),
                                           _f64(res).reshape(-1, Cn) if res is not None else None,
                                           act)
    pc.check_close(yv.reshape(-1, Cn), ref, bound, what + " y")
    assert pc.guard_intact(yv, yb), what + ": y guard band"
    if mask is not None:
      assert pc.guard_intact(mv, mb), what + ": mask guard band"
      bits = _bits_of(mv, pre.shape[0], Cn)
      bad = (bits != (pre > 0)) & ~amb
      assert not bool(bad.any()), "{}: {} mask bits wrong".format(what, int(bad.sum()))
    outs = [yv.clone()] + ([mv.clone()] if mask is not None else [])
    b = [t.clone() if isinstance(t, torch.Tensor) else t for t in saved]
    b[4 if op == "bn_apply" else 2] = yv
    if mask is not None:
      b[6 if op == "bn_apply" else 4] = mv
    _run_k(op, b, not rev)
    assert torch.equal(outs[0].view(torch.int16), yv.view(torch.int16)), what + ": row order"
    if mask is not None:
      assert torch.equal(outs[1], mv), what + ": row order changes the mask"
    return
  if op in ("bn_bwd_reduce", "bn_bwd_apply"):
    if op == "bn_bwd_reduce":
      dy, x, y, mean, invstd, dgam, dbet, relu, fs, fh = a
      # a gradient of mean 1 and inputs above every mean: dgamma and dbeta are then about as large
      # as the sums of magnitudes that bound them, so a missing block of rows exceeds the bound
      dy.copy_(gen.randn(tuple(dy.shape), torch.bfloat16, 0.5, 1.0))
      x.copy_(gen.randn(tuple(x.shape), torch.bfloat16, 0.5, 3.0))
      sum_g = sum_gx = None
      dx = dres = None
    else:
      dy, x, y, gam, mean, invstd, dgam, dbet, dx, dres, relu, fs, fh = a[:13]
      sum_g, sum_gx = (a[13], a[14]) if len(a) > 13 else (None, None)
    Cn = x.shape[-1]
    dy64 = _f64(dy).reshape(-1, Cn)
    x64 = _f64(x).reshape(-1, Cn)
    P = x64.shape[0]
    amb = torch.zeros_like(dy64, dtype=torch.bool)
    if relu == 0:
      keep = torch.ones_like(amb)
    elif relu == 1:
      keep = _f64(y).reshape(-1, Cn) > 0
    elif relu == 2:
      pre = x64 * _f64(fs) + _f64(fh)
      keep = pre > 0
      amb = pre.abs() <= 2 * u * (x64 * _f64(fs)).abs() + 2 * u * _f64(fh).abs()
    else:
      keep = _bits_of(y, P, Cn)
    g = dy64 * keep
    xm = x64 - _f64(mean)
    is64 = _f64(invstd)
    if op == "bn_bwd_reduce":
      dgv, dgb = _guard_out(dgam, False)
      dbv, dbb = _guard_out(dbet, False)
      a[5], a[6] = dgv, dbv
      d0, b0 = _f64(dgam), _f64(dbet)
      _run_k(op, a, rev)
      # fp32 round-to-nearest along bn_bwd_reduce_kernel's tree, plus x - mean and the invstd
      # product for dgamma
      (ref_g, bnd_g), (ref_b, bnd_b) = pc.bn_bwd_reduce_refs(
          g, xm, is64, pc.red_grid_depth(P, Cn, 2), d0, b0, amb_mag=dy64.abs() * amb)
      pc.check_close(dgv, ref_g, bnd_g, what + " dgamma")
      pc.check_close(dbv, ref_b, bnd_b, what + " dbeta")
      assert pc.guard_intact(dgv, dgb) and pc.guard_intact(dbv, dbb), what + ": guard band"
      return
    acc = None
    if kwv:
      # the accumulating variant: this micro-batch's (dgamma, dbeta) v go to dx and are added to
      # the parameter gradient, prefilled with A.  Unfused, v is the scratch the apply reads; on
      # the fused path only the writing variant publishes v, so it runs first on the same inputs
      # (without dres, which may alias dy)
      acc = [gen.randn((Cn,), torch.float32) for _ in range(2)]
      accv = [_guard_out(t, False) for t in acc]
      if sum_g is not None:
        vg, vgb = _guard_out(dgam)
        vb, vbb = _guard_out(dbet)
        w = list(a)
        w[6], w[7], w[8], w[9] = vg, vb, torch.empty_like(dx), None
        _run_k(op, w, rev)
        assert pc.guard_intact(vg, vgb) and pc.guard_intact(vb, vbb), what + ": v guard band"
        dgam, dbet = vg, vb
        a[6], a[7] = accv[0][0], accv[1][0]   # as the trainer passes them: not read
      kwv = {"acc_dgamma": accv[0][0], "acc_dbeta": accv[1][0]}
    dxv, dxb = _guard_out(dx)
    a[8] = dxv
    dresv = None
    if dres is not None:
      if dres.data_ptr() == dy.data_ptr():
        dresv = dy   # the model aliases them: the kernel reads dy before it overwrites it
      else:
        dresv, dresb = _guard_out(dres)
        a[9] = dresv
    saved = [t.clone() if isinstance(t, torch.Tensor) else t for t in a]
    _run_k(op, a, rev, kwv)
    if sum_g is not None:
      db = _f64(sum_g)
      assert torch.equal(dbet, sum_g), what + ": dbeta differs from sum_g"
      dg_ref, dg_bnd = pc.bn_bwd_fused_dgamma_ref(db, _f64(sum_gx), _f64(mean), is64)
      pc.check_close(dgam, dg_ref, dg_bnd, what + " dgamma")
      dg = _f64(dgam)
    else:
      dg, db = _f64(dgam), _f64(dbet)
    if acc is not None:
      if sum_g is None:
        assert torch.equal(dgam, saved[6]) and torch.equal(dbet, saved[7]), \
            what + ": the micro-batch's dgamma / dbeta changed"
      for (t, bk), a0, v, name in zip(accv, acc, (dgam, dbet), ("acc_dgamma", "acc_dbeta")):
        kc.check_accumulated(t, a0, v, what + " " + name)
        assert pc.guard_intact(t, bk), what + ": " + name + " guard band"
    ref, bound = pc.bn_bwd_dx_ref(g, x64, _f64(gam), _f64(mean), is64, dg, db, amb)
    pc.check_close(dxv.reshape(-1, Cn), ref, bound, what + " dx")
    assert pc.guard_intact(dxv, dxb), what + ": dx guard band"
    if dresv is not None:
      got = _f64(dresv).reshape(-1, Cn)
      bad = (got != pc.bf16_rne(g)) & ~amb
      assert not bool(bad.any()), "{}: {} dres elements wrong".format(what, int(bad.sum()))
    first = [dxv.clone()] + ([dresv.clone()] if dresv is not None else [])
    b = [t.clone() if isinstance(t, torch.Tensor) else t for t in saved]
    b[8] = dxv
    if dresv is not None:
      b[9] = dresv
      if dresv is dy:
        b[0] = dy
        dy.copy_(saved[0])
    if acc is not None:
      for (t, _), a0 in zip(accv, acc):
        t.copy_(a0)
      if sum_g is not None:
        b[6], b[7] = accv[0][0], accv[1][0]
    _run_k(op, b, not rev, kwv)
    if acc is not None:
      for (t, _), a0, v in zip(accv, acc, (dgam, dbet)):
        kc.check_accumulated(t, a0, v, what + ": row order")
    assert torch.equal(first[0].view(torch.int16), dxv.view(torch.int16)), \
        what + ": row order changes dx"
    if dresv is not None:
      assert torch.equal(first[1].view(torch.int16), dresv.view(torch.int16)), \
          what + ": row order changes dres"
    return
  if op == "depthwise3x3_fwd":
    x, w, bias, y, stride, act = a
    N, H, W, Cn = x.shape
    OH, OW = y.shape[1], y.shape[2]
    yv, yb = _guard_out(y)
    a[3] = yv
    _run_k(op, a, rev)
    xp = torch.nn.functional.pad(_f64(x), (0, 0, 1, 1, 1, 1))
    acc = torch.zeros(N, OH, OW, Cn, dtype=torch.float64, device=DEV)
    M = torch.zeros_like(acc)
    for kh in range(3):
      for kq in range(3):
        win = xp[:, kh:kh + (OH - 1) * stride + 1:stride, kq:kq + (OW - 1) * stride + 1:stride]
        wt = _f64(w[kh * 3 + kq])
        acc += win * wt
        M += (win * wt).abs()
    if bias is not None:
      acc += _f64(bias)
      M += _f64(bias).abs()
    ref = _act(acc, act)
    # nine fp32 multiply-adds and the bias in round-to-nearest, then the bf16 rounding
    pc.check_close(yv, ref, pc.U_BF16 * ref.abs() + (1 + pc.U_BF16) * pc.gamma(10, u) * M,
                   what + " y")
    assert pc.guard_intact(yv, yb), what + ": guard band"
    return
  if op == "add_act":
    x, r, out, act = a
    pre = _f64(x) + (_f64(r) if r is not None else 0)
    ref = _act(pre, act)
    if out.data_ptr() == x.data_ptr():
      ov = out
    else:
      ov, ob = _guard_out(out)
      a[2] = ov
    _run_k(op, a, rev)
    pc.check_close(ov, ref, pc.U_BF16 * ref.abs() + u * pre.abs(), what + " out")
    if out.data_ptr() != x.data_ptr():
      assert pc.guard_intact(ov, ob), what + ": guard band"
    return
  if op == "colsum":
    x, out = a
    ov, ob = _guard_out(out, False)
    ov.zero_()
    a[1] = ov
    _run_k(op, a, rev)
    Cn = x.shape[-1]
    xx = _f64(x).reshape(-1, Cn)
    pc.check_close(ov, xx.sum(0), pc.gamma(xx.shape[0] + 1, u) * xx.abs().sum(0), what)
    assert pc.guard_intact(ov, ob), what + ": guard band"
    return
  if op == "bn_inference_coeffs":
    gam, bet, rm, rv, scale, shift, eps = a
    rv.abs_()
    sv, sb = _guard_out(scale)
    hv, hb = _guard_out(shift)
    a[4], a[5] = sv, hv
    _run_k(op, a, rev)
    is64 = 1.0 / torch.sqrt(_f64(rv) + eps)
    sc = _f64(gam) * is64
    rel = 5 * u   # rsqrtf: 2 ulp; the + eps: one rounding
    pc.check_close(sv, sc, (rel + u) * sc.abs(), what + " scale")
    sh = _f64(bet) - _f64(rm) * sc
    pc.check_close(hv, sh, (rel + 3 * u) * (_f64(rm) * sc).abs() + u * sh.abs(), what + " shift")
    assert pc.guard_intact(sv, sb) and pc.guard_intact(hv, hb), what + ": guard band"
    return
  raise AssertionError(op)


def test_bn_and_elementwise_launches_match_float64(recorded):
  """Every recorded batch-norm / elementwise launch, replayed on fresh tensors in both row
  orders."""
  import torch
  failures = []
  ops_seen = set()
  for idx, (op, spec, kw, rev, alias) in enumerate(recorded["k"]):
    ops_seen.add(op)
    what = "{}#{} rev{}".format(op, idx, int(rev))
    try:
      _check_k(op, spec, kw, rev, alias, what)
    except AssertionError as e:
      failures.append(str(e))
    torch.cuda.empty_cache()
  print("replayed {} batch-norm / elementwise signatures".format(len(recorded["k"])))
  assert not failures, "\n".join(failures[:20])
  assert ops_seen == set(K_OPS), "ops never recorded: {}".format(set(K_OPS) - ops_seen)

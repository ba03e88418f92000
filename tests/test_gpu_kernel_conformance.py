"""The pooling, fused-stem, input-decode and small MNIST kernels the models launch, replayed on
fresh seeded tensors and checked element by element against float64 (tools/kernel_conformance.py
holds the references, tools/plan_conformance.py the bounds and guard bands).

A module fixture wraps every ``ops.K`` entry point, runs each model once (ResNet-50 training at
256 x 224^2 plus one evaluation batch, its inference and folded serving forwards, ResNet-50 at
8 x 64^2, CIFAR ResNet-20 with one evaluation batch, U-Net training and prediction, MNIST) and
frees the trainers.  Every distinct call of an entry point this file owns becomes a signature
that is replayed; every other entry point must be checked by the plan conformance suite or by the
float64 test ``COVERED_ELSEWHERE`` names.  Synthetic cases add the edges no model reaches: odd
sizes, partial tiles and channel blocks, overlapping and generic windows, ties, all-negative
borders and NaN.

Checks:
  * max pool forward: y bit for bit and idx exactly the selected tap (first maximum, last NaN);
  * max pool backward: bf16 of the float64 sum routed through idx, within gamma(n); pixels no
    window selects are exactly 0;
  * fused stem forward: statistics as bn_apply_finalize, y / idx exact outside the windows whose
    activation interval is open (kc.stem_pool_ref); bit for bit equal to bn_apply_finalize + the
    3x3/2 max pool, the pair evaluation and serving run;
  * fused stem backward: dgamma / dbeta within the probabilistic summation bound, dx within the
    bn_bwd_apply bound, on every run (the sums are atomics);
  * avgpool, decode, copy_channels, relu_bwd, conv3x3_c1, bn_finalize: see each checker;
  * every output lives between guard bands, non-accumulating outputs start as NaN; pool, decode
    and stem forward outputs are bit for bit equal across runs and under CUDA graph replay;
  * the entry points refuse, before any launch, shapes their kernels cannot handle.
"""
import gc
import importlib.util
import math
import os
import re
import zlib

import pytest

pytestmark = pytest.mark.gpu

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
  spec = importlib.util.spec_from_file_location(name, os.path.join(_ROOT, *path))
  m = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(m)
  return m


pc = _load("plan_conformance", "tools", "plan_conformance.py")
kc = _load("kernel_conformance", "tools", "kernel_conformance.py")
_plans = _load("plan_conformance_suite", "tests", "test_gpu_plan_conformance.py")

DEV = "cuda"
U = pc.U_FP32
SMS = 132   # kSmCount: the grid caps of the backward kernels
UNWRITTEN_U8 = 0xEE   # no tap of a k <= 15 window

KERNEL_OPS = ("stem_bn_relu_pool_fwd", "stem_pool_bn_bwd", "maxpool_fwd", "maxpool_bwd",
              "avgpool_fwd", "avgpool_bwd", "decode_normalize", "copy_channels", "relu_bwd",
              "conv3x3_c1_fwd", "conv3x3_c1_wgrad", "bn_finalize", "bn_fold")
# entry points checked against float64 elsewhere: entry -> the test that does it.  A key
# "entry[kw1,kw2]" names the launches that switch on exactly those optional arguments
# (tests/test_gpu_option_conformance.py's variant()), "entry[*]" every variant; a bare "entry"
# covers the launch with no option switched on.
COVERED_ELSEWHERE = {
    "softmax_xent": "test_gpu_resnet_head.py::test_softmax_xent_against_float64",
    "softmax_xent[label_smoothing]": "test_gpu_resnet_head.py::test_softmax_xent_against_float64",
    "pixel_xent": "test_gpu_unet_loss_options.py::test_optioned_pixel_xent_against_float64",
    "pixel_xent[ignore_index,norm,weights]":
        "test_gpu_unet_loss_options.py::test_optioned_pixel_xent_against_float64",
    "pixel_xent[ignore_index,norm]":
        "test_gpu_unet_loss_options.py::test_optioned_pixel_xent_against_float64",
    "pixel_xent[norm,weights]":
        "test_gpu_unet_loss_options.py::test_optioned_pixel_xent_against_float64",
    "seg_label_norm":
        "test_gpu_unet_loss_options.py::test_label_prepass_is_exact_and_bitwise_reproducible",
    "seg_label_norm[*]":
        "test_gpu_unet_loss_options.py::test_label_prepass_is_exact_and_bitwise_reproducible",
    "seg_eval_metrics": "test_gpu_seg_eval.py::test_seg_eval_metrics_against_float64",
    "seg_eval_metrics[*]":
        "test_gpu_unet_loss_options.py::test_optioned_seg_eval_metrics_against_numpy",
    "seg_predict": "test_gpu_serve_unet.py::test_seg_predict_against_host_reference",
    "depthwise3x3_bwd": "test_gpu_unet_finetune.py::test_depthwise_bwd_against_float64",
    "eval_metrics": "test_gpu_eval.py::test_eval_metrics_against_float64",
    "allreduce_opt": "test_gpu_grad_clip.py::test_clipped_steps_match_float64",
    "grad_sumsq": "test_gpu_grad_clip.py::test_clipped_steps_match_float64",
    "clip_finalize": "test_gpu_grad_clip.py::test_clipped_steps_match_float64",
    "lars_norms": "test_gpu_lars.py::test_lars_steps_match_float64_reference",
    "igemm_run": "test_gpu_plan_conformance.py::test_gemm_plans_match_float64",
    "sigmoid_bce": "test_gpu_multilabel.py::test_sigmoid_bce_against_float64",
    "sigmoid_bce[*]": "test_gpu_multilabel.py::test_sigmoid_bce_against_float64",
    "multilabel_eval_metrics":
        "test_gpu_multilabel.py::test_multilabel_eval_metrics_against_reference",
    "seg_loss_grad": "test_gpu_seg_losses.py::test_focal_against_float64",
    "seg_loss_grad[*]": "test_gpu_seg_losses.py::test_focal_against_float64",
    "seg_loss_grad[cross_entropy,dice_coef]": "test_gpu_seg_losses.py::test_dice_against_float64",
    "seg_loss_grad[dice_coef]": "test_gpu_seg_losses.py::test_dice_against_float64",
    "seg_dice_stats": "test_gpu_seg_losses.py::test_dice_against_float64",
    "seg_dice_stats[*]": "test_gpu_seg_losses.py::test_dice_against_float64",
    "ps_push_dense": "test_gpu_ps_kernels.py::test_push_dense_is_bit_exact",
    "ps_push_sparse": "test_gpu_ps_kernels.py::test_push_sparse_against_float64",
    "ps_pull": "test_gpu_ps_kernels.py::test_pull_copies_bitwise",
    "ps_apply": "test_gpu_ps_kernels.py::test_apply_against_float64",
    "ps_push_slot": "test_gpu_ps_kernels.py::test_push_slot_is_bitwise",
    "ps_pull_model": "test_gpu_ps_kernels.py::test_pull_model_is_bitwise",
}


def _mod():
  from tensorflowonspark_b200 import _build
  return _build.load(required=True)


# ----------------------------------------------------------------------------- recording
def _resnet50_train_and_evaluate():
  from tensorflowonspark_b200.models import resnet
  net = resnet.ResNetTrainer(50, batch=256, image=224)
  net.train_step(*net.synthetic_batch())
  net.evaluate([net.synthetic_batch(seed=1)])


def _cifar_and_evaluate():
  from tensorflowonspark_b200.models import resnet
  net = resnet.CifarResNetTrainer(20, batch=128)
  net.step_kernels()
  net.evaluate([net.synthetic_batch(seed=1)])


MODELS = (_resnet50_train_and_evaluate, _plans._resnet50_serving, _plans._resnet50_small,
          _cifar_and_evaluate, _plans._unet_train, _plans._unet_predict, _plans._mnist)


def signatures(rec):
  """The distinct (op, positional spec, keyword spec, aliases) of the entry points this file
  replays, and the names of every entry point launched, from a plan suite recorder."""
  calls = pc.dedup((op, spec, kw, alias) for op, spec, kw, _, alias in rec.k if op in KERNEL_OPS)
  return {"calls": calls, "names": {c[0] for c in rec.k}}


@pytest.fixture(scope="module")
def recorded():
  import torch
  torch.cuda.set_device(0)
  rec = _plans._Recorder()
  _plans._record_models(rec, MODELS)
  return signatures(rec)


# ----------------------------------------------------------------------------- tensors
class _Gen(object):

  def __init__(self, what):
    import torch
    self.g = torch.Generator(device=DEV)
    self.g.manual_seed(zlib.crc32(what.encode()))

  def randn(self, shape, scale=1.0, shift=0.0, dtype=None):
    import torch
    v = torch.randn(tuple(shape), generator=self.g, device=DEV) * scale + shift
    return v.to(dtype or torch.bfloat16)

  def levels(self, shape, negative=False):
    """bf16 values from 32 levels: ties are common."""
    import torch
    v = torch.randint(0, 32, tuple(shape), generator=self.g, device=DEV).float() / 8 - 2
    if negative:
      v = -(v.abs() + 0.125)
    return v.to(torch.bfloat16)

  def positive(self, n):
    import torch
    return torch.rand(n, generator=self.g, device=DEV) + 0.5

  def u8(self, shape):
    import torch
    return torch.randint(0, 256, tuple(shape), generator=self.g, device=DEV, dtype=torch.uint8)


def _out(shape, dtype, fill=True):
  """A guarded output; ``fill``: start as NaN (bf16 / fp32) or 0xEE (uint8)."""
  import torch
  bits = None
  if fill:
    bits = {torch.bfloat16: pc.UNWRITTEN_BF16, torch.float32: pc.UNWRITTEN_FP32}.get(dtype)
  v, b = pc.guarded(tuple(shape), dtype, DEV, bits)
  if fill and dtype == torch.uint8:
    v.fill_(UNWRITTEN_U8)
  return v, b


def _guarded_copy(t):
  v, b = pc.guarded(tuple(t.shape), t.dtype, DEV)
  v.copy_(t)
  return v, b


def _f64(t):
  import torch
  return t.to(torch.float64)


def _sync():
  import torch
  torch.cuda.synchronize()


def _bits(t):
  import torch
  return t.view(torch.int16) if t.dtype == torch.bfloat16 else (
      t.view(torch.int32) if t.dtype == torch.float32 else t)


def _scribble(t):
  import torch
  _bits(t).fill_(255 if t.dtype == torch.uint8 else -1)


def _same_bits(a, b):
  import torch
  return torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------ checkers
def check_maxpool_fwd(N, H, W, C, k, s, p, what, kind="levels"):
  import torch
  gen = _Gen(what)
  OH, OW = kc.pool_out(H, k, s, p), kc.pool_out(W, k, s, p)
  if kind == "randn":
    x = gen.randn((N, H, W, C), 1.5, 0.2)
  else:
    x = gen.levels((N, H, W, C), negative=kind == "negative")
  if kind == "nan":
    nan = torch.rand(x.shape, generator=gen.g, device=DEV) < 0.1
    x[nan] = float("nan")
    x[0, :min(H, k), :min(W, k)] = float("nan")
  y, yb = _out((N, OH, OW, C), torch.bfloat16)
  idx, ib = _out((N, OH, OW, C), torch.uint8)
  _mod().maxpool_fwd(x, y, idx, k, s, p)
  _sync()
  ry, ridx = kc.maxpool_ref(_f64(x), k, s, p)
  y64 = _f64(y)
  bad = ~((y64 == ry) | (torch.isnan(y64) & torch.isnan(ry)))
  assert not bool(bad.any()), "{}: {} of {} y wrong".format(what, int(bad.sum()), bad.numel())
  bad = idx.long() != ridx
  assert not bool(bad.any()), "{}: {} of {} idx wrong".format(what, int(bad.sum()), bad.numel())
  assert pc.guard_intact(y, yb) and pc.guard_intact(idx, ib), what + ": guard band"
  if kind == "nan":
    assert bool(torch.isnan(y64[0, 0, 0]).all()), what + ": an all-NaN window is not NaN"


def check_maxpool_bwd(N, H, W, C, k, s, p, what):
  import torch
  gen = _Gen(what)
  OH, OW = kc.pool_out(H, k, s, p), kc.pool_out(W, k, s, p)
  _, ridx = kc.maxpool_ref(_f64(gen.levels((N, H, W, C))), k, s, p)
  idx = ridx.to(torch.uint8)
  dy = gen.randn((N, OH, OW, C))
  dx, dxb = _out((N, H, W, C), torch.bfloat16)
  _mod().maxpool_bwd(dy, idx, dx, k, s, p)
  _sync()
  ref, mag, cnt = kc.maxpool_bwd_ref(_f64(dy), ridx, H, W, k, s, p)
  n = max(1, int(cnt.max()))
  pc.check_close(dx, ref, pc.U_BF16 * ref.abs() + (1 + pc.U_BF16) * pc.gamma(n, U) * mag,
                 what + " dx")
  assert bool((dx[cnt == 0] == 0).all()), what + ": a pixel no window selects is not 0"
  assert pc.guard_intact(dx, dxb), what + ": guard band"


def _stats_inputs(gen, x, C):
  """Exact fp32 sums of x's channels and the BN parameters / running statistics."""
  import torch
  xx = _f64(x).reshape(-1, C)
  s_sum, s_sq = xx.sum(0).float(), (xx * xx).sum(0).float()
  gam, bet = gen.positive(C), gen.randn((C,), 0.5, 0.0, torch.float32)
  rm, rv = gen.randn((C,), 0.2, 0.0, torch.float32), gen.positive(C)
  return s_sum, s_sq, gam, bet, rm, rv, float(xx.shape[0])


def _check_finalize(s_sum, s_sq, gam, bet, rm0, rv0, rm, rv, mean, invstd, scale, shift, cnt,
                    eps, mom, what):
  """The bounds of the plan conformance suite's bn_apply_finalize check."""
  refs = pc.bn_finalize_refs(_f64(s_sum), _f64(s_sq), _f64(gam), _f64(bet), _f64(rm0),
                             _f64(rv0), cnt, eps, mom, U)
  for name, got in (("mean", mean), ("invstd", invstd), ("scale", scale), ("shift", shift),
                    ("running_mean", rm), ("running_var", rv)):
    pc.check_close(got, refs[name][0], refs[name][1], what + " " + name)


def check_stem_fwd(N, H, W, C, what, eps=1e-3, mom=0.01, compare_unfused=True):
  import torch
  gen = _Gen(what)
  OH, OW = kc.pool_out(H, 3, 2, 1), kc.pool_out(W, 3, 2, 1)
  x = gen.randn((N, H, W, C), 1.5, 0.2)
  s_sum, s_sq, gam, bet, rm0, rv0, cnt = _stats_inputs(gen, x, C)
  rm, rv = rm0.clone(), rv0.clone()
  outs = [_out((C,), torch.float32) for _ in range(4)]
  mean, invstd, scale, shift = (o[0] for o in outs)
  y, yb = _out((N, OH, OW, C), torch.bfloat16)
  idx, ib = _out((N, OH, OW, C), torch.uint8)
  _mod().stem_bn_relu_pool_fwd(x, y, idx, s_sum.clone(), s_sq.clone(), gam, bet, rm, rv, mean,
                               invstd, scale, shift, cnt, eps, mom)
  _sync()
  _check_finalize(s_sum, s_sq, gam, bet, rm0, rv0, rm, rv, mean, invstd, scale, shift, cnt, eps,
                  mom, what)
  assert all(pc.guard_intact(v, b) for v, b in outs), what + ": statistics guard band"
  lo, hi = kc.stem_act_bounds(_f64(x), _f64(scale), _f64(shift))
  ry, ridx, amb = kc.stem_pool_ref(lo, hi)
  y64, i64 = _f64(y), idx.long()
  bad = ((y64 != ry) | (i64 != ridx)) & ~amb
  assert not bool(bad.any()), "{}: {} of {} windows wrong (y or idx)".format(
      what, int(bad.sum()), bad.numel())
  if bool(amb.any()):
    a_lo, a_hi = kc.at_tap(lo, i64, 3, 2, 1), kc.at_tap(hi, i64, 3, 2, 1)
    ok = (y64 >= a_lo) & (y64 <= a_hi) & (y64 >= ry)
    assert bool(ok[amb].all()), what + ": an ambiguous window holds no candidate maximum"
  assert pc.guard_intact(y, yb) and pc.guard_intact(idx, ib), what + ": guard band"
  del lo, hi, ry, ridx, y64, i64
  if compare_unfused:
    # the evaluation / serving path: bn_apply_finalize(act=1), then the tiled 3x3/2 max pool
    act = torch.empty_like(x)
    y2, idx2 = torch.empty_like(y), torch.empty_like(idx)
    sc2, sh2 = torch.empty_like(scale), torch.empty_like(shift)
    _mod().bn_apply_finalize(x, None, act, 1, None, s_sum.clone(), s_sq.clone(), gam, bet,
                             rm0.clone(), rv0.clone(), torch.empty_like(mean),
                             torch.empty_like(invstd), sc2, sh2, cnt, eps, mom)
    _mod().maxpool_fwd(act, y2, idx2, 3, 2, 1)
    _sync()
    assert _same_bits(sc2, scale) and _same_bits(sh2, shift), what + ": scale / shift differ"
    assert _same_bits(y2, y), what + ": fused and unfused y differ"
    assert torch.equal(idx2, idx), what + ": fused and unfused idx differ"
  return int(amb.sum())


def check_stem_bwd(N, H, W, C, what, runs=2, accumulate=False):
  """``accumulate``: the trainer's accumulating launch - dgamma / dbeta reduce into zeroed scratch
  (checked as the writing variant's outputs) and the scratch is added to the parameter gradient,
  prefilled with A: it must end as fl(A + scratch) bit for bit."""
  import torch
  gen = _Gen(what)
  OH, OW = kc.pool_out(H, 3, 2, 1), kc.pool_out(W, 3, 2, 1)
  x = gen.randn((N, H, W, C), 1.5, 0.2)
  mean = gen.randn((C,), 0.3, 0.0, torch.float32)
  invstd, gam = gen.positive(C), gen.positive(C)
  bet = gen.randn((C,), 0.5, 0.0, torch.float32)
  fs = gam * invstd
  fh = bet - mean * fs
  _, ridx = kc.maxpool_ref(_f64(gen.levels((N, H, W, C))), 3, 2, 1)
  idx = ridx.to(torch.uint8)
  dy = gen.randn((N, OH, OW, C))
  x64 = _f64(x)
  gsum, gmag, _ = kc.maxpool_bwd_ref(_f64(dy), ridx, H, W, 3, 2, 1)
  del ridx
  keep, amb = kc.relu_mask(x64, _f64(fs), _f64(fh))
  g = gsum * keep
  gm = gmag * keep
  xm = x64 - _f64(mean)
  is64 = _f64(invstd)
  P = N * H * W
  gp = pc.gamma_prob(kc.stem_bwd_depth(N, H, W, C, SMS))
  dg_ref = (g * xm).reshape(-1, C).sum(0) * is64
  dg_bnd = gp * (gm * xm.abs()).reshape(-1, C).sum(0) * is64 + \
      (gmag * amb * xm.abs()).reshape(-1, C).sum(0) * is64
  db_ref = g.reshape(-1, C).sum(0)
  db_bnd = gp * gm.reshape(-1, C).sum(0) + (gmag * amb).reshape(-1, C).sum(0)
  A = _f64(gam) * is64
  for r in range(runs):
    dgam, dgb = _guarded_copy(torch.zeros(C, device=DEV))
    dbet, dbb = _guarded_copy(torch.zeros(C, device=DEV))
    dx, dxb = _out((N, H, W, C), torch.bfloat16)
    kw, accs, prefill = {}, [], []
    if accumulate:
      prefill = [gen.randn((C,), 1.0, 0.0, torch.float32) for _ in range(2)]
      accs = [_guarded_copy(t) for t in prefill]
      kw = {"acc_dgamma": accs[0][0], "acc_dbeta": accs[1][0]}
    _mod().stem_pool_bn_bwd(dy, idx, x, gam, mean, invstd, fs, fh, dgam, dbet, dx, **kw)
    _sync()
    w = "{} run{}".format(what, r)
    for (t, bk), a0, v, name in zip(accs, prefill, (dgam, dbet), ("acc_dgamma", "acc_dbeta")):
      kc.check_accumulated(t, a0, v, w + " " + name)
      assert pc.guard_intact(t, bk), w + ": " + name + " guard band"
    pc.check_close(dgam, dg_ref, dg_bnd, w + " dgamma")
    pc.check_close(dbet, db_ref, db_bnd, w + " dbeta")
    dg, db = _f64(dgam), _f64(dbet)
    ref = A * (g - db / P - xm * is64 * dg / P)
    Mv = A * gmag + (A * is64 * dg / P).abs() * (x64.abs() + _f64(mean).abs()) + (A * db / P).abs()
    bound = pc.U_BF16 * ref.abs() + (1 + pc.U_BF16) * pc.gamma(10, U) * Mv
    bound = torch.where(amb, torch.full_like(bound, float("inf")), bound)
    pc.check_close(dx, ref, bound, w + " dx")
    del ref, Mv, bound
    assert pc.guard_intact(dgam, dgb) and pc.guard_intact(dbet, dbb), w + ": sums guard band"
    assert pc.guard_intact(dx, dxb), w + ": dx guard band"


def check_avgpool_fwd(xshape, what):
  import torch
  gen = _Gen(what)
  N, C = xshape[0], xshape[-1]
  HW = math.prod(xshape) // (N * C)
  x = gen.randn(xshape, 1.5, 0.2)
  y, yb = _out((N, C), torch.bfloat16)
  _mod().avgpool_fwd(x, y)
  _sync()
  ref, mag = kc.avgpool_ref(_f64(x))
  # HW sequential fp32 additions and the multiply by fl(1 / HW), then the bf16 rounding
  pc.check_close(y, ref, pc.U_BF16 * ref.abs() + (1 + pc.U_BF16) * pc.gamma(HW + 3, U) * mag,
                 what + " y")
  assert pc.guard_intact(y, yb), what + ": guard band"


def check_avgpool_bwd(dxshape, what):
  import torch
  gen = _Gen(what)
  N, C = dxshape[0], dxshape[-1]
  HW = math.prod(dxshape) // (N * C)
  dy = gen.randn((N, C), 1.5)
  dx, dxb = _out(dxshape, torch.bfloat16)
  _mod().avgpool_bwd(dy, dx)
  _sync()
  ref = (_f64(dy) / HW).reshape(N, *([1] * (len(dxshape) - 2)), C).expand(*dxshape)
  pc.check_close(dx, ref, pc.U_BF16 * ref.abs() + (1 + pc.U_BF16) * pc.gamma(2, U) * ref.abs(),
                 what + " dx")
  assert pc.guard_intact(dx, dxb), what + ": guard band"


def check_decode(ishape, oshape, wofs, mean, std, what):
  import torch
  gen = _Gen(what)
  img = gen.u8(ishape)
  out, ob = _out(oshape, torch.bfloat16)
  _mod().decode_normalize(img, out, wofs, list(mean), list(std))
  _sync()
  ref, mag = kc.decode_ref(img, oshape[2], oshape[3], wofs, mean, std)
  # x * fl(1/255), the mean, the scale (and their fp32 products in the RGB kernel): at most six
  # fp32 roundings of terms bounded by mag; zero padding exact
  pc.check_close(out, ref, pc.U_BF16 * ref.abs() + (1 + pc.U_BF16) * pc.gamma(6, U) * mag,
                 what + " out")
  assert pc.guard_intact(out, ob), what + ": guard band"


def check_copy_channels(sshape, dshape, C, soff, doff, what):
  gen = _Gen(what)
  src = gen.randn(sshape)
  dst, db = _guarded_copy(gen.randn(dshape))
  want = dst.clone()
  want.view(-1, dshape[-1])[:, doff:doff + C] = src.view(-1, sshape[-1])[:, soff:soff + C]
  _mod().copy_channels(src, dst, C, soff, doff)
  _sync()
  assert _same_bits(dst, want), what + ": copy or untouched channels wrong"
  assert pc.guard_intact(dst, db), what + ": guard band"


def check_relu_bwd(shape, in_place, what):
  import torch
  gen = _Gen(what)
  dy = gen.randn(shape)
  y = gen.randn(shape)
  y.view(-1)[::7] = 0   # exact zeros: the mask is y > 0
  want = torch.where(y > 0, dy, torch.zeros_like(dy))
  if in_place:
    dy, b = _guarded_copy(dy)
    dx = dy
  else:
    dx, b = _out(shape, torch.bfloat16)
  _mod().relu_bwd(dy, y, dx)
  _sync()
  assert _same_bits(dx, want), what + ": dx wrong"
  assert pc.guard_intact(dx, b), what + ": guard band"


def check_conv3x3_c1_fwd(xshape, Cout, bias, relu, what):
  import torch
  gen = _Gen(what)
  N, H, W = xshape
  x = gen.randn(xshape)
  w = gen.randn((Cout, 9), 0.5)
  b = gen.randn((Cout,), 0.5, 0.0, torch.float32) if bias else None
  y, yb = _out((N, H - 2, W - 2, Cout), torch.bfloat16)
  _mod().conv3x3_c1_fwd(x, w, b, y, relu)
  _sync()
  ref, mag = kc.conv3x3_c1_ref(_f64(x), _f64(w), _f64(b) if bias else None)
  if relu:
    ref = ref.clamp_min(0)
  # nine fp32 multiply-adds onto the bias, then the bf16 rounding
  pc.check_close(y, ref, pc.U_BF16 * ref.abs() + (1 + pc.U_BF16) * pc.gamma(10, U) * mag,
                 what + " y")
  assert pc.guard_intact(y, yb), what + ": guard band"


def check_conv3x3_c1_wgrad(xshape, Cout, bias, what):
  import torch
  gen = _Gen(what)
  N, H, W = xshape
  x = gen.randn(xshape)
  dy = gen.randn((N, H - 2, W - 2, Cout))
  dw, dwb = _guarded_copy(gen.randn((Cout, 9), 1.0, 0.0, torch.float32))
  d0 = _f64(dw)
  db = dbb = b0 = None
  if bias:
    db, dbb = _guarded_copy(gen.randn((Cout,), 1.0, 0.0, torch.float32))
    b0 = _f64(db)
  _mod().conv3x3_c1_wgrad(x, dy, dw, db)
  _sync()
  rw, mw, rb, mb = kc.conv3x3_c1_wgrad_ref(_f64(x), _f64(dy))
  # a thread's pixels, the block's pixel lanes, one atomic per block (conv3x3_c1_wgrad's grid)
  P = N * (H - 2) * (W - 2)
  grid = max(1, min(-(-P // 64), SMS * 2))
  pl = 256 // min(Cout, 256)
  depth = -(-P // (grid * pl)) + pl + grid + 2
  gp = pc.gamma_prob(depth)
  pc.check_close(dw, d0 + rw, gp * (d0.abs() + mw), what + " dw")
  assert pc.guard_intact(dw, dwb), what + ": dw guard band"
  if bias:
    pc.check_close(db, b0 + rb, gp * (b0.abs() + mb), what + " dbias")
    assert pc.guard_intact(db, dbb), what + ": dbias guard band"


def check_bn_finalize(C, rows, what, eps=1e-3, mom=0.01):
  import torch
  gen = _Gen(what)
  x = gen.randn((rows, C), 1.5, 0.2)
  s_sum, s_sq, gam, bet, rm0, rv0, cnt = _stats_inputs(gen, x, C)
  sv, sb = _guarded_copy(s_sum)
  qv, qb = _guarded_copy(s_sq)
  rm, rv = rm0.clone(), rv0.clone()
  outs = [_out((C,), torch.float32) for _ in range(4)]
  mean, invstd, scale, shift = (o[0] for o in outs)
  _mod().bn_finalize(sv, qv, gam, bet, rm, rv, mean, invstd, scale, shift, cnt, eps, mom)
  _sync()
  _check_finalize(s_sum, s_sq, gam, bet, rm0, rv0, rm, rv, mean, invstd, scale, shift, cnt, eps,
                  mom, what)
  assert bool((sv == 0).all() and (qv == 0).all()), what + ": sums not cleared"
  assert all(pc.guard_intact(v, b) for v, b in outs + [(sv, sb), (qv, qb)]), what + ": guard band"


def check_bn_fold(tab, row0, rows, wshape, aux_n, run_n, what):
  """bn_fold over a recorded table (tab, row0: the trainer's values) on fresh seeded filters,
  gamma / beta and running statistics, with variances from 1e-6 to 1e3 (log-uniform) so that eps
  matters for some channels and is negligible for others, and guarded outputs prefilled with
  random values: the elements no unit covers must keep them (kc.check_bn_fold)."""
  import torch
  gen = _Gen(what)
  tab_t = torch.tensor(tab, dtype=torch.int64).reshape(-1, kc.FOLD_COLS)
  row0_t = torch.tensor(row0, dtype=torch.int64)
  eps = torch.full((tab_t.shape[0],), 1e-5, dtype=torch.float32)
  w = gen.randn(wshape, 0.05)
  aux32 = gen.randn((aux_n,), 1.0, 0.0, torch.float32)
  running = gen.randn((run_n,), 0.5, 0.0, torch.float32)
  for wo, cout, per, go, bo, mo, vo, fo in tab_t.tolist():
    running[vo:vo + cout] = torch.pow(10.0, torch.rand(cout, generator=gen.g, device=DEV) * 9 - 6)
  nb = max(r[7] + (r[1] + 7) // 8 * 8 for r in tab_t.tolist())
  wf, wfb = _guarded_copy(gen.randn(wshape))
  bias, bb = _guarded_copy(gen.randn((nb,), 1.0, 0.0, torch.float32))
  wf0, bias0 = wf.clone(), bias.clone()
  _mod().bn_fold(tab_t.to(DEV), eps.to(DEV), row0_t.to(DEV), rows, w, aux32, running, wf, bias)
  _sync()
  kc.check_bn_fold(wf, bias, wf0, bias0, tab_t, eps, row0_t, w, aux32, running, what)
  assert pc.guard_intact(wf, wfb) and pc.guard_intact(bias, bb), what + ": guard band"


# -------------------------------------------------------------------- recorded signatures
def _shape(s):
  assert isinstance(s, tuple) and s and s[0] == "T", s
  return tuple(s[1])


def replay(op, spec, kwspec, alias, what):
  """Run the checker of a recorded call with the recorded shapes, scalar and keyword arguments."""
  a = list(spec)
  kw = dict(kwspec)
  if kw and not (op == "stem_pool_bn_bwd" and sorted(kw) == ["acc_dbeta", "acc_dgamma"]):
    raise AssertionError("{}: no float64 replay for keywords {}".format(what, sorted(kw)))
  if op == "maxpool_fwd":
    N, H, W, C = _shape(a[0])
    k, s, p = a[3:6]
    check_maxpool_fwd(N, H, W, C, k, s, p, what, kind="randn")
    check_maxpool_fwd(N, H, W, C, k, s, p, what + " ties")
  elif op == "maxpool_bwd":
    check_maxpool_bwd(*_shape(a[2]), *a[3:6], what)
  elif op == "stem_bn_relu_pool_fwd":
    check_stem_fwd(*_shape(a[0]), what, eps=a[14], mom=a[15])
  elif op == "stem_pool_bn_bwd":
    check_stem_bwd(*_shape(a[2]), what, runs=1, accumulate=bool(kw))
  elif op == "avgpool_fwd":
    check_avgpool_fwd(_shape(a[0]), what)
  elif op == "avgpool_bwd":
    check_avgpool_bwd(_shape(a[1]), what)
  elif op == "decode_normalize":
    check_decode(_shape(a[0]), _shape(a[1]), a[2], a[3], a[4], what)
  elif op == "copy_channels":
    check_copy_channels(_shape(a[0]), _shape(a[1]), a[2], a[3], a[4], what)
  elif op == "relu_bwd":
    check_relu_bwd(_shape(a[0]), (0, 2) in alias, what)
  elif op == "conv3x3_c1_fwd":
    check_conv3x3_c1_fwd(_shape(a[0]), _shape(a[1])[0], a[2] is not None, bool(a[4]), what)
  elif op == "conv3x3_c1_wgrad":
    check_conv3x3_c1_wgrad(_shape(a[0]), _shape(a[2])[0], a[3] is not None, what)
  elif op == "bn_finalize":
    C = _shape(a[0])[0]
    check_bn_finalize(C, 4096, what, eps=a[11], mom=a[12])
  elif op == "bn_fold":
    check_bn_fold(a[0][3], a[2][3], a[3], _shape(a[4]), _shape(a[5])[0], _shape(a[6])[0], what)
  else:
    raise AssertionError(op)


def test_recorded_launches_match_float64(recorded):
  import torch
  failures = []
  for i, (op, spec, kw, alias) in enumerate(recorded["calls"]):
    what = "{}#{}".format(op, i)
    try:
      replay(op, spec, kw, alias, what)
    except AssertionError as e:
      failures.append(str(e))
    gc.collect()
    torch.cuda.empty_cache()
  print("replayed {} recorded pooling / stem / decode / MNIST signatures".format(
      len(recorded["calls"])))
  assert not failures, "\n".join(failures[:20])
  seen = {c[0] for c in recorded["calls"]}
  assert seen == set(KERNEL_OPS), "entry points never recorded: {}".format(set(KERNEL_OPS) - seen)


def test_every_launched_entry_point_has_a_float64_check(recorded):
  """A new ops.K launch in any model must be added to one of the float64 suites."""
  covered = set(KERNEL_OPS) | set(_plans.K_OPS) | {k.split("[")[0] for k in COVERED_ELSEWHERE}
  missing = sorted(recorded["names"] - covered)
  assert not missing, "ops.K entry points without a float64 check: {}".format(missing)
  for op, test in COVERED_ELSEWHERE.items():
    fname, tname = test.split("::")
    with open(os.path.join(_ROOT, "tests", fname)) as f:
      assert re.search(r"^def {}\(".format(tname), f.read(), re.M), (op, test)


# ---------------------------------------------------------------------- synthetic edges
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
SYNTHETIC = {}
for _C in (8, 72, 128):
  for _kind in ("levels", "negative", "nan"):
    SYNTHETIC["pool3s2_fwd_37x41_c{}_{}".format(_C, _kind)] = (
        check_maxpool_fwd, (2, 37, 41, _C, 3, 2, 1), {"kind": _kind})
  SYNTHETIC["pool3s2_bwd_37x41_c{}".format(_C)] = (check_maxpool_bwd, (2, 37, 41, _C, 3, 2, 1), {})
  SYNTHETIC["stem_fwd_37x41_c{}".format(_C)] = (check_stem_fwd, (2, 37, 41, _C), {})
SYNTHETIC.update({
    "pool3s2_fwd_1x1": (check_maxpool_fwd, (1, 1, 1, 8, 3, 2, 1), {}),
    "pool3s2_fwd_partial_tiles": (check_maxpool_fwd, (3, 9, 17, 64, 3, 2, 1), {}),
    "pool3s2_bwd_1x1": (check_maxpool_bwd, (1, 1, 1, 8, 3, 2, 1), {}),
    "pool3s2_bwd_partial_tiles": (check_maxpool_bwd, (3, 9, 17, 64, 3, 2, 1), {}),
    "pool2s2_fwd_26": (check_maxpool_fwd, (2, 26, 26, 32, 2, 2, 0), {}),
    "pool2s2_fwd_odd": (check_maxpool_fwd, (2, 27, 9, 16, 2, 2, 0), {"kind": "negative"}),
    "pool2s2_fwd_nan": (check_maxpool_fwd, (2, 27, 9, 16, 2, 2, 0), {"kind": "nan"}),
    "pool3s1_fwd_overlap": (check_maxpool_fwd, (2, 10, 13, 24, 3, 1, 1), {}),
    "pool3s1_fwd_overlap_nan": (check_maxpool_fwd, (2, 10, 13, 24, 3, 1, 1), {"kind": "nan"}),
    "pool2s2_bwd_odd": (check_maxpool_bwd, (2, 27, 9, 16, 2, 2, 0), {}),
    "pool3s1_bwd_overlap": (check_maxpool_bwd, (2, 10, 13, 24, 3, 1, 1), {}),
    "stem_fwd_1x1": (check_stem_fwd, (1, 1, 1, 8), {}),
    "stem_fwd_partial_tiles": (check_stem_fwd, (3, 9, 17, 64), {}),
    "stem_bwd_37x41_c8": (check_stem_bwd, (2, 37, 41, 8), {}),
    "stem_bwd_37x41_c128": (check_stem_bwd, (2, 37, 41, 128), {}),
    "stem_bwd_1x1": (check_stem_bwd, (2, 1, 1, 8), {}),
    "stem_bwd_partial_tiles": (check_stem_bwd, (3, 9, 17, 64), {}),
    "avgpool_fwd_hw1": (check_avgpool_fwd, ((5, 1, 1, 16),), {}),
    "avgpool_fwd_hw4": (check_avgpool_fwd, ((5, 2, 2, 72),), {}),
    "avgpool_fwd_hw49": (check_avgpool_fwd, ((5, 7, 7, 136),), {}),
    "avgpool_fwd_hw64": (check_avgpool_fwd, ((5, 8, 8, 8),), {}),
    "avgpool_bwd_hw1": (check_avgpool_bwd, ((5, 1, 1, 16),), {}),
    "avgpool_bwd_hw49": (check_avgpool_bwd, ((5, 7, 7, 136),), {}),
    "avgpool_bwd_hw64": (check_avgpool_bwd, ((5, 8, 8, 8),), {}),
    "decode_rgb8_wofs3": (check_decode, ((2, 5, 9, 3), (2, 5, 15, 8), 3, MEAN, STD), {}),
    "decode_rgb8_odd_wp": (check_decode, ((3, 4, 6, 3), (3, 4, 7, 8), 1, MEAN, STD), {}),
    "decode_generic_cp16": (check_decode, ((2, 5, 9, 3), (2, 5, 12, 16), 2, MEAN, STD), {}),
    "decode_generic_c6": (check_decode, ((2, 5, 9, 6), (2, 5, 9, 8), 0, MEAN, STD), {}),
    "decode_generic_cp5": (check_decode, ((2, 3, 4, 5), (2, 3, 6, 5), 1, MEAN, STD), {}),
    "copy_channels_offsets": (check_copy_channels, ((3, 5, 7, 24), (3, 5, 7, 40), 16, 8, 24), {}),
    "relu_bwd_in_place": (check_relu_bwd, ((4, 13, 13, 32), True), {}),
    "relu_bwd": (check_relu_bwd, ((3, 40), False), {}),
    "conv3x3_c1_fwd_odd": (check_conv3x3_c1_fwd, ((3, 11, 9), 40, True, False), {}),
    "conv3x3_c1_fwd_nobias_relu": (check_conv3x3_c1_fwd, ((2, 7, 30), 8, False, True), {}),
    "conv3x3_c1_wgrad_odd": (check_conv3x3_c1_wgrad, ((3, 11, 9), 40, True), {}),
    "conv3x3_c1_wgrad_wide": (check_conv3x3_c1_wgrad, ((2, 9, 9), 512, False), {}),
    "bn_finalize_c72": (check_bn_finalize, (72, 333), {}),
})


def test_synthetic_edges_match_float64():
  import torch
  failures = []
  for name in sorted(SYNTHETIC):
    fn, args, kw = SYNTHETIC[name]
    try:
      fn(*args, what=name, **kw)
    except AssertionError as e:
      failures.append(str(e))
    torch.cuda.empty_cache()
  print("checked {} synthetic cases".format(len(SYNTHETIC)))
  assert not failures, "\n".join(failures[:20])


# ------------------------------------------------------------- determinism and graph replay
def _pool_launches(gen):
  """(name, run, outputs) of every pooling / decode / stem-forward kernel on fixed inputs."""
  import torch
  m = _mod()
  x = gen.levels((2, 37, 41, 72))
  xs = gen.randn((2, 37, 41, 72), 1.5, 0.2)
  stats = _stats_inputs(gen, xs, 72)
  y3, i3 = torch.empty(2, 19, 21, 72, dtype=torch.bfloat16, device=DEV), \
      torch.empty(2, 19, 21, 72, dtype=torch.uint8, device=DEV)
  y2, i2 = torch.empty(2, 18, 20, 72, dtype=torch.bfloat16, device=DEV), \
      torch.empty(2, 18, 20, 72, dtype=torch.uint8, device=DEV)
  dx3, dx2 = torch.empty_like(x), torch.empty_like(x)
  ys, is_ = torch.empty_like(y3), torch.empty_like(i3)
  vec = [torch.empty(72, device=DEV) for _ in range(4)]
  rm, rv = stats[4].clone(), stats[5].clone()
  av = torch.empty(2, 72, dtype=torch.bfloat16, device=DEV)
  dav = torch.empty_like(x)
  img = gen.u8((2, 9, 11, 3))
  d8 = torch.empty(2, 9, 14, 8, dtype=torch.bfloat16, device=DEV)
  d16 = torch.empty(2, 9, 14, 16, dtype=torch.bfloat16, device=DEV)
  return [
      ("maxpool_fwd 3x3/2", lambda: m.maxpool_fwd(x, y3, i3, 3, 2, 1), (y3, i3)),
      ("maxpool_fwd 2x2/2", lambda: m.maxpool_fwd(x, y2, i2, 2, 2, 0), (y2, i2)),
      ("maxpool_bwd 3x3/2", lambda: m.maxpool_bwd(y3, i3, dx3, 3, 2, 1), (dx3,)),
      ("maxpool_bwd 2x2/2", lambda: m.maxpool_bwd(y2, i2, dx2, 2, 2, 0), (dx2,)),
      ("stem_bn_relu_pool_fwd",
       lambda: m.stem_bn_relu_pool_fwd(xs, ys, is_, stats[0], stats[1], stats[2], stats[3], rm, rv,
                                       *vec, stats[6], 1e-3, 0.01), (ys, is_)),
      ("avgpool_fwd", lambda: m.avgpool_fwd(x, av), (av,)),
      ("avgpool_bwd", lambda: m.avgpool_bwd(av, dav), (dav,)),
      ("decode rgb8", lambda: m.decode_normalize(img, d8, 2, list(MEAN), list(STD)), (d8,)),
      ("decode generic", lambda: m.decode_normalize(img, d16, 1, list(MEAN), list(STD)), (d16,)),
  ]


def test_pool_outputs_bitwise_across_runs_and_graph_replay():
  import torch
  launches = _pool_launches(_Gen("determinism"))
  first = []
  for _, run, outs in launches:
    run()
    torch.cuda.synchronize()
    first.append([o.clone() for o in outs])
  for (name, run, outs), ref in zip(launches, first):
    for o in outs:
      _scribble(o)
    run()
    torch.cuda.synchronize()
    assert all(_same_bits(o, r) for o, r in zip(outs, ref)), name + ": second run differs"
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.stream(s):
    with torch.cuda.graph(graph, stream=s):
      for _, run, _ in launches:
        run()
  torch.cuda.current_stream().wait_stream(s)
  for _, _, outs in launches:
    for o in outs:
      _scribble(o)
  graph.replay()
  torch.cuda.synchronize()
  for (name, _, outs), ref in zip(launches, first):
    assert all(_same_bits(o, r) for o, r in zip(outs, ref)), name + ": graph replay differs"


# ---------------------------------------------------------------------------- refusals
def _bad_calls():
  """(what, entry point, arguments) the entry points must refuse before launching anything."""
  import torch
  m = _mod()
  bf = lambda *s: torch.zeros(*s, dtype=torch.bfloat16, device=DEV)  # noqa: E731
  u8 = lambda *s: torch.zeros(*s, dtype=torch.uint8, device=DEV)  # noqa: E731
  f32 = lambda *s: torch.zeros(*s, dtype=torch.float32, device=DEV)  # noqa: E731
  v = lambda C: [f32(C) for _ in range(10)]  # noqa: E731
  return [
      ("maxpool_fwd C % 8", m.maxpool_fwd, (bf(1, 8, 8, 12), bf(1, 4, 4, 12), u8(1, 4, 4, 12), 3, 2, 1)),
      ("maxpool_fwd y shape", m.maxpool_fwd, (bf(1, 8, 8, 8), bf(1, 3, 4, 8), u8(1, 3, 4, 8), 3, 2, 1)),
      ("maxpool_fwd y channels", m.maxpool_fwd, (bf(1, 8, 8, 16), bf(1, 4, 4, 8), u8(1, 4, 4, 8), 3, 2, 1)),
      ("maxpool_fwd y dtype", m.maxpool_fwd, (bf(1, 8, 8, 8), f32(1, 4, 4, 8), u8(1, 4, 4, 8), 3, 2, 1)),
      ("maxpool_fwd idx dtype", m.maxpool_fwd, (bf(1, 8, 8, 8), bf(1, 4, 4, 8), bf(1, 4, 4, 8), 3, 2, 1)),
      ("maxpool_fwd idx numel", m.maxpool_fwd, (bf(1, 8, 8, 8), bf(1, 4, 4, 8), u8(1, 4, 4, 4), 3, 2, 1)),
      ("maxpool_fwd k > 15", m.maxpool_fwd, (bf(1, 16, 16, 8), bf(1, 1, 1, 8), u8(1, 1, 1, 8), 16, 1, 0)),
      ("maxpool_fwd pad > k / 2", m.maxpool_fwd, (bf(1, 4, 4, 8), bf(1, 7, 7, 8), u8(1, 7, 7, 8), 2, 1, 2)),
      ("maxpool_bwd C % 8", m.maxpool_bwd, (bf(1, 4, 4, 12), u8(1, 4, 4, 12), bf(1, 8, 8, 12), 3, 2, 1)),
      ("maxpool_bwd dy shape", m.maxpool_bwd, (bf(1, 5, 4, 8), u8(1, 5, 4, 8), bf(1, 8, 8, 8), 3, 2, 1)),
      ("maxpool_bwd idx numel", m.maxpool_bwd, (bf(1, 4, 4, 8), u8(1, 4, 4, 4), bf(1, 8, 8, 8), 3, 2, 1)),
      ("maxpool_bwd dx dtype", m.maxpool_bwd, (bf(1, 4, 4, 8), u8(1, 4, 4, 8), f32(1, 8, 8, 8), 3, 2, 1)),
      ("maxpool_bwd generic C % 8", m.maxpool_bwd, (bf(1, 4, 4, 4), u8(1, 4, 4, 4), bf(1, 8, 8, 4), 2, 2, 0)),
      ("avgpool_fwd C % 8", m.avgpool_fwd, (bf(2, 7, 7, 12), bf(2, 12))),
      ("avgpool_fwd y numel", m.avgpool_fwd, (bf(2, 7, 7, 16), bf(2, 8))),
      ("avgpool_fwd y dtype", m.avgpool_fwd, (bf(2, 7, 7, 16), f32(2, 16))),
      ("avgpool_bwd dy dtype", m.avgpool_bwd, (f32(2, 16), bf(2, 7, 7, 16))),
      ("avgpool_bwd dy numel", m.avgpool_bwd, (bf(2, 8), bf(2, 7, 7, 16))),
      ("avgpool_bwd C % 8", m.avgpool_bwd, (bf(2, 12), bf(2, 7, 7, 12))),
      ("decode out N", m.decode_normalize, (u8(2, 4, 6, 3), bf(1, 4, 6, 8), 0, [0.5], [0.5])),
      ("decode out H", m.decode_normalize, (u8(2, 4, 6, 3), bf(2, 3, 6, 8), 0, [0.5], [0.5])),
      ("decode wofs + W > Wp", m.decode_normalize, (u8(2, 4, 6, 3), bf(2, 4, 8, 8), 3, [0.5], [0.5])),
      ("decode wofs < 0", m.decode_normalize, (u8(2, 4, 6, 3), bf(2, 4, 8, 8), -1, [0.5], [0.5])),
      ("decode C > Cp", m.decode_normalize, (u8(2, 4, 6, 9), bf(2, 4, 6, 8), 0, [0.5], [0.5])),
      ("stem fwd C % 8", m.stem_bn_relu_pool_fwd,
       (bf(1, 8, 8, 12), bf(1, 4, 4, 12), u8(1, 4, 4, 12), *v(12), 64.0, 1e-3, 0.01)),
      ("stem fwd y shape", m.stem_bn_relu_pool_fwd,
       (bf(1, 8, 8, 8), bf(1, 4, 5, 8), u8(1, 4, 5, 8), *v(8), 64.0, 1e-3, 0.01)),
      ("stem fwd idx dtype", m.stem_bn_relu_pool_fwd,
       (bf(1, 8, 8, 8), bf(1, 4, 4, 8), bf(1, 4, 4, 8), *v(8), 64.0, 1e-3, 0.01)),
      ("stem bwd C = 72", m.stem_pool_bn_bwd,
       (bf(1, 4, 4, 72), u8(1, 4, 4, 72), bf(1, 8, 8, 72), *v(72)[:7], bf(1, 8, 8, 72))),
      ("stem bwd dy_pool shape", m.stem_pool_bn_bwd,
       (bf(1, 5, 4, 8), u8(1, 5, 4, 8), bf(1, 8, 8, 8), *v(8)[:7], bf(1, 8, 8, 8))),
      ("stem bwd dx shape", m.stem_pool_bn_bwd,
       (bf(1, 4, 4, 8), u8(1, 4, 4, 8), bf(1, 8, 8, 8), *v(8)[:7], bf(1, 8, 4, 16))),
  ]


def test_bad_shapes_are_refused():
  import torch
  accepted = []
  for what, fn, args in _bad_calls():
    try:
      fn(*args)
    except (RuntimeError, ValueError):
      continue
    accepted.append(what)
  torch.cuda.synchronize()
  assert not accepted, "accepted: {}".format(accepted)

"""CPU tier of the U-Net's focal and Dice losses (``UNetTrainer(loss=...)``): the float64 references
of tools/seg_loss_reference.py (used by tests/test_gpu_seg_losses.py) against torch.autograd,
their finite limits, argument checks before anything touches a device, the examples' flags (with
the stand-in trainer of test_unet_finetune_host) and ptxas' resource report of the new kernels
(needs nvcc, not a GPU)."""
import importlib.util
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_unet_classes_host as uc  # noqa: E402
import test_unet_finetune_host as ft  # noqa: E402


def _ref():
  spec = importlib.util.spec_from_file_location(
      "seg_loss_reference", os.path.join(uc.ROOT, "tools", "seg_loss_reference.py"))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


R = _ref()
GAMMAS = [0.0, 0.5, 1.0, 2.0, 5.0]


# ----------------------------------------------------------------------------- references
def _case(kind, V=5, P=60, seed=0):
  """(logits [P, V + 3] with junk padding, labels, class weights or None, ignore or None)."""
  g = torch.Generator().manual_seed(seed)
  l = torch.randn(P, V + 3, generator=g, dtype=torch.float64) * 2
  l[:, V:] = 1e4
  y = torch.randint(0, V, (P,), generator=g)
  w, ignore = None, None
  if kind == "ignored":
    ignore = 255
    y[::4] = 255
  elif kind == "zero_weights":
    w = torch.rand(V, generator=g, dtype=torch.float64) + 0.5
    w[1] = 0.0
    ignore = 255
    y[::7] = 255
  elif kind == "out_of_range":
    y[::5] = V
    y[1::9] = -1
  elif kind == "empty":
    ignore = 3
    y[:] = 3
  return l, y, w, ignore


def _autograd_focal(l, y, V, gamma, w, ignore):
  x = l[:, :V].clone().requires_grad_(True)
  ok = (y >= 0) & (y < V)
  logp = torch.log_softmax(x, dim=1)
  lpy = logp.gather(1, y.clamp(0, V - 1)[:, None])[:, 0]
  s = R.pixel_scale(y, V, w, ignore)
  fl = -(1 - lpy.exp()) ** gamma * lpy
  ce = torch.logsumexp(x, 1)      # a label outside [0, V): the cross-entropy term lse - 0
  loss = (s * torch.where(ok, fl, ce)).sum()
  loss.backward()
  return float(loss), x.grad


def _autograd_dice(l, y, V, smooth, w, ignore):
  x = l[:, :V].clone().requires_grad_(True)
  S = torch.ones(len(y), dtype=torch.bool) if ignore is None else y != ignore
  ok = (y >= 0) & (y < V)
  p = torch.softmax(x, 1)[S]
  oh = torch.zeros(len(y), V, dtype=torch.float64)
  oh[ok, y[ok]] = 1.0
  oh = oh[S]
  I, P, Y = (p * oh).sum(0), p.sum(0), oh.sum(0)
  wt = torch.ones(V, dtype=torch.float64) if w is None else w
  loss = (wt / wt.sum() * (1 - (2 * I + smooth) / (P + Y + smooth))).sum()
  loss.backward()
  return float(loss), x.grad


KINDS = ["random", "ignored", "zero_weights", "out_of_range", "empty"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("gamma", GAMMAS)
def test_focal_reference_matches_autograd(kind, gamma):
  V = 5
  l, y, w, ignore = _case(kind, V, seed=GAMMAS.index(gamma))
  loss, d = R.focal(l, y, V, gamma, w, ignore)
  want_loss, want = _autograd_focal(l, y, V, gamma, w, ignore)
  assert loss == pytest.approx(want_loss, rel=1e-12, abs=1e-15)
  assert torch.allclose(d, want, rtol=1e-10, atol=1e-14)
  if kind == "empty":
    assert loss == 0.0 and not d.any()


def test_focal_at_gamma_zero_is_cross_entropy():
  import torch.nn.functional as F
  l, y, w, ignore = _case("zero_weights", 6, seed=3)
  loss, d = R.focal(l, y, 6, 0.0, w, ignore)
  x = l[:, :6].clone().requires_grad_(True)
  ref = F.cross_entropy(x, y, weight=w, ignore_index=ignore)
  ref.backward()
  assert loss == pytest.approx(float(ref), rel=1e-12)
  assert torch.allclose(d, x.grad, rtol=1e-10, atol=1e-15)


@pytest.mark.parametrize("gamma", GAMMAS)
def test_focal_reference_is_finite_at_the_singularities(gamma):
  V = 4
  l = torch.zeros(3, V, dtype=torch.float64)
  l[0, 0] = 1000.0      # p_y = 1 exactly (q underflows to 0)
  l[1, 0] = -1000.0     # p_y = 0 exactly
  l[2, 0] = 40.0        # q = 3 e^-40: tiny but not 0
  y = torch.zeros(3, dtype=torch.long)
  loss, d = R.focal(l, y, V, gamma, options=True)
  assert math.isfinite(loss) and bool(torch.isfinite(d).all())
  p, ok, onehot, py, q, lp = R._softmax_parts(l, y, V)
  F, qg = R.focal_factor(py, q, lp, gamma)
  assert float(q[0]) == 0.0 and float(py[1]) == 0.0
  assert float(F[0]) == (1.0 if gamma == 0 else 0.0)     # q^gamma (1 + gamma p_y) at q = 0
  assert float(F[1]) == 1.0                               # p_y log p_y -> 0
  qq = 3 * math.exp(-40)
  assert float(F[2]) == pytest.approx(qq ** gamma * (1 + gamma * (1 - qq)), rel=1e-9)
  assert not d[0].any() or gamma == 0


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("smooth", [1e-5, 1.0])
def test_dice_reference_matches_autograd(kind, smooth):
  V = 5
  l, y, w, ignore = _case(kind, V, seed=7)
  loss, d, A, B = R.dice(l, y, V, smooth, w, ignore)
  want_loss, want = _autograd_dice(l, y, V, smooth, w, ignore)
  assert loss == pytest.approx(want_loss, rel=1e-12, abs=1e-15)
  assert torch.allclose(d, want, rtol=1e-9, atol=1e-15)
  if ignore is not None:
    assert not d[y == ignore].any()
  if kind == "empty":
    assert loss == 0.0 and not d.any()


def test_dice_reference_statistics():
  V = 4
  l, y, w, ignore = _case("out_of_range", V, seed=2)
  I, P, Y = R.dice_stats(l, y, V, w, ignore)
  ok = (y >= 0) & (y < V)
  assert float(P.sum()) == pytest.approx(len(y), rel=1e-12)      # every pixel adds to P_c
  assert torch.equal(Y, torch.bincount(y[ok], minlength=V).double())
  assert float(I.sum()) <= float(Y.sum())


# ----------------------------------------------------------------------------- validation
BAD = [
    {"loss": "tversky"}, {"loss": None}, {"loss": 1},
    {"loss": "focal", "focal_gamma": float("nan")}, {"loss": "focal", "focal_gamma": -0.5},
    {"loss": "focal", "focal_gamma": float("inf")}, {"loss": "focal", "focal_gamma": True},
    {"loss": "focal", "focal_gamma": "2"},
    {"loss": "dice", "dice_smooth": 0.0}, {"loss": "dice", "dice_smooth": -1e-5},
    {"loss": "dice_ce", "dice_smooth": float("nan")}, {"loss": "dice", "dice_smooth": float("inf")},
    {"focal_gamma": 1.0}, {"loss": "dice", "focal_gamma": 1.0},
    {"dice_smooth": 1.0}, {"loss": "focal", "dice_smooth": 1.0},
]


@pytest.mark.parametrize("kw", BAD, ids=[repr(k) for k in BAD])
@pytest.mark.parametrize("training", [True, False])
def test_bad_loss_raises_before_any_allocation(kw, training, monkeypatch):
  from tensorflowonspark_b200.models import unet

  def no_alloc(*a, **k):
    raise AssertionError("allocated before validating its arguments")
  monkeypatch.setattr(unet, "_buf", no_alloc)
  monkeypatch.setattr(unet, "MobileNetV2Encoder", no_alloc)
  monkeypatch.setattr(torch, "zeros", no_alloc)
  with pytest.raises(ValueError):
    unet.UNetTrainer(batch=2, device="cuda:0", classes=3, training=training, **kw)


@pytest.mark.parametrize("loss", ["focal", "dice", "dice_ce"])
def test_inference_only_trainer_takes_only_the_default_loss(loss, monkeypatch):
  from tensorflowonspark_b200.models import unet

  def no_alloc(*a, **k):
    raise AssertionError("allocated before validating its arguments")
  monkeypatch.setattr(unet, "_buf", no_alloc)
  monkeypatch.setattr(unet, "MobileNetV2Encoder", no_alloc)
  with pytest.raises(ValueError, match="training=True"):
    unet.UNetTrainer(batch=2, device="cuda:0", classes=3, training=False, loss=loss)
  # the defaults, spelled out, are accepted
  assert unet._loss_args("cross_entropy", 2, 1e-5, False, unet.UNetTrainer.LOSS_DEFAULTS) == \
      ("cross_entropy", 2.0, 1e-5)


def test_good_loss_arguments_are_normalised():
  from tensorflowonspark_b200.models import unet
  d = unet.UNetTrainer.LOSS_DEFAULTS
  assert d == ("cross_entropy", 2.0, 1e-5)
  assert unet._loss_args("focal", 0, 1e-5, True, d) == ("focal", 0.0, 1e-5)
  assert unet._loss_args("dice_ce", 2.0, 1, True, d) == ("dice_ce", 2.0, 1.0)
  assert unet._loss_args("focal", 0.5, 1e-5, True, d) == ("focal", 0.5, 1e-5)
  assert set(unet.LOSSES) == {"cross_entropy", "focal", "dice", "dice_ce"}


# ----------------------------------------------------------------------------- examples
drivers = ft.drivers


def test_segmentation_loss_flags_reach_the_trainer(drivers):
  drivers.seg.train(ft._seg_args(drivers.seg))
  kw = ft._Trainer.made[-1].kw
  assert not {"loss", "focal_gamma", "dice_smooth"} & set(kw)
  drivers.seg.train(ft._seg_args(drivers.seg, "--loss", "focal", "--focal_gamma", "0.5"))
  kw = ft._Trainer.made[-1].kw
  assert kw["loss"] == "focal" and kw["focal_gamma"] == 0.5 and "dice_smooth" not in kw


def test_segmentation_trainer_kwargs_give_the_loss_names_only_when_set(monkeypatch):
  monkeypatch.syspath_prepend(os.path.join(uc.ROOT, "examples", "segmentation"))
  sys.modules.pop("segmentation", None)
  try:
    import segmentation
    a = segmentation.define_flags().parse_args([])
    assert a.loss is None and a.focal_gamma is None and a.dice_smooth is None
    assert segmentation.trainer_kwargs(a) == {}
    a = segmentation.define_flags().parse_args(["--loss", "dice_ce", "--dice_smooth", "1"])
    assert segmentation.trainer_kwargs(a) == {"loss": "dice_ce", "dice_smooth": 1.0}
    with pytest.raises(SystemExit):
      segmentation.define_flags().parse_args(["--loss", "lovasz"])
  finally:
    sys.modules.pop("segmentation", None)


def test_segmentation_spark_passes_the_loss(drivers):
  class Args(object):
    batch_size, learning_rate, input_mode, steps, epochs, num_examples = 2, 1e-3, "tf", 2, 1, 8

  drivers.spark.main_fun(Args(), ft._Ctx())
  kw = ft._Trainer.made[-1].kw
  assert not {"loss", "focal_gamma", "dice_smooth"} & set(kw)
  Args.loss, Args.dice_smooth = "dice", 0.5
  drivers.spark.main_fun(Args(), ft._Ctx())
  kw = ft._Trainer.made[-1].kw
  assert kw["loss"] == "dice" and kw["dice_smooth"] == 0.5 and "focal_gamma" not in kw
  a = drivers.spark.define_flags().parse_args(["--loss", "focal", "--focal_gamma", "3"])
  assert (a.loss, a.focal_gamma, a.dice_smooth) == ("focal", 3.0, None)


# ----------------------------------------------------------------------------- kernel resources
@pytest.mark.skipif(not os.path.exists(uc.NVCC), reason="nvcc not found")
@pytest.mark.parametrize("kernel,instances", [("seg_dice_stats_kernel", 6),
                                              ("seg_loss_grad_kernel", 12)])
def test_loss_kernels_have_no_stack_frame_or_spills(kernel, instances, tmp_path):
  # seg_dice_stats: G = 1 (8 channels), 2, 4, 8, 16, 32; seg_loss_grad: those G x kOpt
  kernels = {k: v for k, v in uc._ptxas("elementwise.cu", tmp_path).items() if kernel in k}
  assert len(kernels) == instances, sorted(kernels)
  bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
  assert not bad, "stack frame / spill stores / spill loads (bytes): {}".format(bad)

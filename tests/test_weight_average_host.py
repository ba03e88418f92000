"""Weight averaging (``ema_decay``), host side (no GPU): the argument checks of the three trainers,
the example flags, the exportable ``averaged()`` views, loading optimizer states written without an
average, and the float64 reference recurrence (with its error bound) that the GPU tests compare
the fused kernels against."""
import importlib
import math
import os
import sys

import numpy as np
import pytest
import torch

from tensorflowonspark_b200.models import engine, resnet, unet
from tensorflowonspark_b200.parallel import fused_optim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_example_drivers_dryrun as dry  # noqa: E402
from test_example_drivers_dryrun import fake_gpu  # noqa: E402,F401  (fixture)
from test_resnet_head_host import cpu_plans  # noqa: E402,F401  (fixture)


# ------------------------------------------------------------------ the reference
def ema_reference(masters, d):
  """float64 average after each update of the fp32 ``masters`` (one tensor per update, the
  master just written): Keras's rule, avg_1 = w_1, avg_n = d avg_(n-1) + (1 - d) w_n, with d
  rounded to fp32 as the kernel reads it from the hyper-parameter vector."""
  d = float(np.float32(d))
  out, avg = [], None
  for w in masters:
    w = w.double()
    avg = w.clone() if avg is None else d * avg + (1.0 - d) * w
    out.append(avg)
  return out


def ema_bound(masters, d):
  """Per-element bound on |fp32 average - float64 reference| after the last of ``masters``, for
  every d in [0, 1).  The kernel computes fmaf(d, avg, fl(om * w)) with om = fl(1 - d).  With
  M = max_k |w_k| (the average is a convex combination of the masters, so |avg| <= M too),
  update k >= 2 adds at most 2^-24 (1 - d) M from rounding 1 - d (0 when d = 0 or d >= 0.5, where
  1 - d is exact), 2^-24 (1 - d) M from rounding om * w and 2^-24 M from the fma, and decays the
  error it inherits by d; update 1 is an exact copy.  After n updates the error is therefore at
  most 2^-24 M (3 - 2 d) (1 + d + ... + d^(n-2)).  (A tiny term covers the float64 reference's
  own rounding.)"""
  n = len(masters)
  m = torch.stack([w.double().abs() for w in masters]).amax(0)
  d = float(np.float32(d))
  geo = sum(d ** k for k in range(n - 1))
  return 2.0 ** -24 * m * (3.0 - 2.0 * d) * geo + (2.0 ** -50 * m if n > 1 else 0.0)


def _fma32(a, b, c):
  """fp32 fma emulated in float64 (exact product; one rounding of the sum, then to fp32)."""
  return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def _kernel_emulation(masters, d):
  """The kernel's fp32 arithmetic on the host."""
  d32 = np.float32(d)
  om = np.float32(1.0) - d32
  avg = None
  for w in masters:
    w = w.numpy().astype(np.float32)
    avg = w.copy() if avg is None else _fma32(np.full_like(w, d32), avg, (om * w).astype(np.float32))
  return torch.from_numpy(avg)


@pytest.mark.parametrize("d", [0.0, 0.1, 0.3, 0.5, 0.9, 0.999])
def test_reference_matches_the_closed_form_and_bounds_the_fp32_recurrence(d):
  gen = torch.Generator().manual_seed(3)
  masters = [(torch.randn(4096, generator=gen) * (1 + k)).float() for k in range(20)]
  ref = ema_reference(masters, d)
  assert torch.equal(ref[0], masters[0].double())                       # update 1 copies
  d64 = float(np.float32(d))
  closed = d64 ** 19 * masters[0].double() + sum(
      (1 - d64) * d64 ** (19 - k) * masters[k].double() for k in range(1, 20))
  assert torch.allclose(ref[-1], closed, rtol=1e-12, atol=1e-12)
  got = _kernel_emulation(masters, d).double()
  err = (got - ref[-1]).abs()
  assert bool((err <= ema_bound(masters, d)).all())
  if d == 0.0:
    assert torch.equal(got.float(), masters[-1])                        # d = 0 is the master


def test_bound_is_zero_after_one_update_and_grows_with_the_steps():
  w = [torch.ones(3)]
  assert float(ema_bound(w, 0.9).max()) == 0.0
  assert float(ema_bound(w * 3, 0.9).max()) == pytest.approx(2.0 ** -24 * 1.2 * 1.9, rel=1e-6)


# ------------------------------------------------------------------ argument checks
class _Allocated(Exception):
  pass


@pytest.fixture
def no_alloc(monkeypatch):
  """Building a parameter store is the first allocation of every trainer: make it fail loudly."""
  def boom(*a, **k):
    raise _Allocated()
  monkeypatch.setattr(resnet, "ParamStore", boom)
  monkeypatch.setattr(unet, "ParamStore", boom)


BAD = [True, False, float("nan"), -0.1, 1.0, 1.5, math.inf, "0.9", [0.9]]


def _make(trainer, **kw):
  if trainer == "UNetTrainer":
    return unet.UNetTrainer(device="cpu", **kw)
  return getattr(resnet, trainer)(device="cpu", **kw)


@pytest.mark.parametrize("trainer", ["ResNetTrainer", "CifarResNetTrainer", "UNetTrainer"])
@pytest.mark.parametrize("d", BAD, ids=repr)
def test_bad_ema_decay_raises_before_allocation(no_alloc, trainer, d):
  with pytest.raises(ValueError, match="ema_decay"):
    _make(trainer, ema_decay=d)


@pytest.mark.parametrize("trainer", ["ResNetTrainer", "UNetTrainer"])
def test_ema_decay_needs_training(no_alloc, trainer):
  with pytest.raises(ValueError, match="ema_decay needs training=True"):
    _make(trainer, ema_decay=0.9, training=False)
  with pytest.raises(_Allocated):                 # None is fine without training
    _make(trainer, ema_decay=None, training=False)


@pytest.mark.parametrize("trainer", ["ResNetTrainer", "CifarResNetTrainer", "UNetTrainer"])
@pytest.mark.parametrize("d", [0, 0.0, 0.5, 0.999, np.float32(0.9)], ids=repr)
def test_good_ema_decay_passes_the_checks(no_alloc, trainer, d):
  with pytest.raises(_Allocated):
    _make(trainer, ema_decay=d)


def test_optimizer_checks_the_decay_too():
  from tensorflowonspark_b200.models.engine import ParamStore, constant
  st = ParamStore()
  st.register("w", (16,), True, constant(1.0))
  st.finalize(torch.device("cpu"))
  for d in (True, 1.0, -1e-9, float("nan")):
    with pytest.raises(ValueError, match="ema_decay"):
      fused_optim.FusedOptimizer(st, ema_decay=d)
  opt = fused_optim.FusedOptimizer(st, ema_decay=0.9)
  assert opt.ema.shape == (st.total,) and len(opt.hyper) == fused_optim.HYPER_EMA
  assert float(opt.hyper[8]) == pytest.approx(0.9) and opt.average_count() == 0
  plain = fused_optim.FusedOptimizer(st)
  assert plain.ema is None and len(plain.hyper) == fused_optim.HYPER
  assert "ema" not in plain._args[0] and opt._args[0]["ema"] == opt.ema.data_ptr()
  with pytest.raises(RuntimeError, match="no weight average"):
    plain.averaged_weights()


# ------------------------------------------------------------------ optimizer state
def _cpu_opt(**kw):
  from tensorflowonspark_b200.models.engine import ParamStore, normal
  st = ParamStore()
  st.register("w", (40,), True, normal(0.1))
  st.register("b", (8,), False, normal(0.1))
  st.finalize(torch.device("cpu"), seed=2)
  return fused_optim.FusedOptimizer(st, **kw)


@pytest.mark.parametrize("opt", ["sgd", "momentum", "adam", "lars"])
def test_an_eight_entry_hyper_from_an_old_checkpoint_loads(opt):
  old = _cpu_opt(opt=opt, lr=0.3).state_dict()
  assert len(old["hyper"]) == 8 and "ema" not in old
  new = _cpu_opt(opt=opt, lr=0.1, ema_decay=0.99)
  new.hyper[9] = 5.0
  new.load_state_dict(old)
  assert float(new.hyper[0]) == pytest.approx(0.3)
  assert float(new.hyper[8]) == pytest.approx(0.99) and new.average_count() == 0   # reset
  # and the other way round: an averaged optimizer's state into one without an average
  src = _cpu_opt(opt=opt, lr=0.7, ema_decay=0.9)
  src.hyper[9] = 3.0
  sd = src.state_dict()
  assert len(sd["hyper"]) == 10 and sd["ema_count"] == 3 and sd["ema"].shape == (src.store.total,)
  plain = _cpu_opt(opt=opt)
  plain.load_state_dict(sd)
  assert len(plain.hyper) == 8 and float(plain.hyper[0]) == pytest.approx(0.7)
  again = _cpu_opt(opt=opt, ema_decay=0.5)
  sd["ema"] = torch.arange(src.store.total, dtype=torch.float32)
  again.load_state_dict(sd)
  assert again.average_count() == 3 and torch.equal(again.ema, sd["ema"])
  assert float(again.hyper[8]) == pytest.approx(0.5)          # the decay stays the optimizer's


# ------------------------------------------------------------------ averaged() views
def test_resnet_views_carry_the_export_attributes(cpu_plans):
  net = resnet.ResNetTrainer(depth=50, batch=2, image=32, num_classes=37, device="cpu",
                             ema_decay=0.9)
  view = net.averaged()
  assert view.export_builder == net.export_builder == "tensorflowonspark_b200.models.resnet:build_served"
  assert view.export_builder_args == {"depth": 50, "image": 32, "num_classes": 37}
  assert view.export_signatures == net.export_signatures
  sd, live = view.state_dict(), net.state_dict()
  assert set(sd) == set(live)
  for k in live:                       # no update yet: the average is the current parameters
    assert torch.equal(sd[k], live[k]), k
  with pytest.raises(RuntimeError, match="no weight average"):
    resnet.ResNetTrainer(depth=50, batch=2, image=32, device="cpu").averaged()


def test_cifar_view_and_reset(cpu_plans):
  net = resnet.CifarResNetTrainer(depth=20, batch=1, device="cpu", ema_decay=0.5)
  assert net.averaged().export_builder is None and net.optim.ema is not None
  net.optim.hyper[9] = 4.0
  net.load_state_dict(net.state_dict())        # a parameter-only load resets the average
  assert net.optim.average_count() == 0
  net.optim.hyper[9] = 4.0
  net.load_backbone(net.state_dict())
  assert net.optim.average_count() == 0
  with pytest.raises(RuntimeError, match="no weight average"):
    resnet.CifarResNetTrainer(depth=20, batch=1, device="cpu").eval_begin(averaged=True)


# ------------------------------------------------------------------ example flags
def test_resnet_spark_ema_flag(fake_gpu, tmp_path):
  mod = importlib.import_module("resnet_spark")
  assert mod.parse([]).ema_decay is None
  base = ["resnet_spark.py", "--batch_size", "8", "--image", "64", "--train_steps", "2",
          "--metrics_port", "0"]
  mod.main_fun(base, dry._Ctx())
  assert "ema_decay" not in dry._Trainer.made[-1].kw
  mod.main_fun(base + ["--ema_decay", "0.99"], dry._Ctx())
  assert dry._Trainer.made[-1].kw["ema_decay"] == 0.99


def test_resnet_cifar_ema_flag(fake_gpu):
  mod = importlib.import_module("resnet_cifar_main")
  assert mod.define_flags().parse_args([]).ema_decay is None
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "2"], mod.LocalContext())
  assert "ema_decay" not in dry._Trainer.made[-1].kw
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "2", "--ema_decay", "0.9"],
               mod.LocalContext())
  assert dry._Trainer.made[-1].kw["ema_decay"] == 0.9


@pytest.mark.parametrize("name", ["segmentation", "segmentation_dist", "segmentation_spark"])
def test_segmentation_examples_take_the_ema_flag(name):
  path = os.path.join(ROOT, "examples", "segmentation")
  sys.path.insert(0, path)
  try:
    sys.modules.pop(name, None)
    mod = importlib.import_module(name)
    # (segmentation_dist parses segmentation.py's flags)
    parser = (mod.segmentation if name == "segmentation_dist" else mod).define_flags()
    assert parser.parse_args([]).ema_decay is None
    assert parser.parse_args(["--ema_decay", "0.95"]).ema_decay == 0.95
    assert "live" in parser.format_help()       # the help says what model_dir serves
  finally:
    sys.path.remove(path)
    sys.modules.pop(name, None)

"""Gradient clipping by global norm (``clip_norm``), host side (no GPU): the argument checks of the
optimizer and the three trainers, the example flags, the float64 reference that the GPU tests
compare the fused kernels against (checked here against ``torch.nn.utils.clip_grad_norm_``
followed by ``torch.optim``), and the ptxas report of the new kernels."""
import importlib
import math
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from tensorflowonspark_b200 import _build
from tensorflowonspark_b200.models import resnet, unet
from tensorflowonspark_b200.parallel import fused_optim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_example_drivers_dryrun as dry  # noqa: E402
from test_example_drivers_dryrun import fake_gpu  # noqa: E402,F401  (fixture)

NVCC = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin",
                                            "nvcc")


# ------------------------------------------------------------------ the reference
def clip_coef(gsum, scale, c):
  """(N, coefficient, clipped scale) of the kernels' rule in float64: N = ||scale * gsum||,
  coef = c / (N + 1e-6) clamped to at most 1 (NaN stays NaN, inf gives 0), and the scale the
  update kernels read, fl32(scale * coef)."""
  s = float(np.float32(scale))
  norm = math.sqrt(float((gsum.double() ** 2).sum())) * abs(s)
  q = c / (norm + 1e-6) if not math.isnan(norm) else float("nan")
  coef = 1.0 if q >= 1.0 else q
  return norm, coef, float(np.float32(s * coef))


def step_reference(opt, w, gsum, state, hyper, decay_end, c, lars_bounds=None):
  """One clipped update in float64.  ``w`` master, ``gsum`` the unscaled gradient sum (float64
  or fp32 tensors), ``state`` {"state1", "state2"} (updated in place, float64), ``hyper`` the
  fp32 vector the step reads (Adam's step already counted).  Returns (new w, N, coef)."""
  h = [float(x) for x in hyper]
  lr, mom, wd, scale, b1, b2, eps, t = h[:8]
  norm, coef, s = clip_coef(gsum, scale, c)
  w = w.double()
  g = gsum.double() * s
  dec = torch.zeros_like(w, dtype=torch.bool)
  dec[:decay_end] = True
  if opt == "lars":
    v = state["state1"]
    lrt = torch.full_like(w, lr)
    for t0, t1 in zip(lars_bounds[:-1], lars_bounds[1:]):
      gn = math.sqrt(float((gsum[t0:t1].double() ** 2).sum())) * abs(s)
      wn = math.sqrt(float((w[t0:t1] ** 2).sum()))
      trust = b1 * wn / (gn + wd * wn) if (wn > 0 and gn > 0) else 1.0
      lrt[t0:t1] = lr * trust
    v.copy_(torch.where(dec, mom * v + lrt * (g + wd * w), mom * v + lr * g))
    return w - v, norm, coef
  g = torch.where(dec, g + wd * w, g)
  if opt == "sgd":
    return w - lr * g, norm, coef
  if opt == "momentum":
    m = state["state1"]
    m.copy_(mom * m + g)
    return w - lr * m, norm, coef
  m, v = state["state1"], state["state2"]
  m.copy_(b1 * m + (1 - b1) * g)
  v.copy_(b2 * v + (1 - b2) * g * g)
  c1, c2 = 1 - b1 ** t, 1 - b2 ** t
  return w - lr * (m / c1) / (torch.sqrt(v / c2) + eps), norm, coef


@pytest.mark.parametrize("opt", ["momentum", "adam"])
@pytest.mark.parametrize("frac", [0.1, 0.5, 2.0, math.inf])
def test_reference_matches_torch_clip_then_optimizer(opt, frac):
  """clip_grad_norm_ then torch.optim.SGD(momentum) / Adam in float64, several steps.  Scale 1
  (the gradient is already the average) keeps fl32(scale * coef) within 2^-24 of coef."""
  gen = torch.Generator().manual_seed(3)
  n, decay_end = 300, 300           # torch's weight decay covers every element
  w0 = torch.randn(n, generator=gen, dtype=torch.float64)
  grads = [torch.randn(n, generator=gen, dtype=torch.float64) * 0.3 for _ in range(4)]
  lr, wd = (0.05, 1e-3) if opt == "momentum" else (1e-2, 1e-3)
  p = torch.nn.Parameter(w0.clone())
  tor = (torch.optim.SGD([p], lr=lr, momentum=0.9, weight_decay=wd) if opt == "momentum"
         else torch.optim.Adam([p], lr=lr, betas=(0.9, 0.999), eps=1e-7, weight_decay=wd))
  w = w0.clone()
  state = {"state1": torch.zeros(n, dtype=torch.float64), "state2": torch.zeros(n, dtype=torch.float64)}
  for k, g in enumerate(grads):
    c = frac * float(g.norm())
    p.grad = g.clone()
    total = torch.nn.utils.clip_grad_norm_([p], max_norm=c)
    tor.step()
    hyper = [lr, 0.9, wd, 1.0, 0.9, 0.999, 1e-7, k + 1]
    w, norm, coef = step_reference(opt, w, g, state, hyper, decay_end, c)
    assert norm == pytest.approx(float(total), rel=1e-12)
    assert (coef == 1.0) == (frac >= 1.0)
    assert torch.allclose(w, p.detach(), rtol=1e-6, atol=1e-9), k


def test_reference_coefficient_edge_cases():
  g = torch.tensor([3.0, 4.0])
  assert clip_coef(g, 1.0, 5.0 + 1e-6)[1] == 1.0            # threshold reached exactly: 1
  assert clip_coef(g, 1.0, math.inf)[1] == 1.0
  assert clip_coef(g, 1.0, 2.5)[1] == pytest.approx(0.5, rel=1e-6)
  assert clip_coef(g, 0.5, 2.5)[0] == pytest.approx(2.5)    # the norm is of the scaled gradient
  assert math.isnan(clip_coef(torch.tensor([float("nan"), 1.0]), 1.0, 1.0)[1])
  assert clip_coef(torch.tensor([float("inf"), 1.0]), 1.0, 1.0)[1] == 0.0
  # torch agrees on both
  for bad, want in ((float("nan"), math.isnan), (float("inf"), lambda x: x == 0.0)):
    p = torch.nn.Parameter(torch.ones(2))
    p.grad = torch.tensor([bad, 1.0])
    torch.nn.utils.clip_grad_norm_([p], max_norm=1.0)
    assert want(float(p.grad[1]))


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


BAD = [True, False, float("nan"), 0, 0.0, -1.0, -math.inf, "1.0", [1.0]]


def _make(trainer, **kw):
  if trainer == "UNetTrainer":
    return unet.UNetTrainer(device="cpu", **kw)
  return getattr(resnet, trainer)(device="cpu", **kw)


@pytest.mark.parametrize("trainer", ["ResNetTrainer", "CifarResNetTrainer", "UNetTrainer"])
@pytest.mark.parametrize("c", BAD, ids=repr)
def test_bad_clip_norm_raises_before_allocation(no_alloc, trainer, c):
  with pytest.raises(ValueError, match="clip_norm"):
    _make(trainer, clip_norm=c)


@pytest.mark.parametrize("trainer", ["ResNetTrainer", "CifarResNetTrainer", "UNetTrainer"])
@pytest.mark.parametrize("c", [1, 0.5, 1e-30, math.inf, np.float32(2.0)], ids=repr)
def test_good_clip_norm_passes_the_checks(no_alloc, trainer, c):
  with pytest.raises(_Allocated):
    _make(trainer, clip_norm=c)


@pytest.mark.parametrize("trainer", ["ResNetTrainer", "UNetTrainer"])
def test_clip_norm_needs_training(no_alloc, trainer):
  with pytest.raises(ValueError, match="clip_norm needs training=True"):
    _make(trainer, clip_norm=1.0, training=False)
  with pytest.raises(_Allocated):                 # None is fine without training
    _make(trainer, clip_norm=None, training=False)


def _cpu_store():
  from tensorflowonspark_b200.models.engine import ParamStore, normal
  st = ParamStore()
  st.register("w", (40,), True, normal(0.1))
  st.register("b", (8,), False, normal(0.1))
  st.finalize(torch.device("cpu"), seed=2)
  return st


def test_optimizer_checks_the_threshold():
  st = _cpu_store()
  for c in BAD:
    with pytest.raises(ValueError, match="clip_norm"):
      fused_optim.FusedOptimizer(st, clip_norm=c)
  assert fused_optim.check_clip_norm(None) is None
  assert fused_optim.check_clip_norm(3) == 3.0 and isinstance(fused_optim.check_clip_norm(3), float)


@pytest.mark.parametrize("opt", ["sgd", "momentum", "adam", "lars"])
def test_optimizer_layout_and_state_dict_are_unchanged(opt):
  plain = fused_optim.FusedOptimizer(_cpu_store(), opt=opt, ema_decay=0.9)
  clip = fused_optim.FusedOptimizer(_cpu_store(), opt=opt, ema_decay=0.9, clip_norm=1.0)
  assert plain.grad_norm is None and clip.grad_norm.shape == (1,)
  # the default launches get the same arguments (no clipping keys)
  assert [sorted(d) for d in plain._args] == [sorted(d) for d in clip._args]
  # the updates read the per-step copy of hyper; the saved state is the same as without clipping
  assert all(d["hyper"] == clip.hyper_step.data_ptr() for d in clip._clip_update)
  a, b = plain.state_dict(), clip.state_dict()
  assert set(a) == set(b) and all(torch.equal(torch.as_tensor(a[k]), torch.as_tensor(b[k])) for k in a)
  clip.load_state_dict(a)


def test_one_bucket_of_several_cannot_step_alone():
  st = _cpu_store()
  o = fused_optim.FusedOptimizer(st, buckets=[(0, 40, "a"), (40, st.total, "b")], clip_norm=1.0)
  with pytest.raises(ValueError, match="every bucket"):
    o.step(0)


# ------------------------------------------------------------------ example flags
def test_resnet_spark_clip_flag(fake_gpu):
  mod = importlib.import_module("resnet_spark")
  assert mod.parse([]).clip_norm is None
  base = ["resnet_spark.py", "--batch_size", "8", "--image", "64", "--train_steps", "2",
          "--metrics_port", "0"]
  mod.main_fun(base, dry._Ctx())
  assert "clip_norm" not in dry._Trainer.made[-1].kw
  mod.main_fun(base + ["--clip_norm", "1.5"], dry._Ctx())
  assert dry._Trainer.made[-1].kw["clip_norm"] == 1.5


def test_resnet_cifar_clip_flag(fake_gpu, monkeypatch, capsys):
  monkeypatch.setattr(dry._Trainer, "grad_norm", torch.tensor([2.5]), raising=False)
  mod = importlib.import_module("resnet_cifar_main")
  assert mod.define_flags().parse_args([]).clip_norm is None
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "2"], mod.LocalContext())
  assert "clip_norm" not in dry._Trainer.made[-1].kw
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "2", "--clip_norm", "inf"],
               mod.LocalContext())
  assert dry._Trainer.made[-1].kw["clip_norm"] == math.inf
  assert "grad_norm 2.5000" in capsys.readouterr().out     # printed next to the loss


@pytest.mark.parametrize("name", ["segmentation", "segmentation_spark"])
def test_segmentation_examples_take_the_clip_flag(name):
  path = os.path.join(ROOT, "examples", "segmentation")
  sys.path.insert(0, path)
  try:
    sys.modules.pop(name, None)
    mod = importlib.import_module(name)
    parser = mod.define_flags()
    assert parser.parse_args([]).clip_norm is None
    assert parser.parse_args(["--clip_norm", "0.5"]).clip_norm == 0.5
    if name == "segmentation":
      assert "clip_norm" not in mod.trainer_kwargs(parser.parse_args([]))
      assert mod.trainer_kwargs(parser.parse_args(["--clip_norm", "2"])) == {"clip_norm": 2.0}
  finally:
    sys.path.remove(path)


# ------------------------------------------------------------------ kernel resources
NEW_KERNELS = ("allreduce_opt_kernelILi0ELb0ELi3ELb0E", "allreduce_opt_kernelILi0ELb1ELi3ELb0E",
               "grad_sumsq_kernel", "clip_finalize_kernel")


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not found")
def test_clip_kernels_have_no_stack_frame_or_spills(tmp_path):
  out = tmp_path / "optim_comm.o"
  cmd = [NVCC] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", _build.CSRC_DIR, "-c",
                                      os.path.join(_build.CSRC_DIR, "optim_comm.cu"), "-o", str(out)]
  r = subprocess.run(cmd, capture_output=True, text=True)
  assert r.returncode == 0, r.stderr[-4000:]
  kernels, cur = {}, None
  for line in r.stderr.splitlines():
    m = re.search(r"Compiling entry function '(\S+)'", line)
    if m:
      cur = m.group(1)
      continue
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
    if m and cur is not None:
      kernels[cur] = tuple(int(x) for x in m.groups())
  for k in NEW_KERNELS:
    hit = {n: v for n, v in kernels.items() if k in n}
    assert len(hit) == 1, (k, sorted(kernels))
    assert list(hit.values()) == [(0, 0, 0)], hit

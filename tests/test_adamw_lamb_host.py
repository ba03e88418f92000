"""AdamW and LAMB, host side (no GPU): the float64 references the GPU tests compare the fused
kernels against (AdamW checked against ``torch.optim.AdamW``, also after ``clip_grad_norm_``; LAMB
against a case worked out by hand), the argument checks of the three trainers, the example flags
and the ptxas report of the new kernel instances."""
import importlib
import inspect
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
def adam_family_reference(opt, w, g_sum, m, v, hyper, decay_end, bounds=None, scale=None):
  """One adamw | lamb step in float64.  ``w`` the master before the step, ``g_sum`` the unscaled
  gradient sum, ``m`` / ``v`` the moments before the step, ``hyper`` the vector the step reads
  (its step t already counted), ``bounds`` the adapted tensors [bounds[k], bounds[k + 1]) tiling
  [0, decay_end) (LAMB), ``scale`` the gradient scale when it is not hyper[3] (clipping).
  Returns (w, m, v)."""
  h = [float(x) for x in hyper]
  lr, _, wd, s, b1, b2, eps, t = h[:8]
  s = s if scale is None else float(scale)
  w, m, v = w.double().clone(), m.double().clone(), v.double().clone()
  g = g_sum.double() * s
  m = b1 * m + (1 - b1) * g
  v = b2 * v + (1 - b2) * g * g
  u = (m / (1 - b1 ** t)) / (torch.sqrt(v / (1 - b2 ** t)) + eps)
  dec = torch.zeros_like(w, dtype=torch.bool)
  dec[:decay_end] = True
  if opt == "adamw":
    w = torch.where(dec, w * (1 - lr * wd), w)
    return w - lr * u, m, v
  assert opt == "lamb"
  r = torch.where(dec, u + wd * w, u)
  ratio = torch.ones_like(w)
  for t0, t1 in zip(bounds[:-1], bounds[1:]):
    wn, rn = float(w[t0:t1].norm()), float(r[t0:t1].norm())
    ratio[t0:t1] = wn / rn if (wn > 0 and rn > 0) else 1.0
  return w - lr * ratio * r, m, v


@pytest.mark.parametrize("frac", [None, 0.3, math.inf])
def test_adamw_reference_matches_torch(frac):
  """torch.optim.AdamW in float64 over several steps, two parameter groups (the decayed head with
  wd, the tail with 0); ``frac``: clip_grad_norm_ to frac * |g| first (scale = clipped coef)."""
  gen = torch.Generator().manual_seed(7)
  n, decay_end = 300, 200
  w0 = torch.randn(n, generator=gen, dtype=torch.float64)
  grads = [torch.randn(n, generator=gen, dtype=torch.float64) * 0.3 for _ in range(5)]
  lr, wd, b1, b2, eps = 1e-2, 0.05, 0.9, 0.99, 1e-7
  head = torch.nn.Parameter(w0[:decay_end].clone())
  tail = torch.nn.Parameter(w0[decay_end:].clone())
  tor = torch.optim.AdamW([{"params": [head], "weight_decay": wd},
                           {"params": [tail], "weight_decay": 0.0}],
                          lr=lr, betas=(b1, b2), eps=eps)
  w, m, v = w0.clone(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
  for k, g in enumerate(grads):
    head.grad, tail.grad = g[:decay_end].clone(), g[decay_end:].clone()
    scale = 1.0
    if frac is not None:
      c = frac * float(g.norm())
      total = float(torch.nn.utils.clip_grad_norm_([head, tail], max_norm=c))
      q = c / (total + 1e-6)
      scale = 1.0 if q >= 1.0 else q
    tor.step()
    hyper = [lr, 0.9, wd, 1.0, b1, b2, eps, k + 1]
    w, m, v = adam_family_reference("adamw", w, g, m, v, hyper, decay_end, scale=scale)
    got = torch.cat([head.detach(), tail.detach()])
    assert torch.allclose(w, got, rtol=1e-12, atol=1e-14), k


def test_adamw_with_zero_decay_is_adam():
  gen = torch.Generator().manual_seed(1)
  w, g = torch.randn(50, generator=gen), torch.randn(50, generator=gen)
  p = torch.nn.Parameter(w.double().clone())
  p.grad = g.double().clone()
  torch.optim.Adam([p], lr=0.1, betas=(0.9, 0.999), eps=1e-7).step()
  z = torch.zeros(50, dtype=torch.float64)
  got, _, _ = adam_family_reference("adamw", w, g, z, z, [0.1, 0, 0.0, 1, 0.9, 0.999, 1e-7, 1], 50)
  assert torch.allclose(got, p.detach(), rtol=1e-14, atol=0)


def test_lamb_reference_hand_worked_case():
  """Step 1 (t = 1, beta1 = 0.5, beta2 = 0.75, eps = 0): m / c1 = g and v / c2 = g^2, so the Adam
  direction is sign(g).  Tensors: A = [3, 4] (|w| = 5), g = [1, -2] -> r = [1 + 3 wd, -1 + 4 wd];
  B = [0, 0] (|w| = 0: ratio 1), g = [1, 1] -> r = [1, 1]; C = [1, 0] with g = 0 and wd = 0
  (a second run) -> r = 0: ratio 1, no change; tail D = [2] (never decayed or adapted), g = -1."""
  hyper = [0.1, 0.0, 0.5, 1.0, 0.5, 0.75, 0.0, 1.0]       # lr, -, wd, scale, b1, b2, eps, t
  w = torch.tensor([3.0, 4.0, 0.0, 0.0, 2.0], dtype=torch.float64)
  g = torch.tensor([1.0, -2.0, 1.0, 1.0, -1.0], dtype=torch.float64)
  z = torch.zeros(5, dtype=torch.float64)
  got, m, v = adam_family_reference("lamb", w, g, z, z, hyper, 4, bounds=[0, 2, 4])
  # A: r = [2.5, 1.0], |r| = sqrt(7.25), ratio = 5 / sqrt(7.25)
  ra = 5.0 / math.sqrt(7.25)
  want = [3.0 - 0.1 * ra * 2.5, 4.0 - 0.1 * ra * 1.0,
          -0.1, -0.1,                                   # B: ratio 1, r = [1, 1] (wd * 0 = 0)
          2.0 + 0.1]                                    # D: r = sign(-1) = -1
  assert torch.allclose(got, torch.tensor(want, dtype=torch.float64), rtol=1e-15, atol=1e-15)
  assert torch.allclose(m, 0.5 * g) and torch.allclose(v, 0.25 * g * g)
  # r = 0 on a whole tensor (zero gradient, no decay): ratio 1 and the tensor does not move
  hyper0 = list(hyper)
  hyper0[2], hyper0[6] = 0.0, 1e-8        # (eps > 0: 0 / 0 would be NaN)
  w2 = torch.tensor([1.0, 0.0, 3.0, 4.0], dtype=torch.float64)
  g2 = torch.tensor([0.0, 0.0, 1.0, -1.0], dtype=torch.float64)
  z4 = torch.zeros(4, dtype=torch.float64)
  got2, _, _ = adam_family_reference("lamb", w2, g2, z4, z4, hyper0, 4, bounds=[0, 2, 4])
  # second tensor: r = [u, -u] with u = 1 / (1 + eps), |w| = 5: ratio * r = 5 / sqrt(2) [1, -1]
  r2 = 5.0 / math.sqrt(2.0)
  want2 = [1.0, 0.0, 3.0 - 0.1 * r2, 4.0 + 0.1 * r2]
  assert torch.allclose(got2, torch.tensor(want2, dtype=torch.float64), rtol=1e-13, atol=0)


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


def _make(trainer, **kw):
  if trainer == "UNetTrainer":
    return unet.UNetTrainer(device="cpu", **kw)
  return getattr(resnet, trainer)(device="cpu", **kw)


TRAINERS = ["ResNetTrainer", "CifarResNetTrainer", "UNetTrainer"]
BAD_BETA = [True, -0.1, 1.0, 1.5, float("nan"), math.inf, "0.9", None]
BAD_EPS = [True, 0, 0.0, -1e-7, float("nan"), math.inf, "1e-7", None]


@pytest.mark.parametrize("trainer", TRAINERS)
@pytest.mark.parametrize("name", ["beta1", "beta2"])
@pytest.mark.parametrize("b", BAD_BETA, ids=repr)
def test_bad_beta_raises_before_allocation(no_alloc, trainer, name, b):
  with pytest.raises(ValueError, match=name):
    _make(trainer, **{name: b})


@pytest.mark.parametrize("trainer", TRAINERS)
@pytest.mark.parametrize("e", BAD_EPS, ids=repr)
def test_bad_epsilon_raises_before_allocation(no_alloc, trainer, e):
  with pytest.raises(ValueError, match="epsilon"):
    _make(trainer, epsilon=e)


@pytest.mark.parametrize("trainer", TRAINERS)
@pytest.mark.parametrize("kw", [dict(beta1=0.0, beta2=0.5, epsilon=1e-30),
                                dict(beta1=np.float32(0.8), beta2=0.9999, epsilon=1)], ids=repr)
def test_good_adam_args_pass_the_checks(no_alloc, trainer, kw):
  with pytest.raises(_Allocated):
    _make(trainer, **kw)


@pytest.mark.parametrize("wd", [True, -1e-4, float("nan"), math.inf, "0.1", None])
def test_unet_bad_weight_decay(no_alloc, wd):
  with pytest.raises(ValueError, match="weight_decay"):
    _make("UNetTrainer", weight_decay=wd)


@pytest.mark.parametrize("o", ["sgd", "momentum", "lars", "Adam", None, 2])
def test_unet_bad_optimizer(no_alloc, o):
  with pytest.raises(ValueError, match="optimizer"):
    _make("UNetTrainer", optimizer=o)


@pytest.mark.parametrize("o", ["adam", "adamw", "lamb"])
def test_unet_optimizers_pass_the_checks(no_alloc, o):
  with pytest.raises(_Allocated):
    _make("UNetTrainer", optimizer=o, weight_decay=1e-4)


@pytest.mark.parametrize("kw", [dict(optimizer="adamw"), dict(optimizer="lamb"),
                                dict(weight_decay=1e-4), dict(beta1=0.8), dict(beta2=0.99),
                                dict(epsilon=1e-8)], ids=repr)
def test_unet_optimizer_args_need_training(no_alloc, kw):
  with pytest.raises(ValueError, match="needs training=True"):
    _make("UNetTrainer", training=False, **kw)
  with pytest.raises(_Allocated):                      # the defaults are fine without training
    _make("UNetTrainer", training=False)


def test_unet_defaults_are_the_optimizers_adam():
  """UNetTrainer() hands FusedOptimizer today's Adam: opt adam, weight_decay 0 and the
  optimizer's own beta1 / beta2 / eps defaults."""
  sig = inspect.signature(fused_optim.FusedOptimizer.__init__).parameters
  tsig = inspect.signature(unet.UNetTrainer.__init__).parameters
  assert unet.UNetTrainer.OPT_DEFAULTS == ("adam", 0.0, sig["beta1"].default,
                                           sig["beta2"].default, sig["eps"].default)
  assert tuple(tsig[n].default for n in ("optimizer", "weight_decay", "beta1", "beta2", "epsilon")) \
      == unet.UNetTrainer.OPT_DEFAULTS
  for cls in (resnet.ResNetTrainer, resnet.CifarResNetTrainer):
    p = inspect.signature(cls.__init__).parameters
    assert (p["beta1"].default, p["beta2"].default, p["epsilon"].default) == \
        (sig["beta1"].default, sig["beta2"].default, sig["eps"].default)


def _cpu_store():
  from tensorflowonspark_b200.models.engine import ParamStore, normal
  st = ParamStore()
  st.register("w", (40,), True, normal(0.1))
  st.register("v", (24,), True, normal(0.1))
  st.register("b", (8,), False, normal(0.1))
  st.finalize(torch.device("cpu"), seed=2)
  return st


def test_optimizer_codes_state_and_checkpoints():
  assert fused_optim.OPTIMIZERS == {"sgd": 0, "momentum": 1, "adam": 2, "lars": 3, "adamw": 4,
                                    "lamb": 5}
  adam = fused_optim.FusedOptimizer(_cpu_store(), opt="adam", lr=1e-3, weight_decay=1e-2)
  adam.state1.fill_(0.5)
  adam.state2.fill_(0.25)
  adam.hyper[7] = 3.0
  sd = adam.state_dict()
  for name in ("adamw", "lamb"):
    o = fused_optim.FusedOptimizer(_cpu_store(), opt=name, lr=1e-3, weight_decay=1e-2,
                                   trust_coefficient=0.5)
    assert o.state2 is not None and float(o.hyper[4]) == pytest.approx(0.9)  # beta1, not eta
    a, b = o.state_dict(), adam.state_dict()
    assert set(a) == set(b)                          # the same layout as adam's
    o.load_state_dict(sd)
    assert torch.equal(o.state1, adam.state1) and torch.equal(o.state2, adam.state2)
    assert torch.equal(o.hyper, adam.hyper)
    back = fused_optim.FusedOptimizer(_cpu_store(), opt="adam")
    back.load_state_dict(o.state_dict())
    assert torch.equal(back.state2, adam.state2) and torch.equal(back.hyper, adam.hyper)


def test_lamb_tables_and_bucket_rules():
  st = _cpu_store()
  o = fused_optim.FusedOptimizer(st, opt="lamb")
  assert o._lars_bounds == [0, 40, 64] and len(o._lars_args) == 1
  nd = o._lars_args[0]
  assert nd["lamb"] == 1 and nd["hyper"] == o.hyper.data_ptr()
  assert nd["state1"] == o.state1.data_ptr() and nd["state2"] == o.state2.data_ptr()
  with pytest.raises(ValueError, match="inside an adapted tensor"):
    fused_optim.FusedOptimizer(_cpu_store(), opt="lamb", buckets=[(0, 16, "a"), (16, 72, "b")])
  # LARS's norm-pass arguments are unchanged (no LAMB keys)
  lars = fused_optim.FusedOptimizer(_cpu_store(), opt="lars")
  assert not {"lamb", "hyper", "state1", "state2"} & set(lars._lars_args[0])
  # with clipping the LAMB norm pass reads the clipped scale
  c = fused_optim.FusedOptimizer(_cpu_store(), opt="lamb", clip_norm=1.0)
  assert [d["hyper"] for d in c._clip_lamb_norms] == [c.hyper_step.data_ptr()]
  assert fused_optim.FusedOptimizer(_cpu_store(), opt="lars", clip_norm=1.0)._clip_lamb_norms is None


def test_step_counts_for_the_adam_family():
  for name in ("adam", "adamw", "lamb"):
    o = fused_optim.FusedOptimizer(_cpu_store(), opt=name)
    o._bump_step()
    assert float(o.hyper[7]) == 1.0 and o.step_count == 1
  o = fused_optim.FusedOptimizer(_cpu_store(), opt="lars")
  o._bump_step()
  assert float(o.hyper[7]) == 0.0


# ------------------------------------------------------------------ example flags
def test_resnet_spark_optimizer_flags(fake_gpu):
  mod = importlib.import_module("resnet_spark")
  a = mod.parse([])
  assert (a.optimizer, a.weight_decay, a.beta1, a.beta2, a.epsilon) == ("momentum", None, None,
                                                                        None, None)
  base = ["resnet_spark.py", "--batch_size", "8", "--image", "64", "--train_steps", "2",
          "--metrics_port", "0"]
  mod.main_fun(base, dry._Ctx())
  plain = dict(dry._Trainer.made[-1].kw)
  for k in ("optimizer", "weight_decay", "beta1", "beta2", "epsilon", "trust_coefficient"):
    assert k not in plain
  for name in ("adamw", "lamb"):
    mod.main_fun(base + ["--optimizer", name, "--weight_decay", "0.05", "--beta1", "0.8",
                         "--beta2", "0.99", "--epsilon", "1e-6"], dry._Ctx())
    kw = dry._Trainer.made[-1].kw
    assert kw["optimizer"] == name and "trust_coefficient" not in kw
    assert (kw["weight_decay"], kw["beta1"], kw["beta2"], kw["epsilon"]) == (0.05, 0.8, 0.99, 1e-6)
  mod.main_fun(base + ["--optimizer", "lars"], dry._Ctx())
  kw = dry._Trainer.made[-1].kw
  assert kw["optimizer"] == "lars" and "weight_decay" not in kw


def test_resnet_spark_lamb_uses_the_large_batch_schedule(fake_gpu, monkeypatch):
  mod = importlib.import_module("resnet_spark")
  seen = []
  monkeypatch.setattr(resnet, "poly_warmup_lr", lambda *a: seen.append(a) or 0.1)
  base = ["resnet_spark.py", "--batch_size", "8", "--image", "64", "--train_steps", "3",
          "--metrics_port", "0"]
  mod.main_fun(base + ["--optimizer", "adamw"], dry._Ctx())
  assert not seen
  mod.main_fun(base + ["--optimizer", "lamb", "--warmup_steps", "1"], dry._Ctx())
  assert len(seen) == 3


@pytest.mark.parametrize("name", ["segmentation", "segmentation_spark"])
def test_segmentation_examples_take_the_optimizer_flags(name):
  path = os.path.join(ROOT, "examples", "segmentation")
  sys.path.insert(0, path)
  try:
    sys.modules.pop(name, None)
    mod = importlib.import_module(name)
    parser = mod.define_flags()
    a = parser.parse_args([])
    assert a.optimizer is None and a.weight_decay is None
    a = parser.parse_args(["--optimizer", "lamb", "--weight_decay", "1e-4"])
    assert a.optimizer == "lamb" and a.weight_decay == 1e-4
    with pytest.raises(SystemExit):
      parser.parse_args(["--optimizer", "sgd"])
    if name == "segmentation":
      assert mod.trainer_kwargs(parser.parse_args([])) == {}
      assert mod.trainer_kwargs(parser.parse_args(["--optimizer", "adamw", "--weight_decay", "0"])) \
          == {"optimizer": "adamw", "weight_decay": 0.0}
  finally:
    sys.path.remove(path)


# ------------------------------------------------------------------ kernel resources
NEW_KERNELS = tuple("allreduce_opt_kernelILi4ELb%dELi%dELb%dE" % (mc, ph, ema)
                    for mc, ph in ((0, 0), (1, 0), (0, 2)) for ema in (0, 1)) + \
    tuple("allreduce_opt_kernelILi5ELb%dELi%dELb%dE" % (mc, ph, ema)
          for mc, ph in ((0, 0), (0, 2), (1, 2)) for ema in (0, 1)) + \
    ("lars_norms_kernelILb1E",)


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not found")
def test_new_kernels_have_no_stack_frame_or_spills(tmp_path):
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
  assert len(NEW_KERNELS) == 13
  for k in NEW_KERNELS:
    hit = {n: v for n, v in kernels.items() if k in n}
    assert len(hit) == 1, (k, sorted(kernels))
    assert list(hit.values()) == [(0, 0, 0)], hit

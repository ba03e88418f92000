"""Gradient accumulation without a GPU: the trainers' argument checks, the optimizer's grad scale
and checkpoint rules, the window bookkeeping, the example flags and the ptxas report of the
accumulating kernels."""
import importlib
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

from tensorflowonspark_b200 import _build
from tensorflowonspark_b200.models import engine, resnet, unet
from tensorflowonspark_b200.parallel import fused_optim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_example_drivers_dryrun as dry  # noqa: E402
from test_example_drivers_dryrun import fake_gpu  # noqa: E402,F401  (fixture)

NVCC = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin",
                                            "nvcc")
BAD = [0, -1, 2.0, 1.5, True, False, "2", None]


# ------------------------------------------------------------------ argument checks
@pytest.mark.parametrize("k", BAD)
def test_checker_rejects(k):
  with pytest.raises(ValueError, match="gradient_accumulation_steps"):
    engine.check_gradient_accumulation_steps(k)


def test_checker_accepts_ints():
  import numpy as np
  assert engine.check_gradient_accumulation_steps(1) == 1
  assert engine.check_gradient_accumulation_steps(np.int64(4)) == 4
  assert engine.check_gradient_accumulation_steps(1, training=False) == 1
  with pytest.raises(ValueError, match="training=True"):
    engine.check_gradient_accumulation_steps(2, training=False)


@pytest.mark.parametrize("k", BAD)
@pytest.mark.parametrize("make", [
    lambda k: resnet.ResNetTrainer(depth=50, batch=8, image=64, gradient_accumulation_steps=k),
    lambda k: resnet.CifarResNetTrainer(depth=20, batch=8, gradient_accumulation_steps=k),
    lambda k: unet.UNetTrainer(batch=2, gradient_accumulation_steps=k),
], ids=["resnet", "cifar", "unet"])
def test_trainers_reject_before_allocating(make, k, monkeypatch):
  """ValueError before anything is allocated (building a parameter store would be the first)."""
  def boom(*a, **kw):
    raise AssertionError("allocated before the argument check")
  monkeypatch.setattr(engine.ParamStore, "finalize", boom)
  with pytest.raises(ValueError, match="gradient_accumulation_steps"):
    make(k)


def test_inference_trainers_take_only_k1(monkeypatch):
  monkeypatch.setattr(engine.ParamStore, "finalize",
                      lambda *a, **k: (_ for _ in ()).throw(AssertionError("allocated")))
  with pytest.raises(ValueError, match="training=True"):
    unet.UNetTrainer(batch=2, training=False, gradient_accumulation_steps=2)
  with pytest.raises(ValueError, match="training=True"):
    resnet.ResNetTrainer(depth=50, batch=8, image=64, training=False, gradient_accumulation_steps=3)


# ------------------------------------------------------------------ grad scale and checkpoints
def _cpu_store():
  st = engine.ParamStore()
  st.register("a.w", (40,), True, engine.constant(0.5))
  st.register("b.w", (24,), True, engine.constant(-0.25))
  st.register("c.b", (16,), False, engine.constant(0.0))
  st.finalize("cpu", grads=True)
  return st


def test_scale_is_one_over_world_k_and_checkpoints_are_k_free():
  o = fused_optim.FusedOptimizer(_cpu_store(), opt="adam")
  assert float(o.hyper[3]) == 1.0
  o.set_accumulation(3)
  assert float(o.hyper[3]) == float(torch.tensor(1.0 / 3, dtype=torch.float32))
  sd = o.state_dict()
  assert float(sd["hyper"][3]) == 1.0 and float(o.hyper[3]) != 1.0   # saved k-free, live kept
  one = fused_optim.FusedOptimizer(_cpu_store(), opt="adam")
  one.load_state_dict(sd)
  assert float(one.hyper[3]) == 1.0
  sd1 = one.state_dict()
  four = fused_optim.FusedOptimizer(_cpu_store(), opt="adam")
  four.set_accumulation(4)
  four.load_state_dict(sd1)
  assert float(four.hyper[3]) == 0.25


def test_window_bookkeeping():
  o = fused_optim.FusedOptimizer(_cpu_store(), opt="sgd")
  w = engine.GradAccumulation(3)
  assert [w.phase(i) for i in range(3)] == [(True, False), (False, False), (False, True)]
  seen = []
  for _ in range(7):
    seen.append(w.micro_step)
    w.advance()
  assert seen == [0, 1, 2, 0, 1, 2, 0]
  o.store.grads.fill_(1.0)
  w.restart(o)
  assert w.micro_step == 0 and not o.store.grads.any()
  one = engine.GradAccumulation(1)
  assert one.phase() == (True, True)
  o.store.grads.fill_(1.0)
  one.restart(o)   # k = 1: nothing to restart, every step zeroes the gradients itself
  assert o.store.grads.all()


# ------------------------------------------------------------------ example flags
class _AccTrainer(dry._Trainer):
  """The dry-run trainer with an accumulation window."""

  def __init__(self, **kw):
    super().__init__(**kw)
    self.k, self.micro_step = kw.get("gradient_accumulation_steps", 1), 0

  def train_step(self, *a):
    self.micro_step = (self.micro_step + 1) % self.k
    return super().train_step(*a)


def test_resnet_spark_flag(fake_gpu, monkeypatch):
  mod = importlib.import_module("resnet_spark")
  assert mod.parse([]).gradient_accumulation_steps == 1
  base = ["resnet_spark.py", "--batch_size", "8", "--image", "64", "--train_steps", "3",
          "--metrics_port", "0"]
  mod.main_fun(base, dry._Ctx())
  assert "gradient_accumulation_steps" not in dry._Trainer.made[-1].kw
  monkeypatch.setattr(resnet, "ResNetTrainer", _AccTrainer)
  lrs = []
  monkeypatch.setattr(resnet, "poly_warmup_lr", lambda step, *a: lrs.append(step) or 0.1)
  mod.main_fun(base + ["--gradient_accumulation_steps", "4", "--optimizer", "lars"], dry._Ctx())
  net = dry._Trainer.made[-1]
  assert net.kw["gradient_accumulation_steps"] == 4
  # warm-up step + capture, the window finished, then 3 updates of 4 micro-steps each
  assert net.micro_step == 0 and net.steps % 4 == 0 and net.steps >= 3 * 4
  assert lrs == [0, 1, 2]   # the schedule counts updates


@pytest.mark.parametrize("name", ["segmentation", "segmentation_spark"])
def test_segmentation_flags(name):
  path = os.path.join(ROOT, "examples", "segmentation")
  sys.path.insert(0, path)
  try:
    sys.modules.pop(name, None)
    mod = importlib.import_module(name)
    parser = mod.define_flags()
    assert parser.parse_args([]).gradient_accumulation_steps is None
    assert parser.parse_args(["--gradient_accumulation_steps", "4"]).gradient_accumulation_steps == 4
    if name == "segmentation":
      assert mod.trainer_kwargs(parser.parse_args([])) == {}
      assert mod.trainer_kwargs(parser.parse_args(["--gradient_accumulation_steps", "2"])) == \
          {"gradient_accumulation_steps": 2}
  finally:
    sys.path.remove(path)


# ------------------------------------------------------------------ kernel resources
def _ptxas(source, tmp_path):
  out = tmp_path / (source + ".o")
  cmd = [NVCC] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", _build.CSRC_DIR, "-c",
                                      os.path.join(_build.CSRC_DIR, source), "-o", str(out)]
  r = subprocess.run(cmd, capture_output=True, text=True)
  assert r.returncode == 0, r.stderr[-4000:]
  kernels, cur = {}, None
  for line in r.stderr.splitlines():
    m = re.search(r"Compiling entry function '(\S+)'", line)
    if m:
      cur = m.group(1)
      continue
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                  line)
    if m and cur is not None:
      kernels[cur] = tuple(int(x) for x in m.groups())
  return kernels


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not found")
@pytest.mark.parametrize("source,count", [("bn_bwd.cu", 1), ("stem_fused.cu", 1),
                                          ("smallops.cu", 3)])
def test_accumulating_kernels_have_no_stack_frame_or_spills(source, count, tmp_path):
  kernels = _ptxas(source, tmp_path)
  acc = {k: v for k, v in kernels.items() if "_acc_kernel" in k}
  assert len(acc) == count, sorted(kernels)
  bad = {k: v for k, v in acc.items() if v != (0, 0, 0)}
  assert not bad, "stack frame / spill stores / spill loads (bytes): {}".format(bad)

"""CPU tier of U-Net encoder fine-tuning: argument validation of
``UNetTrainer(encoder_trainable_from=...)`` before anything touches a device, the example drivers'
``--encoder_trainable_from`` flag (with a stand-in trainer), and ptxas' resource report of the
depthwise backward kernel (needs nvcc, not a GPU)."""
import importlib
import os
import re
import shutil
import subprocess
import sys
import types

import pytest
import torch

from tensorflowonspark_b200 import _build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin",
                                            "nvcc")


# ----------------------------------------------------------------------------- validation
@pytest.mark.parametrize("kw", [dict(encoder_trainable_from=17), dict(encoder_trainable_from=-1),
                                dict(encoder_trainable_from=1.0), dict(encoder_trainable_from="3"),
                                dict(encoder_trainable_from=True),
                                dict(encoder_trainable_from=0, training=False),
                                dict(encoder_trainable_from=16, training=False)])
def test_bad_encoder_trainable_from_raises_before_any_allocation(kw, monkeypatch):
  from tensorflowonspark_b200.models import unet

  def no_alloc(*a, **k):
    raise AssertionError("allocated before validating its arguments")
  monkeypatch.setattr(unet, "_buf", no_alloc)
  monkeypatch.setattr(unet, "MobileNetV2Encoder", no_alloc)
  monkeypatch.setattr(torch, "zeros", no_alloc)
  with pytest.raises(ValueError):
    unet.UNetTrainer(batch=2, device="cuda:0", **kw)


def test_block_numbering_and_depthwise_shapes():
  from tensorflowonspark_b200.models import unet
  shapes = unet.encoder_depthwise_shapes(128)
  assert unet.NUM_BLOCKS == len(shapes) == 17
  assert shapes[0] == (0, 64, 32, 1) and shapes[13] == (13, 8, 576, 2)
  assert shapes[16] == (16, 4, 960, 1)
  assert all(C % 8 == 0 for _, _, C, _ in shapes)


# ----------------------------------------------------------------------------- example drivers
class _Optim(object):
  def __init__(self):
    self.loaded = None

  def state_dict(self):
    return {"step": 3}

  def load_state_dict(self, sd):
    self.loaded = sd


class _Trainer(object):
  made = []
  params = {"up0.w": torch.zeros(2)}

  def __init__(self, **kw):
    self.kw, self.optim, self.loaded, self.steps = kw, _Optim(), None, 0
    self.store = types.SimpleNamespace(order=[{"name": k} for k in _Trainer.params])
    _Trainer.made.append(self)

  def synthetic_batch(self, seed=0):
    return torch.zeros(2, 8, 8, 3, dtype=torch.uint8), None

  def set_input(self, x, y=None):
    pass

  def train_step(self, *a):
    self.steps += 1
    return torch.tensor(1.0)

  def capture(self):
    pass

  def state_dict(self):
    return dict(_Trainer.params)

  def load_state_dict(self, sd):
    self.loaded = sd


@pytest.fixture
def drivers(monkeypatch):
  from tensorflowonspark_b200.models import unet
  _Trainer.made = []
  monkeypatch.setattr(unet, "UNetTrainer", _Trainer)
  monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
  monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
  monkeypatch.syspath_prepend(os.path.join(ROOT, "examples", "segmentation"))
  names = ("segmentation", "segmentation_spark")
  for n in names:
    sys.modules.pop(n, None)
  yield types.SimpleNamespace(seg=importlib.import_module("segmentation"),
                              spark=importlib.import_module("segmentation_spark"))
  for n in names:
    sys.modules.pop(n, None)


def _seg_args(mod, *extra):
  return mod.define_flags().parse_args(["--epochs", "1", "--steps_per_epoch", "2", "--eval_steps",
                                        "0", "--batch_size", "2"] + list(extra))


def test_segmentation_flag_reaches_the_trainer_and_the_default_is_unchanged(drivers):
  drivers.seg.train(_seg_args(drivers.seg))
  assert "encoder_trainable_from" not in _Trainer.made[-1].kw
  drivers.seg.train(_seg_args(drivers.seg, "--encoder_trainable_from", "13"))
  assert _Trainer.made[-1].kw["encoder_trainable_from"] == 13


def test_resuming_a_frozen_checkpoint_for_fine_tuning_skips_the_optimizer_state(drivers, tmp_path,
                                                                               capsys):
  from tensorflowonspark_b200.utils import checkpoint
  md = str(tmp_path / "ckpt")
  drivers.seg.train(_seg_args(drivers.seg, "--model_dir", md))      # frozen run: no encoder.*
  assert checkpoint.load(md)[0] == 2
  net = _Trainer.made[-1]
  assert net.loaded is None and net.optim.loaded is None
  drivers.seg.train(_seg_args(drivers.seg, "--model_dir", md))      # resumes as before
  assert _Trainer.made[-1].optim.loaded == {"step": 3}
  capsys.readouterr()
  # the fine-tuning trainer's parameters include encoder.*: so does the checkpoint it writes
  _Trainer.params = {"up0.w": torch.zeros(2), "encoder.stem.w": torch.zeros(3)}
  try:
    drivers.seg.train(_seg_args(drivers.seg, "--model_dir", md, "--encoder_trainable_from", "0"))
    net = _Trainer.made[-1]
    assert net.kw["encoder_trainable_from"] == 0
    assert net.loaded is not None and net.optim.loaded is None
    assert "fresh optimizer state" in capsys.readouterr().out
    # a fine-tuning checkpoint resumes with its optimizer state
    drivers.seg.train(_seg_args(drivers.seg, "--model_dir", md, "--encoder_trainable_from", "0"))
    assert _Trainer.made[-1].optim.loaded == {"step": 3}
    assert "fresh optimizer state" not in capsys.readouterr().out
    # a checkpoint that fine-tuned other blocks (k = 0) resumed with k = 13: fresh optimizer
    _Trainer.params = {"up0.w": torch.zeros(2), "encoder.block13.dw.w": torch.zeros(3)}
    drivers.seg.train(_seg_args(drivers.seg, "--model_dir", md, "--encoder_trainable_from", "13"))
    assert _Trainer.made[-1].optim.loaded is None
    assert "fresh optimizer state" in capsys.readouterr().out
    drivers.seg.train(_seg_args(drivers.seg, "--model_dir", md, "--encoder_trainable_from", "13"))
    assert _Trainer.made[-1].optim.loaded == {"step": 3}
  finally:
    _Trainer.params = {"up0.w": torch.zeros(2)}


class _Ctx(object):
  rank, world_size, is_chief, num_workers = 0, 1, True, 1

  def gradient_comm(self):
    return None

  def absolute_path(self, p):
    return os.path.abspath(p)


def test_segmentation_spark_flag(drivers):
  class Args(object):
    batch_size, learning_rate, input_mode, steps, epochs, num_examples = 2, 1e-3, "tf", 2, 1, 8

  drivers.spark.main_fun(Args(), _Ctx())
  assert "encoder_trainable_from" not in _Trainer.made[-1].kw
  Args.encoder_trainable_from = 5
  drivers.spark.main_fun(Args(), _Ctx())
  assert _Trainer.made[-1].kw["encoder_trainable_from"] == 5


# ----------------------------------------------------------------------------- kernel resources
@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not found")
def test_depthwise_backward_has_no_stack_frame_or_spills(tmp_path):
  out = tmp_path / "smallops.o"
  cmd = [NVCC] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", _build.CSRC_DIR, "-c",
                                      os.path.join(_build.CSRC_DIR, "smallops.cu"), "-o", str(out)]
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
  bwd = {k: v for k, v in kernels.items() if "depthwise3x3_bwd_kernel" in k}
  assert len(bwd) == 3, sorted(kernels)     # one instance per channel-group chunking (4, 2, 1)
  bad = {k: v for k, v in bwd.items() if v != (0, 0, 0)}
  assert not bad, "stack frame / spill stores / spill loads (bytes): {}".format(bad)

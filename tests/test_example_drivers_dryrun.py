"""Driver logic of the GPU-only example programs, dry-run on CPU.

examples/resnet/{resnet_spark,resnet_cifar_main}.py can only train on an H100, but everything
around the trainer - flag parsing, communicator selection and initial broadcast, resume from
``model_dir``, LR schedule, periodic checkpoints, JSONL metrics and TensorBoard events - is plain
Python.  Here the native trainers are replaced by a stand-in with the same surface, so that a typo
in that glue fails on the CPU tier instead of on the first GPU run (reference scripts:
examples/resnet/resnet_cifar_{main,dist,spark}.py)."""
import importlib
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Optim(object):
  def __init__(self):
    self.loaded = None

  def state_dict(self):
    return {"step": 3}

  def load_state_dict(self, sd):
    self.loaded = sd


class _Trainer(object):
  made = []

  def __init__(self, **kw):
    self.kw, self.optim, self.steps, self.lrs, self.loaded, self.captured = kw, _Optim(), 0, [], None, False
    _Trainer.made.append(self)

  def synthetic_batch(self, seed=0):
    return torch.zeros(2, dtype=torch.uint8), torch.zeros(2, dtype=torch.int32)

  def set_input(self, x, y=None):
    pass

  def train_step(self, *a):
    self.steps += 1
    return torch.tensor(1.0 / self.steps)

  def capture(self):
    self.captured = True

  def set_lr(self, lr):
    self.lrs.append(lr)

  def state_dict(self):
    return {"w": torch.full((3,), float(self.steps))}

  def load_state_dict(self, sd):
    self.loaded = sd


class _Comm(object):
  world, rank = 2, 0

  def __init__(self):
    self.broadcasts = []

  def broadcast(self, name, root=0):
    self.broadcasts.append((name, root))


@pytest.fixture
def fake_gpu(monkeypatch):
  from tensorflowonspark_b200.models import resnet
  _Trainer.made = []
  monkeypatch.setattr(resnet, "ResNetTrainer", _Trainer)
  monkeypatch.setattr(resnet, "CifarResNetTrainer", _Trainer)
  monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
  monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
  monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
  monkeypatch.syspath_prepend(os.path.join(ROOT, "examples", "resnet"))
  for name in ("resnet_spark", "resnet_cifar_main"):
    sys.modules.pop(name, None)
  yield
  for name in ("resnet_spark", "resnet_cifar_main"):
    sys.modules.pop(name, None)


class _Ctx(object):
  def __init__(self, world=1, comm=None):
    self.rank, self.world_size, self.is_chief, self.gpus = 0, world, True, [0]
    self.job_name, self.task_index, self._comm = "chief", 0, comm

  def absolute_path(self, p):
    return os.path.abspath(p)

  def gradient_comm(self):
    return self._comm


def test_resnet_spark_driver_checkpoints_metrics_events_and_resume(fake_gpu, tmp_path):
  from tensorflowonspark_b200.utils import checkpoint, metrics, summary
  mod = importlib.import_module("resnet_spark")
  md, mt = str(tmp_path / "ckpt"), str(tmp_path / "steps.jsonl")
  argv = ["resnet_spark.py", "--batch_size", "8", "--image", "64", "--train_steps", "25", "--model_dir", md,
          "--save_steps", "10", "--metrics", mt, "--epochs_per_step", "10", "--metrics_port", "0"]
  mod.main_fun(argv, _Ctx())
  net = _Trainer.made[-1]
  assert net.kw["depth"] == 50 and net.kw["batch"] == 8 and net.kw["comm"] is None and net.captured
  assert net.steps == 1 + 25 and len(net.lrs) == 25 and net.lrs[-1] < net.lrs[0]   # piecewise schedule
  step, state = checkpoint.load(md)
  assert step == 20 and set(state) == {"params", "optim"}
  recs = metrics.read(mt + ".rank0")
  assert [r["step"] for r in recs] == [10, 20] and recs[-1]["images_per_s"] > 0
  (ev,) = summary.event_files(md)
  assert [e["step"] for e in summary.read_events(ev) if e["scalars"]] == [10, 20]
  # a second run resumes where the checkpoint left off, on two "ranks" through the communicator
  comm = _Comm()
  mod.main_fun(argv + ["--model", "resnet56", "--no_graph"], _Ctx(world=2, comm=comm))
  net = _Trainer.made[-1]
  assert comm.broadcasts == [("weights", 0), ("aux32", 0)] and net.kw["comm"] is comm and not net.captured
  assert net.loaded is not None and net.optim.loaded == {"step": 3}
  assert checkpoint.load(md)[0] == 40                                        # steps 21 .. 45, saved at 30, 40


def test_resnet_cifar_entry_points_share_main_fun_and_local_context(fake_gpu, tmp_path):
  from tensorflowonspark_b200.utils import checkpoint
  mod = importlib.import_module("resnet_cifar_main")
  md = str(tmp_path / "cifar")
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "7", "--resnet_size", "20", "--model_dir", md],
               mod.LocalContext())
  net = _Trainer.made[-1]
  assert net.kw["depth"] == 20 and net.kw["comm"] is None and net.captured and net.steps == 1 + 7
  assert checkpoint.load(md)[0] == 7
  comm = _Comm()                       # what resnet_cifar_dist.py builds under torchrun
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "9", "--model_dir", md, "--no_graph"],
               mod.LocalContext(0, 2, comm))
  net = _Trainer.made[-1]
  assert net.kw["comm"] is comm and comm.broadcasts == [("weights", 0), ("aux32", 0)]
  assert net.loaded is not None and net.steps == 1 + 2                       # resumed at step 7 of 9
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "3", "--ds", "off"], mod.LocalContext(0, 2, comm))
  assert _Trainer.made[-1].kw["comm"] is None                                # --ds off: no collective
  img = __import__("numpy").zeros((4, 32, 32, 3), dtype="uint8")
  assert mod.augment(img, __import__("numpy").random.RandomState(0)).shape == img.shape


def test_segmentation_spark_driver_tf_mode_with_a_communicator(fake_gpu, monkeypatch):
  from tensorflowonspark_b200.models import unet
  monkeypatch.setattr(unet, "UNetTrainer", _Trainer)
  monkeypatch.syspath_prepend(os.path.join(ROOT, "examples", "segmentation"))
  sys.modules.pop("segmentation_spark", None)
  mod = importlib.import_module("segmentation_spark")

  class Args(object):
    batch_size, learning_rate, input_mode, steps, epochs, num_examples = 4, 1e-3, "tf", 12, 1, 64

  real_batch = _Trainer.synthetic_batch
  monkeypatch.setattr(_Trainer, "synthetic_batch",
                      lambda self, seed=0: (torch.zeros(4, 8, 8, 3, dtype=torch.uint8), None))
  comm = _Comm()
  ctx = _Ctx(world=2, comm=comm)
  ctx.num_workers = 2
  mod.main_fun(Args(), ctx)
  net = _Trainer.made[-1]
  assert net.kw["comm"] is comm and net.kw["classes"] == 3 and net.captured and net.steps == 1 + 12
  assert comm.broadcasts == [("weights", 0), ("aux32", 0)]
  assert real_batch is not _Trainer.synthetic_batch
  sys.modules.pop("segmentation_spark", None)

"""Held-out evaluation of the segmentation U-Net, host side (no GPU): the metric arithmetic of
``unet.seg_eval_result`` and the evaluation schedule, TensorBoard scalars and checkpoints of the
segmentation drivers, with a stand-in trainer that has the evaluation surface."""
import argparse
import importlib
import math
import os
import sys

import pytest
import torch

from tensorflowonspark_b200.models import unet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_example_drivers_dryrun as dry  # noqa: E402
from test_example_drivers_dryrun import fake_gpu  # noqa: E402,F401  (fixture)


def _totals(cm, count=None, correct=None, invalid=0, loss=0.0, images=1):
  """Accumulator layout of seg_eval_metrics: [count, correct, invalid, loss, confusion[8 x 8]],
  then the image count at unet.SEG_IMAGES."""
  t = [0.0] * unet.SEG_ACC
  for y, row in enumerate(cm):
    for p, v in enumerate(row):
      t[unet.SEG_CONFUSION + 8 * y + p] = float(v)
  n = sum(sum(r) for r in cm)
  t[unet.SEG_COUNT] = float(n if count is None else count)
  t[unet.SEG_CORRECT] = float(sum(cm[i][i] for i in range(len(cm))) if correct is None else correct)
  t[unet.SEG_INVALID], t[unet.SEG_LOSS], t[unet.SEG_IMAGES] = float(invalid), loss, float(images)
  return t


def test_iou_from_the_confusion_matrix():
  cm = [[3, 1, 0], [1, 4, 0], [0, 1, 2]]   # rows: label, columns: prediction
  r = unet.seg_eval_result(_totals(cm, loss=6.0, images=2), 3)
  assert r["count"] == 12 and r["images"] == 2
  assert r["accuracy"] == 9 / 12 and r["loss"] == 0.5
  assert r["iou"] == pytest.approx([3 / 5, 4 / 7, 2 / 3])
  assert r["mean_iou"] == pytest.approx((3 / 5 + 4 / 7 + 2 / 3) / 3)


def test_absent_class_has_nan_iou_and_is_left_out_of_the_mean():
  cm = [[3, 1, 0], [1, 4, 0], [0, 0, 0]]   # class 2: neither a label nor a prediction
  r = unet.seg_eval_result(_totals(cm), 3)
  assert math.isnan(r["iou"][2])
  assert r["mean_iou"] == pytest.approx((3 / 5 + 4 / 6) / 2)
  # predicted but never labelled: union > 0, IoU 0, part of the mean
  r = unet.seg_eval_result(_totals([[3, 1, 1], [1, 4, 0], [0, 0, 0]]), 3)
  assert r["iou"][2] == 0.0 and r["mean_iou"] == pytest.approx((3 / 6 + 4 / 6 + 0) / 3)


def test_nothing_scored():
  r = unet.seg_eval_result(_totals([[0, 0], [0, 0]], images=0), 2)
  assert r["count"] == 0 and r["images"] == 0
  assert math.isnan(r["loss"]) and math.isnan(r["accuracy"]) and math.isnan(r["mean_iou"])
  assert len(r["iou"]) == 2 and all(math.isnan(v) for v in r["iou"])


def test_invalid_labels_raise():
  with pytest.raises(ValueError, match="3 mask value"):
    unet.seg_eval_result(_totals([[1, 0], [0, 1]], invalid=3), 2)


def test_masks_are_never_narrowed():
  m = unet._widen(torch.tensor([[-1, 0, 2, 256, 2 ** 40]], dtype=torch.int64))
  assert m.tolist() == [[-1, 0, 2, 256, 2 ** 31 - 1]]
  u8 = torch.tensor([0, 255], dtype=torch.uint8)
  assert unet._widen(u8) is u8 or unet._widen(u8).dtype == torch.uint8


# ------------------------------------------------------------------------- drivers
class _SegTrainer(dry._Trainer):
  def __init__(self, **kw):
    super().__init__(**kw)
    self.evals = []      # (train steps so far, images per evaluation)

  def synthetic_batch(self, seed=0):
    return torch.full((2, 4, 4, 3), seed % 256, dtype=torch.uint8), None

  def evaluate(self, batches):
    n = 0
    for x, y in batches:
      assert y.shape == x.shape[:3]
      n += len(x)
    self.evals.append((self.steps, n))
    return {"count": n * 16, "images": n, "loss": 0.5, "accuracy": 0.25, "mean_iou": 0.75,
            "iou": [0.5, 1.0]}


@pytest.fixture
def seg_drivers(fake_gpu, monkeypatch):
  monkeypatch.setattr(unet, "UNetTrainer", _SegTrainer)
  monkeypatch.syspath_prepend(os.path.join(ROOT, "examples", "segmentation"))
  for name in ("segmentation", "segmentation_spark"):
    sys.modules.pop(name, None)
  yield
  for name in ("segmentation", "segmentation_spark"):
    sys.modules.pop(name, None)


def test_segmentation_evaluates_every_epoch_with_scalars_and_checkpoints(seg_drivers, tmp_path,
                                                                         capsys):
  from tensorflowonspark_b200.utils import checkpoint, summary
  mod = importlib.import_module("segmentation")
  md, ex = str(tmp_path / "md"), str(tmp_path / "export")
  args = mod.define_flags().parse_args(["--batch_size", "2", "--epochs", "3", "--steps_per_epoch",
                                        "4", "--eval_steps", "2", "--model_dir", md,
                                        "--export_dir", ex])
  net = mod.train(args)
  assert net.evals == [(4, 4), (8, 4), (12, 4)]          # 2 held-out batches of 2 per epoch
  out = capsys.readouterr().out
  assert "epoch 3 loss 0.0833 val_loss 0.5000 val_accuracy 0.2500 val_mean_iou 0.7500" in out
  (ev,) = summary.event_files(os.path.join(md, "eval"))
  recs = [e for e in summary.read_events(ev) if e["scalars"]]
  assert [e["step"] for e in recs] == [4, 8, 12]
  assert recs[-1]["scalars"] == {"loss": 0.5, "accuracy": 0.25, "mean_iou": 0.75}
  step, state = checkpoint.load(md)                       # net.state_dict(), not store's
  assert step == 12 and torch.equal(state["params"]["w"], torch.full((3,), 12.0))
  assert os.path.isdir(ex)
  # resume: the checkpoint goes through load_state_dict
  net2 = mod.train(mod.define_flags().parse_args(["--epochs", "1", "--steps_per_epoch", "2",
                                                  "--model_dir", md]))
  assert torch.equal(net2.loaded["w"], torch.full((3,), 12.0)) and net2.optim.loaded == {"step": 3}
  assert net2.evals == [(2, 2)]                           # default: one held-out batch per rank


def test_segmentation_eval_steps_zero_and_non_chief_ranks(seg_drivers, tmp_path, capsys):
  mod = importlib.import_module("segmentation")
  md = str(tmp_path / "md")
  args = mod.define_flags().parse_args(["--epochs", "2", "--steps_per_epoch", "3", "--eval_steps",
                                        "0", "--model_dir", md])
  assert mod.train(args).evals == []
  assert not os.path.exists(os.path.join(md, "eval"))
  assert "val_loss" not in capsys.readouterr().out
  # evaluation is collective: a non-chief rank evaluates its own shard too, and prints nothing
  args = mod.define_flags().parse_args(["--epochs", "1", "--steps_per_epoch", "3", "--eval_steps", "3"])
  net = mod.train(args, rank=1, world=2, comm=dry._Comm(), is_chief=False)
  assert net.evals == [(3, 6)]
  assert capsys.readouterr().out == ""


def _spark_args(**kw):
  a = argparse.Namespace(batch_size=4, learning_rate=1e-3, input_mode="tf", steps=12, epochs=1,
                         num_examples=64)
  for k, v in kw.items():
    setattr(a, k, v)
  return a


def test_segmentation_spark_eval_steps_and_eval_every(seg_drivers, capsys):
  import re
  mod = importlib.import_module("segmentation_spark")
  ctx = dry._Ctx(world=2, comm=dry._Comm())
  ctx.num_workers = 2
  mod.main_fun(_spark_args(eval_steps=2, eval_every=5), ctx)
  net = _SegTrainer.made[-1]
  assert net.evals == [(1 + 5, 4), (1 + 10, 4), (1 + 12, 4)]   # warm-up step + 5, 10, last
  out = capsys.readouterr().out
  assert "eval: step 10 val_loss=0.5000 val_accuracy=0.2500 val_mean_iou=0.7500 (4 images)" in out
  # the evaluation lines add nothing to what a "loss <value>" scan of the training log finds
  assert all("eval:" not in line for line in out.splitlines() if re.search(r"loss ([\d.]+)", line))
  mod.main_fun(_spark_args(eval_steps=1, eval_every=4), ctx)   # the last step is on the schedule
  assert _SegTrainer.made[-1].evals == [(1 + 4, 2), (1 + 8, 2), (1 + 12, 2)]
  mod.main_fun(_spark_args(eval_steps=1, eval_every=0), ctx)
  assert _SegTrainer.made[-1].evals == [(1 + 12, 2)]
  mod.main_fun(_spark_args(), ctx)                           # off by default
  assert _SegTrainer.made[-1].evals == []

"""CPU tier of the U-Net's loss options (``ignore_index``, ``class_weights``): validation before
anything touches a device, the weighted evaluation loss of seg_eval_result, the examples' flags
(with the stand-in trainer of test_unet_finetune_host) and ptxas' resource report of the optioned
kernel instances (needs nvcc, not a GPU)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_unet_classes_host as uc  # noqa: E402
import test_unet_finetune_host as ft  # noqa: E402


# ----------------------------------------------------------------------------- validation
BAD = [
    {"ignore_index": 2.0}, {"ignore_index": True}, {"ignore_index": "255"},
    {"ignore_index": 2 ** 31}, {"ignore_index": -2 ** 31 - 1},
    {"class_weights": [1.0, 1.0]}, {"class_weights": [1.0] * 4}, {"class_weights": 1.0},
    {"class_weights": True}, {"class_weights": "1,1,1"}, {"class_weights": [1.0, True, 1.0]},
    {"class_weights": [1.0, float("nan"), 1.0]}, {"class_weights": [1.0, float("inf"), 1.0]},
    {"class_weights": [1.0, -0.5, 1.0]}, {"class_weights": [0.0, 0.0, 0.0]},
    {"class_weights": [1.0, "2", 1.0]},
]


@pytest.mark.parametrize("kw", BAD, ids=[repr(k) for k in BAD])
@pytest.mark.parametrize("training", [True, False])
def test_bad_loss_option_raises_before_any_allocation(kw, training, monkeypatch):
  from tensorflowonspark_b200.models import unet

  def no_alloc(*a, **k):
    raise AssertionError("allocated before validating its arguments")
  monkeypatch.setattr(unet, "_buf", no_alloc)
  monkeypatch.setattr(unet, "MobileNetV2Encoder", no_alloc)
  monkeypatch.setattr(torch, "zeros", no_alloc)
  with pytest.raises(ValueError):
    unet.UNetTrainer(batch=2, device="cuda:0", classes=3, training=training, **kw)


def test_good_loss_options_are_normalised():
  from tensorflowonspark_b200.models import unet
  assert unet._ignore_index(None) is None and unet._class_weights(None, 3) is None
  assert unet._ignore_index(np.int64(255)) == 255 and unet._ignore_index(-2 ** 31) == -2 ** 31
  w = unet._class_weights(np.array([0.1, 0, 3]), 3)
  assert w == (float(np.float32(0.1)), 0.0, 3.0)
  assert unet._class_weights(torch.tensor([1.0, 2.0]), 2) == (1.0, 2.0)


# ----------------------------------------------------------------------------- host metrics
def _narrow_totals(cm8, loss, images=1):
  from tensorflowonspark_b200.models import unet
  t = [0.0] * unet.SEG_ACC
  t[unet.SEG_COUNT] = float(cm8.sum())
  t[unet.SEG_CORRECT] = float(np.trace(cm8))
  t[unet.SEG_LOSS] = loss
  t[unet.SEG_IMAGES] = images
  t[unet.SEG_CONFUSION:unet.SEG_CONFUSION + 64] = cm8.reshape(-1).tolist()
  return t


def test_seg_eval_result_weighted_loss_narrow():
  from tensorflowonspark_b200.models import unet
  cm = np.zeros((8, 8))
  cm[0, 0], cm[0, 2], cm[1, 1], cm[2, 2], cm[2, 1] = 5, 1, 4, 2, 3   # rows 6, 4, 5
  w = (0.5, 2.0, 0.0)
  res = unet.seg_eval_result(_narrow_totals(cm, 9.0), 3, w)
  assert res["loss"] == 9.0 / (0.5 * 6 + 2.0 * 4 + 0.0 * 5)
  plain = unet.seg_eval_result(_narrow_totals(cm, 9.0), 3)
  assert plain["loss"] == 9.0 / 15
  assert {k: v for k, v in res.items() if k != "loss"} == \
      {k: v for k, v in plain.items() if k != "loss"}, "IoU and accuracy stay unweighted"
  assert set(plain) == {"count", "images", "loss", "accuracy", "mean_iou", "iou"}


def test_seg_eval_result_weighted_loss_wide_and_empty_denominator():
  from tensorflowonspark_b200.models import unet
  V = 21
  cm = np.zeros((V, V))
  cm[0, 0], cm[0, 1], cm[3, 3], cm[20, 5] = 6, 2, 3, 4     # rows: 8, 3, 4
  w = [1.0] * V
  w[0], w[3], w[20] = 0.25, 4.0, 1.5
  res = unet.seg_eval_result(uc._wide_totals(V, cm, loss=12.0), V, w)
  assert res["loss"] == pytest.approx(12.0 / (0.25 * 8 + 4.0 * 3 + 1.5 * 4), rel=1e-15)
  assert res["accuracy"] == 9 / 15
  assert unet.seg_eval_result(uc._wide_totals(V, cm, loss=12.0), V)["loss"] == 12.0 / 15
  w0 = [0.0] * V
  w0[7] = 1.0                                                # no pixel of class 7: sum w = 0
  assert np.isnan(unet.seg_eval_result(uc._wide_totals(V, cm, loss=0.0), V, w0)["loss"])


# ----------------------------------------------------------------------------- examples
drivers = ft.drivers


def test_segmentation_loss_flags_reach_the_trainer(drivers):
  drivers.seg.train(ft._seg_args(drivers.seg))
  kw = ft._Trainer.made[-1].kw
  assert "ignore_index" not in kw and "class_weights" not in kw
  drivers.seg.train(ft._seg_args(drivers.seg, "--classes", "4", "--ignore_index", "255",
                                 "--class_weights", "1,0.5,2,0"))
  kw = ft._Trainer.made[-1].kw
  assert kw["ignore_index"] == 255 and kw["class_weights"] == [1.0, 0.5, 2.0, 0.0]
  assert "encoder_trainable_from" not in kw


def test_segmentation_dist_parses_loss_flags(monkeypatch):
  monkeypatch.syspath_prepend(os.path.join(uc.ROOT, "examples", "segmentation"))
  sys.modules.pop("segmentation", None)
  try:
    import segmentation
    a = segmentation.define_flags().parse_args([])
    assert a.ignore_index is None and a.class_weights is None
    a = segmentation.define_flags().parse_args(["--ignore_index", "-1", "--class_weights", "3,1"])
    assert segmentation.trainer_kwargs(a) == {"ignore_index": -1, "class_weights": [3.0, 1.0]}
  finally:
    sys.modules.pop("segmentation", None)


def test_segmentation_spark_loss_options(drivers):
  class Args(object):
    batch_size, learning_rate, input_mode, steps, epochs, num_examples = 2, 1e-3, "tf", 2, 1, 8

  drivers.spark.main_fun(Args(), ft._Ctx())
  kw = ft._Trainer.made[-1].kw
  assert "ignore_index" not in kw and "class_weights" not in kw
  Args.ignore_index, Args.class_weights = 255, [1.0, 2.0, 3.0]
  drivers.spark.main_fun(Args(), ft._Ctx())
  kw = ft._Trainer.made[-1].kw
  assert kw["ignore_index"] == 255 and kw["class_weights"] == [1.0, 2.0, 3.0]
  src = open(os.path.join(uc.ROOT, "examples", "segmentation", "segmentation_spark.py")).read()
  assert '"--ignore_index"' in src and '"--class_weights"' in src


# ----------------------------------------------------------------------------- kernel resources
@pytest.mark.skipif(not os.path.exists(uc.NVCC), reason="nvcc not found")
@pytest.mark.parametrize("source,kernel,instances", [
    ("elementwise.cu", "pixel_xent_kernel", 1),
    ("elementwise.cu", "pixel_xent_wide_kernel", 5),
    ("elementwise.cu", "seg_label_norm_kernel", 1),
    ("eval.cu", "seg_eval_metrics_kernel", 1),
    ("eval.cu", "seg_eval_wide_kernel", 5)])
def test_loss_option_kernels_have_no_stack_frame_or_spills(source, kernel, instances, tmp_path):
  # the option instances: Lb0E in the mangled name is the template argument kOpt = false (the
  # default instances; tests/test_unet_classes_host.py has the wide ones)
  kernels = {k: v for k, v in uc._ptxas(source, tmp_path).items()
             if kernel in k and "Lb0E" not in k}
  assert len(kernels) == instances, sorted(kernels)
  bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
  assert not bad, "stack frame / spill stores / spill loads (bytes): {}".format(bad)

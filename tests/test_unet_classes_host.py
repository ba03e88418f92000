"""CPU tier of the U-Net beyond eight classes: class-count validation before anything touches a
device, the host metrics of the wide accumulator layout, the examples' ``--classes`` flag (with
the stand-in trainer of test_unet_finetune_host), the synthetic V-class labels and ptxas'
resource report of the wide kernels (needs nvcc, not a GPU)."""
import importlib
import math
import os
import re
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from tensorflowonspark_b200 import _build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin",
                                            "nvcc")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_unet_finetune_host as ft  # noqa: E402


# ----------------------------------------------------------------------------- validation
@pytest.mark.parametrize("classes", [0, 257, -3, 3.0, True, "21", None])
def test_bad_class_count_raises_before_any_allocation(classes, monkeypatch):
  from tensorflowonspark_b200.models import unet

  def no_alloc(*a, **k):
    raise AssertionError("allocated before validating its arguments")
  monkeypatch.setattr(unet, "_buf", no_alloc)
  monkeypatch.setattr(unet, "MobileNetV2Encoder", no_alloc)
  monkeypatch.setattr(torch, "zeros", no_alloc)
  with pytest.raises(ValueError):
    unet.UNetTrainer(batch=2, device="cuda:0", classes=classes)


def test_padded_classes():
  from tensorflowonspark_b200.models import unet
  assert [unet.padded_classes(v) for v in (1, 3, 8, 9, 16, 17, 21, 150, 255, 256)] == \
      [8, 8, 8, 16, 16, 24, 24, 152, 256, 256]


# ----------------------------------------------------------------------------- host metrics
def _wide_totals(V, cm, count=None, invalid=0, loss=0.0, images=2):
  from tensorflowonspark_b200.models import unet
  images_slot, conf, ld, n = unet.seg_eval_layout(V)
  assert (images_slot, conf, ld, n) == (4, 5, V, 5 + V * V)
  t = [0.0] * n
  t[unet.SEG_COUNT] = float(cm.sum()) if count is None else count
  t[unet.SEG_CORRECT] = float(np.trace(cm))
  t[unet.SEG_INVALID] = invalid
  t[unet.SEG_LOSS] = loss
  t[images_slot] = images
  t[conf:] = cm.reshape(-1).astype(np.float64).tolist()
  return t


def test_seg_eval_result_on_wide_totals():
  from tensorflowonspark_b200.models import unet
  V = 21
  cm = np.zeros((V, V))
  cm[0, 0], cm[0, 1], cm[1, 1], cm[2, 0] = 6, 2, 3, 1     # classes 3..20: empty unions
  cm[20, 20] = 4
  res = unet.seg_eval_result(_wide_totals(V, cm, loss=8.0), V)
  assert res["count"] == 16 and res["images"] == 2
  assert res["loss"] == 0.5 and res["accuracy"] == 13 / 16
  assert len(res["iou"]) == V
  want = {0: 6 / (8 + 7 - 6), 1: 3 / 5, 2: 0.0, 20: 1.0}
  for c, v in want.items():
    assert res["iou"][c] == pytest.approx(v, rel=1e-15)
  assert all(math.isnan(res["iou"][c]) for c in range(3, 20))
  assert res["mean_iou"] == pytest.approx(sum(want.values()) / 4, rel=1e-15)


def test_seg_eval_result_wide_raises_on_invalid_labels_and_handles_no_pixels():
  from tensorflowonspark_b200.models import unet
  V = 150
  cm = np.zeros((V, V))
  with pytest.raises(ValueError, match="outside"):
    unet.seg_eval_result(_wide_totals(V, cm, invalid=3), V)
  res = unet.seg_eval_result(_wide_totals(V, cm, count=0, images=0), V)
  assert res["count"] == 0 and math.isnan(res["loss"]) and math.isnan(res["mean_iou"])


def test_narrow_layout_is_unchanged():
  from tensorflowonspark_b200.models import unet
  assert unet.seg_eval_layout(3) == (unet.SEG_IMAGES, unet.SEG_CONFUSION, 8, unet.SEG_ACC) == \
      (68, 4, 8, 72)


# ----------------------------------------------------------------------------- examples
drivers = ft.drivers


def test_segmentation_classes_flag(drivers):
  drivers.seg.train(ft._seg_args(drivers.seg))
  assert ft._Trainer.made[-1].kw["classes"] == 3
  default_kw = dict(ft._Trainer.made[-1].kw)
  drivers.seg.train(ft._seg_args(drivers.seg, "--classes", "21"))
  assert ft._Trainer.made[-1].kw == dict(default_kw, classes=21)


def test_segmentation_dist_parses_classes():
  sys.path.insert(0, os.path.join(ROOT, "examples", "segmentation"))
  try:
    sys.modules.pop("segmentation", None)
    seg = importlib.import_module("segmentation")
    assert seg.define_flags().parse_args([]).classes == 3
    assert seg.define_flags().parse_args(["--classes", "150"]).classes == 150
  finally:
    sys.path.pop(0)
    sys.modules.pop("segmentation", None)


def test_segmentation_spark_classes(drivers):
  class Args(object):
    batch_size, learning_rate, input_mode, steps, epochs, num_examples = 2, 1e-3, "tf", 2, 1, 8

  drivers.spark.main_fun(Args(), ft._Ctx())
  assert ft._Trainer.made[-1].kw["classes"] == 3
  Args.classes = 150
  drivers.spark.main_fun(Args(), ft._Ctx())
  assert ft._Trainer.made[-1].kw["classes"] == 150
  rows = drivers.spark.synth_rows(3, 0, 150)
  assert rows[0][1].dtype == np.uint8 and rows[0][1].max() < 150


def test_inference_example_scores_the_classes_masks(monkeypatch):
  monkeypatch.syspath_prepend(os.path.join(ROOT, "examples", "segmentation"))
  sys.modules.pop("segmentation_inference", None)
  inf = importlib.import_module("segmentation_inference")
  from tensorflowonspark_b200.models import unet
  imgs, masks = inf.synth(2, 0)
  assert np.array_equal(masks, unet.synthetic_labels(imgs, 3))
  imgs, masks = inf.synth(2, 0, 21)
  assert np.array_equal(masks, unet.synthetic_labels(imgs, 21))
  src = open(os.path.join(ROOT, "examples", "segmentation", "segmentation_inference.py")).read()
  assert '"--classes"' in src


# ----------------------------------------------------------------------------- synthetic labels
def test_synthetic_labels():
  from tensorflowonspark_b200.models import unet
  g = torch.Generator().manual_seed(0)
  x = torch.randint(0, 256, (4, 64, 64, 3), dtype=torch.uint8, generator=g)
  tri = (x[..., 0] > 127).int() + (x[..., 1] > 200).int()
  assert torch.equal(unet.synthetic_labels(x, 3), tri)
  assert np.array_equal(unet.synthetic_labels(x.numpy(), 3), tri.numpy().astype(np.uint8))
  for V in (1, 2, 9, 21, 150, 256):
    y = unet.synthetic_labels(x, V)
    assert y.dtype == torch.int32
    assert set(y.unique().tolist()) == set(range(V)), V
    assert np.array_equal(unet.synthetic_labels(x.numpy(), V), y.numpy().astype(np.uint8))


# ----------------------------------------------------------------------------- kernel resources
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
@pytest.mark.parametrize("source,kernel", [("elementwise.cu", "pixel_xent_wide_kernel"),
                                           ("eval.cu", "seg_eval_wide_kernel"),
                                           ("eval.cu", "seg_predict_wide_kernel")])
def test_wide_kernels_have_no_stack_frame_or_spills(source, kernel, tmp_path):
  # the default instances: Lb1E in the mangled name is the template argument kOpt = true (the loss
  # options; tests/test_unet_loss_options_host.py has those)
  kernels = {k: v for k, v in _ptxas(source, tmp_path).items() if kernel in k and "Lb1E" not in k}
  assert len(kernels) == 5, sorted(kernels)     # one instance per group width 2, 4, 8, 16, 32
  bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
  assert not bad, "stack frame / spill stores / spill loads (bytes): {}".format(bad)

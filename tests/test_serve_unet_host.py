"""Host side of serving the segmentation U-Net: raw-bytes outputs and output selection in
pipeline._run_model, the export attributes of UNetTrainer, the checkpoint / export of
segmentation_spark.py (dry run with a stand-in trainer) and the resources of seg_predict."""
import importlib
import json
import os
import sys

import numpy as np
import pytest
import torch

from test_kernel_resources import NVCC, ptxas_report

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNET_SIG = {"serving_default": {
    "inputs": {"image": "image"}, "outputs": {"mask": "mask", "logits": "logits"},
    "input_dtypes": {"image": "uint8"}, "output_dtypes": {"mask": "uint8", "logits": "float32"}}}


class _Seg(object):
  """Stand-in replica: mask = first H*W bytes of the row, logits = those bytes as float32 / 2,
  score = the row sum (an output without a declared dtype)."""

  def __init__(self):
    self.selected, self.calls = None, 0

  def select_outputs(self, names):
    self.selected = list(names)
    self.calls += 1

  def __call__(self, image):
    x = np.asarray(image).reshape(len(image), -1)
    m = x[:, :6].reshape(-1, 2, 3)
    return {"mask": m.astype(np.uint8), "logits": m.astype(np.float32) / 2,
            "score": x.astype(np.int64).sum(1)}


def _args(outputs, batch=4):
  from tensorflowonspark_b200 import pipeline
  return pipeline.Namespace({"export_dir": "seg", "model_dir": None, "tag_set": None,
                             "signature_def_key": None, "batch_size": batch,
                             "input_mapping": {"image": "image"}, "output_mapping": outputs,
                             "num_gpus": 0})


def _run(model, outputs, cells):
  from tensorflowonspark_b200 import pipeline
  pipeline._model_cache.update(key=("seg", None, None, None), model=model, sig={"signatures": UNET_SIG})
  try:
    args = _args(outputs)
    return list(pipeline._run_model(iter([(c,) for c in cells]), args, args))
  finally:
    pipeline._model_cache.update(key=None, model=None, sig=None)


def test_declared_outputs_travel_as_bytes_in_row_order():
  rng = np.random.RandomState(1)
  cells = [rng.randint(0, 256, size=12, dtype=np.uint8).tobytes() for _ in range(11)]   # ragged tail
  m = _Seg()
  out = _run(m, {"mask": "m", "logits": "l", "score": "s"}, cells)
  assert m.selected == ["logits", "mask", "score"] and m.calls == 1    # once per partition
  assert len(out) == len(cells)
  for (lg, mk, sc), c in zip(out, cells):   # columns in sorted output-tensor order
    x = np.frombuffer(c, dtype=np.uint8)
    assert type(mk) is bytes and len(mk) == 6 and mk == x[:6].tobytes()
    assert type(lg) is bytes and len(lg) == 24
    assert np.array_equal(np.frombuffer(lg, dtype=np.float32), x[:6].astype(np.float32) / 2)
    assert type(sc) is int and sc == int(x.astype(np.int64).sum())    # undeclared: a plain value
  only = _run(_Seg(), {"mask": "mask"}, cells)
  assert [r[0] for r in only] == [c[:6] for c in cells]


def test_models_without_output_selection_are_unaffected():
  class Plain(object):
    def __call__(self, image):
      return {"mask": np.asarray(image).reshape(len(image), -1)[:, :2]}
  cells = [bytes([i, i + 1, 7]) for i in range(5)]
  assert [r[0] for r in _run(Plain(), {"mask": "mask"}, cells)] == [c[:2] for c in cells]


def test_unet_export_attributes():
  from tensorflowonspark_b200.models import unet
  assert unet.UNetTrainer.export_builder == "tensorflowonspark_b200.models.unet:build_served"
  assert unet.UNetTrainer.export_signatures == UNET_SIG
  assert set(unet.UNetTrainer.export_builder_args.fget(
      type("T", (), {"image": 128, "classes": 3})())) == {"image", "classes"}
  assert callable(unet.build_served) and hasattr(unet.ServedUNet, "select_outputs")


class _Trainer(object):
  """Stand-in with the U-Net's export attributes."""
  made = []
  export_builder = "tensorflowonspark_b200.models.unet:build_served"
  export_signatures = UNET_SIG
  export_builder_args = {"image": 128, "classes": 3}

  def __init__(self, **kw):
    self.kw, self.steps = kw, 0
    _Trainer.made.append(self)

  def synthetic_batch(self, seed=0):
    return torch.zeros(4, 8, 8, 3, dtype=torch.uint8), None

  def set_input(self, x, y=None):
    pass

  def train_step(self, *a):
    self.steps += 1
    return torch.tensor(1.0)

  def capture(self):
    pass

  def state_dict(self):
    return {"w": torch.full((3,), float(self.steps))}


class _Ctx(object):
  def __init__(self, rank):
    self.rank, self.world_size, self.num_workers, self.is_chief = rank, 1, 1, rank == 0

  def absolute_path(self, p):
    return os.path.abspath(p)

  def gradient_comm(self):
    return None


@pytest.fixture
def seg_spark(monkeypatch):
  from tensorflowonspark_b200.models import unet
  monkeypatch.setattr(unet, "UNetTrainer", _Trainer)
  monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
  monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
  monkeypatch.syspath_prepend(os.path.join(ROOT, "examples", "segmentation"))
  sys.modules.pop("segmentation_spark", None)
  yield importlib.import_module("segmentation_spark")
  sys.modules.pop("segmentation_spark", None)


def test_segmentation_spark_checkpoints_and_exports_on_the_chief(seg_spark, tmp_path):
  from tensorflowonspark_b200.utils import checkpoint
  md, ed = str(tmp_path / "model"), str(tmp_path / "export")

  class Args(object):
    batch_size, learning_rate, input_mode, steps, epochs, num_examples = 4, 1e-3, "tf", 5, 1, 64
    model_dir, export_dir = md, ed

  seg_spark.main_fun(Args(), _Ctx(rank=1))              # a worker writes nothing
  assert not os.path.exists(md) and not os.path.exists(ed)
  seg_spark.main_fun(Args(), _Ctx(rank=0))
  step, state = checkpoint.load(md)
  assert step == 5 and torch.equal(state["w"], torch.full((3,), 6.0))
  for d in (md, ed):
    sig = json.load(open(os.path.join(d, "signature.json")))
    assert sig["builder"] == "tensorflowonspark_b200.models.unet:build_served"
    assert sig["builder_args"] == {"image": 128, "classes": 3}
    assert sig["signatures"] == UNET_SIG
  assert os.path.exists(os.path.join(ed, "weights.pt"))


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not found")
def test_seg_predict_does_not_spill(tmp_path):
  kernels = ptxas_report("eval.cu", tmp_path)
  pred = {k: v for k, v in kernels.items() if "seg_predict" in k}
  assert pred, "no seg_predict kernel in the ptxas report of eval.cu"
  assert all(v == (0, 0, 0) for v in pred.values()), pred

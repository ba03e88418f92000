"""Multi-label ResNet classifiers, host side (no GPU): argument checks, binding refusals, the
float64 binary cross-entropy and evaluation references the GPU tests compare against, eval_end's
keys on hand-built totals, the multi-label head and labels, load_backbone between softmax and
multi-label trainers, the export arguments and signature, and the example's --multi_label flag."""
import importlib
import json
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from tensorflowonspark_b200.models import resnet
from tensorflowonspark_b200.ops import igemm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_example_drivers_dryrun as dry  # noqa: E402
import test_unet_classes_host as uc  # noqa: E402
from test_example_drivers_dryrun import fake_gpu  # noqa: E402,F401  (fixture)

NAN = float("nan")


class _Plan(object):
  def set_reverse(self, flag):
    pass


@pytest.fixture
def cpu_plans(monkeypatch):
  """Trainers built on the CPU: every igemm plan builder returns a placeholder."""
  for name in ("conv_fprop", "conv_dgrad", "conv_wgrad", "stem_fprop", "stem_wgrad", "gemm",
               "gemm_wgrad"):
    monkeypatch.setattr(igemm, name, lambda *a, **k: _Plan())


class _Allocated(Exception):
  pass


@pytest.fixture
def no_alloc(monkeypatch):
  """Building a parameter store is the first allocation of both trainers: make it fail loudly."""
  def boom(*a, **k):
    raise _Allocated()
  monkeypatch.setattr(resnet, "ParamStore", boom)


# ------------------------------------------------------------------ float64 references
def softplus(x):
  return x.clamp(min=0) + torch.log1p(torch.exp(-x.abs()))


def ref_bce(logits, targets, V, eps=0.0, pos_weight=None):
  """float64 per-element loss p t softplus(-l) + (1 - t) softplus(l) and its gradient
  sigmoid(l) (p t + 1 - t) - p t over the first V columns, t = y (1 - eps) + eps / 2 with y the
  nonzero bytes of ``targets``."""
  l = logits[:, :V].double().cpu()
  y = (targets[:, :V].cpu() != 0).double()
  t = y * (1 - eps) + eps / 2
  p = torch.ones(V, dtype=torch.float64) if pos_weight is None else \
      torch.as_tensor(pos_weight, dtype=torch.float64).cpu()
  pt = p * t
  loss = pt * softplus(-l) + (1 - t) * softplus(l)
  grad = torch.sigmoid(l) * (pt + 1 - t) - pt
  return loss, grad


def ref_exact_rows(logits, targets, V):
  """Rows whose prediction (l > 0 per class) equals the target (nonzero byte) everywhere."""
  return int(((logits[:, :V].cpu() > 0) == (targets[:, :V].cpu() != 0)).all(1).sum())


def ref_multilabel_acc(logits, targets, n, V):
  """The multilabel_eval_metrics accumulator (8 + 3 V float64 values) of rows [0, n)."""
  L = logits[:n, :V].double().cpu()
  Y = targets[:n, :V].cpu().long()
  bad = (Y > 1).any(1)
  L, Y = L[~bad], Y[~bad]
  pred, pos = L > 0, Y == 1
  loss = torch.where(pos, softplus(-L), softplus(L))
  ok = pred == pos
  acc = [float((~bad).sum()), float(bad.sum()), float(loss.sum()), float(ok.sum()),
         float(ok.all(1).sum()), 0.0, 0.0, 0.0]
  acc += (pred & pos).sum(0).double().tolist()
  acc += (pred & ~pos).sum(0).double().tolist()
  acc += (~pred & pos).sum(0).double().tolist()
  return acc


def _same_nan(a, b):
  return (a != a and b != b) or a == b


def _assert_totals(got, want):
  assert set(got) == set(want)
  for k in want:
    if k == "f1_per_class":
      assert len(got[k]) == len(want[k]) and all(_same_nan(a, b) for a, b in zip(got[k], want[k]))
    else:
      assert _same_nan(got[k], want[k]) or math.isclose(got[k], want[k], rel_tol=1e-12), k


# ------------------------------------------------------------------ argument checks
@pytest.mark.parametrize("trainer", ["ResNetTrainer", "CifarResNetTrainer"])
@pytest.mark.parametrize("kw,match", [
    ({"multi_label": 1}, "multi_label must be a bool"),
    ({"multi_label": "yes"}, "multi_label must be a bool"),
    ({"multi_label": None}, "multi_label must be a bool"),
    ({"pos_weight": [1.0] * 5}, "needs multi_label=True"),
    ({"multi_label": True, "pos_weight": [1.0] * 4}, "one value per class"),
    ({"multi_label": True, "pos_weight": [1.0] * 6}, "one value per class"),
    ({"multi_label": True, "pos_weight": [1.0, 2.0, NAN, 1.0, 1.0]}, "finite and >= 0"),
    ({"multi_label": True, "pos_weight": [1.0, math.inf, 1.0, 1.0, 1.0]}, "finite and >= 0"),
    ({"multi_label": True, "pos_weight": [1.0, 1.0, -0.5, 1.0, 1.0]}, "finite and >= 0"),
    ({"multi_label": True, "pos_weight": 3.0}, "sequence of 5 numbers"),
    ({"multi_label": True, "pos_weight": ["a"] * 5}, "sequence of 5 numbers"),
])
def test_bad_multilabel_arguments_raise_before_allocation(no_alloc, trainer, kw, match):
  with pytest.raises(ValueError, match=match):
    getattr(resnet, trainer)(device="cpu", num_classes=5, **kw)


def test_pos_weight_is_refused_on_an_inference_trainer(no_alloc):
  with pytest.raises(ValueError, match="training=False"):
    resnet.ResNetTrainer(device="cpu", num_classes=5, training=False, multi_label=True,
                         pos_weight=[1.0] * 5)


@pytest.mark.parametrize("kw", [{"multi_label": True}, {"multi_label": False},
                                {"multi_label": True, "pos_weight": [0.0, 1.0, 2.5, 1e3, 1]},
                                {"multi_label": True, "pos_weight": torch.ones(5)},
                                {"multi_label": True, "training": False}])
def test_good_multilabel_arguments_pass_the_checks(no_alloc, kw):
  with pytest.raises(_Allocated):
    resnet.ResNetTrainer(device="cpu", num_classes=5, **kw)


# ------------------------------------------------------------------ binding refusals
def _C():
  from tensorflowonspark_b200 import ops
  return ops.C()


@pytest.mark.parametrize("case,match", [
    ({"label_smoothing": -0.1}, "label_smoothing must be in"),
    ({"label_smoothing": NAN}, "label_smoothing must be in"),
    ({"label_smoothing": 1.5}, "label_smoothing must be in"),
    ({"V": 0}, r"need 1 <= V <= ld"),
    ({"V": 17}, r"need 1 <= V <= ld"),
    ({"targets": torch.zeros(4, 9, dtype=torch.uint8)}, r"targets must be \[rows, V\]"),
    ({"targets": torch.zeros(3, 10, dtype=torch.uint8)}, r"targets must be \[rows, V\]"),
    ({"dlogits": torch.zeros(4, 8, dtype=torch.bfloat16)}, r"ldd >= V"),
    ({"pos_weight": torch.ones(9)}, r"pos_weight must hold V = 10"),
])
def test_sigmoid_bce_binding_refuses_before_the_launch(case, match):
  """Shapes and values are checked before the tensors' devices: CPU tensors reach no launch."""
  a = {"logits": torch.zeros(4, 16), "targets": torch.zeros(4, 10, dtype=torch.uint8),
       "dlogits": None, "loss_sum": torch.zeros(1), "correct": None, "V": 10, "scale": 0.025}
  a.update(case)
  with pytest.raises(ValueError, match=match):
    _C().sigmoid_bce(**a)
  good = dict(a, V=10, label_smoothing=0.1, targets=torch.zeros(4, 10, dtype=torch.uint8),
              dlogits=None, pos_weight=None)
  with pytest.raises(RuntimeError, match="CUDA tensor"):   # good arguments get to the tensor checks
    _C().sigmoid_bce(**good)


@pytest.mark.parametrize("case,match", [
    ({"V": 0}, r"need 1 <= V <= ld"),
    ({"V": 17}, r"need 1 <= V <= ld"),
    ({"targets": torch.zeros(4, 11, dtype=torch.uint8)}, r"targets must be \[rows, V\]"),
    ({"acc": torch.zeros(37, dtype=torch.float64)}, r"acc needs 8 \+ 3 V = 38 slots"),
])
def test_multilabel_eval_metrics_binding_refuses_before_the_launch(case, match):
  a = {"logits": torch.zeros(4, 16), "targets": torch.zeros(4, 10, dtype=torch.uint8),
       "n_valid": torch.zeros(1, dtype=torch.int32), "acc": torch.zeros(38, dtype=torch.float64),
       "V": 10}
  a.update(case)
  with pytest.raises(ValueError, match=match):
    _C().multilabel_eval_metrics(*a.values())
  assert _C().multilabel_eval_slots(10) == 38


# ------------------------------------------------------------------ ptxas
@pytest.mark.skipif(not os.path.exists(uc.NVCC), reason="nvcc not found")
@pytest.mark.parametrize("source,kernel,instances", [
    ("elementwise.cu", "sigmoid_bce_kernel", 4),          # plain, smoothed, pos_weight, both
    ("eval.cu", "multilabel_eval_metrics_kernel", 1)])
def test_multilabel_kernels_have_no_stack_frame_or_spills(source, kernel, instances, tmp_path):
  kernels = {k: v for k, v in uc._ptxas(source, tmp_path).items() if kernel in k}
  assert len(kernels) == instances, sorted(kernels)
  bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
  assert not bad, "stack frame / spill stores / spill loads (bytes): {}".format(bad)


# ------------------------------------------------------------------ the references
@pytest.mark.parametrize("V", [1, 7, 20, 1001])
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("weighted", [False, True])
def test_bce_reference_matches_torch(V, eps, weighted):
  g = torch.Generator().manual_seed(V)
  logits = torch.randn(16, V + 3, generator=g, dtype=torch.float64) * 4
  logits[0, :V] = 1e4              # saturated rows: the stable softplus keeps them finite
  logits[1, :V] = -1e4
  y = torch.randint(0, 2, (16, V), generator=g, dtype=torch.uint8)
  y[2] = 7                         # any nonzero byte is a positive in training
  pw = torch.rand(V, generator=g, dtype=torch.float64) * 3 if weighted else None
  loss, grad = ref_bce(logits, y, V, eps, pw)
  x = logits[:, :V].clone().requires_grad_(True)
  t = (y != 0).double() * (1 - eps) + eps / 2
  want = F.binary_cross_entropy_with_logits(x, t, pos_weight=pw, reduction="none")
  want.sum().backward()
  assert bool(torch.isfinite(loss).all() and torch.isfinite(grad).all())
  torch.testing.assert_close(loss, want.detach(), rtol=1e-12, atol=1e-12)
  torch.testing.assert_close(grad, x.grad, rtol=1e-12, atol=1e-12)
  # the mean over B x V is BCEWithLogitsLoss(reduction="mean")
  mean = F.binary_cross_entropy_with_logits(logits[:, :V], t, pos_weight=pw)
  assert math.isclose(float(loss.mean()), float(mean), rel_tol=1e-12)


def _hand_case():
  """5 rows x 4 classes: class 3 is empty (never a target, never predicted), row 1 is
  all-negative and right, row 2 holds a NaN logit (predicts negative), row 4 has an invalid byte."""
  L = torch.tensor([[2.0, -1.0, 0.5, -3.0],
                    [-1.0, -2.0, -0.5, -1.0],
                    [NAN, 1.0, -1.0, -2.0],
                    [0.0, 3.0, 2.0, -0.1],
                    [1.0, 1.0, 1.0, 1.0]])
  Y = torch.tensor([[1, 0, 0, 0],
                    [0, 0, 0, 0],
                    [1, 1, 0, 0],
                    [1, 0, 1, 0],
                    [1, 2, 0, 0]], dtype=torch.uint8)
  return L, Y


def test_eval_reference_and_totals_on_a_hand_built_case():
  L, Y = _hand_case()
  acc = ref_multilabel_acc(L, Y, 4, 4)   # rows 0 .. 3: all valid
  # predictions: [1,0,1,0] [0,0,0,0] [0,1,0,0] [0,1,1,0]; row 2's NaN predicts negative
  assert acc[:2] == [4.0, 0.0] and acc[3:5] == [12.0, 1.0]
  assert acc[8:12] == [1.0, 1.0, 1.0, 0.0]       # TP per class
  assert acc[12:16] == [0.0, 1.0, 1.0, 0.0]      # FP
  assert acc[16:20] == [2.0, 0.0, 0.0, 0.0]      # FN
  assert acc[2] != acc[2]                        # the NaN logit makes the loss NaN
  f1 = [2 / 4, 2 / 3, 2 / 3, NAN]
  TP, FP, FN = 3.0, 2.0, 2.0
  _assert_totals(resnet.multilabel_totals(acc, 4), {
      "count": 4, "loss": NAN, "binary_accuracy": 12 / 16, "exact_match": 1 / 4,
      "precision": TP / (TP + FP), "recall": TP / (TP + FN), "f1": 2 * TP / (2 * TP + FP + FN),
      "macro_f1": sum(f1[:3]) / 3, "f1_per_class": f1})
  # without the NaN row: a finite loss, the mean over count * V
  L2 = L.clone()
  L2[2, 0] = -4.0
  acc = ref_multilabel_acc(L2, Y, 4, 4)
  want = float(torch.where(Y[:4] == 1, softplus(-L2[:4].double()), softplus(L2[:4].double())).sum())
  got = resnet.multilabel_totals(acc, 4)
  assert math.isclose(got["loss"], want / 16, rel_tol=1e-12)
  # partial n_valid: rows [0, 2) only; classes 1 and 3 are empty there, class 2 has one FP
  acc = ref_multilabel_acc(L, Y, 2, 4)
  got = resnet.multilabel_totals(acc, 4)
  assert got["count"] == 2 and got["exact_match"] == 0.5 and got["recall"] == 1.0
  assert got["precision"] == 0.5 and got["f1"] == 2 / 3
  assert all(_same_nan(a, b) for a, b in zip(got["f1_per_class"], [1.0, NAN, 0.0, NAN]))
  assert got["macro_f1"] == 0.5


def test_invalid_bytes_raise_and_empty_totals_are_nan():
  L, Y = _hand_case()
  acc = ref_multilabel_acc(L, Y, 5, 4)
  assert acc[:2] == [4.0, 1.0]                   # row 4 is counted as invalid, not scored
  with pytest.raises(ValueError, match="1 row\\(s\\) with a label byte other than 0 or 1"):
    resnet.multilabel_totals(acc, 4)
  got = resnet.multilabel_totals([0.0] * (8 + 3 * 4), 4)
  assert got["count"] == 0 and all(got[k] != got[k] for k in (
      "loss", "binary_accuracy", "exact_match", "precision", "recall", "f1", "macro_f1"))
  # all-negative targets predicted negative: every class is empty, accuracy is perfect
  acc = ref_multilabel_acc(-torch.ones(3, 4), torch.zeros(3, 4, dtype=torch.uint8), 3, 4)
  got = resnet.multilabel_totals(acc, 4)
  assert got["binary_accuracy"] == 1.0 and got["exact_match"] == 1.0
  assert got["precision"] != got["precision"] and got["macro_f1"] != got["macro_f1"]


# ------------------------------------------------------------------ head layout and labels
@pytest.mark.parametrize("V,VP", [(1, 8), (20, 24), (1001, 1008)])
@pytest.mark.parametrize("training", [True, False])
def test_multilabel_head_is_the_padded_head(cpu_plans, V, VP, training):
  net = resnet.ResNetTrainer(depth=50, batch=2, image=32, num_classes=V, device="cpu",
                             training=training, multi_label=True)
  ref = resnet.ResNetTrainer(depth=50, batch=2, image=32, num_classes=V, device="cpu",
                             training=training)
  st = net.store
  assert net.VP == VP and st.by_name["fc.w"]["shape"] == (VP, 2048)
  assert torch.equal(st.master, ref.store.master)       # the head (and all else) is unchanged
  assert not st.m(st.by_name["fc.w"])[V:].any() and not st.m(st.by_name["fc.b"]).any()
  assert net.labels.shape == (2, V) and net.labels.dtype == torch.uint8
  assert ref.labels.shape == (2,) and ref.labels.dtype == torch.int32
  assert net.pos_weight is None
  assert net.state_dict().keys() == ref.state_dict().keys()


def test_synthetic_batch_and_labels(cpu_plans):
  net = resnet.CifarResNetTrainer(depth=20, batch=64, num_classes=20, device="cpu",
                                  multi_label=True, pos_weight=[2.0] * 20)
  assert net.labels.shape == (64, 20) and net.labels.dtype == torch.uint8
  assert net.pos_weight.dtype == torch.float32 and net.pos_weight.tolist() == [2.0] * 20
  x, y = net.synthetic_batch(seed=3)
  assert x.shape == (64, 32, 32, 3) and y.shape == (64, 20) and y.dtype == torch.uint8
  assert set(y.unique().tolist()) == {0, 1} and 0.4 < float(y.float().mean()) < 0.6
  assert torch.equal(y, net.synthetic_batch(seed=3)[1])
  assert not torch.equal(y, net.synthetic_batch(seed=4)[1])
  net.set_input(x, y.bool())                            # bool targets are staged as 0 / 1 bytes
  assert torch.equal(net.labels, y)


# ------------------------------------------------------------------ load_backbone
def _cifar(V, multi_label, seed):
  net = resnet.CifarResNetTrainer(depth=20, batch=1, num_classes=V, device="cpu", seed=seed,
                                  multi_label=multi_label)
  net.running.tensor().uniform_(0.5, 2.0)
  return net


@pytest.mark.parametrize("src_ml,dst_ml", [(False, True), (True, False)])
def test_load_backbone_between_softmax_and_multilabel(cpu_plans, src_ml, dst_ml):
  src = _cifar(10, src_ml, seed=1)
  with torch.no_grad():
    src.store.master.add_(torch.randn(src.store.total, generator=torch.Generator().manual_seed(0)))
  sd = src.state_dict()
  dst, fresh = _cifar(20, dst_ml, seed=2), _cifar(20, dst_ml, seed=2)
  dst.load_backbone(sd)
  for s in dst.store.order:
    want = fresh.store.m(s) if s["name"] in ("fc.w", "fc.b") else sd[s["name"]]
    assert torch.equal(dst.store.m(s), want), s["name"]
  assert torch.equal(dst.running.tensor(), sd["__running__"])


def test_load_backbone_resnet50_1000_softmax_to_20_multilabel(cpu_plans):
  src = resnet.ResNetTrainer(depth=50, batch=1, image=32, device="cpu", training=False, seed=1)
  dst = resnet.ResNetTrainer(depth=50, batch=1, image=32, num_classes=20, device="cpu",
                             training=False, seed=2, multi_label=True)
  head = [dst.store.m(dst.store.by_name[n]).clone() for n in ("fc.w", "fc.b")]
  sd = src.state_dict()
  dst.load_backbone(sd)
  assert torch.equal(dst.store.m(dst.store.by_name["layer4.2.u3.conv.w"]), sd["layer4.2.u3.conv.w"])
  assert all(torch.equal(dst.store.m(dst.store.by_name[n]), t)
             for n, t in zip(("fc.w", "fc.b"), head))


# ------------------------------------------------------------------ export
def test_export_args_signature_and_old_exports(cpu_plans, monkeypatch, tmp_path):
  from tensorflowonspark_b200.utils import checkpoint
  made = []

  class _Served(object):
    def __init__(self, state, **kw):
      made.append(kw)

  monkeypatch.setattr(resnet, "ServedResNet", _Served)
  ml = resnet.ResNetTrainer(depth=50, batch=1, image=32, num_classes=20, device="cpu",
                            training=False, multi_label=True)
  sm = resnet.ResNetTrainer(depth=50, batch=1, image=32, num_classes=20, device="cpu",
                            training=False)
  assert sm.export_builder_args == {"depth": 50, "image": 32, "num_classes": 20}
  assert ml.export_builder_args == dict(sm.export_builder_args, multi_label=True)
  assert sm.export_signatures == {"serving_default": {
      "inputs": {"image": "image"}, "outputs": {"logits": "logits", "prediction": "prediction"},
      "input_dtypes": {"image": "uint8"}}}
  sig = ml.export_signatures["serving_default"]
  assert sig["outputs"] == {"logits": "logits", "prediction": "prediction"}
  assert sig["output_dtypes"] == {"prediction": "uint8"}
  assert sig["output_shapes"] == {"logits": [-1, 20], "prediction": [-1, 20]}
  for net, want in ((ml, True), (sm, False)):
    d = str(tmp_path / ("ml" if want else "sm"))
    checkpoint.export_model(net, d)
    with open(os.path.join(d, "signature.json")) as f:
      assert json.load(f)["signatures"] == net.export_signatures
    checkpoint.load_model(d)
    assert made[-1]["multi_label"] is want and made[-1]["num_classes"] == 20
  # an export written before multi-label heads existed: no key, served as softmax
  resnet.build_served({}, depth=50, image=32, num_classes=20, batch=4)
  assert made[-1]["multi_label"] is False


# ------------------------------------------------------------------ the example's flag
class _EvalTrainer(dry._Trainer):
  def evaluate(self, batches, averaged=False):
    keys = ("binary_accuracy", "exact_match", "f1", "macro_f1")
    if self.kw.get("multi_label"):
      return dict({k: 0.5 for k in keys}, count=8, loss=0.25, precision=0.5, recall=0.5,
                  f1_per_class=[0.5])
    return {"count": 8, "loss": 0.25, "top1": 0.5, "top5": 0.75}


def test_resnet_spark_multi_label_flag(fake_gpu, monkeypatch, tmp_path, capsys):
  from tensorflowonspark_b200.utils import metrics
  monkeypatch.setattr(resnet, "ResNetTrainer", _EvalTrainer)
  monkeypatch.setattr(resnet, "CifarResNetTrainer", _EvalTrainer)
  mod = importlib.import_module("resnet_spark")
  assert mod.parse([]).multi_label is False
  mt = str(tmp_path / "steps.jsonl")
  base = ["resnet_spark.py", "--batch_size", "4", "--image", "64", "--train_steps", "10",
          "--eval_steps", "2", "--metrics", mt]
  mod.main_fun(base, dry._Ctx())
  net = dry._Trainer.made[-1]
  assert set(net.kw) == {"depth", "batch", "image", "device", "comm", "lr"}   # as before
  assert "top1 0.5000 top5 0.7500 (8 images)" in capsys.readouterr().out
  mod.main_fun(base + ["--multi_label", "--ema_decay", "0.9"], dry._Ctx())
  net = dry._Trainer.made[-1]
  assert net.kw["multi_label"] is True
  out = capsys.readouterr().out
  assert "loss 0.2500 binary_accuracy 0.5000 exact_match 0.5000 f1 0.5000 macro_f1 0.5000" in out
  (rec,) = [r for r in metrics.read(mt + ".rank0") if "eval_f1" in r]
  assert {k for k in rec if k.startswith("eval_")} == {
      "eval_loss", "eval_binary_accuracy", "eval_exact_match", "eval_f1", "eval_macro_f1",
      "eval_count", "eval_avg_loss", "eval_avg_binary_accuracy", "eval_avg_exact_match",
      "eval_avg_f1", "eval_avg_macro_f1"}
  mod.main_fun(base + ["--multi_label", "--model", "resnet56"], dry._Ctx())
  assert dry._Trainer.made[-1].kw["multi_label"] is True

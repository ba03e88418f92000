"""ResNet classifiers for any label set, host side (no GPU): argument checks, the padded head's
layout, load_backbone's key selection and checks, the float64 label-smoothed cross-entropy the GPU
tests compare against, and the example flags."""
import hashlib
import importlib
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
from test_example_drivers_dryrun import fake_gpu  # noqa: E402,F401  (fixture)


class _Plan(object):
  def set_reverse(self, flag):
    pass


@pytest.fixture
def cpu_plans(monkeypatch):
  """Trainers built on the CPU: every igemm plan builder returns a placeholder."""
  for name in ("conv_fprop", "conv_dgrad", "conv_wgrad", "stem_fprop", "stem_wgrad", "gemm",
               "gemm_wgrad"):
    monkeypatch.setattr(igemm, name, lambda *a, **k: _Plan())


def ref_smoothed_xent(logits, labels, V, eps):
  """float64 per-row loss lse - (1 - eps) l_y - (eps / V) sum_j l_j and its gradient
  softmax - (1 - eps) onehot - eps / V over the first V columns of ``logits``."""
  l = logits[:, :V].double()
  y = labels.long()
  loss = torch.logsumexp(l, 1) - (1 - eps) * l.gather(1, y[:, None])[:, 0] - eps / V * l.sum(1)
  target = torch.full_like(l, eps / V)
  target[torch.arange(len(y)), y] += 1 - eps
  return loss, torch.softmax(l, 1) - target


# ------------------------------------------------------------------ argument checks
class _Allocated(Exception):
  pass


@pytest.fixture
def no_alloc(monkeypatch):
  """Building a parameter store is the first allocation of both trainers: make it fail loudly."""
  def boom(*a, **k):
    raise _Allocated()
  monkeypatch.setattr(resnet, "ParamStore", boom)


@pytest.mark.parametrize("trainer", ["ResNetTrainer", "CifarResNetTrainer"])
@pytest.mark.parametrize("kw", [{"num_classes": 0}, {"num_classes": -3}, {"num_classes": True},
                                {"num_classes": 10.0}, {"num_classes": "10"},
                                {"label_smoothing": -0.1}, {"label_smoothing": 1.5},
                                {"label_smoothing": float("nan")}, {"label_smoothing": math.inf},
                                {"label_smoothing": "0.1"}, {"label_smoothing": None},
                                {"label_smoothing": True}])
def test_bad_head_arguments_raise_before_allocation(no_alloc, trainer, kw):
  with pytest.raises(ValueError, match=next(iter(kw))):
    getattr(resnet, trainer)(device="cpu", **kw)


@pytest.mark.parametrize("kw", [{"num_classes": 1}, {"num_classes": 37},
                                {"label_smoothing": 0}, {"label_smoothing": 1},
                                {"label_smoothing": 0.1}])
def test_good_head_arguments_pass_the_checks(no_alloc, kw):
  with pytest.raises(_Allocated):
    resnet.ResNetTrainer(device="cpu", **kw)


@pytest.mark.parametrize("eps", [-0.1, 1.01, float("nan"), float("inf"), -float("inf")])
def test_softmax_xent_rejects_bad_label_smoothing_before_the_launch(eps):
  """The binding checks eps first, so CPU tensors reach no launch and no other check."""
  from tensorflowonspark_b200 import ops
  logits, labels, loss = torch.zeros(2, 16), torch.zeros(2, dtype=torch.int32), torch.zeros(1)
  with pytest.raises(ValueError, match="label_smoothing must be in"):
    ops.C().softmax_xent(logits, labels, None, loss, None, 10, 0.5, label_smoothing=eps)
  with pytest.raises(RuntimeError, match="logits"):    # a good eps gets to the tensor checks
    ops.C().softmax_xent(logits, labels, None, loss, None, 10, 0.5, label_smoothing=0.1)


def test_label_smoothing_is_stored_as_float(cpu_plans):
  net = resnet.CifarResNetTrainer(depth=20, batch=1, device="cpu", label_smoothing=1)
  assert net.label_smoothing == 1.0 and type(net.label_smoothing) is float
  assert resnet.CifarResNetTrainer(depth=20, batch=1, device="cpu").label_smoothing == 0.0


# ------------------------------------------------------------------ head layout
# (store.total, store.decay_end, sha256 of [(name, shape, offset)]) of ResNet-50 before heads were
# padded: a class count that is a multiple of 8 must keep exactly this layout
UNPADDED_LAYOUT = {8: (23543688, 23490560, "2c1fcfd0d4c892b7"),
                   1000: (25576296, 25522176, "3d2a821863e2208c")}


def _layout(st):
  lay = repr([(s["name"], s["shape"], s["offset"]) for s in st.order]).encode()
  return st.total, st.decay_end, hashlib.sha256(lay).hexdigest()[:16]


@pytest.mark.parametrize("V,VP", [(1, 8), (7, 8), (8, 8), (37, 40), (1000, 1000), (1001, 1008)])
@pytest.mark.parametrize("training", [True, False])
def test_head_is_padded_to_a_multiple_of_8_with_zero_rows(cpu_plans, V, VP, training):
  net = resnet.ResNetTrainer(depth=50, batch=2, image=32, num_classes=V, device="cpu",
                             training=training)
  st = net.store
  assert net.num_classes == V and net.VP == VP
  assert st.by_name["fc.w"]["shape"] == (VP, 2048) and st.by_name["fc.b"]["shape"] == (VP,)
  assert tuple(net.logits.shape) == (2, VP) and net.logits.dtype == torch.float32
  if training:
    assert tuple(net.dlogits.shape) == (2, VP) and net.dlogits.dtype == torch.bfloat16
  w, b = st.m(st.by_name["fc.w"]), st.m(st.by_name["fc.b"])
  assert not w[V:].any() and not b.any() and not st.w(st.by_name["fc.w"])[V:].any()
  assert w[:V].abs().amax(1).min() > 0 and 0.005 < float(w[:V].std()) < 0.02   # normal(0.01)
  if V in UNPADDED_LAYOUT:
    assert _layout(st) == UNPADDED_LAYOUT[V]


# ------------------------------------------------------------------ load_backbone
def _snapshot(net):
  st = net.store
  return [t.clone() for t in (st.master, st.weights, st.aux32, net.running.tensor())]


def _same(a, b):
  return all(torch.equal(x, y) for x, y in zip(a, b))


def _cifar(depth=20, V=10, seed=1234):
  net = resnet.CifarResNetTrainer(depth=depth, batch=1, num_classes=V, device="cpu", seed=seed)
  net.running.tensor().uniform_(0.5, 2.0)   # something other than the initial statistics
  return net


def test_load_backbone_takes_everything_but_the_head(cpu_plans):
  src = _cifar(V=100, seed=1)
  with torch.no_grad():
    src.store.master.add_(torch.randn(src.store.total, generator=torch.Generator().manual_seed(0)))
  sd = src.state_dict()
  dst, fresh = _cifar(V=37, seed=2), _cifar(V=37, seed=2)
  dst.optim.state1.uniform_()   # momentum: load_backbone leaves it alone
  before = {k: v.clone() for k, v in dst.optim.state_dict().items() if torch.is_tensor(v)}
  dst.load_backbone(sd)
  st = dst.store
  for s in st.order:
    got = st.m(s)
    if s["name"] in ("fc.w", "fc.b"):
      assert torch.equal(got, fresh.store.m(s)), s["name"]
    else:
      assert torch.equal(got, sd[s["name"]]), s["name"]
  assert torch.equal(dst.running.tensor(), sd["__running__"])
  assert torch.equal(st.weights, st.master.to(torch.bfloat16))
  assert torch.equal(st.aux32[:st.total - st.decay_end], st.master[st.decay_end:])
  after = {k: v for k, v in dst.optim.state_dict().items() if torch.is_tensor(v)}
  assert before.keys() == after.keys() and all(torch.equal(before[k], after[k]) for k in before)


def test_load_backbone_bottleneck_1000_to_37(cpu_plans):
  src = resnet.ResNetTrainer(depth=50, batch=1, image=32, device="cpu", training=False, seed=1)
  dst = resnet.ResNetTrainer(depth=50, batch=1, image=32, num_classes=37, device="cpu",
                             training=False, seed=2)
  fc = [dst.store.m(dst.store.by_name[n]).clone() for n in ("fc.w", "fc.b")]
  sd = src.state_dict()
  dst.load_backbone(sd)
  conv = dst.store.by_name["layer4.2.u3.conv.w"]
  assert torch.equal(dst.store.m(conv), sd["layer4.2.u3.conv.w"])
  assert all(torch.equal(dst.store.m(dst.store.by_name[n]), t) for n, t in zip(("fc.w", "fc.b"), fc))


def _mutate(sd, name, fn):
  sd = dict(sd)
  fn(sd, name)
  return sd


@pytest.mark.parametrize("case,match", [
    ("deeper_source", r"stage1\.3\.\S+ is not a tensor of this trainer"),
    ("shallower_source", r"is missing from the state"),
    ("missing_tensor", r"stage2\.0\.u1\.bn\.gamma \(32,\) is missing"),
    ("missing_running", r"__running__ .* is missing"),
    ("wrong_shape", r"stage3\.1\.u2\.conv\.w has shape \(64, 3, 3, 32\) in the state, "
                    r"\(64, 3, 3, 64\) in this trainer"),
    ("wrong_running", r"__running__ has shape"),
])
def test_failed_load_backbone_names_the_tensor_and_leaves_the_trainer_unchanged(cpu_plans, case,
                                                                                 match):
  dst = _cifar(V=37, seed=2)
  src = _cifar(depth={"deeper_source": 32, "shallower_source": 14}.get(case, 20), V=10, seed=1)
  sd = src.state_dict()
  if case == "missing_tensor":
    del sd["stage2.0.u1.bn.gamma"]
  elif case == "missing_running":
    del sd["__running__"]
  elif case == "wrong_shape":
    sd["stage3.1.u2.conv.w"] = torch.zeros(64, 3, 3, 32)
  elif case == "wrong_running":
    sd["__running__"] = sd["__running__"][:-8]
  before = _snapshot(dst)
  with pytest.raises(ValueError, match=match):
    dst.load_backbone(sd)
  assert _same(before, _snapshot(dst))


def test_load_state_dict_still_takes_the_head(cpu_plans):
  src, dst = _cifar(V=37, seed=1), _cifar(V=37, seed=2)
  dst.load_state_dict(src.state_dict())
  assert torch.equal(dst.store.master, src.store.master)


# ------------------------------------------------------------------ float64 reference
@pytest.mark.parametrize("V", [1, 10, 37, 1001])
@pytest.mark.parametrize("eps", [0.0, 0.1, 0.5, 1.0])
def test_reference_matches_torch_cross_entropy(V, eps):
  g = torch.Generator().manual_seed(V)
  logits = torch.randn(16, V + 5, generator=g, dtype=torch.float64) * 4
  y = torch.randint(0, V, (16,), generator=g, dtype=torch.int32)
  loss, grad = ref_smoothed_xent(logits, y, V, eps)
  x = logits[:, :V].clone().requires_grad_(True)
  want = F.cross_entropy(x, y.long(), label_smoothing=eps, reduction="none")
  want.sum().backward()
  torch.testing.assert_close(loss, want.detach(), rtol=1e-12, atol=1e-12)
  torch.testing.assert_close(grad, x.grad, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------ example flags
class _BackboneTrainer(dry._Trainer):
  def load_backbone(self, sd):
    self.backbone = sd


def _spark(argv, world=1):
  mod = importlib.import_module("resnet_spark")
  mod.main_fun(["resnet_spark.py", "--batch_size", "4", "--image", "64"] + argv, dry._Ctx(world))
  return dry._Trainer.made[-1]


def test_resnet_spark_flags(fake_gpu, monkeypatch, tmp_path):
  monkeypatch.setattr(resnet, "ResNetTrainer", _BackboneTrainer)
  monkeypatch.setattr(resnet, "CifarResNetTrainer", _BackboneTrainer)
  args = importlib.import_module("resnet_spark").parse([])
  assert (args.num_classes, args.label_smoothing, args.init_checkpoint) == (None, 0.0, None)
  # defaults: the trainer gets the arguments it always got
  net = _spark(["--train_steps", "2"])
  assert set(net.kw) == {"depth", "batch", "image", "device", "comm", "lr"}
  net = _spark(["--train_steps", "2", "--model", "resnet56"])
  assert set(net.kw) == {"depth", "batch", "device", "comm", "lr"}
  net = _spark(["--train_steps", "2", "--num_classes", "37", "--label_smoothing", "0.1"])
  assert net.kw["num_classes"] == 37 and net.kw["label_smoothing"] == 0.1
  # --init_checkpoint: the backbone of the newest checkpoint there, unless model_dir resumes
  src, dst = str(tmp_path / "imagenet"), str(tmp_path / "pets")
  _spark(["--train_steps", "20", "--model_dir", src, "--save_steps", "10"])
  net = _spark(["--train_steps", "2", "--num_classes", "37", "--model_dir", dst,
                "--init_checkpoint", src, "--save_steps", "2"])
  assert torch.equal(net.backbone["w"], torch.full((3,), 21.0)) and net.loaded is None
  net = _spark(["--train_steps", "2", "--model_dir", dst, "--init_checkpoint", src])
  assert not hasattr(net, "backbone") and net.loaded is not None
  with pytest.raises(ValueError, match="no checkpoint"):
    _spark(["--train_steps", "2", "--init_checkpoint", str(tmp_path / "empty")])


def test_resnet_cifar_label_smoothing_flag(fake_gpu):
  mod = importlib.import_module("resnet_cifar_main")
  assert mod.define_flags().parse_args([]).label_smoothing == 0.0
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "2"], mod.LocalContext())
  assert "label_smoothing" not in dry._Trainer.made[-1].kw
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "2", "--label_smoothing", "0.1"],
               mod.LocalContext())
  assert dry._Trainer.made[-1].kw["label_smoothing"] == 0.1

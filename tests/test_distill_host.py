"""Knowledge distillation for the ResNet trainers, host side (no GPU): the option and teacher-state
checks (all refused before anything is allocated), the float64 reference of the distillation loss
and its gradient that tests/test_gpu_distill.py compares the kernel against, the binding's refusals,
ptxas on csrc/distill.cu and the examples' distillation flags."""
import importlib
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from tensorflowonspark_b200.models import engine, resnet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_example_drivers_dryrun as dry  # noqa: E402
import test_unet_classes_host as uc  # noqa: E402
from test_example_drivers_dryrun import fake_gpu  # noqa: E402,F401  (fixture)
from test_mixup_host import _Allocated, cpu_plans, no_alloc  # noqa: E402,F401  (fixtures)

NAN = float("nan")
DISTILL_KW = ("teacher", "teacher_depth", "distill_alpha", "distill_temperature")
TRAINERS = {"ResNetTrainer": 50, "CifarResNetTrainer": 20}


def teacher_state(cls, depth, V):
  """A state_dict() of a ``cls`` trainer of ``depth`` with V classes, as zeros on the host."""
  return {k: torch.zeros(s) for k, s in resnet._state_shapes(cls, depth, V).items()}


# ------------------------------------------------------------------ float64 reference
def soft_target(labels, V, eps, lam, mixing):
  """Row i's hard target: s(y_i), or lam s(y_i) + (1 - lam) s(y_p(i)) with p(i) = B - 1 - i when
  mixing; s(y) = (1 - eps) onehot(y) + eps / V (timm's mixup_target)."""
  s = F.one_hot(labels.long(), V).double() * (1.0 - eps) + eps / V
  if not mixing:
    return s
  return lam * s + (1.0 - lam) * s.flip(0)


def ref_distill(s, z, labels, V, eps, alpha, T, lam=1.0, mixing=False, scale=None):
  """float64 (loss_sum, dlogits [B, V]) of the distillation loss of student logits s and teacher
  logits z (first V columns), scale 1 / B by default."""
  s, z = s[:, :V].double(), z[:, :V].double()
  B = s.shape[0]
  scale = 1.0 / B if scale is None else scale
  t = soft_target(labels, V, eps, lam, mixing)
  ls, lsT, lq = F.log_softmax(s, 1), F.log_softmax(s / T, 1), F.log_softmax(z / T, 1)
  q = lq.exp()
  ce = -(t * ls).sum(1)
  kl = (q * (lq - lsT)).sum(1)
  loss = ((1 - alpha) * ce + alpha * T * T * kl).sum() * scale
  d = ((1 - alpha) * (ls.exp() - t) + alpha * T * (lsT.exp() - q)) * scale
  return float(loss), d


def ref_hits(s, labels, V, lam=1.0, mixing=False):
  """The student's lowest-index arg-max against the dominant label (the row's own when lam >= 0.5
  or without a mix, its partner's otherwise)."""
  am = s[:, :V].argmax(1)
  dom = labels.long() if (not mixing or lam >= 0.5) else labels.long().flip(0)
  return int((am == dom).sum())


def torch_loss(s, z, y, V, eps, alpha, T, lam, mixing):
  """The loss as the issue states it in torch terms: F.cross_entropy (timm's soft-target
  cross-entropy when mixing) plus T^2 F.kl_div(batchmean)."""
  if mixing:
    hard = (-soft_target(y, V, eps, lam, True) * F.log_softmax(s, 1)).sum(1).mean()
  else:
    hard = F.cross_entropy(s, y.long(), label_smoothing=eps)
  kd = F.kl_div(F.log_softmax(s / T, 1), F.log_softmax(z / T, 1), log_target=True,
                reduction="batchmean")
  return (1 - alpha) * hard + alpha * T * T * kd


MIXES = [("none", 1.0), ("mixup", 0.3), ("cutmix", 0.75)]


@pytest.mark.parametrize("V", [10, 37, 1000])
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("T", [1.0, 4.0])
@pytest.mark.parametrize("alpha", [0.5, 1.0])
@pytest.mark.parametrize("mode,lam", MIXES)
def test_reference_matches_torch_autograd(V, eps, T, alpha, mode, lam):
  g = torch.Generator().manual_seed(V + int(10 * T))
  B = 6
  s = (torch.randn(B, V, generator=g, dtype=torch.float64) * 3).requires_grad_(True)
  z = torch.randn(B, V, generator=g, dtype=torch.float64) * 3
  y = torch.randint(0, V, (B,), generator=g, dtype=torch.int32)
  mixing = mode != "none"
  want = torch_loss(s, z, y, V, eps, alpha, T, lam, mixing)
  want.backward()
  loss, d = ref_distill(s.detach(), z, y, V, eps, alpha, T, lam, mixing)
  assert loss == pytest.approx(float(want.detach()), rel=1e-12, abs=1e-12)
  torch.testing.assert_close(d, s.grad, rtol=1e-10, atol=1e-12)


def test_reference_padding_columns_are_ignored():
  g = torch.Generator().manual_seed(3)
  s, z = torch.randn(4, 40, generator=g), torch.randn(4, 48, generator=g)
  y = torch.randint(0, 37, (4,), generator=g, dtype=torch.int32)
  a = ref_distill(s, z, y, 37, 0.1, 0.5, 2.0)
  s[:, 37:], z[:, 37:] = 1e4, -1e4
  b = ref_distill(s, z, y, 37, 0.1, 0.5, 2.0)
  assert a[0] == b[0] and torch.equal(a[1], b[1])


def test_dominant_label_rule():
  s = torch.tensor([[0.0, 5.0], [5.0, 0.0]])
  y = torch.tensor([1, 1], dtype=torch.int32)
  assert ref_hits(s, y, 2) == 1 and ref_hits(s, y, 2, 0.2, True) == 1
  y = torch.tensor([1, 0], dtype=torch.int32)
  assert ref_hits(s, y, 2, 0.6, True) == 2 and ref_hits(s, y, 2, 0.4, True) == 0


# ------------------------------------------------------------------ option checks
@pytest.mark.parametrize("trainer", sorted(TRAINERS))
@pytest.mark.parametrize("kw,match", [
    ({"distill_alpha": 0.0}, r"distill_alpha must be a real number in \(0, 1\]"),
    ({"distill_alpha": 1.5}, "distill_alpha"),
    ({"distill_alpha": -0.1}, "distill_alpha"),
    ({"distill_alpha": NAN}, "distill_alpha"),
    ({"distill_alpha": True}, "distill_alpha"),
    ({"distill_alpha": "0.5"}, "distill_alpha"),
    ({"distill_temperature": 0.0}, "distill_temperature must be a finite real number > 0"),
    ({"distill_temperature": -2.0}, "distill_temperature"),
    ({"distill_temperature": math.inf}, "distill_temperature"),
    ({"distill_temperature": NAN}, "distill_temperature"),
    ({"distill_temperature": None}, "distill_temperature"),
    ({"distill_temperature": 1e-50}, "that fp32 holds"),
    ({"distill_temperature": 1e39}, "that fp32 holds"),
    ({"teacher_depth": "50"}, "teacher_depth must be an int"),
    ({"teacher_depth": True}, "teacher_depth must be an int"),
    ({"teacher": [1, 2]}, "teacher must be a state_dict"),
])
def test_bad_distillation_options_raise_before_allocation(no_alloc, trainer, kw, match):
  with pytest.raises(ValueError, match=match):
    getattr(resnet, trainer)(device="cpu", num_classes=5, **kw)


@pytest.mark.parametrize("trainer", sorted(TRAINERS))
@pytest.mark.parametrize("kw", [{"distill_alpha": 0.7}, {"distill_temperature": 4.0},
                                {"teacher_depth": 50}, {"distill_alpha": 1.0,
                                                        "distill_temperature": 2}])
def test_distillation_options_need_a_teacher(no_alloc, trainer, kw):
  with pytest.raises(ValueError, match="need a teacher"):
    getattr(resnet, trainer)(device="cpu", num_classes=5, **kw)


@pytest.mark.parametrize("kw", [{"distill_alpha": 0.7}, {"distill_temperature": 4.0},
                                {"teacher_depth": 50}, {"teacher": "T"}])
def test_distillation_options_are_refused_on_an_inference_trainer(no_alloc, kw):
  if kw.get("teacher") == "T":
    kw = {"teacher": teacher_state(resnet.ResNetTrainer, 50, 5)}
  with pytest.raises(ValueError, match="training=True"):
    resnet.ResNetTrainer(device="cpu", num_classes=5, training=False, **kw)


@pytest.mark.parametrize("trainer", sorted(TRAINERS))
def test_teacher_is_refused_with_multi_label(no_alloc, trainer):
  cls = getattr(resnet, trainer)
  with pytest.raises(ValueError, match="multi_label"):
    cls(device="cpu", num_classes=5, multi_label=True,
        teacher=teacher_state(cls, TRAINERS[trainer], 5))


def _bad_states():
  R, C = resnet.ResNetTrainer, resnet.CifarResNetTrainer
  out = []
  st = teacher_state(R, 50, 5)
  del st["layer3.2.u2.conv.w"]
  out.append(("ResNetTrainer", {}, st, "layer3.2.u2.conv.w .* is missing"))
  st = teacher_state(R, 50, 5)
  del st["__running__"]
  out.append(("ResNetTrainer", {}, st, "__running__ .* missing .* running statistics"))
  st = teacher_state(R, 50, 5)
  st["extra.w"] = torch.zeros(3)
  out.append(("ResNetTrainer", {}, st, "extra.w is not a tensor of this model"))
  st = teacher_state(R, 50, 5)
  st["layer1.0.u2.bn.gamma"] = torch.zeros(65)
  out.append(("ResNetTrainer", {}, st, r"layer1.0.u2.bn.gamma has shape \(65,\)"))
  out.append(("ResNetTrainer", {}, teacher_state(R, 50, 20), "fc.w .* another class count"))
  out.append(("ResNetTrainer", {}, teacher_state(R, 101, 5), "is not a tensor|missing"))
  out.append(("ResNetTrainer", {"teacher_depth": 101}, teacher_state(R, 50, 5), "missing"))
  out.append(("ResNetTrainer", {"teacher_depth": 34}, teacher_state(R, 50, 5),
              "teacher_depth 34 is not a depth of ResNetTrainer"))
  out.append(("ResNetTrainer", {}, teacher_state(C, 20, 5), "has shape|not a tensor|missing"))
  out.append(("CifarResNetTrainer", {}, teacher_state(C, 56, 5), "missing|not a tensor"))
  out.append(("CifarResNetTrainer", {"teacher_depth": 21}, teacher_state(C, 20, 5),
              "teacher_depth 21 is not a depth of CifarResNetTrainer"))
  out.append(("CifarResNetTrainer", {}, teacher_state(C, 20, 12), "fc.w .* another class count"))
  out.append(("CifarResNetTrainer", {}, teacher_state(R, 50, 5), "not a tensor|missing"))
  return out


@pytest.mark.parametrize("trainer,kw,state,match", _bad_states())
def test_bad_teacher_states_raise_before_allocation(no_alloc, trainer, kw, state, match):
  depth = TRAINERS[trainer]
  with pytest.raises(ValueError, match=match):
    getattr(resnet, trainer)(depth=depth, device="cpu", num_classes=5, teacher=state, **kw)


@pytest.mark.parametrize("trainer,depth,tdepth", [("ResNetTrainer", 50, None),
                                                  ("ResNetTrainer", 50, 101),
                                                  ("ResNetTrainer", 50, 152),
                                                  ("CifarResNetTrainer", 20, 56),
                                                  ("CifarResNetTrainer", 20, None),
                                                  ("CifarResNetTrainer", 56, 110)])
def test_good_teachers_pass_the_checks(no_alloc, trainer, depth, tdepth):
  cls = getattr(resnet, trainer)
  kw = {} if tdepth is None else {"teacher_depth": tdepth}
  with pytest.raises(_Allocated):
    cls(depth=depth, device="cpu", num_classes=5, distill_alpha=1, distill_temperature=4,
        teacher=teacher_state(cls, tdepth or depth, 5), **kw)


def test_check_distill_args_returns_floats():
  assert engine.check_distill_args() == (None, 0.5, 1.0)
  got = engine.check_distill_args({}, 101, 1, 4)
  assert got == (101, 1.0, 4.0) and type(got[1]) is float and type(got[2]) is float


@pytest.mark.parametrize("depth,V", [(20, 10), (32, 37), (56, 100)])
def test_state_shapes_are_the_cifar_trainers(cpu_plans, depth, V):
  net = resnet.CifarResNetTrainer(depth=depth, batch=2, num_classes=V, device="cpu")
  sd = net.state_dict()
  assert {k: tuple(v.shape) for k, v in sd.items()} == \
      resnet._state_shapes(resnet.CifarResNetTrainer, depth, V)
  assert net.teacher is None and (net.distill_alpha, net.distill_temperature) == (0.5, 1.0)


@pytest.mark.parametrize("depth,V", [(50, 1000), (101, 37)])
def test_state_shapes_are_the_resnet_trainers(cpu_plans, depth, V):
  net = resnet.ResNetTrainer(depth=depth, batch=1, image=32, num_classes=V, device="cpu",
                             training=False)
  sd = net.state_dict()
  assert {k: tuple(v.shape) for k, v in sd.items()} == \
      resnet._state_shapes(resnet.ResNetTrainer, depth, V)


# ------------------------------------------------------------------ binding refusals
def _C():
  from tensorflowonspark_b200 import ops
  return ops.C()


def _args(**over):
  a = {"logits": torch.zeros(4, 16), "teacher_logits": torch.zeros(4, 16),
       "labels": torch.zeros(4, dtype=torch.int32), "dlogits": torch.zeros(4, 16,
                                                                           dtype=torch.bfloat16),
       "loss_sum": torch.zeros(1), "correct": torch.zeros(1), "V": 10, "scale": 0.25,
       "label_smoothing": 0.0, "alpha": 0.5, "temperature": 1.0, "mix": None}
  a.update(over)
  return a


@pytest.mark.parametrize("over,match", [
    ({"teacher_logits": torch.zeros(4, 16, dtype=torch.bfloat16)}, "teacher_logits must be fp32"),
    ({"teacher_logits": torch.zeros(4, 16, dtype=torch.float64)}, "teacher_logits must be fp32"),
    ({"teacher_logits": torch.zeros(5, 16)}, "teacher_logits must have the student's 4 rows"),
    ({"teacher_logits": torch.zeros(4, 8)}, "ldt >= V"),
    ({"teacher_logits": torch.zeros(64)}, r"teacher_logits must be contiguous \[rows, ldt\]"),
    ({"logits": torch.zeros(4, 16, dtype=torch.bfloat16)}, "logits must be contiguous fp32"),
    ({"V": 17}, "1 <= V <= ld"),
    ({"V": 0}, "1 <= V <= ld"),
    ({"labels": torch.zeros(5, dtype=torch.int32)}, "one label per row"),
    ({"labels": torch.zeros(4, dtype=torch.int64)}, "labels must be contiguous int32"),
    ({"dlogits": torch.zeros(4, 16)}, "dlogits must be contiguous bf16"),
    ({"alpha": 0.0}, r"alpha must be in \(0, 1\]"),
    ({"alpha": 1.01}, "alpha must be in"),
    ({"alpha": NAN}, "alpha must be in"),
    ({"temperature": 0.0}, "temperature must be finite and > 0"),
    ({"temperature": -1.0}, "temperature must be finite"),
    ({"temperature": math.inf}, "temperature must be finite"),
    ({"temperature": NAN}, "temperature must be finite"),
    ({"temperature": 1e-50}, "temperature must be finite and > 0 in fp32"),
    ({"temperature": 1e39}, "temperature must be finite and > 0 in fp32"),
    ({"label_smoothing": 1.5}, "label_smoothing must be in"),
    ({"mix": torch.zeros(8, dtype=torch.float64)}, "mix must be float32"),
    ({"mix": torch.zeros(7)}, "vector of 8 values"),
    ({"mix": torch.zeros(16)[::2]}, "vector of 8 values"),
    ({"mix": torch.zeros(8)}, "mix must be on the CUDA device"),
    ({}, "logits must be a CUDA tensor"),
])
def test_distill_xent_refuses_bad_arguments_before_the_launch(over, match):
  with pytest.raises(ValueError, match=match):
    _C().distill_xent(**_args(**over))


def test_every_entry_point_of_bind_distill_has_a_float64_check():
  """bind_distill registers outside the m.def list the kernel registry test scans: the same guard
  here.  Every entry point it defines must be a variant this feature's GPU tests check against
  float64 (tests/test_gpu_distill.py CHECKED_HERE)."""
  import re
  with open(os.path.join(ROOT, "csrc", "binding.cpp")) as f:
    src = f.read()
  body = src[src.index("void bind_distill("):]
  body = body[:body.index("\n}\n")]
  defs = set(re.findall(r'\bmod\.def\("(\w+)"', body))
  assert defs == {"distill_xent"}, defs
  assert not re.findall(r'\bmod\.def\(', src.replace(body, "")), "mod.def outside bind_distill"
  import test_gpu_distill as gd
  assert defs <= {op for op, _ in gd.CHECKED_HERE}


# ------------------------------------------------------------------ ptxas
@pytest.mark.skipif(not os.path.exists(uc.NVCC), reason="nvcc not found")
def test_distill_kernels_have_no_stack_frame_or_spills(tmp_path):
  kernels = uc._ptxas("distill.cu", tmp_path)
  assert len(kernels) == 2 and all("distill_xent_kernel" in k for k in kernels), sorted(kernels)
  bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
  assert not bad, "stack frame / spill stores / spill loads (bytes): {}".format(bad)


def test_new_kernel_name_contains_no_existing_kernel_name():
  import re
  csrc = os.path.join(ROOT, "csrc")
  old = set()
  for f in os.listdir(csrc):
    if f.endswith((".cu", ".cuh")) and f != "distill.cu":
      with open(os.path.join(csrc, f)) as fh:
        old |= set(re.findall(r"\b(\w+_kernel)\b", fh.read()))
  assert not [o for o in old if o in "distill_xent_kernel"]


# ------------------------------------------------------------------ example flags
def _spark(argv):
  mod = importlib.import_module("resnet_spark")
  mod.main_fun(["resnet_spark.py", "--batch_size", "4", "--image", "64"] + argv, dry._Ctx(1))
  return dry._Trainer.made[-1]


def _teacher_dir(tmp_path, state):
  from tensorflowonspark_b200.utils import checkpoint
  d = str(tmp_path / "teacher")
  checkpoint.save(d, 7, {"params": state, "optim": {}})
  return d


def test_resnet_spark_distillation_flags(fake_gpu, tmp_path):
  args = importlib.import_module("resnet_spark").parse([])
  assert [getattr(args, k) for k in DISTILL_KW] == [None] * 4
  net = _spark(["--train_steps", "2"])
  assert not set(DISTILL_KW) & set(net.kw)
  d = _teacher_dir(tmp_path, {"w": torch.arange(3.0)})
  net = _spark(["--train_steps", "2", "--teacher", d, "--teacher_depth", "152",
                "--distill_alpha", "0.9", "--distill_temperature", "4"])
  assert torch.equal(net.kw["teacher"]["w"], torch.arange(3.0))
  assert [net.kw[k] for k in DISTILL_KW[1:]] == [152, 0.9, 4.0]
  net = _spark(["--train_steps", "2", "--teacher", d])
  assert "teacher" in net.kw and not set(DISTILL_KW[1:]) & set(net.kw)
  with pytest.raises(ValueError, match="no checkpoint there"):
    _spark(["--train_steps", "2", "--teacher", str(tmp_path / "empty")])


def test_resnet_cifar_distillation_flags(fake_gpu, tmp_path):
  mod = importlib.import_module("resnet_cifar_main")
  args = mod.define_flags().parse_args([])
  assert [getattr(args, k) for k in DISTILL_KW] == [None] * 4
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "2"], mod.LocalContext())
  assert not set(DISTILL_KW) & set(dry._Trainer.made[-1].kw)
  d = _teacher_dir(tmp_path, {"w": torch.ones(2)})
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "2", "--teacher", d,
                "--teacher_depth", "110", "--distill_temperature", "2"], mod.LocalContext())
  kw = dry._Trainer.made[-1].kw
  assert torch.equal(kw["teacher"]["w"], torch.ones(2))
  assert kw["teacher_depth"] == 110 and kw["distill_temperature"] == 2.0
  assert "distill_alpha" not in kw

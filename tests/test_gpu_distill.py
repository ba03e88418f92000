"""Knowledge distillation on one H100: the distillation loss kernel against the float64 reference of
tests/test_distill_host.py, captured CIFAR ResNet and ResNet-50 steps whose teacher logits are its
folded forward pass on that step's (mixed) student input bit for bit and whose loss and gradient
are the float64 loss of that step's logits, a teacher that stays frozen and out of the student's
state, the launches a teacher adds, the float64 coverage of every distillation launch, and a
student that moves towards its teacher.

The module's name sorts it after tests/test_gpu_cluster.py (see tests/test_gpu_grad_accum.py).
"""
import gc
import importlib.util
import itertools
import math
import os
import sys
import types

import pytest
import torch

pytestmark = pytest.mark.gpu

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(_ROOT, "tests"))

import test_distill_host as ref  # noqa: E402


def _load(name, *path):
  spec = importlib.util.spec_from_file_location(name, os.path.join(_ROOT, *path))
  m = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(m)
  return m


sc = _load("step_conformance", "tools", "step_conformance.py")
LR, MOMENTUM, WD = 0.1, 0.9, 1e-4
DEV = "cuda"
MODES = {"none": 0.0, "mixup": 1.0, "cutmix": 2.0}


def _C():
  from tensorflowonspark_b200 import ops
  return ops.C()


def _pad8(v):
  return (v + 7) // 8 * 8


def _bits(t):
  return t.view(torch.int16) if t.dtype == torch.bfloat16 else t


def _free():
  torch.cuda.synchronize()
  gc.collect()
  torch.cuda.empty_cache()


def _mixvec(mode, lam):
  v = torch.zeros(8, dtype=torch.float32, device=DEV)
  v[0], v[1] = MODES[mode], lam
  return v


def f32(v):
  return float(torch.tensor(v, dtype=torch.float32))


# ----------------------------------------------------------------------------- kernel
def _case(B, V, ld, ldt, seed):
  g = torch.Generator().manual_seed(seed)
  s = torch.randn(B, ld, generator=g) * 3
  z = torch.randn(B, ldt, generator=g) * 3
  s[:, V:], z[:, V:] = 1e4, -1e4               # padding columns must not be read
  s[0, :V] = 0.5                               # a tie: the lowest index is the arg-max
  y = torch.randint(0, V, (B,), generator=g, dtype=torch.int32)
  y[1] = int(s[1, :V].argmax())                # at least one hit
  return s.to(DEV), z.to(DEV), y.to(DEV)


def _run(s, z, y, V, ldd, scale, **kw):
  dl = torch.full((s.shape[0], ldd), 7.0, dtype=torch.bfloat16, device=DEV)
  loss = torch.zeros(1, dtype=torch.float32, device=DEV)
  correct = torch.zeros(1, dtype=torch.float32, device=DEV)
  _C().distill_xent(s, z, y, dl, loss, correct, V, scale, **kw)
  torch.cuda.synchronize()
  return dl, loss, correct


def _rows(s, z, y, V, eps, alpha, T, lam, mixing):
  """Per-row float64 losses (for the loss bound's magnitude)."""
  s, z = s[:, :V].double().cpu(), z[:, :V].double().cpu()
  t = ref.soft_target(y.cpu(), V, eps, lam, mixing)
  ls, lsT, lq = torch.log_softmax(s, 1), torch.log_softmax(s / T, 1), torch.log_softmax(z / T, 1)
  return (1 - alpha) * -(t * ls).sum(1) + alpha * T * T * (lq.exp() * (lq - lsT)).sum(1)


def _check_kernel(s, z, y, V, ldd, eps, alpha, T, mode, lam, what):
  B = s.shape[0]
  scale = 1.0 / B
  mixing = mode in ("mixup", "cutmix")
  lam = f32(lam) if mixing else 1.0
  kw = {} if mode == "plain" else {"mix": _mixvec(mode, lam)}   # plain: no mix vector at all
  dl, loss, correct = _run(s, z, y, V, ldd, scale, label_smoothing=eps, alpha=alpha,
                           temperature=T, **kw)
  want, grad = ref.ref_distill(s.cpu(), z.cpu(), y.cpu(), V, eps, alpha, T, lam, mixing)
  mag = float(_rows(s, z, y, V, eps, alpha, T, lam, mixing).abs().sum()) * scale
  assert abs(float(loss) - want) <= 4e-5 * mag + 1e-6, (what, float(loss), want)
  got = dl[:, :V].double().cpu()
  bound = 2.0 ** -8 * grad.abs() + 1e-5 * (1 + T) * scale
  err = (got - grad).abs() - bound
  assert bool((err <= 0).all()), (what, float(err.max()))
  assert not dl[:, V:].float().any(), "padding columns of dlogits must be 0"
  assert int(correct) == ref.ref_hits(s.cpu(), y.cpu(), V, lam, mixing), what
  return correct


@pytest.mark.parametrize("V,ld,ldt", [(10, 16, 24), (37, 40, 40), (37, 40, 48), (1000, 1000, 1008),
                                      (1001, 1008, 1008)])
@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_distill_xent_against_float64(V, ld, ldt, eps):
  B = 256
  s, z, y = _case(B, V, ld, ldt, seed=V + ld + ldt + int(10 * eps))
  for T, alpha, (mode, lam) in itertools.product((1.0, 4.0), (0.5, 1.0),
                                                 (("none", 1.0), ("mixup", 0.3),
                                                  ("cutmix", 0.75), ("plain", 1.0))):
    c = _check_kernel(s, z, y, V, ld, eps, alpha, T, mode, lam, (T, alpha, mode))
    if alpha == 1.0 and mode in ("none", "plain"):     # correct is softmax_xent's count
      other = torch.zeros(1, device=DEV)
      _C().softmax_xent(s, y, None, torch.zeros(1, device=DEV), other, V, 1.0 / B,
                        label_smoothing=eps)
      torch.cuda.synchronize()
      assert torch.equal(c, other)


def test_distill_xent_odd_batch_pairs_the_middle_row_with_itself():
  B, V = 255, 37
  s, z, y = _case(B, V, 40, 40, seed=5)
  _check_kernel(s, z, y, V, 40, 0.1, 0.5, 2.0, "mixup", 0.4, "odd batch")


def test_distill_xent_refuses_a_teacher_on_another_device():
  s, z, y = _case(4, 10, 16, 16, 1)
  with pytest.raises(ValueError, match="teacher_logits must be on the device of logits"):
    _C().distill_xent(s, z.cpu(), y, None, torch.zeros(1, device=DEV), None, 10, 0.25)
  with pytest.raises(ValueError, match="labels must be on the device"):
    _C().distill_xent(s, z, y.cpu(), None, torch.zeros(1, device=DEV), None, 10, 0.25)
  with pytest.raises(ValueError, match="mix must be on the CUDA device"):
    _C().distill_xent(s, z, y, None, torch.zeros(1, device=DEV), None, 10, 0.25,
                      mix=torch.zeros(8))


# ----------------------------------------------------------------------------- trainers
def _teacher_state(cls, **kw):
  """A teacher that has trained three steps (non-trivial running statistics and residual
  branches)."""
  net = cls(device=DEV, **kw)
  x, y = net.synthetic_batch(seed=99)
  for _ in range(3):
    net.train_step(x, y)
  sd = net.state_dict()
  del net
  _free()
  return sd


_STATES = {}


def _cifar_teacher():
  from tensorflowonspark_b200.models import resnet
  if "c56" not in _STATES:
    _STATES["c56"] = _teacher_state(resnet.CifarResNetTrainer, depth=56, batch=32, seed=7)
  return _STATES["c56"]


def _r101_teacher():
  from tensorflowonspark_b200.models import resnet
  if "r101" not in _STATES:
    _STATES["r101"] = _teacher_state(resnet.ResNetTrainer, depth=101, batch=8, image=64, seed=7)
  return _STATES["r101"]


def _cifar(**kw):
  from tensorflowonspark_b200.models import resnet
  return resnet.CifarResNetTrainer(20, batch=32, device=DEV, **kw)


def _r50(**kw):
  from tensorflowonspark_b200.models import resnet
  return resnet.ResNetTrainer(50, batch=8, image=64, device=DEV, **kw)


def _distilled(kind, **kw):
  if kind == "cifar":
    return _cifar(teacher=_cifar_teacher(), teacher_depth=56, **kw)
  return _r50(teacher=_r101_teacher(), teacher_depth=101, **kw)


def _input(net):
  return net.xp if hasattr(net, "xp") else net.x8


def _replica(net):
  """An independent folded teacher built from the same state, whose stem reads a scratch copy of
  the student's decoded input."""
  from tensorflowonspark_b200.models import resnet
  copy = torch.zeros_like(_input(net))
  fake = types.SimpleNamespace(B=net.B, image=net.image, num_classes=net.num_classes,
                               device=net.device, xp=copy, x8=copy)
  if hasattr(net, "xp"):
    return resnet._ResNetTeacher(fake, _r101_teacher(), 101), copy
  return resnet._CifarTeacher(fake, _cifar_teacher(), 56), copy


def _check_step(net, rep, copy, what):
  torch.cuda.synchronize()
  copy.copy_(_input(net))
  rep.run()
  torch.cuda.synchronize()
  assert torch.equal(rep.logits, net.teacher.logits), (what, "teacher logits")
  mode, lam, _ = net.last_mix
  mixing = mode != "none"
  lam = f32(lam) if mixing else 1.0
  V, eps = net.num_classes, net.label_smoothing
  a, T = net.distill_alpha, net.distill_temperature
  s, z, y = net.logits.cpu(), net.teacher.logits.cpu(), net.labels.cpu()
  want, grad = ref.ref_distill(s, z, y, V, eps, a, T, lam, mixing)
  mag = float(_rows(s, z, y, V, eps, a, T, lam, mixing).abs().sum()) / net.B
  got = float(net.loss_sum)
  assert math.isfinite(got) and abs(got - want) <= 4e-5 * mag + 1e-6, (what, got, want)
  d = net.dlogits[:, :V].double().cpu()
  err = (d - grad).abs() - (2.0 ** -8 * grad.abs() + 1e-5 * (1 + T) / net.B)
  assert bool((err <= 0).all()), (what, float(err.max()))
  assert not net.dlogits[:, V:].float().any()


@pytest.mark.parametrize("kind", ["cifar", "r50"])
@pytest.mark.parametrize("k", [1, 2])
def test_every_replay_distils_from_its_own_input(kind, k):
  net = _distilled(kind, mixup_alpha=0.4, cutmix_alpha=1.0, label_smoothing=0.1, seed=21,
                   distill_alpha=0.7, distill_temperature=3.0, gradient_accumulation_steps=k)
  rep, copy = _replica(net)
  x, y = net.synthetic_batch()
  net.set_input(x, y)
  net.train_step()                       # eager
  _check_step(net, rep, copy, "eager")
  net.capture()
  seen = set()
  for i in range(6):
    net.train_step(*net.synthetic_batch(seed=100 + i))
    _check_step(net, rep, copy, "replay {} (micro-step {})".format(i, i % k))
    seen.add(net.last_mix[0])
  assert seen >= {"mixup", "cutmix"}, seen
  del net, rep
  _free()


def _teacher_tensors(t):
  n = t.net
  out = {"master": n.store.master, "weights": n.store.weights, "aux32": n.store.aux32,
         "running": n.running.tensor(), "wf": n.wf, "bf": n.bf}
  return {k: v.clone() for k, v in out.items()}


@pytest.mark.parametrize("kind", ["cifar", "r50"])
def test_teacher_stays_frozen_and_out_of_the_student(kind):
  from tensorflowonspark_b200.models import resnet
  net = _distilled(kind, mixup_alpha=0.2, seed=4)
  before = _teacher_tensors(net.teacher)
  x, y = net.synthetic_batch()
  net.set_input(x, y)
  net.capture()
  for i in range(4):
    net.train_step(*net.synthetic_batch(seed=i))
  torch.cuda.synchronize()
  after = _teacher_tensors(net.teacher)
  for name in before:
    assert torch.equal(before[name], after[name]), name
  sd = net.state_dict()
  plain = _cifar() if kind == "cifar" else _r50()
  assert set(sd) == set(plain.state_dict())
  assert sd["__running__"].shape == plain.state_dict()["__running__"].shape
  plain.load_state_dict(sd)
  batches = [net.synthetic_batch(seed=50 + i) for i in range(2)]
  assert net.evaluate(batches) == plain.evaluate(batches)
  if kind == "r50":
    assert net.export_builder_args == plain.export_builder_args
    served = [resnet.build_served(m.state_dict(), batch=8, **m.export_builder_args)
              for m in (net, plain)]
    for s in served:
      s.net.set_input(batches[0][0])
      s._run()
    torch.cuda.synchronize()
    assert torch.equal(served[0].net.logits, served[1].net.logits)
  del net, plain
  _free()


# ----------------------------------------------------------------------------- launches
# the distillation variants this file checks against float64 (the option suite's notation)
CHECKED_HERE = {("distill_xent", tuple(sorted(("alpha", "temperature") + extra)))
                for extra in ((), ("label_smoothing",), ("mix",), ("label_smoothing", "mix"))}


def r50_plain():
  net = _r50(mixup_alpha=0.2, label_smoothing=0.1)
  net.train_step(*net.synthetic_batch())


def r50_teacher():
  net = _r50(mixup_alpha=0.2, label_smoothing=0.1, teacher=_r101_teacher(), teacher_depth=101)
  net.train_step(*net.synthetic_batch())


def cifar_plain():
  net = _cifar()
  net.train_step(*net.synthetic_batch())


def cifar_teacher():
  net = _cifar(teacher=_cifar_teacher(), teacher_depth=56, distill_alpha=1.0)
  net.train_step(*net.synthetic_batch())


@pytest.fixture(scope="module")
def recorded():
  opt = _load("option_conformance_suite", "tests", "test_gpu_option_conformance.py")
  torch.cuda.set_device(0)
  _r101_teacher(), _cifar_teacher()     # (their own training is not recorded)
  out = {}
  for fn in (r50_plain, r50_teacher, cifar_plain, cifar_teacher):
    rec = opt.plans._Recorder()
    opt.plans._record_models(rec, [fn])
    out[fn.__name__] = rec
  return opt, out


def _no_addresses(spec):
  if isinstance(spec, tuple):
    return tuple(_no_addresses(v) for v in spec)
  return "address" if isinstance(spec, int) and not isinstance(spec, bool) and spec >= 2 ** 32 \
      else spec


@pytest.mark.parametrize("family,teacher_launches", [("r50", ["maxpool_fwd", "avgpool_fwd"]),
                                                     ("cifar", ["avgpool_fwd"])])
def test_teacher_launches_are_the_plain_launches_plus_its_forward(recorded, family,
                                                                  teacher_launches):
  """The student's plans and launches are the plain trainer's in the same order with the same
  arguments; the teacher's folded forward runs right after the decode, and distill_xent takes
  softmax_xent's place."""
  opt, rec = recorded
  a, b = rec[family + "_plain"], rec[family + "_teacher"]
  n = len(a.gemm)
  assert [(op, args) for op, args, _ in a.gemm] == [(op, args) for op, args, _ in b.gemm[:n]]
  assert len(b.gemm) > n
  ka = [(op, _no_addresses(spec), kw) for op, spec, kw, _, _ in a.k]
  kb = [(op, _no_addresses(spec), kw) for op, spec, kw, _, _ in b.k]
  dec = [op for op, _, _ in kb].index("decode_normalize")
  assert [op for op, _, _ in kb[dec + 1:dec + 1 + len(teacher_launches)]] == teacher_launches
  del kb[dec + 1:dec + 1 + len(teacher_launches)]
  # launches made while the teacher is built (before the first step) come after the student's
  deca = [op for op, _, _ in ka].index("decode_normalize")
  assert deca == dec, "launches while the teacher is built: {}".format(
      [c[0] for c in kb[deca:dec]])
  assert len(ka) == len(kb)
  swapped = []
  for x, y in zip(ka, kb):
    if x == y:
      continue
    assert (x[0], y[0]) == ("softmax_xent", "distill_xent"), (x[0], y[0])
    swapped.append(y)
  assert len(swapped) == 1


def _step_launches(net):
  """The launches of one recorded train_step (tools/step_conformance.py's recorder: every plan
  run, ops.K call and host clear, with the plan object of each plan run)."""
  launches, _ = sc.record_step(net, net.synthetic_batch(seed=5), [])
  return launches


@pytest.mark.parametrize("family", ["r50", "cifar"])
def test_teacher_plans_run_right_after_the_decode(family):
  """Between the decode and the student's first launch run exactly the teacher's folded forward
  plans in order, its pools and its head, and nothing else."""
  net = _distilled("cifar" if family == "cifar" else "r50")
  net.train_step(*net.synthetic_batch(seed=1))
  t = net.teacher
  if family == "r50":
    want = [("plan", t.net._f_plans[0]), ("k", "maxpool_fwd")] + \
        [("plan", p) for p in t.net._f_plans[1:]] + [("k", "avgpool_fwd"), ("plan", t.net.fc.fwd)]
  else:
    want = [("plan", p) for p in t.plans] + [("k", "avgpool_fwd"), ("plan", t.net.fc.fwd)]
  launches = _step_launches(net)
  dec = [la.name for la in launches].index("decode_normalize")
  got = launches[dec + 1:dec + 1 + len(want)]
  for la, (kind, what) in zip(got, want):
    assert la.kind == kind and (la.plan is what if kind == "plan" else la.name == what), (la, what)
  nxt = launches[dec + 1 + len(want)]
  first = net.p_stem if family == "r50" else net.stem.conv.fwd
  assert nxt.kind == "plan" and nxt.plan is first, nxt
  teacher_plans = {id(p) for kind, p in want if kind == "plan"}
  assert sum(1 for la in launches if la.plan is not None and id(la.plan) in teacher_plans) == \
      sum(1 for kind, _ in want if kind == "plan")
  del net, t
  _free()


def test_a_trainer_without_a_teacher_passes_the_plain_step_check():
  """No teacher: a trainer built with every distillation option at its default passes the step
  suite's plain ResNet-50 check, whose launch sequence (every launch claimed, in order, with
  softmax_xent) and references describe the trainer as it was before distillation existed."""
  from tensorflowonspark_b200.models import resnet
  net = resnet.ResNetTrainer(50, batch=8, image=64, device=DEV, lr=LR, momentum=MOMENTUM,
                             weight_decay=WD, teacher=None, teacher_depth=None,
                             distill_alpha=0.5, distill_temperature=1.0)
  assert net.teacher is None
  rep, claimed, launches = _checked_third_step(net)
  assert claimed == len(launches) and not rep.failures, sorted(rep.failures)[:5]
  assert "distill_xent" not in [la.name for la in launches]
  assert not [n for n in rep.layers if n.startswith("teacher.")]
  del net
  _free()


# ----------------------------------------------------------------------------- whole step
def _checked_third_step(net, mutate=None):
  for seed in (1, 2):
    net.train_step(*net.synthetic_batch(seed=seed))
  if mutate is not None:
    mutate(net)
  phase = net.accum.phase()
  buffers = sc.resnet_buffers(net)
  if net.teacher is not None:
    buffers += sc.teacher_buffers(net.teacher)
  launches, snaps = sc.record_step(net, net.synthetic_batch(seed=3), buffers)
  rep, claimed = sc.check_resnet_step(net, launches, snaps, LR, MOMENTUM, WD, phase)
  return rep, claimed, launches


def test_distilled_resnet50_step_matches_float64_layer_by_layer():
  """A ResNet-50 step with a ResNet-101 teacher (alpha 0.7, T 3, label smoothing 0.1): every
  launch claimed in order, the teacher's folded convolutions, pools and head against float64 on
  the student's decoded input, distill_xent on the two layers' logits, and no teacher launch
  writing a student buffer (nor a student launch a teacher buffer)."""
  _free()
  torch.cuda.reset_peak_memory_stats()
  net = _distilled("r50", lr=LR, momentum=MOMENTUM, weight_decay=WD, label_smoothing=0.1,
                   distill_alpha=0.7, distill_temperature=3.0)
  rep, claimed, launches = _checked_third_step(net)
  print("\ndistilled ResNet-50 8 x 64^2: {} launches, {} claimed; peak {:.2f} GB".format(
      len(launches), claimed, torch.cuda.max_memory_allocated() / 1e9))
  print(rep.table())
  assert claimed == len(launches)
  assert not rep.failures, "\n".join(m for _, _, m in sorted(rep.failures)[:10])
  assert {"teacher conv", "teacher pool", "teacher head", "distill loss"} <= set(rep.classes)
  teacher_layers = [n for n in rep.layers if n.startswith("teacher.")]
  # stem, max pool, 3 or 4 convolutions per block (33 blocks), average pool, head
  assert len(teacher_layers) == 4 + 3 * 33 + 4, len(teacher_layers)
  del net
  _free()


def _teacher_stem_reads_its_own_input(net):
  """The teacher's stem reads the teacher replica's own input buffer, which nothing decodes,
  instead of the student's decoded xp."""
  from tensorflowonspark_b200.ops import igemm
  t = net.teacher.net
  t._f_plans[0] = igemm.stem_fprop(t.xp, t.store._view(t.wf, t.stem_w), t.stem_act,
                                   bias=t.bf[:64], relu=True)


def test_teacher_stem_wiring_mutant_is_caught_at_the_teacher_stem():
  _free()
  net = _distilled("r50", lr=LR, momentum=MOMENTUM, weight_decay=WD)
  rep, _, _ = _checked_third_step(net, _teacher_stem_reads_its_own_input)
  failing = rep.failing_layers()
  print("\nteacher stem mutant: first failures {}".format(failing[:4]))
  assert failing, "the step checker passed a miswired teacher"
  assert failing[0] == "teacher.stem.conv", "\n".join(m for _, _, m in sorted(rep.failures)[:4])
  del net
  _free()


def test_every_distillation_variant_has_a_float64_check(recorded):
  opt, rec = recorded
  defaults = set(opt.plans.K_OPS) | set(opt.kern.KERNEL_OPS)
  launched, missing = set(), set()
  for name, r in rec.items():
    for op, spec, kw, _, _ in r.k:
      if op in opt.NO_KERNEL:
        continue
      v = opt.variant(op, spec, kw)
      launched.add(v)
      key = "{}[{}]".format(op, ",".join(v[1])) if v[1] else op
      if op == "distill_xent":
        if v not in CHECKED_HERE:
          missing.add(key)
        continue
      if "mix" in v[1]:
        continue        # tests/test_gpu_mixup.py's
      if not (v in opt.REPLAYED_HERE or (not v[1] and op in defaults) or
              key in opt.kern.COVERED_ELSEWHERE or op + "[*]" in opt.kern.COVERED_ELSEWHERE):
        missing.add(key)
  assert not missing, "launched variants without a float64 check: {}".format(sorted(missing))
  assert ("distill_xent", ("alpha", "label_smoothing", "mix", "temperature")) in launched
  assert ("distill_xent", ("alpha", "temperature")) in launched


def test_distill_xent_is_bound_and_registered_here():
  """The entry point the trainers launch is the extension's, and this file is its float64 check."""
  assert callable(getattr(_C(), "distill_xent"))
  assert {v[0] for v in CHECKED_HERE} == {"distill_xent"}


# ----------------------------------------------------------------------------- training
# The teacher is a ResNet-56 trained on the fixed batch until it predicts it confidently, so that
# the student starts far from it, far above the loss's fp32 resolution.  Measured on one H100
# 80GB HBM3 (700 W), two runs: the teacher's training loss ended at 0.0075-0.0076 with 64 / 64
# hits; the student's mean KL was 1.11-1.12 over the first 10 steps and 0.014 over the last 10
# (ratio 0.012).  The test asks for a first KL above 0.02 and a ratio below 0.1.
TEACHER_STEPS = 80
KL_FIRST_MIN = 0.02
KL_RATIO_MAX = 0.1


def _confident_cifar_teacher(x, y):
  from tensorflowonspark_b200.models import resnet
  net = resnet.CifarResNetTrainer(56, batch=x.shape[0], device=DEV, seed=3)
  net.set_input(x, y)
  net.capture()
  for _ in range(TEACHER_STEPS):
    net.train_step()
  torch.cuda.synchronize()
  print("\nteacher: training loss {:.4f}, hits {} / {}".format(float(net.loss_sum),
                                                              int(net.correct), x.shape[0]))
  sd = net.state_dict()
  del net
  _free()
  return sd


def test_student_moves_towards_its_teacher():
  from tensorflowonspark_b200.models import resnet
  x, y = resnet.CifarResNetTrainer.synthetic_batch(types.SimpleNamespace(
      B=64, image=32, num_classes=10, multi_label=False, device=torch.device(DEV)), seed=8)
  teacher = _confident_cifar_teacher(x, y)
  net = resnet.CifarResNetTrainer(20, batch=64, device=DEV, teacher=teacher, teacher_depth=56,
                                  distill_alpha=1.0, distill_temperature=4.0, seed=1, lr=0.05)
  net.set_input(x, y)
  net.capture()
  kl = []
  for _ in range(100):
    net.train_step()
    kl.append(net.loss_sum.clone())
  torch.cuda.synchronize()
  kl = [float(v) / 16.0 for v in kl]          # loss = T^2 KL at alpha = 1
  first, last = sum(kl[:10]) / 10, sum(kl[-10:]) / 10
  print("distillation KL: first 10 steps {:.5f}, last 10 {:.5f}, ratio {:.3f}".format(
      first, last, last / first))
  assert all(math.isfinite(v) for v in kl)
  assert first > KL_FIRST_MIN, first
  assert last < KL_RATIO_MAX * first, (first, last)
  del net
  _free()

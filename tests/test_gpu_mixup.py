"""Mixup and CutMix on one H100: the mixing decode and the two mixed-target losses against the
float64 references of tests/test_mixup_host.py, mode none bit for bit against the plain kernels,
captured ResNet steps whose every replay uses that step's draw, evaluation that never mixes, and
the float64 coverage of every (entry point, options) the mixing trainers launch.

The module's name sorts it after tests/test_gpu_cluster.py (see tests/test_gpu_grad_accum.py).
"""
import importlib.util
import math
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(_ROOT, "tests"))

import test_mixup_host as ref  # noqa: E402


def _load(name, *path):
  spec = importlib.util.spec_from_file_location(name, os.path.join(_ROOT, *path))
  m = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(m)
  return m


pc = _load("plan_conformance", "tools", "plan_conformance.py")
DEV = "cuda"
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


def _C():
  from tensorflowonspark_b200 import ops
  return ops.C()


def _mixvec(draw):
  from tensorflowonspark_b200.models import engine
  return torch.tensor(engine.MixDraws.vector(draw), dtype=torch.float32, device=DEV)


def _bits(t):
  return t.view(torch.int16) if t.dtype == torch.bfloat16 else t


# ----------------------------------------------------------------------------- decode
def _stem(H):
  from tensorflowonspark_b200.ops import igemm
  return igemm.stem_geometry(H, H)[2], igemm.STEM_PAD


def _layouts():
  out = []
  for name, B, H in (("stem224", 4, 224), ("stem64", 5, 64)):
    out.append((name, B, H, "stem"))
  out.append(("cifar32", 7, 32, "cifar"))
  return out


def _draws(H, W):
  d = [("none", 1.0, (0, 0, 0, 0)), ("mixup", 0.0, (0, 0, 0, 0)), ("mixup", 0.3, (0, 0, 0, 0)),
       ("mixup", 1.0, (0, 0, 0, 0)),
       ("cutmix", 0.0, (H // 2, H // 2, 0, W)),              # empty
       ("cutmix", 0.0, (0, H, 0, W)),                        # the whole image
       ("cutmix", 0.5, (0, H // 3, 3, W // 2)),              # touching the top
       ("cutmix", 0.5, (H // 2, H, 1, W - 2)),               # the bottom
       ("cutmix", 0.5, (2, H - 1, 0, W // 4)),               # the left
       ("cutmix", 0.5, (1, H // 2, W // 3, W)),              # the right
       ("cutmix", 0.5, (H // 2, H // 2 + 1, W - 1, W)),      # a single pixel
       ("cutmix", 0.5, (-7, H + 9, W - 3, 10 * W))]          # out of range: clamped
  return d


@pytest.mark.parametrize("name,B,H,layout", _layouts())
def test_mixing_decode_against_float64(name, B, H, layout):
  Wp, wofs = _stem(H) if layout == "stem" else (H, 0)
  g = torch.Generator().manual_seed(H + B)
  img = torch.randint(0, 256, (B, H, H, 3), dtype=torch.uint8, generator=g).to(DEV)
  plain, pb = pc.guarded((B, H, Wp, 8), torch.bfloat16, DEV, pc.UNWRITTEN_BF16)
  _C().decode_normalize(img, plain, wofs, MEAN, STD)
  for draw in _draws(H, H):
    what = "{} {}".format(name, draw)
    out, ob = pc.guarded((B, H, Wp, 8), torch.bfloat16, DEV, pc.UNWRITTEN_BF16)
    _C().decode_normalize(img, out, wofs, MEAN, STD, mix=_mixvec(draw))
    torch.cuda.synchronize()
    want, mag = ref.ref_mix_decode(img, Wp, wofs, MEAN, STD, draw)
    got = out.double().cpu()
    # one bf16 rounding of the value on top of a few fp32 roundings of terms bounded by mag
    bound = pc.U_BF16 * want.abs() + 1e-6 * mag
    err = (got - want).abs() - bound
    assert bool((err <= 0).all()), (what, float(err.max()))
    assert not got[..., 3:].any() and not got[:, :, :wofs].any() and \
        not got[:, :, wofs + H:].any(), what + ": padding"
    assert pc.guard_intact(out, ob), what + ": guard band"
    if draw[0] == "none":
      assert torch.equal(_bits(out), _bits(plain)), what + ": none is not the plain decode"
  # any other mode code is none
  out = torch.empty_like(plain)
  v = _mixvec(("none", 1.0, (0, H, 0, H)))
  v[0] = 7.0
  _C().decode_normalize(img, out, wofs, MEAN, STD, mix=v)
  torch.cuda.synchronize()
  assert torch.equal(_bits(out), _bits(plain))
  assert pc.guard_intact(plain, pb)


# ----------------------------------------------------------------------------- losses
def _pad8(v):
  return (v + 7) // 8 * 8


def _xent_case(B, V, ld, seed):
  g = torch.Generator().manual_seed(seed)
  logits = torch.randn(B, ld, generator=g) * 3
  logits[:, V:] = 1e4
  labels = torch.randint(0, V, (B,), generator=g, dtype=torch.int32)
  for r in range(0, min(B, 40), 4):        # planted ties: the lower index is the arg-max
    y = max(1, int(labels[r]))
    labels[r] = y
    top = float(logits[r, :V].max()) + 1.0
    logits[r, y] = logits[r, y - 1 if r % 8 == 0 else min(y + 1, V - 1)] = top
  for r in range(40, min(B, 80)):          # rows that predict their own or their partner's label
    logits[r, int(labels[r if r % 2 else B - 1 - r])] += 20.0
  return logits.to(DEV), labels.to(DEV)


def _run_xent(logits, labels, V, ldd, scale, **kw):
  dl = torch.full((logits.shape[0], ldd), 7.0, dtype=torch.bfloat16, device=DEV)
  loss = torch.zeros(1, dtype=torch.float32, device=DEV)
  correct = torch.zeros(1, dtype=torch.float32, device=DEV)
  _C().softmax_xent(logits, labels, dl, loss, correct, V, scale, **kw)
  torch.cuda.synchronize()
  return dl, loss, correct


MIXES = [("mixup", 0.3, (0, 0, 0, 0)), ("cutmix", 0.75, (0, 0, 0, 0)), ("mixup", 0.5, (0, 0, 0, 0)),
         ("mixup", 0.0, (0, 0, 0, 0))]


@pytest.mark.parametrize("V", [10, 37, 1000, 1001])
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("B", [256, 255])
def test_mixed_softmax_xent_against_float64(V, eps, B):
  ld = _pad8(V) + 8
  scale = 1.0 / B
  logits, labels = _xent_case(B, V, ld, seed=V + int(eps * 10) + B)
  for draw in MIXES:
    lam = ref.f32(draw[1])
    dl, loss, correct = _run_xent(logits, labels, V, ld, scale, label_smoothing=eps,
                                  mix=_mixvec(draw))
    ref_loss, ref_grad = ref.ref_mixed_xent(logits, labels, V, eps, lam)
    want = float(ref_loss.sum()) * scale
    assert abs(float(loss) - want) <= 2e-5 * float(ref_loss.abs().sum()) * scale + 1e-6, (
        draw, float(loss), want)
    ref_grad = ref_grad * scale
    got = dl[:, :V].double().cpu()
    bound = 2.0 ** -8 * ref_grad.abs() + 1e-5 * scale
    err = (got - ref_grad).abs() - bound
    assert bool((err <= 0).all()), (draw, float(err.max()))
    assert not dl[:, V:].float().any(), "padding columns of dlogits must be 0"
    assert int(correct) == ref.ref_hits(logits, labels, V, lam), draw


@pytest.mark.parametrize("V", [10, 1001])
@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_mixed_softmax_xent_mode_none_is_the_plain_kernel(V, eps):
  B, ld = 256, _pad8(V)
  logits, labels = _xent_case(B, V, ld, seed=3 * V)
  a = _run_xent(logits, labels, V, ld, 1.0 / B, label_smoothing=eps)
  for code in (0.0, 5.0, float("nan")):
    v = _mixvec(("none", 1.0, (0, 0, 0, 0)))
    v[0] = code
    v[1] = 0.25                 # lam is ignored without a mixing mode
    b = _run_xent(logits, labels, V, ld, 1.0 / B, label_smoothing=eps, mix=v)
    assert torch.equal(_bits(a[0]), _bits(b[0])) and torch.equal(a[2], b[2]), code
    rows, _ = ref.ref_mixed_xent(logits, labels, V, eps, 1.0)
    assert abs(float(a[1]) - float(b[1])) <= 2 * pc.gamma(B) * float(rows.abs().sum()) / B, code
  for r in (0, 77, 255):        # one row: one atomic add onto 0, bit for bit
    one = [_run_xent(logits[r:r + 1], labels[r:r + 1], V, ld, 0.5, label_smoothing=eps, **kw)[1]
           for kw in ({}, {"mix": _mixvec(("none", 1.0, (0, 0, 0, 0)))})]
    assert torch.equal(one[0], one[1]), r


def _bce_case(B, V, ld, seed, weighted):
  g = torch.Generator().manual_seed(seed)
  logits = torch.randn(B, ld, generator=g) * 3
  logits[:, V:] = 1e4
  logits[0, :V], logits[1, :V] = 1e4, -1e4
  targets = torch.randint(0, 2, (B, V), generator=g, dtype=torch.uint8)
  targets[3] *= 5
  targets[4] = (logits[4, :V] > 0).to(torch.uint8)              # exact on its own target
  targets[B - 1 - 5] = (logits[5, :V] > 0).to(torch.uint8)      # exact on its partner's
  pw = (torch.rand(V, generator=g) * 3).to(DEV) if weighted else None
  return logits.to(DEV), targets.to(DEV), pw


def _run_bce(logits, targets, V, ldd, scale, **kw):
  dl = torch.full((logits.shape[0], ldd), 7.0, dtype=torch.bfloat16, device=DEV)
  loss = torch.zeros(1, dtype=torch.float32, device=DEV)
  correct = torch.zeros(1, dtype=torch.float32, device=DEV)
  _C().sigmoid_bce(logits, targets, dl, loss, correct, V, scale, **kw)
  torch.cuda.synchronize()
  return dl, loss, correct


@pytest.mark.parametrize("V", [10, 37, 1000, 1001])
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("weighted", [False, True])
def test_mixed_sigmoid_bce_against_float64(V, eps, weighted):
  for B in (256, 255):
    ld = _pad8(V) + 8
    scale = 1.0 / (B * V)
    logits, targets, pw = _bce_case(B, V, ld, V + int(eps * 10) + 100 * weighted + B, weighted)
    for draw in MIXES:
      lam = ref.f32(draw[1])
      dl, loss, correct = _run_bce(logits, targets, V, ld, scale, label_smoothing=eps,
                                   pos_weight=pw, mix=_mixvec(draw))
      ref_loss, ref_grad = ref.ref_mixed_bce(logits, targets, V, eps, lam, pw)
      want = float(ref_loss.sum()) * scale
      assert math.isfinite(float(loss)) and bool(torch.isfinite(dl.float()).all())
      assert abs(float(loss) - want) <= 2e-5 * want + 1e-7, (draw, float(loss), want)
      ref_grad = ref_grad * scale
      got = dl[:, :V].double().cpu()
      pmax = 1.0 if pw is None else float(pw.max())
      bound = 2.0 ** -8 * ref_grad.abs() + 1e-6 * (1 + pmax) * scale
      err = (got - ref_grad).abs() - bound
      assert bool((err <= 0).all()), (draw, float(err.max()))
      assert not dl[:, V:].float().any(), "padding columns of dlogits must be 0"
      assert int(correct) == ref.ref_exact_rows(logits, targets, V, lam) >= 1, draw


@pytest.mark.parametrize("eps,weighted", [(0.0, False), (0.1, True)])
def test_mixed_sigmoid_bce_mode_none_is_the_plain_kernel(eps, weighted):
  B, V = 256, 1001
  logits, targets, pw = _bce_case(B, V, 1008, 9, weighted)
  a = _run_bce(logits, targets, V, 1008, 1.0 / (B * V), label_smoothing=eps, pos_weight=pw)
  b = _run_bce(logits, targets, V, 1008, 1.0 / (B * V), label_smoothing=eps, pos_weight=pw,
               mix=_mixvec(("none", 1.0, (0, 0, 0, 0))))
  assert torch.equal(_bits(a[0]), _bits(b[0])) and torch.equal(a[2], b[2])
  rows, _ = ref.ref_mixed_bce(logits, targets, V, eps, 1.0, pw)
  assert abs(float(a[1]) - float(b[1])) <= 2 * pc.gamma(B) * float(rows.abs().sum()) / (B * V)


# ----------------------------------------------------------------------------- captured steps
def _cifar(**kw):
  from tensorflowonspark_b200.models import resnet
  return resnet.CifarResNetTrainer(20, batch=32, device=DEV, **kw)


def _r50(**kw):
  from tensorflowonspark_b200.models import resnet
  return resnet.ResNetTrainer(50, batch=8, image=64, device=DEV, **kw)


def _decoded(net):
  """(decoded input buffer, Wp, wofs) of a trainer."""
  from tensorflowonspark_b200.ops import igemm
  if hasattr(net, "xp"):
    return net.xp, net.xp.shape[2], igemm.STEM_PAD
  return net.x8, 32, 0


def _check_step(net, what):
  """The decoded input is the float64 mix of in_u8 under last_mix, and the reported loss is the
  float64 mixed loss of the logits buffer."""
  torch.cuda.synchronize()
  buf, Wp, wofs = _decoded(net)
  want, mag = ref.ref_mix_decode(net.in_u8, Wp, wofs, net.mean, net.std, net.last_mix)
  err = (buf.double().cpu() - want).abs() - (pc.U_BF16 * want.abs() + 1e-6 * mag)
  assert bool((err <= 0).all()), (what, net.last_mix, float(err.max()))
  lam, V, eps = ref.f32(net.last_mix[1]), net.num_classes, net.label_smoothing
  if net.multi_label:
    rows, _ = ref.ref_mixed_bce(net.logits, net.labels, V, eps, lam, net.pos_weight)
    rows = rows.sum(1) / V
  else:
    rows, _ = ref.ref_mixed_xent(net.logits, net.labels, V, eps, lam)
  want = float(rows.sum()) / net.B
  got = float(net.loss_sum)
  assert math.isfinite(got) and abs(got - want) <= 2e-5 * float(rows.abs().sum()) / net.B + 1e-6, \
      (what, net.last_mix, got, want)


@pytest.mark.parametrize("make", [_cifar, _r50], ids=["cifar20_b32", "r50_b8_64"])
def test_every_replay_uses_its_own_draw(make):
  net = make(mixup_alpha=0.2, cutmix_alpha=1.0, label_smoothing=0.1, seed=21)
  x, y = net.synthetic_batch()
  net.set_input(x, y)
  net.capture()
  assert net.graph is not None and net.last_mix is not None   # the warm-up steps drew
  seen = set()
  for i in range(6):
    x, y = net.synthetic_batch(seed=100 + i)
    net.train_step(x, y)
    _check_step(net, "replay {}".format(i))
    seen.add((net.last_mix[0], net.last_mix[1]))
  assert len(seen) == 6 and {m for m, _ in seen} == {"mixup", "cutmix"}


def test_accumulation_micro_steps_draw_on_their_own():
  net = _cifar(mixup_alpha=0.4, cutmix_alpha=1.0, gradient_accumulation_steps=3, seed=5)
  x, y = net.synthetic_batch()
  net.set_input(x, y)
  net.capture()
  draws = []
  for i in range(6):
    net.train_step(*net.synthetic_batch(seed=i))
    _check_step(net, "micro-step {}".format(i))
    draws.append(net.last_mix)
  assert len({(m, lam) for m, lam, _ in draws}) == 6


def test_multilabel_pos_weight_trains_with_finite_losses():
  V = 12
  net = _cifar(multi_label=True, num_classes=V, pos_weight=[0.5 + 0.2 * i for i in range(V)],
               mixup_alpha=0.2, cutmix_alpha=1.0, label_smoothing=0.1)
  x, y = net.synthetic_batch()
  net.set_input(x, y)
  net.capture()
  losses = []
  for i in range(5):
    net.train_step(x, y)
    _check_step(net, "multi-label {}".format(i))
    losses.append(float(net.loss_sum))
  assert all(math.isfinite(v) for v in losses)


def test_first_eager_steps_and_plain_trainer_launches():
  """Without capture too each step stages its draw; a trainer with mix_prob = 0 mixes nothing."""
  net = _cifar(cutmix_alpha=1.0, mix_prob=0.0)
  x, y = net.synthetic_batch()
  net.train_step(x, y)
  assert net.last_mix == ("none", 1.0, (0, 0, 0, 0))
  _check_step(net, "mix_prob 0")
  net = _cifar(mixup_alpha=1.0, seed=3)
  for i in range(3):
    net.train_step(x, y)
    _check_step(net, "eager {}".format(i))


def test_evaluation_does_not_mix():
  mixed = _cifar(mixup_alpha=0.2, cutmix_alpha=1.0)
  for i in range(3):
    mixed.train_step(*mixed.synthetic_batch(seed=i))
  plain = _cifar()
  plain.load_state_dict(mixed.state_dict())
  batches = [mixed.synthetic_batch(seed=50 + i) for i in range(2)]
  a, b = mixed.evaluate(batches), plain.evaluate(batches)
  assert a == b, (a, b)


# ----------------------------------------------------------------------------- coverage
# the mixing variants this file checks against float64 (the option suite's notation)
CHECKED_HERE = {("decode_normalize", ("mix",)), ("softmax_xent", ("mix",)),
                ("softmax_xent", ("label_smoothing", "mix")), ("sigmoid_bce", ("mix",)),
                ("sigmoid_bce", ("mix", "pos_weight")), ("sigmoid_bce", ("label_smoothing", "mix")),
                ("sigmoid_bce", ("label_smoothing", "mix", "pos_weight"))}


def r50_mix_smoothed():
  net = _r50(mixup_alpha=0.2, cutmix_alpha=1.0, label_smoothing=0.1)
  net.train_step(*net.synthetic_batch())


def r50_plain():
  net = _r50()
  net.train_step(*net.synthetic_batch())


def cifar_mix():
  net = _cifar(cutmix_alpha=1.0)
  net.train_step(*net.synthetic_batch())


def cifar_multilabel_mix():
  net = _cifar(multi_label=True, num_classes=20, pos_weight=[1.0] * 20, mixup_alpha=0.2)
  net.train_step(*net.synthetic_batch())


@pytest.fixture(scope="module")
def recorded():
  opt = _load("option_conformance_suite", "tests", "test_gpu_option_conformance.py")
  torch.cuda.set_device(0)
  out = {}
  for fn in (r50_plain, r50_mix_smoothed, cifar_mix, cifar_multilabel_mix):
    rec = opt.plans._Recorder()
    opt.plans._record_models(rec, [fn])
    out[fn.__name__] = rec
  return opt, out


def _no_addresses(spec):
  """A launch spec with the device addresses some launches take as integers masked."""
  if isinstance(spec, tuple):
    return tuple(_no_addresses(v) for v in spec)
  return "address" if isinstance(spec, int) and not isinstance(spec, bool) and spec >= 2 ** 32 \
      else spec


def test_mixing_launches_are_the_plain_launches_plus_mix(recorded):
  """Same plans, same launches in the same order; only the training decode and the loss gain the
  mix vector."""
  opt, rec = recorded
  a, b = rec["r50_plain"], rec["r50_mix_smoothed"]
  assert [(op, args) for op, args, _ in a.gemm] == [(op, args) for op, args, _ in b.gemm]
  assert len(a.k) == len(b.k)
  gained = []
  for ca, cb in zip(a.k, b.k):
    assert ca[0] == cb[0] and _no_addresses(ca[1]) == _no_addresses(cb[1]) and ca[3] == cb[3], \
        (ca[0], cb[0])
    kwa, kwb = dict(ca[2]), dict(cb[2])
    if kwa != kwb:
      kwb.pop("mix")
      kwb.pop("label_smoothing", None), kwa.pop("label_smoothing", None)
      assert kwa == kwb, cb[0]
      gained.append(cb[0])
  assert gained == ["decode_normalize", "softmax_xent"]


def test_every_mixing_variant_has_a_float64_check(recorded):
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
      if "mix" in v[1]:
        if v not in CHECKED_HERE:
          missing.add(key)
        continue
      if not (v in opt.REPLAYED_HERE or (not v[1] and op in defaults) or
              key in opt.kern.COVERED_ELSEWHERE or op + "[*]" in opt.kern.COVERED_ELSEWHERE):
        missing.add(key)
  assert not missing, "launched variants without a float64 check: {}".format(sorted(missing))
  for want in (("decode_normalize", ("mix",)), ("softmax_xent", ("label_smoothing", "mix")),
               ("sigmoid_bce", ("mix", "pos_weight")), ("softmax_xent", ("mix",))):
    assert want in launched, want

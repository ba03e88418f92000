"""GPU tier: gradient clipping by global norm (``clip_norm``) fused into the gradient all-reduce +
optimizer kernels.  The kernels against the float64 reference of test_grad_clip_host.py for sgd /
momentum / adam / lars with and without the weight average, bitwise-unclipped steps below the
threshold (eager and graph replay), the bucket ordering of the overlapped launches, replays with
changing gradients, NaN gradients, launch counts, checkpoints, and the three trainers.  The
multi-rank paths are tools/gpu_check_grad_clip.py (2+ GPUs)."""
import math
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_grad_clip_host import step_reference  # noqa: E402
from test_weight_average_host import ema_bound, ema_reference  # noqa: E402

SIZES = (1, 7, 8, 9, 4096, 300_003)
OPT_KW = {"sgd": dict(lr=0.05, weight_decay=1e-3), "momentum": dict(lr=0.05, weight_decay=1e-3),
          "adam": dict(lr=1e-3, weight_decay=1e-3),
          "lars": dict(lr=0.8, weight_decay=1e-3, trust_coefficient=0.02)}
NAMES = {0: "sgd", 1: "momentum", 2: "adam", 3: "lars"}


@pytest.fixture(scope="module", autouse=True)
def _ext():
  from tensorflowonspark_b200 import _build
  _build.load(required=True)


def _store():
  from tensorflowonspark_b200.models import engine
  st = engine.ParamStore()
  for i, n in enumerate(SIZES):
    st.register("w%d" % i, (n,), True, engine.normal(0.05))
  for i, n in enumerate((64, 10, 3)):
    st.register("bn%d" % i, (n,), False, engine.constant(1.0))
  st.finalize(torch.device("cuda", 0), seed=5)
  return st


def _optimizer(st, opt, ema=None, clip=None):
  """Two buckets (the overlapped launch / finish path), cut at a tensor start."""
  from tensorflowonspark_b200.parallel.fused_optim import FusedOptimizer
  cut = st.by_name["w4"]["offset"]
  return FusedOptimizer(st, opt=opt, buckets=[(cut, st.total, "late"), (0, cut, "early")],
                        ema_decay=ema, clip_norm=clip, **OPT_KW[opt])


def _grads(st, steps, seed=42):
  """Random gradients on every real element, 0 on the padding (as a trainer's)."""
  gen = torch.Generator().manual_seed(seed)
  mask = torch.zeros(st.total)
  for s in st.order:
    mask[s["offset"]:s["offset"] + s["numel"]] = 1.0
  return [(torch.randn(st.total, generator=gen) * 0.1 * mask).cuda() for _ in range(steps)]


def _norm64(g, scale=1.0):
  return math.sqrt(float((g.double() ** 2).sum())) * abs(scale)


def _step(opt, st, g):
  opt.zero_grads()
  st.grads.copy_(g)
  opt.finish()


def _state(o):
  return {"state1": o.state1.detach().cpu().double().clone() if o.state1 is not None else None,
          "state2": o.state2.detach().cpu().double().clone() if o.state2 is not None else None}


def _lars_bounds(st):
  return [s["offset"] for s in st.order if s["decay"]] + [st.decay_end]


# ------------------------------------------------------------------ the kernels vs float64
@pytest.mark.parametrize("ema", [None, 0.9], ids=["plain", "ema"])
@pytest.mark.parametrize("frac", [0.1, 0.5])
@pytest.mark.parametrize("opt", ["sgd", "momentum", "adam", "lars"])
def test_clipped_steps_match_float64(opt, frac, ema):
  """Each step from the kernel's own state before it: master, state and grad_norm against the
  float64 clip + update within bounds derived from fp32 rounding of each term."""
  st = _store()
  grads = _grads(st, 4)
  o = _optimizer(st, opt, ema, clip=1.0)
  masters = []
  for g in grads:
    c = frac * _norm64(g)
    o.clip_norm = c                     # (configuration: the next finalise reads it)
    w0, s0 = st.master.detach().cpu().clone(), _state(o)
    h = o.hyper.detach().cpu().clone()
    if opt == "adam":
      h[7] += 1                         # the step counts itself before the update
    _step(o, st, g)
    torch.cuda.synchronize()
    old1 = s0["state1"].clone() if s0["state1"] is not None else None
    ref, norm, coef = step_reference(opt, w0, g.cpu(), s0, h, st.decay_end, c, _lars_bounds(st))
    assert coef < 1.0
    assert float(o.grad_norm) == pytest.approx(norm, rel=2e-6)
    w = st.master.detach().cpu().double()
    bound = 2.0 ** -22 * (w0.double().abs() + ref.abs()) + 2e-4 * (ref - w0.double()).abs() + 1e-12
    assert bool(((w - ref).abs() <= bound).all()), float(((w - ref).abs() - bound).max())
    if opt != "sgd":
      # (s0 now holds the reference's new state; the fp32 terms of the sum bound the rounding)
      s1, r1 = o.state1.detach().cpu().double(), s0["state1"]
      terms = old1.abs() + r1.abs() + g.cpu().double().abs() + w0.double().abs()
      assert bool(((s1 - r1).abs() <= 2e-4 * r1.abs() + 2.0 ** -20 * terms + 1e-12).all())
    masters.append(st.master.detach().cpu().clone())
    # slot 3 of the step's copy is the clipped scale; the saved vector is untouched
    assert float(o.hyper[3]) == 1.0
    assert float(o.hyper_step[3]) == pytest.approx(coef, rel=2e-6)
  if ema is not None:
    err = (o.ema.detach().cpu().double() - ema_reference(masters, ema)[-1]).abs()
    assert bool((err <= ema_bound(masters, ema)).all())


def _run(opt, ema, clip, capture, grads=None, order=False):
  st = _store()
  o = _optimizer(st, opt, ema, clip)
  grads = grads if grads is not None else _grads(st, 5)
  norms = []
  if capture:
    o.zero_grads()
    st.grads.copy_(grads[0])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      o.finish()
    o.reset_average()
    for gr in grads:
      st.grads.copy_(gr)
      g.replay()
      if o.grad_norm is not None:
        norms.append(o.grad_norm.clone())
  else:
    for gr in grads:
      if order:
        # bucket A's gradients final -> launch(A); then B's -> launch(B); then finish()
        cut = st.by_name["w4"]["offset"]
        o.zero_grads()
        st.grads[cut:].copy_(gr[cut:])
        o.launch("late")
        st.grads[:cut].copy_(gr[:cut])
        o.launch("early")
        o.finish()
      else:
        _step(o, st, gr)
      if o.grad_norm is not None:
        norms.append(o.grad_norm.clone())
  torch.cuda.synchronize()
  out = [st.master, st.weights, st.aux32] + [t for t in (o.state1, o.state2, o.ema) if t is not None]
  return [t.clone() for t in out], o.hyper.clone(), norms


@pytest.mark.parametrize("capture", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("ema", [None, 0.9], ids=["plain", "ema"])
@pytest.mark.parametrize("opt", ["sgd", "momentum", "adam", "lars"])
def test_inactive_threshold_is_bitwise_the_unclipped_step(opt, ema, capture):
  grads = _grads(_store(), 5)
  big = 2.0 * max(_norm64(g) for g in grads)
  plain, h0, _ = _run(opt, ema, None, capture, grads)
  for c in (math.inf, big):
    got, h1, norms = _run(opt, ema, c, capture, grads)
    for a, b in zip(plain, got):
      assert torch.equal(a, b), c
    assert torch.equal(h0, h1)
    assert len(norms) == len(grads)
    for n, g in zip(norms, grads):
      assert float(n) == pytest.approx(_norm64(g), rel=2e-6)


@pytest.mark.parametrize("opt", ["momentum", "adam", "lars"])
def test_no_bucket_updates_before_every_bucket_is_reduced(opt):
  """launch(A) with only A's gradients final, then B's, then finish(): the same bits as the
  whole gradient at once, i.e. the coefficient of both buckets' gradients."""
  grads = _grads(_store(), 3)
  c = 0.3 * _norm64(grads[0])
  ref, _, n0 = _run(opt, None, c, False, grads)
  got, _, n1 = _run(opt, None, c, False, grads, order=True)
  for a, b in zip(ref, got):
    assert torch.equal(a, b)
  assert all(torch.equal(a, b) for a, b in zip(n0, n1))


@pytest.mark.parametrize("opt", ["momentum", "adam"])
def test_replays_use_their_own_gradients_and_repeat_bitwise(opt):
  grads = _grads(_store(), 5, seed=7)
  for k in range(len(grads)):
    grads[k] = grads[k] * (0.5 + k)       # norms that differ from replay to replay
  c = 0.2 * _norm64(grads[0])
  eager, he, ne = _run(opt, 0.9, c, False, grads)
  graph, hg, ng = _run(opt, 0.9, c, True, grads)
  for a, b in zip(eager, graph):
    assert torch.equal(a, b)
  assert torch.equal(he, hg)
  assert all(torch.equal(a, b) for a, b in zip(ne, ng))
  assert len({float(n) for n in ng}) == len(grads)
  again, _, na = _run(opt, 0.9, c, True, grads)
  assert all(torch.equal(a, b) for a, b in zip(graph, again))
  assert all(torch.equal(a, b) for a, b in zip(ng, na))


def test_nan_gradient_gives_nan_norm_and_is_not_clipped_silently():
  st = _store()
  o = _optimizer(st, "momentum", clip=1.0)
  g = _grads(st, 1)[0]
  g[st.by_name["w5"]["offset"] + 3] = float("nan")
  _step(o, st, g)
  torch.cuda.synchronize()
  assert math.isnan(float(o.grad_norm))
  assert not bool(torch.isfinite(st.master[:st.by_name["w4"]["offset"]]).any())   # every element
  assert math.isnan(float(o.hyper_step[3]))
  # an infinite threshold too: inf / NaN is NaN (torch's clip_grad_norm_ gives NaN gradients)
  st2 = _store()
  o2 = _optimizer(st2, "momentum", clip=math.inf)
  _step(o2, st2, g)
  torch.cuda.synchronize()
  assert math.isnan(float(o2.grad_norm)) and not bool(torch.isfinite(st2.master).all())


def test_launch_counts():
  from tensorflowonspark_b200 import ops
  counts = {}
  for clip in (None, 1.0):
    st = _store()
    o = _optimizer(st, "adam", clip=clip)
    g = _grads(st, 1)[0]
    c0 = ops.launch_count()
    _step(o, st, g)
    counts[clip] = ops.launch_count() - c0
  assert counts[None] == 1 + 2                 # zero_grads + one fused kernel per bucket
  assert counts[1.0] == 1 + 2 + 1 + 2          # + a sum of squares per bucket, the finaliser


def test_checkpoint_continues_bitwise():
  N, k = 8, 3
  for opt in ("momentum", "adam", "lars"):
    st = _store()
    grads = _grads(st, N)
    c = 0.4 * _norm64(grads[0])
    a = _optimizer(st, opt, 0.9, clip=c)
    for g in grads[:k]:
      _step(a, st, g)
    params, optim = st.state_dict(), a.state_dict()
    for g in grads[k:]:
      _step(a, st, g)
    st2 = _store()
    b = _optimizer(st2, opt, 0.9, clip=c)
    st2.load_state_dict(params)
    b.load_state_dict(optim)
    for g in grads[k:]:
      _step(b, st2, g)
    torch.cuda.synchronize()
    assert torch.equal(st2.master, st.master) and torch.equal(b.ema, a.ema), opt
    assert torch.equal(b.grad_norm, a.grad_norm) and torch.equal(b.hyper, a.hyper)


# ------------------------------------------------------------------ trainers
def _resnet50(**kw):
  from tensorflowonspark_b200.models import resnet
  return resnet.ResNetTrainer(depth=50, batch=8, image=64, num_classes=37, seed=3, **kw)


def _cifar(**kw):
  from tensorflowonspark_b200.models import resnet
  return resnet.CifarResNetTrainer(depth=20, batch=32, seed=4, **kw)


def _unet(k):
  def make(**kw):
    from tensorflowonspark_b200.models import unet
    return unet.UNetTrainer(batch=4, image=128, classes=21, seed=9, lr=2e-3,
                            encoder_trainable_from=k, **kw)
  return make


def _batches(net, n):
  from tensorflowonspark_b200.models import unet
  out = []
  for i in range(n):
    x, y = net.synthetic_batch(seed=i)
    if isinstance(net, unet.UNetTrainer):
      y = unet.synthetic_labels(x, net.classes)
    out.append((x, y))
  return out


TRAINERS = {"resnet50": _resnet50, "cifar20": _cifar, "unet21_frozen": _unet(None),
            "unet21_finetune13": _unet(13)}


@pytest.mark.parametrize("name", list(TRAINERS))
def test_trainer_inf_threshold_is_bitwise_the_unclipped_update(name):
  """Captured steps with clip_norm=inf: each step's update is bit for bit the unclipped fused
  update of the same gradients from the same state (a trainer's gradients themselves are not
  bit-reproducible from run to run: batch-norm sums use float atomics), and grad_norm is the
  float64 norm of the gradients."""
  from tensorflowonspark_b200.parallel.fused_optim import FusedOptimizer
  net = TRAINERS[name](clip_norm=math.inf)
  batches = _batches(net, 2)
  net.set_input(*batches[0])
  net.capture()
  st, o = net.store, net.optim
  s = float(o.hyper[3])
  for k in range(3):
    net.set_input(*batches[k % 2])
    before = [t.clone() for t in (st.master, o.state1, o.state2, o.hyper) if t is not None]
    net.train_step()
    torch.cuda.synchronize()
    assert float(o.grad_norm) == pytest.approx(_norm64(st.grads, s), rel=2e-6)
    after = [t.clone() for t in (st.master, st.weights, st.aux32, o.state1, o.state2) if t is not None]
    # replay the update with an optimizer that does not clip, on the trainer's gradients
    p = FusedOptimizer(st, opt=NAMES[o.opt])
    st.master.copy_(before[0])
    p.state1 is not None and p.state1.copy_(before[1])
    p.state2 is not None and p.state2.copy_(before[2])
    p.hyper.copy_(before[-1][:8])
    p.step()
    torch.cuda.synchronize()
    want = [t for t in (st.master, st.weights, st.aux32, p.state1, p.state2) if t is not None]
    for a, b in zip(after, want):
      assert torch.equal(a, b), (name, k)
    st._assemble = o.assemble


@pytest.mark.parametrize("name", list(TRAINERS))
def test_trainer_active_threshold(name):
  """clip_norm = 0.5 N of the first step: that step matches the float64 clip + update of the
  trainer's own gradients, training still reduces the loss and the weight average still tracks."""
  probe = TRAINERS[name](clip_norm=math.inf)
  batches = _batches(probe, 1)
  probe.train_step(*batches[0])
  torch.cuda.synchronize()
  c = 0.5 * float(probe.grad_norm)
  del probe
  net = TRAINERS[name](clip_norm=c, ema_decay=0.9)
  st, o = net.store, net.optim
  w0, s0 = st.master.detach().cpu().clone(), _state(o)
  h = o.hyper.detach().cpu().clone()
  loss0 = float(net.train_step(*batches[0]))
  torch.cuda.synchronize()
  h[7] = o.hyper[7]
  ref, norm, coef = step_reference(NAMES[o.opt], w0, st.grads.cpu(), s0, h, st.decay_end, c)
  assert 0.3 < coef < 0.8 and float(o.grad_norm) == pytest.approx(norm, rel=2e-6)
  w = st.master.detach().cpu().double()
  bound = 2.0 ** -22 * (w0.double().abs() + ref.abs()) + 2e-4 * (ref - w0.double()).abs() + 1e-12
  assert bool(((w - ref).abs() <= bound).all()), float(((w - ref).abs() - bound).max())
  masters = [st.master.detach().cpu().clone()]
  for _ in range(5):
    loss = float(net.train_step(*batches[0]))
    torch.cuda.synchronize()
    masters.append(st.master.detach().cpu().clone())
  assert loss < loss0
  sd = net.averaged().state_dict()
  ref_avg, bound_avg = ema_reference(masters, 0.9)[-1], ema_bound(masters, 0.9)
  for s in st.order:
    sl = slice(s["offset"], s["offset"] + s["numel"])
    assert bool(((sd[s["name"]].reshape(-1).double() - ref_avg[sl]).abs() <= bound_avg[sl]).all())


def test_trainer_checkpoint_round_trip():
  """A clipped CIFAR ResNet-20 saved and loaded: the same optimizer state and hyper-parameters
  (the threshold is configuration), and the continued step clips with the loaded state."""
  a = _cifar(clip_norm=0.5)
  batches = _batches(a, 2)
  for k in range(3):
    a.train_step(*batches[k % 2])
  params, optim = a.state_dict(), a.optim.state_dict()
  assert "clip_norm" not in optim and len(optim["hyper"]) == 8
  b = _cifar(clip_norm=0.5)
  b.load_state_dict(params)
  b.optim.load_state_dict(optim)
  assert torch.equal(b.store.master, a.store.master) and torch.equal(b.optim.hyper, a.optim.hyper)
  assert torch.equal(b.optim.state1, a.optim.state1)
  # the next update from identical gradients is bitwise identical
  for net in (a, b):
    net.optim.zero_grads()
    net.store.grads.copy_(a.store.grads * 0 + torch.linspace(-1, 1, a.store.total, device="cuda"))
    net.optim.step()
  torch.cuda.synchronize()
  assert torch.equal(a.store.master, b.store.master) and torch.equal(a.optim.grad_norm, b.optim.grad_norm)

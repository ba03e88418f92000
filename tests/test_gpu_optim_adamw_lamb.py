"""GPU tier: AdamW and LAMB in the fused all-reduce + optimizer kernels against the float64
reference of test_adamw_lamb_host.py - one and two overlapped buckets, eager and CUDA-graph
replay, AdamW with zero decay bitwise Adam, checkpoints continued from Adam, the weight average,
gradient clipping (LAMB's norms from the clipped gradient) - the ResNet-50, CIFAR ResNet-20 and
U-Net trainers with ``optimizer="adamw" | "lamb"``, and (2+ GPUs) the multi-rank paths through
tools/gpu_check_adamw_lamb.py.

(The file name sorts after test_gpu_cluster.py: the cluster tests ask gpu_info for a GPU that no
process holds, and the CUDA context these tests create lives as long as the pytest process.)"""
import inspect
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_adamw_lamb_host import adam_family_reference  # noqa: E402
from test_weight_average_host import ema_bound, ema_reference  # noqa: E402

AWKWARD = (1, 7, 8, 9, 4096, 1_000_003)
OPT_KW = {"adamw": dict(lr=2e-3, weight_decay=0.05), "lamb": dict(lr=1e-2, weight_decay=0.01)}


@pytest.fixture(scope="module", autouse=True)
def _ext():
  from tensorflowonspark_b200 import _build
  _build.load(required=True)


def rel(a, b):
  return float((a.double().cpu() - b.double().cpu()).abs().max()
               / (b.double().cpu().abs().max() + 1e-12))


def _bounds(st):
  return [s["offset"] for s in st.order if s["decay"]] + [st.decay_end]


def _store():
  from tensorflowonspark_b200.models import engine
  st = engine.ParamStore()
  for i, n in enumerate(AWKWARD):
    st.register("w%d" % i, (n,), True, engine.normal(0.05))
  st.register("zero_grad", (100,), True, engine.normal(0.05))
  st.register("zero_w", (200,), True, engine.constant(0.0))
  for i, n in enumerate((64, 64, 10, 3)):
    st.register("bn%d" % i, (n,), False, engine.constant(1.0))
  st.finalize(torch.device("cuda", 0), seed=5)
  return st


def _grads(st, steps, seed=42):
  """Per-step gradients: random on every real element, 0 on the padding and on 'zero_grad'."""
  gen = torch.Generator().manual_seed(seed)
  mask = torch.zeros(st.total)
  for s in st.order:
    if s["name"] != "zero_grad":
      mask[s["offset"]:s["offset"] + s["numel"]] = 1.0
  return [(torch.randn(st.total, generator=gen) * 0.1 * mask).cuda() for _ in range(steps)]


def _optimizer(st, opt, split, **kw):
  from tensorflowonspark_b200.parallel.fused_optim import FusedOptimizer
  buckets = None
  if split:   # two buckets -> the overlapped (launch / finish) path on the communication stream
    cut = _bounds(st)[4]
    buckets = [(cut, st.total, "late"), (0, cut, "early")]
  args = dict(OPT_KW.get(opt, {}))
  args.update(kw)
  return FusedOptimizer(st, opt=opt, buckets=buckets, **args)


def _step(o, st, g):
  o.zero_grads()
  st.grads.copy_(g)
  o.finish()


def _ref(opt, st, o, w, m, v, g, scale=None):
  h = o.hyper.detach().cpu()
  return adam_family_reference(opt, w, g.cpu(), m, v, h, st.decay_end, _bounds(st), scale=scale)


def _snapshot(st, o):
  return [t.detach().cpu().double().clone() for t in (st.master, o.state1, o.state2)]


def _check(st, o, w, m, v, what):
  """master, m, v within 1e-5 of the float64 step taken from the kernel's own state before it
  (each step on its own: the bias corrections' __powf carries ~1e-4 relative error at t = 1, so a
  chained float64 run would drift by that much per step), bf16 weights and the fp32 tail copy."""
  assert rel(st.master, w) <= 1e-5, what + " master"
  assert rel(o.state1, m) <= 1e-5, what + " m"
  assert rel(o.state2, v) <= 1e-5, what + " v"
  assert rel(st.weights, w) <= 1e-2, what + " bf16 weights"
  n = st.total - st.decay_end
  assert rel(st.aux32[:n], w[st.decay_end:]) <= 1e-5, what + " aux32"


# ------------------------------------------------------------------ the kernels vs float64
@pytest.mark.parametrize("split", [False, True], ids=["one_bucket", "two_buckets"])
@pytest.mark.parametrize("opt", ["adamw", "lamb"])
def test_steps_match_float64_reference(opt, split):
  st = _store()
  o = _optimizer(st, opt, split)
  zw = st.by_name["zero_w"]["offset"]
  assert float(st.master[zw:zw + 200].abs().max()) == 0.0
  for step, g in enumerate(_grads(st, 5)):
    w, m, v = _snapshot(st, o)
    _step(o, st, g)
    torch.cuda.synchronize()
    assert float(o.hyper[7]) == step + 1
    w, m, v = _ref(opt, st, o, w, m, v, g)
    _check(st, o, w, m, v, "step %d" % step)


def _run(opt, split, capture, **kw):
  st = _store()
  o = _optimizer(st, opt, split, **kw)
  grads = _grads(st, 5)
  if capture:
    o.zero_grads()
    st.grads.copy_(grads[0])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      o.finish()                       # (the step count's increment is part of the graph)
    for step_grads in grads:
      st.grads.copy_(step_grads)
      g.replay()
  else:
    for step_grads in grads:
      _step(o, st, step_grads)
  torch.cuda.synchronize()
  out = [st.master, o.state1, o.state2, st.weights, st.aux32]
  if o.ema is not None:
    out.append(o.ema)
  return [t.clone() for t in out]


@pytest.mark.parametrize("opt", ["adamw", "lamb"])
def test_buckets_eager_and_graph_replay_bitwise_equal(opt):
  one, two = _run(opt, False, False), _run(opt, True, False)
  graph = _run(opt, True, True)
  again = _run(opt, True, False)
  for a, b, c, d in zip(one, two, graph, again):
    assert torch.equal(a, b), "one bucket differs from two"
    assert torch.equal(b, c), "graph replay differs from eager"
    assert torch.equal(b, d), "two eager runs differ"


@pytest.mark.parametrize("split", [False, True])
def test_adamw_without_decay_is_bitwise_adam(split):
  a = _run("adam", split, False, lr=2e-3, weight_decay=0.0)
  b = _run("adamw", split, False, lr=2e-3, weight_decay=0.0)
  for x, y in zip(a, b):
    assert torch.equal(x, y)


@pytest.mark.parametrize("opt", ["adamw", "lamb"])
def test_adam_checkpoint_continues(opt):
  """An adam state_dict (m, v, t and the hyper vector) loaded into adamw / lamb continues from
  that state: the next steps match the float64 reference started from it."""
  st = _store()
  grads = _grads(st, 5)
  adam = _optimizer(st, "adam", False, lr=2e-3, weight_decay=0.0)
  for g in grads[:2]:
    _step(adam, st, g)
  sd = adam.state_dict()
  other = _optimizer(st, opt, False)
  other.load_state_dict(sd)
  assert float(other.hyper[7]) == 2.0 and torch.equal(other.state2, adam.state2)
  other.hyper[2] = OPT_KW[opt]["weight_decay"]      # the checkpoint carried adam's (zero) decay
  m, v = sd["state1"].double(), sd["state2"].double()
  for k, g in enumerate(grads[2:]):
    w = st.master.detach().cpu().double().clone()
    if k:
      _, m, v = _snapshot(st, other)
    _step(other, st, g)
    torch.cuda.synchronize()
    w, m, v = _ref(opt, st, other, w, m, v, g)
    _check(st, other, w, m, v, "step %d" % k)


@pytest.mark.parametrize("opt", ["adamw", "lamb"])
def test_weight_average(opt):
  plain = _run(opt, True, False)
  st = _store()
  o = _optimizer(st, opt, True, ema_decay=0.9)
  masters = []
  for g in _grads(st, 5):
    _step(o, st, g)
    torch.cuda.synchronize()
    masters.append(st.master.detach().cpu().clone())
  for a, b in zip(plain, [st.master, o.state1, o.state2, st.weights, st.aux32]):
    assert torch.equal(a, b), "the average changed training"
  err = (o.ema.detach().cpu().double() - ema_reference(masters, 0.9)[-1]).abs()
  assert bool((err <= ema_bound(masters, 0.9)).all())


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("opt", ["adamw", "lamb"])
def test_inf_threshold_is_bitwise_unclipped(opt, split):
  a = _run(opt, split, False)
  b = _run(opt, split, False, clip_norm=math.inf)
  for x, y in zip(a, b):
    assert torch.equal(x, y)


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("opt", ["adamw", "lamb"])
def test_clipped_steps_match_float64(opt, split):
  """A binding threshold: the update (LAMB's norms included) sees the clipped gradient."""
  st = _store()
  o = _optimizer(st, opt, split, clip_norm=1.0)
  for step, g in enumerate(_grads(st, 4)):
    n64 = math.sqrt(float((g.double() ** 2).sum()))
    c = 0.4 * n64
    o.clip_norm = c                     # (configuration: the next finalise reads it)
    w, m, v = _snapshot(st, o)
    _step(o, st, g)
    torch.cuda.synchronize()
    assert float(o.grad_norm) == pytest.approx(n64, rel=2e-6)
    scale = float(o.hyper_step[3])      # the clipped scale the kernels read
    assert scale == pytest.approx(c / (n64 + 1e-6), rel=2e-6) and scale < 0.5
    w, m, v = _ref(opt, st, o, w, m, v, g, scale=scale)
    _check(st, o, w, m, v, "step %d" % step)


# ------------------------------------------------------------------ trainers
def _trainer_step_matches(net, opt, batch):
  """One eager step against the float64 reference from a snapshot + the step's gradients (the
  optimizer reads the gradient buffer and leaves it as it is)."""
  st, o = net.store, net.optim
  net.train_step(*batch)               # non-zero moments before the checked step
  torch.cuda.synchronize()
  w0, m0, v0 = (t.detach().cpu().clone() for t in (st.master, o.state1, o.state2))
  net.train_step(*batch)
  torch.cuda.synchronize()
  w, m, v = _ref(opt, st, o, w0, m0, v0, st.grads)
  _check(st, o, w, m, v, "trainer step")
  return w0, w


def _head_padding_is_zero(net):
  st, V = net.store, net.num_classes
  for spec in (net.fc.sw, net.fc.sbias):
    rows = slice(spec["offset"] + V * (spec["numel"] // spec["shape"][0]),
                 spec["offset"] + spec["numel"])
    assert not st.master[rows].any() and not st.weights[rows].any(), spec["name"]
    assert not net.optim.state1[rows].any() and not net.optim.state2[rows].any(), spec["name"]
  assert not st.f32(net.fc.sbias)[V:].any()


@pytest.mark.parametrize("opt", ["adamw", "lamb"])
def test_resnet50_trainer(opt):
  from tensorflowonspark_b200.models import resnet
  torch.cuda.set_device(0)
  net = resnet.ResNetTrainer(depth=50, batch=8, image=64, num_classes=37, device="cuda:0",
                             optimizer=opt, lr=1e-3 if opt == "adamw" else 5e-3,
                             weight_decay=0.01, beta1=0.85, beta2=0.99, epsilon=1e-6)
  h = net.optim.hyper.cpu()
  assert [float(x) for x in h[4:7]] == pytest.approx([0.85, 0.99, 1e-6])
  batch = net.synthetic_batch(seed=3)
  _trainer_step_matches(net, opt, batch)
  for _ in range(3):
    net.train_step(*batch)
  torch.cuda.synchronize()
  assert math.isfinite(float(net.loss_sum))
  _head_padding_is_zero(net)


def test_cifar_resnet20_trainer_lamb_learns():
  from tensorflowonspark_b200.models import resnet
  torch.cuda.set_device(0)
  net = resnet.CifarResNetTrainer(depth=20, batch=32, device="cuda:0", optimizer="lamb", lr=2e-2,
                                  weight_decay=1e-3)
  x, y = net.synthetic_batch(seed=9)
  net.set_input(x, y)
  net.capture()
  losses = [float(net.train_step()) for _ in range(20)]
  torch.cuda.synchronize()
  assert all(math.isfinite(l) for l in losses), losses
  assert sum(losses[-3:]) / 3 < losses[0], losses


def _unet(**kw):
  from tensorflowonspark_b200.models import unet
  return unet.UNetTrainer(batch=4, image=128, classes=21, seed=9, lr=2e-3, **kw)


def _unet_batch(net):
  from tensorflowonspark_b200.models import unet
  x, _ = net.synthetic_batch(seed=1)
  return x, unet.synthetic_labels(x, net.classes)


def test_unet_finetune_adamw_decays_only_the_filters():
  net = _unet(encoder_trainable_from=13, optimizer="adamw", weight_decay=0.05)
  st = net.store
  assert float(net.optim.hyper[2]) == pytest.approx(0.05)
  enc = [s for s in st.order if s["name"].startswith("encoder.")]
  assert enc and all(s["decay"] == s["name"].endswith(".w") for s in enc)
  assert all(s["name"].endswith(".w") for s in st.order if s["decay"])
  # (the reference decays [0, decay_end) only: the filters; biases and the tail take Adam's step)
  _trainer_step_matches(net, "adamw", _unet_batch(net))


def test_unet_lamb_step_matches_float64():
  net = _unet(optimizer="lamb", weight_decay=0.01)
  _trainer_step_matches(net, "lamb", _unet_batch(net))


def test_unet_default_builds_todays_adam(monkeypatch):
  """UNetTrainer() without the new keywords hands FusedOptimizer the same resolved arguments as
  before they existed: opt adam, weight_decay 0 and the optimizer's beta / eps defaults."""
  from tensorflowonspark_b200.parallel import fused_optim
  seen = []
  real = fused_optim.FusedOptimizer

  class Recording(real):
    def __init__(self, *a, **k):
      seen.append(inspect.signature(real.__init__).bind(self, *a, **k))
      super().__init__(*a, **k)
  monkeypatch.setattr(fused_optim, "FusedOptimizer", Recording)
  _unet()
  args = seen[-1]
  args.apply_defaults()
  got = {k: v for k, v in args.arguments.items() if k not in ("self", "store")}
  assert got == dict(comm=None, opt="adam", lr=2e-3, momentum=0.9, weight_decay=0.0, beta1=0.9,
                     beta2=0.999, eps=1e-7, buckets=None, trust_coefficient=0.001, ema_decay=None,
                     clip_norm=None)


def _free_port():
  import socket
  with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as sk:
    sk.bind(("127.0.0.1", 0))
    return str(sk.getsockname()[1])


def test_adamw_lamb_two_ranks():
  """Peer-to-peer, NVLS (when available), HierComm and GroupComm with overlapped buckets: replicas
  bitwise identical, results equal within tolerance to one rank on the summed gradients."""
  if torch.cuda.device_count() < 2:
    pytest.skip("needs 2 GPUs")
  p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node",
                      "2", "--master-addr", "127.0.0.1", "--master-port", _free_port(),
                      os.path.join(ROOT, "tools", "gpu_check_adamw_lamb.py")],
                     capture_output=True, text=True, timeout=900, cwd=ROOT)
  print(p.stdout[-4000:], p.stderr[-2000:])
  assert p.returncode == 0 and "ADAMW LAMB CHECK PASSED" in p.stdout

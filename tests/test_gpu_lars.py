"""GPU tier: the LARS optimizer (norm pass + LARS update of the fused optimizer kernel) against a
float64 PyTorch reference, its determinism and CUDA-graph replay, the two ResNet trainers with
``optimizer="lars"``, and (2+ GPUs) the multi-rank paths through tools/gpu_check_lars.py."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

AWKWARD = (1, 7, 8, 9, 4096, 1_000_003)
HYPER = dict(lr=0.8, momentum=0.9, weight_decay=1e-3, trust_coefficient=0.02)


def rel(a, b):
  return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-12))


def lars_reference(w, v, g_sum, bounds, decay_end, lr, momentum, weight_decay, eta, scale=1.0):
  """One LARS step in float64: adapted tensors [bounds[t], bounds[t + 1]) below decay_end get
  v = m v + lr trust (g + wd w) with trust = eta |w| / (|g| + wd |w|) (1 if a norm is 0), the
  tail v = m v + lr g; w = w - v.  Returns (w, v)."""
  w, v, g = w.double().clone(), v.double().clone(), g_sum.double() * scale
  for t in range(len(bounds) - 1):
    sl = slice(bounds[t], bounds[t + 1])
    wn, gn = float(w[sl].norm()), float(g[sl].norm())
    trust = eta * wn / (gn + weight_decay * wn) if (wn > 0 and gn > 0) else 1.0
    v[sl] = momentum * v[sl] + lr * trust * (g[sl] + weight_decay * w[sl])
  v[decay_end:] = momentum * v[decay_end:] + lr * g[decay_end:]
  return w - v, v


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


def _grads(st, steps):
  """Per-step gradients: random on every real element, 0 on the padding and on 'zero_grad'."""
  gen = torch.Generator(device="cpu")
  gen.manual_seed(42)
  mask = torch.zeros(st.total, dtype=torch.bool)
  for s in st.order:
    if s["name"] != "zero_grad":
      mask[s["offset"]:s["offset"] + s["numel"]] = True
  return [(torch.randn(st.total, generator=gen) * mask).cuda() for _ in range(steps)]


def _optimizer(st, split):
  from tensorflowonspark_b200.parallel.fused_optim import FusedOptimizer
  buckets = None
  if split:   # two buckets -> the overlapped (launch / finish) path on the communication stream
    cut = _bounds(st)[4]
    buckets = [(cut, st.total, "late"), (0, cut, "early")]
  return FusedOptimizer(st, opt="lars", buckets=buckets, **HYPER)


@pytest.mark.parametrize("split", [False, True])
def test_lars_steps_match_float64_reference(split):
  from tensorflowonspark_b200 import _build
  _build.load(required=True)
  st = _store()
  opt = _optimizer(st, split)
  bounds = _bounds(st)
  w = st.master.clone().double()
  v = torch.zeros_like(w)
  assert float(w[st.by_name["zero_w"]["offset"]:][:200].abs().max()) == 0.0
  for step, g in enumerate(_grads(st, 5)):
    opt.zero_grads()                 # (also re-arms launch() for the next step)
    st.grads.copy_(g)
    opt.finish()
    torch.cuda.synchronize()
    w, v = lars_reference(w, v, g, bounds, st.decay_end, HYPER["lr"], HYPER["momentum"],
                          HYPER["weight_decay"], HYPER["trust_coefficient"])
    assert rel(st.master, w) <= 1e-5, "step %d master" % step
    assert rel(opt.state1, v) <= 1e-5, "step %d velocity" % step
    assert rel(st.weights, w) <= 1e-2, "step %d bf16 weights" % step
    n = st.total - st.decay_end
    assert rel(st.aux32[:n], w[st.decay_end:]) <= 1e-5, "step %d aux32" % step


def _run(split, capture):
  st = _store()
  opt = _optimizer(st, split)
  grads = _grads(st, 5)
  if capture:
    opt.zero_grads()
    st.grads.copy_(grads[0])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      opt.finish()
    for step_grads in grads:
      st.grads.copy_(step_grads)
      g.replay()
  else:
    for step_grads in grads:
      opt.zero_grads()
      st.grads.copy_(step_grads)
      opt.finish()
  torch.cuda.synchronize()
  return [t.clone() for t in (st.master, opt.state1, st.weights, st.aux32, opt.lars_norms)]


@pytest.mark.parametrize("split", [False, True])
def test_lars_deterministic_and_graph_replay_bitwise_equal(split):
  from tensorflowonspark_b200 import _build
  _build.load(required=True)
  eager1, eager2 = _run(split, False), _run(split, False)
  graph = _run(split, True)
  for a, b, c in zip(eager1, eager2, graph):
    assert torch.equal(a, b), "two eager runs differ"
    assert torch.equal(a, c), "graph replay differs from eager"


def _check_trainer_step(net):
  """One eager step against the float64 reference rebuilt from a snapshot + the step's
  gradients (the optimizer reads the gradient buffer and leaves it as it is)."""
  st, opt = net.store, net.optim
  x, y = net.synthetic_batch(seed=3)
  net.train_step(x, y)               # non-zero velocity before the checked step
  torch.cuda.synchronize()
  w0, v0 = st.master.clone(), opt.state1.clone()
  net.train_step(x, y)
  torch.cuda.synchronize()
  h = [float(t) for t in opt.hyper.cpu()]
  w, v = lars_reference(w0, v0, st.grads, _bounds(st), st.decay_end, h[0], h[1], h[2], h[4], h[3])
  assert rel(st.master, w) <= 1e-5
  assert rel(opt.state1, v) <= 1e-5
  assert rel(st.weights, w) <= 1e-2
  n = st.total - st.decay_end
  assert rel(st.aux32[:n], w[st.decay_end:]) <= 1e-5


def _check_trainer_learns(net):
  x, y = net.synthetic_batch(seed=9)
  net.set_input(x, y)
  net.capture()
  losses = []
  for _ in range(20):
    losses.append(float(net.train_step()))
  torch.cuda.synchronize()
  assert all(l == l and abs(l) < float("inf") for l in losses), losses
  assert sum(losses[-3:]) / 3 < losses[0], losses


def test_resnet50_trainer_lars():
  from tensorflowonspark_b200.models import resnet
  torch.cuda.set_device(0)
  net = resnet.ResNetTrainer(depth=50, batch=8, image=64, device="cuda:0", optimizer="lars",
                             lr=4.0, trust_coefficient=0.001, weight_decay=5e-5)
  assert net.optim.lars and float(net.optim.hyper[4]) == pytest.approx(0.001)
  _check_trainer_step(net)
  _check_trainer_learns(net)


def test_cifar_resnet20_trainer_lars():
  from tensorflowonspark_b200.models import resnet
  torch.cuda.set_device(0)
  net = resnet.CifarResNetTrainer(depth=20, batch=32, device="cuda:0", optimizer="lars", lr=4.0,
                                  trust_coefficient=0.001, weight_decay=5e-5)
  _check_trainer_step(net)
  _check_trainer_learns(net)


def _free_port():
  import socket
  with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as sk:
    sk.bind(("127.0.0.1", 0))
    return str(sk.getsockname()[1])


def test_lars_two_ranks():
  """Peer-to-peer, NVLS (when available), HierComm (1 host x 2 GPUs, 2 one-GPU hosts) and
  GroupComm against NCCL all_reduce + the float64 reference; replicas bitwise identical."""
  if torch.cuda.device_count() < 2:
    pytest.skip("needs 2 GPUs")
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node",
                      "2", "--master-addr", "127.0.0.1", "--master-port", _free_port(),
                      os.path.join(root, "tools", "gpu_check_lars.py")],
                     capture_output=True, text=True, timeout=600, cwd=root)
  print(p.stdout[-4000:], p.stderr[-2000:])
  assert p.returncode == 0 and "LARS CHECK PASSED" in p.stdout

"""GPU tier: ResNet classifiers for any label set - the label-smoothed softmax_xent kernel against
float64, the default instance unchanged, padded heads of 37 and 1001 classes trained, evaluated and
served, a 1000-class backbone moved under a 37-class head, and a smoothed CIFAR ResNet-20."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from test_gpu_eval import _check_totals, _eval_batches, _rel_l2  # noqa: E402
from test_resnet_head_host import ref_smoothed_xent  # noqa: E402

pytestmark = pytest.mark.gpu


def _C():
  from tensorflowonspark_b200 import ops
  return ops.C()


def _pad8(v):
  return (v + 7) // 8 * 8


def _case(B, V, ld, dtype, seed):
  g = torch.Generator().manual_seed(seed)
  logits = torch.randn(B, ld, generator=g) * 3
  logits[:, V:] = 1e4                      # padding columns hold large values: never read
  labels = torch.randint(0, V, (B,), generator=g, dtype=torch.int32)
  for r in range(0, min(B, 40), 4):        # planted ties: the lower index is the arg-max
    y = max(1, int(labels[r]))
    labels[r] = y
    top = float(logits[r, :V].max()) + 1.0
    logits[r, y] = logits[r, y - 1 if r % 8 == 0 else min(y + 1, V - 1)] = top
  return logits.to(dtype).cuda(), labels.cuda()


def _run(logits, labels, V, ldd, scale, **kw):
  dl = torch.full((logits.shape[0], ldd), 7.0, dtype=torch.bfloat16, device="cuda")
  loss = torch.zeros(1, dtype=torch.float32, device="cuda")
  correct = torch.zeros(1, dtype=torch.float32, device="cuda")
  _C().softmax_xent(logits, labels, dl, loss, correct, V, scale, **kw)
  torch.cuda.synchronize()
  return dl, loss, correct


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("V", [10, 37, 1000, 1001])
@pytest.mark.parametrize("eps", [0.0, 0.1, 0.5, 1.0])
def test_softmax_xent_against_float64(dtype, V, eps):
  B, ld = 256, _pad8(V) + 8
  ldd, scale = ld, 1.0 / 256
  logits, labels = _case(B, V, ld, dtype, seed=V + int(eps * 10))
  dl, loss, correct = _run(logits, labels, V, ldd, scale, label_smoothing=eps)
  ref_loss, ref_grad = ref_smoothed_xent(logits.double(), labels, V, eps)
  want = float(ref_loss.sum()) * scale
  assert abs(float(loss) - want) <= 2e-5 * float(ref_loss.abs().sum()) * scale + 1e-6, (
      float(loss), want)
  ref_grad = ref_grad * scale
  got = dl[:, :V].double()
  # bf16 rounding of each element (8 significant bits: 2^-8 relative) on top of fp32 softmax
  # errors (absolute, below 1e-6 of the row's probabilities, which sum to 1)
  bound = 2.0 ** -8 * ref_grad.abs() + 1e-5 * scale
  assert bool(((got - ref_grad).abs() <= bound).all()), float(((got - ref_grad).abs() - bound).max())
  assert not dl[:, V:].float().any(), "padding columns of dlogits must be 0"
  amax = logits[:, :V].double().argmax(1)   # first index of the maximum
  assert int(correct) == int((amax == labels.long()).sum())
  assert int(correct) < B                   # the planted ties count as misses


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_zero_smoothing_is_the_default_instance_bit_for_bit(dtype):
  V = 1001
  logits, labels = _case(256, V, 1008, dtype, seed=5)
  a = _run(logits, labels, V, 1008, 1.0 / 256)
  b = _run(logits, labels, V, 1008, 1.0 / 256, label_smoothing=0.0)
  assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
  # the loss of one row is one atomic add onto 0: compare it bit for bit row by row
  for r in (0, 1, 77, 255):
    one = [_run(logits[r:r + 1], labels[r:r + 1], V, 1008, 0.5, **kw)[1]
           for kw in ({}, {"label_smoothing": 0.0})]
    assert torch.equal(one[0], one[1]), r


def test_smoothed_results_replay_bitwise_under_a_cuda_graph():
  V, B = 1001, 256
  logits, labels = _case(B, V, 1008, torch.float32, seed=6)
  C = _C()
  for rows in (B, 1):
    dl = torch.zeros(rows, 1008, dtype=torch.bfloat16, device="cuda")
    loss = torch.zeros(1, dtype=torch.float32, device="cuda")
    correct = torch.zeros(1, dtype=torch.float32, device="cuda")
    args = (logits[:rows], labels[:rows], dl, loss, correct, V, 1.0 / B)
    C.softmax_xent(*args, label_smoothing=0.1)
    torch.cuda.synchronize()
    eager = [t.clone() for t in (dl, loss, correct)]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      loss.zero_()
      correct.zero_()
      C.softmax_xent(*args, label_smoothing=0.1)
    for _ in range(3):
      dl.fill_(3.0)
      g.replay()
      torch.cuda.synchronize()
      assert torch.equal(dl, eager[0]) and torch.equal(correct, eager[2])
      if rows == 1:    # a single atomic add: the loss is bitwise too
        assert torch.equal(loss, eager[1])
      else:
        assert abs(float(loss) - float(eager[1])) <= 1e-6 * abs(float(eager[1]))


# --------------------------------------------------------------------------- trainers
def _resnet(V, **kw):
  from tensorflowonspark_b200.models import resnet
  kw.setdefault("seed", 3)
  return resnet.ResNetTrainer(depth=50, batch=8, image=64, num_classes=V, device="cuda:0",
                              label_smoothing=0.1, **kw)


def _fc_grads_against_autograd(net):
  """fc gradients of the last eager step against float64 autograd of F.cross_entropy(
  label_smoothing) on the step's own pooled features and logits (the optimizer only reads the
  gradient buffer; the weights are already updated, the gradient does not depend on them)."""
  st, V = net.store, net.num_classes
  avg = net.avg.double()
  logits = net.logits.double().clone().requires_grad_(True)
  loss = F.cross_entropy(logits[:, :V], net.labels.long(), label_smoothing=net.label_smoothing)
  loss.backward()
  want = float(loss.detach())
  assert abs(float(net.loss_sum) - want) <= 1e-5 * want, (float(net.loss_sum), want)
  gw_ref, gb_ref = logits.grad.t() @ avg, logits.grad.sum(0)
  gw, gb = st.g(net.fc.sw), st.g(net.fc.sbias)
  assert _rel_l2(gw[:V], gw_ref[:V]) <= 1e-2, _rel_l2(gw[:V], gw_ref[:V])
  assert _rel_l2(gb[:V], gb_ref[:V]) <= 1e-2, _rel_l2(gb[:V], gb_ref[:V])
  assert not gw[V:].any() and not gb[V:].any()


def _head_padding_is_zero(net):
  st, V = net.store, net.num_classes
  for spec in (net.fc.sw, net.fc.sbias):
    rows = slice(spec["offset"] + V * (spec["numel"] // spec["shape"][0]),
                 spec["offset"] + spec["numel"])
    assert not st.master[rows].any() and not st.weights[rows].any(), spec["name"]
    if net.optim.state1 is not None:
      assert not net.optim.state1[rows].any(), spec["name"]
  assert not st.f32(net.fc.sbias)[V:].any()


@pytest.mark.parametrize("V", [37, 1001])
def test_padded_head_gradients_padding_and_learning(V):
  net = _resnet(V, lr=0.05)
  assert net.VP == _pad8(V) and net.logits.shape == (8, net.VP)
  x, y = net.synthetic_batch(seed=1)
  first = float(net.train_step(x, y))
  assert abs(first - np.log(V)) < 1.0, first      # small initial logits: about log V
  _fc_grads_against_autograd(net)
  net.capture()
  losses = [float(net.train_step()) for _ in range(12)]
  assert all(np.isfinite(losses)) and losses[-1] < 0.6 * first, (first, losses)
  _head_padding_is_zero(net)
  # LARS (momentum, weight decay, per-layer trust ratios over ||w|| and ||g||)
  lars = _resnet(V, optimizer="lars", lr=1.0)
  for _ in range(4):
    lars.train_step(x, y)
  torch.cuda.synchronize()
  assert np.isfinite(float(lars.loss_sum))
  _head_padding_is_zero(lars)


@pytest.mark.parametrize("V", [37, 1001])
def test_padded_head_evaluation_and_serving(V):
  from tensorflowonspark_b200.models import resnet
  net = _resnet(V, lr=0.05, seed=4)
  x, y = net.synthetic_batch(seed=1)
  for _ in range(3):
    net.train_step(x, y)
  batches = _eval_batches(net, (8, 5), seed=40)
  got = _check_totals(net, batches)      # plain cross-entropy and top-1 / top-5 vs float64
  assert got["count"] == 13
  # the folded evaluation forward against the served export of the same state
  n = 5
  xs, ys = batches[1]
  net.eval_begin()
  net.eval_step(xs, ys)
  ref = net.logits[:n, :V].clone()
  served = resnet.build_served(net.state_dict(), **dict(net.export_builder_args, batch=8))
  for _ in range(2):                      # eager, then captured
    out = served(image=xs.cpu().numpy())
  assert out["logits"].shape == (n, V) and out["logits"].dtype == np.float32
  logits = torch.from_numpy(out["logits"]).cuda()
  assert _rel_l2(logits, ref) <= 2e-2, _rel_l2(logits, ref)
  pred = torch.from_numpy(out["prediction"])
  assert pred.shape == (n,) and int(pred.min()) >= 0 and int(pred.max()) < V
  assert torch.equal(pred.cuda(), logits.argmax(1))


def test_backbone_transfer_1000_to_37():
  src = _resnet(1000, lr=0.05, seed=1)
  x, y = src.synthetic_batch(seed=1)
  for _ in range(2):
    src.train_step(x, y)
  sd = src.state_dict()
  src.load_state_dict(sd)       # bf16 weights = the rounded masters, as a load leaves them
  dst = _resnet(37, seed=2)
  dst.load_backbone(sd)
  fresh = _resnet(37, seed=2)
  st = dst.store
  for spec in (dst.fc.sw, dst.fc.sbias):
    assert torch.equal(st.m(spec), fresh.store.m(spec)) and torch.equal(st.w(spec),
                                                                        fresh.store.w(spec))
  xe, ye = _eval_batches(src, (8,), seed=60)[0]
  ye = ye % 37
  feats = []
  for net in (src, dst):
    net.eval_begin()
    net.eval_step(xe, ye)
    torch.cuda.synchronize()
    feats.append(net.avg.clone())
  assert torch.equal(feats[0], feats[1])
  assert np.isfinite(float(dst.train_step(x, y % 37)))


def test_cifar_resnet20_100_classes_smoothed():
  from tensorflowonspark_b200.models import resnet
  net = resnet.CifarResNetTrainer(depth=20, batch=64, num_classes=100, device="cuda:0", seed=5,
                                  lr=0.1, label_smoothing=0.1)
  assert net.VP == 104
  x, y = net.synthetic_batch(seed=1)
  first = float(net.train_step(x, y))
  _fc_grads_against_autograd(net)
  net.capture()
  losses = [float(net.train_step()) for _ in range(40)]
  assert all(np.isfinite(losses)) and losses[-1] < first - 0.3, (first, losses)

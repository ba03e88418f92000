"""GPU tier: multi-label ResNet classifiers - sigmoid_bce and multilabel_eval_metrics against
float64 references, a multi-label ResNet-50 head trained (gradients against autograd, zero padding
rows, launch counts), a CIFAR ResNet-20 learning a synthetic tagging task, a softmax backbone moved
under a multi-label head, the composition with accumulation / clipping / averaging, and serving."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from test_gpu_eval import _rel_l2  # noqa: E402
from test_gpu_resnet_head import _head_padding_is_zero  # noqa: E402
from test_multilabel_host import ref_bce, ref_exact_rows, ref_multilabel_acc  # noqa: E402


def _load_pc():
  import importlib.util
  spec = importlib.util.spec_from_file_location(
      "plan_conformance", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                       "tools", "plan_conformance.py"))
  m = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(m)
  return m


pc = _load_pc()

pytestmark = pytest.mark.gpu

KEYS = {"count", "loss", "binary_accuracy", "exact_match", "precision", "recall", "f1",
        "macro_f1", "f1_per_class"}


def _C():
  from tensorflowonspark_b200 import ops
  return ops.C()


def _pad8(v):
  return (v + 7) // 8 * 8


def _bce_case(B, V, ld, seed, weighted):
  g = torch.Generator().manual_seed(seed)
  logits = torch.randn(B, ld, generator=g) * 3
  logits[:, V:] = 1e4                          # padding columns: never read
  logits[0, :V], logits[1, :V] = 1e4, -1e4     # saturated rows: finite loss and gradient
  logits[2, :V] = torch.where(torch.arange(V) % 2 == 0, 1e4, -1e4)
  targets = torch.randint(0, 2, (B, V), generator=g, dtype=torch.uint8)
  targets[3] *= 5                              # any nonzero byte is a positive
  targets[4] = (logits[4, :V] > 0).to(torch.uint8)   # an exact-match row
  pw = (torch.rand(V, generator=g) * 3).cuda() if weighted else None
  return logits.cuda(), targets.cuda(), pw


def _run_bce(logits, targets, V, ldd, scale, **kw):
  dl = torch.full((logits.shape[0], ldd), 7.0, dtype=torch.bfloat16, device="cuda")
  loss = torch.zeros(1, dtype=torch.float32, device="cuda")
  correct = torch.zeros(1, dtype=torch.float32, device="cuda")
  _C().sigmoid_bce(logits, targets, dl, loss, correct, V, scale, **kw)
  torch.cuda.synchronize()
  return dl, loss, correct


@pytest.mark.parametrize("V", [1, 7, 20, 1000, 1001])
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("weighted", [False, True])
def test_sigmoid_bce_against_float64(V, eps, weighted):
  B, ld = 256, _pad8(V) + 8
  scale = 1.0 / (B * V)
  logits, targets, pw = _bce_case(B, V, ld, seed=V + int(eps * 10) + 100 * weighted,
                                  weighted=weighted)
  dl, loss, correct = _run_bce(logits, targets, V, ld, scale, label_smoothing=eps, pos_weight=pw)
  ref_loss, ref_grad = ref_bce(logits, targets, V, eps, pw)
  want = float(ref_loss.sum()) * scale
  assert np.isfinite(float(loss)) and bool(torch.isfinite(dl.float()).all())
  assert abs(float(loss) - want) <= 2e-5 * want + 1e-7, (float(loss), want)
  ref_grad = ref_grad * scale
  got = dl[:, :V].double().cpu()
  pmax = 1.0 if pw is None else float(pw.max())
  # one bf16 rounding (2^-8 relative) on top of fp32 sigmoid errors (absolute, ~1e-7 of p t + 1)
  bound = 2.0 ** -8 * ref_grad.abs() + 1e-6 * (1 + pmax) * scale
  err = (got - ref_grad).abs() - bound
  assert bool((err <= 0).all()), float(err.max())
  assert not dl[:, V:].float().any(), "padding columns of dlogits must be 0"
  assert int(correct) == ref_exact_rows(logits, targets, V) and int(correct) >= 1


def test_sigmoid_bce_replays_bitwise_under_a_cuda_graph():
  V, B = 1001, 256
  logits, targets, pw = _bce_case(B, V, 1008, seed=6, weighted=True)
  C = _C()
  for rows in (B, 1):
    dl = torch.zeros(rows, 1008, dtype=torch.bfloat16, device="cuda")
    loss = torch.zeros(1, dtype=torch.float32, device="cuda")
    correct = torch.zeros(1, dtype=torch.float32, device="cuda")
    args = (logits[:rows], targets[:rows], dl, loss, correct, V, 1.0 / (B * V))
    kw = {"label_smoothing": 0.1, "pos_weight": pw}
    C.sigmoid_bce(*args, **kw)
    torch.cuda.synchronize()
    eager = [t.clone() for t in (dl, loss, correct)]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      loss.zero_()
      correct.zero_()
      C.sigmoid_bce(*args, **kw)
    for _ in range(3):
      dl.fill_(3.0)
      g.replay()
      torch.cuda.synchronize()
      assert torch.equal(dl, eager[0]) and torch.equal(correct, eager[2])
      if rows == 1:    # one atomic add onto 0: bitwise too
        assert torch.equal(loss, eager[1])
      else:
        # the same rows' losses (each >= 0, so their sum bounds the magnitudes) added with one
        # float atomic per row in any order: each total is within gamma_prob(rows - 1) of the
        # exact sum, so two totals within twice that
        bound = 2 * pc.gamma_prob(rows - 1) * abs(float(eager[1])) * (1 + 2.0 ** -20)
        assert abs(float(loss) - float(eager[1])) <= bound, (float(loss), float(eager[1]), bound)


# --------------------------------------------------------------------------- evaluation kernel
def _eval_case(B, V, ld, seed):
  g = torch.Generator().manual_seed(seed)
  logits = torch.randn(B, ld, generator=g) * 3
  logits[:, V:] = 1e4
  logits[:, :V][torch.rand(B, V, generator=g) < 0.02] = 0.0     # exactly 0 predicts negative
  targets = torch.randint(0, 2, (B, V), generator=g, dtype=torch.uint8)
  targets[7, 0] = 2                                              # invalid rows
  targets[B // 2, V - 1] = 255
  targets[9] = 0                                                 # an all-negative row
  return logits.cuda(), targets.cuda()


def _run_eval(logits, targets, n, V, acc=None):
  from tensorflowonspark_b200 import ops
  acc = torch.zeros(8 + 3 * V, dtype=torch.float64, device="cuda") if acc is None else acc
  nv = torch.tensor([n], dtype=torch.int32, device="cuda")
  ops.K.multilabel_eval_metrics(logits, targets, nv, acc, V)
  return acc


def _check_acc(got, want, V):
  got = got.cpu().tolist()
  for i in (0, 1, 3, 4):
    assert got[i] == want[i], (i, got[i], want[i])
  assert got[8:8 + 3 * V] == want[8:8 + 3 * V]
  assert got[5:8] == [0.0, 0.0, 0.0]
  assert abs(got[2] - want[2]) <= 1e-5 * max(1.0, abs(want[2])), (got[2], want[2])


@pytest.mark.parametrize("B,V", [(256, 20), (256, 1000), (256, 1001), (2100, 20)])
def test_multilabel_eval_metrics_against_reference(B, V):
  logits, targets = _eval_case(B, V, _pad8(V) + 8, seed=B + V)
  for n in (0, 1, 10, B - 1, B):
    _check_acc(_run_eval(logits, targets, n, V), ref_multilabel_acc(logits, targets, n, V), V)
  # a NaN logit predicts negative and makes the loss NaN; the counts stay exact
  bad = logits.clone()
  bad[3, :5] = float("nan")
  got, want = _run_eval(bad, targets, B, V).cpu().tolist(), ref_multilabel_acc(bad, targets, B, V)
  assert got[2] != got[2] and [got[i] for i in (0, 1, 3, 4)] == [want[i] for i in (0, 1, 3, 4)]
  assert got[8:] == want[8:]


def test_multilabel_eval_metrics_bitwise_across_runs_and_graph_replay():
  V, B = 1000, 2100
  logits, targets = _eval_case(B, V, 1008, seed=3)
  a = _run_eval(logits, targets, B - 3, V)
  b = _run_eval(logits, targets, B - 3, V)
  from tensorflowonspark_b200 import ops
  acc = torch.zeros(8 + 3 * V, dtype=torch.float64, device="cuda")
  nv = torch.tensor([B - 3], dtype=torch.int32, device="cuda")
  ops.K.multilabel_eval_metrics(logits, targets, nv, acc, V)    # warm-up outside the capture
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    acc.zero_()
    ops.K.multilabel_eval_metrics(logits, targets, nv, acc, V)
  for _ in range(2):
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(a, acc)


# --------------------------------------------------------------------------- ResNet-50
def _resnet(V=20, **kw):
  from tensorflowonspark_b200.models import resnet
  kw.setdefault("seed", 3)
  kw.setdefault("multi_label", True)
  return resnet.ResNetTrainer(depth=50, batch=8, image=64, num_classes=V, device="cuda:0", **kw)


def _fc_grads_against_autograd(net, pos_weight=None):
  """fc gradients of the last eager step against float64 autograd of
  F.binary_cross_entropy_with_logits on the step's own pooled features and logits."""
  st, V, eps = net.store, net.num_classes, net.label_smoothing
  avg = net.avg.double()
  logits = net.logits.double().clone().requires_grad_(True)
  t = (net.labels != 0).double() * (1 - eps) + eps / 2
  pw = None if pos_weight is None else torch.tensor(pos_weight, dtype=torch.float64, device="cuda")
  loss = F.binary_cross_entropy_with_logits(logits[:, :V], t, pos_weight=pw)
  loss.backward()
  want = float(loss.detach())
  assert abs(float(net.loss_sum) - want) <= 1e-5 * want, (float(net.loss_sum), want)
  gw_ref, gb_ref = logits.grad.t() @ avg, logits.grad.sum(0)
  gw, gb = st.g(net.fc.sw), st.g(net.fc.sbias)
  assert _rel_l2(gw[:V], gw_ref[:V]) <= 1e-2, _rel_l2(gw[:V], gw_ref[:V])
  assert _rel_l2(gb[:V], gb_ref[:V]) <= 1e-2, _rel_l2(gb[:V], gb_ref[:V])
  assert not gw[V:].any() and not gb[V:].any()


def test_resnet50_multilabel_gradients_padding_and_learning():
  pw = [0.5 + 0.1 * j for j in range(20)]
  net = _resnet(lr=0.1, label_smoothing=0.1, pos_weight=pw)
  assert net.VP == 24 and net.logits.shape == (8, 24) and net.labels.shape == (8, 20)
  x, y = net.synthetic_batch(seed=1)
  first = float(net.train_step(x, y))
  assert abs(first - float(np.log(2) * np.mean([(1 + p) / 2 for p in pw]))) < 0.2, first
  _fc_grads_against_autograd(net, pw)
  eager = [float(net.train_step()) for _ in range(3)]
  net.capture()
  captured = [float(net.train_step()) for _ in range(12)]
  losses = [first] + eager + captured
  # measured on one H100: 0.866 -> 0.617 after 3 eager steps -> 0.252 after 12 captured ones
  assert all(np.isfinite(losses)), losses
  assert eager[-1] < first and captured[-1] < captured[0] < first, losses
  assert captured[-1] < 0.5 * first, losses
  _head_padding_is_zero(net)
  lars = _resnet(optimizer="lars", lr=1.0)
  for _ in range(4):
    lars.train_step(x, y)
  torch.cuda.synchronize()
  assert np.isfinite(float(lars.loss_sum))
  _head_padding_is_zero(lars)


def test_multilabel_step_launches_as_many_kernels_as_the_default():
  from tensorflowonspark_b200 import ops
  counts = []
  for ml in (False, True):
    net = _resnet(multi_label=ml)
    x, y = net.synthetic_batch(seed=1)
    net.set_input(x, y)
    net.train_step()
    torch.cuda.synchronize()
    l0 = ops.launch_count()
    net.train_step()
    counts.append(ops.launch_count() - l0)
  assert counts[0] == counts[1], counts


# --------------------------------------------------------------------------- learning
PATCH_CLASSES = 8
PATCH_P = 0.3


def _patch_batch(B, gen):
  """A coloured 8x8 patch per class at its own place of a 4 x 4 grid (classes 0 .. 7 in cells
  0, 2, 5, 7, 8, 10, 13, 15), present with probability PATCH_P, on a noisy grey image."""
  cells = (0, 2, 5, 7, 8, 10, 13, 15)
  colours = torch.tensor([[255, 0, 0], [0, 255, 0], [0, 0, 255], [255, 255, 0], [255, 0, 255],
                          [0, 255, 255], [255, 255, 255], [0, 0, 0]], dtype=torch.float32)
  x = 128 + 20 * torch.randn(B, 32, 32, 3, generator=gen)
  y = (torch.rand(B, PATCH_CLASSES, generator=gen) < PATCH_P).to(torch.uint8)
  for c, cell in enumerate(cells):
    r0, c0 = (cell // 4) * 8, (cell % 4) * 8
    on = y[:, c].bool()
    x[on, r0:r0 + 8, c0:c0 + 8] = colours[c] + 10 * torch.randn(int(on.sum()), 8, 8, 3,
                                                                 generator=gen)
  return x.clamp(0, 255).to(torch.uint8), y


def test_cifar_resnet20_learns_a_synthetic_tagging_task():
  from tensorflowonspark_b200.models import resnet
  B = 128
  net = resnet.CifarResNetTrainer(depth=20, batch=B, num_classes=PATCH_CLASSES, device="cuda:0",
                                  seed=5, lr=0.1, multi_label=True)
  gen = torch.Generator().manual_seed(0)
  train = [_patch_batch(B, gen) for _ in range(16)]
  held = [_patch_batch(B, gen) for _ in range(4)]
  train = [(x.cuda(), y.cuda()) for x, y in train]
  net.train_step(*train[0])
  net.capture()
  for i in range(300):
    loss = net.train_step(*train[i % len(train)])
  res = net.evaluate([(x.numpy(), y.numpy().astype(bool)) for x, y in held])  # host bool targets
  assert set(res) == KEYS and res["count"] == 4 * B
  chance = 2 * PATCH_P / (1 + PATCH_P)     # micro-F1 of predicting every class present: 0.46
  # measured on one H100: held-out micro-F1 1.000 (macro 1.000, exact match 1.000) after 300
  # steps, training loss 0.011
  assert res["f1"] > 0.9 > chance, (res, float(loss))
  assert res["macro_f1"] > 0.9 and res["exact_match"] > 0.8, res


# --------------------------------------------------------------------------- transfer
def test_backbone_transfer_1000_softmax_to_20_multilabel():
  src = _resnet(V=1000, multi_label=False, lr=0.05, seed=1)
  x, y = src.synthetic_batch(seed=1)
  for _ in range(2):
    src.train_step(x, y)
  sd = src.state_dict()
  src.load_state_dict(sd)       # bf16 weights = the rounded masters, as a load leaves them
  dst = _resnet(seed=2)
  dst.load_backbone(sd)
  xm, ym = dst.synthetic_batch(seed=7)
  feats = []
  for net, lab in ((src, y), (dst, ym)):
    net.eval_begin()
    net.eval_step(xm, lab)
    torch.cuda.synchronize()
    feats.append(net.avg.clone())
  assert torch.equal(feats[0], feats[1])
  losses = [float(dst.train_step(xm, ym)) for _ in range(4)]
  assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses


# --------------------------------------------------------------------------- composition
def test_accumulation_clipping_and_average_with_multilabel():
  from tensorflowonspark_b200.models import resnet
  net = _resnet(lr=0.05, gradient_accumulation_steps=2, clip_norm=1.0, ema_decay=0.9)
  x, y = net.synthetic_batch(seed=1)
  net.set_input(x, y)
  net.capture()
  losses = [float(net.train_step()) for _ in range(16)]
  # measured on one H100: 0.658 -> 0.334 over 8 updates
  assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
  assert np.isfinite(float(net.grad_norm))
  xe, ye = net.synthetic_batch(seed=9)
  for averaged in (False, True):
    res = net.evaluate([(xe, ye)], averaged=averaged)
    assert set(res) == KEYS and res["count"] == 8 and len(res["f1_per_class"]) == 20
  # the totals of a partial batch against the float64 reference on the batch's own logits
  net.eval_begin()
  net.eval_step(xe[:5], ye[:5])
  got = net.eval_end()
  want = resnet.multilabel_totals(ref_multilabel_acc(net.logits, ye, 5, 20), 20)
  for k in KEYS - {"f1_per_class", "loss"}:
    assert (got[k] != got[k] and want[k] != want[k]) or got[k] == want[k], k
  assert abs(got["loss"] - want["loss"]) <= 1e-5 * want["loss"]
  bad = ye.clone()
  bad[2, 3] = 2
  with pytest.raises(ValueError, match="label byte other than 0 or 1"):
    net.evaluate([(xe, bad)])


# --------------------------------------------------------------------------- serving
def test_serving_multilabel_and_softmax_exports():
  from tensorflowonspark_b200.models import resnet
  n = 5
  for ml in (True, False):
    net = _resnet(multi_label=ml, lr=0.05, seed=4)
    x, y = net.synthetic_batch(seed=1)
    for _ in range(3):
      net.train_step(x, y)
    xs, ys = net.synthetic_batch(seed=11)
    net.eval_begin()
    net.eval_step(xs[:n], ys[:n])
    ref = net.logits[:n, :20].clone()
    served = resnet.build_served(net.state_dict(), **dict(net.export_builder_args, batch=8))
    for _ in range(2):                      # eager, then captured
      out = served(image=xs[:n].cpu().numpy())
    logits = torch.from_numpy(out["logits"])
    assert logits.shape == (n, 20) and _rel_l2(logits.cuda(), ref) <= 2e-2, _rel_l2(
        logits.cuda(), ref)
    pred = torch.from_numpy(out["prediction"])
    if ml:
      assert pred.shape == (n, 20) and pred.dtype == torch.uint8
      assert torch.equal(pred, (logits > 0).to(torch.uint8))
      assert torch.equal(served.net.logits[:n, :20].cpu(), logits)
    else:
      assert pred.shape == (n,) and torch.equal(pred, logits.argmax(1))

"""GPU tier: held-out evaluation of the ResNet trainers - the eval_metrics kernel against a float64
reference, the folded evaluation forward on a training trainer's buffers against fp32 PyTorch,
that evaluation leaves the training state untouched, that the totals do not depend on how the
images are batched, and (2+ GPUs) the totals across ranks through tools/gpu_check_eval.py."""
import os
import socket
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def ref_metrics(logits, labels, n, V):
  """float64 totals with the kernel's rules: rows >= n and columns >= V are never read; rank =
  #{l_j > l_y} + #{j < y : l_j == l_y}; a NaN label logit is wrong and makes the loss NaN."""
  L = logits[:n, :V].double().cpu()
  y = labels[:n].long().cpu()
  valid = (y >= 0) & (y < V)
  L, y = L[valid], y[valid]
  ly = L.gather(1, y[:, None])[:, 0]
  j = torch.arange(V)
  rank = (L > ly[:, None]).sum(1) + ((L == ly[:, None]) & (j[None, :] < y[:, None])).sum(1)
  ok = ~torch.isnan(ly)
  return {"count": int(valid.sum()), "top1": int(((rank < 1) & ok).sum()),
          "top5": int(((rank < 5) & ok).sum()), "invalid": int((~valid).sum()),
          "loss": float((torch.logsumexp(L, 1) - ly).sum())}


def run_metrics(logits, labels, n, V, acc=None):
  from tensorflowonspark_b200 import ops
  acc = torch.zeros(8, dtype=torch.float64, device="cuda") if acc is None else acc
  nv = torch.tensor([n], dtype=torch.int32, device="cuda")
  ops.K.eval_metrics(logits, labels, nv, acc, V)
  return acc


def unpack(acc):
  a = acc.cpu().tolist()
  return {"count": int(a[0]), "top1": int(a[1]), "top5": int(a[2]), "invalid": int(a[3]),
          "loss": a[4]}


def _case(B, ld, V, seed):
  g = torch.Generator().manual_seed(seed)
  logits = torch.randn(B, ld, generator=g) * 3
  logits[:, V:] = 1e4                      # padding columns hold large values: never read
  labels = torch.randint(0, V, (B,), generator=g, dtype=torch.int32)
  for r in range(0, 40, 4):                # planted ties on both sides of the label
    y = int(labels[r]) if 0 < int(labels[r]) < V - 1 else 1
    labels[r] = y
    top = float(logits[r, :V].max()) + 1.0
    logits[r, y] = top
    logits[r, y - 1 if r % 8 == 0 else y + 1] = top     # lower index wins: wrong at top-1
  logits[-1] = float("nan")                # beyond n_valid in every case but n = B
  return logits.cuda(), labels.cuda()


@pytest.mark.parametrize("B,ld,V", [(256, 1000, 1000), (256, 16, 10)])
def test_eval_metrics_against_float64(B, ld, V):
  logits, labels = _case(B, ld, V, seed=B + V)
  for n in (0, 1, B - 1):
    got, ref = unpack(run_metrics(logits, labels, n, V)), ref_metrics(logits, labels, n, V)
    for k in ("count", "top1", "top5", "invalid"):
      assert got[k] == ref[k], (n, k, got, ref)
    assert abs(got["loss"] - ref["loss"]) <= 1e-6 * max(1.0, abs(ref["loss"])), (n, got, ref)
  assert ref_metrics(logits, labels, B - 1, V)["top1"] < B - 1   # the planted ties count
  # a NaN label logit: the row is wrong and the loss is NaN
  bad = logits.clone()
  bad[3, int(labels[3])] = float("nan")
  got, ref = unpack(run_metrics(bad, labels, B - 1, V)), ref_metrics(bad, labels, B - 1, V)
  assert (got["count"], got["top1"], got["top5"]) == (ref["count"], ref["top1"], ref["top5"])
  assert got["loss"] != got["loss"]
  # out-of-range labels are counted as invalid, not scored
  lab = labels.clone()
  lab[5], lab[9] = V, -1
  got, ref = unpack(run_metrics(logits, lab, B - 1, V)), ref_metrics(logits, lab, B - 1, V)
  assert got["invalid"] == 2 and (got["count"], got["top1"], got["top5"]) == (
      ref["count"], ref["top1"], ref["top5"])


def test_eval_metrics_bitwise_across_runs_and_graph_replay():
  logits, labels = _case(256, 1000, 1000, seed=3)
  a = run_metrics(logits, labels, 255, 1000)
  b = run_metrics(logits, labels, 255, 1000)
  acc = torch.zeros(8, dtype=torch.float64, device="cuda")
  nv = torch.tensor([255], dtype=torch.int32, device="cuda")
  from tensorflowonspark_b200 import ops
  ops.K.eval_metrics(logits, labels, nv, acc, 1000)   # warm-up outside the capture
  acc.zero_()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    ops.K.eval_metrics(logits, labels, nv, acc, 1000)
  g.replay()
  torch.cuda.synchronize()
  assert torch.equal(a, b) and torch.equal(a, acc)


# --------------------------------------------------------------------------- networks
def _perturb(net, seed):
  """Non-trivial batch-norm parameters and running statistics (as tools/gpu_check.py does)."""
  gen = torch.Generator().manual_seed(seed)
  sd = net.state_dict()
  for k in list(sd):
    if k.endswith(".gamma"):
      sd[k] = 0.3 + 0.6 * torch.rand(sd[k].shape, generator=gen)
    elif k.endswith(".beta"):
      sd[k] = 0.1 * torch.randn(sd[k].shape, generator=gen)
  sd["__running__"] = 0.05 * torch.randn(sd["__running__"].shape, generator=gen)
  net.load_state_dict(sd)
  for _, bn in net._fold_units():
    bn.running_var.copy_(0.5 + torch.rand(bn.C, generator=gen).cuda())


def _rel_l2(a, b):
  return float((a.double() - b.double()).norm() / b.double().norm())


def _eval_batches(net, sizes, seed):
  out = []
  for i, n in enumerate(sizes):
    x, y = net.synthetic_batch(seed=seed + i)
    out.append((x[:n], y[:n]))
  return out


def _check_totals(net, batches, tv_forward=None):
  """eval_step over ``batches`` (eager, then captured, then replayed); the totals must equal the
  float64 metrics of the logits each step left in ``net.logits``."""
  net.eval_begin()
  ref = {"count": 0, "top1": 0, "top5": 0, "loss": 0.0}
  for x, y in batches:
    net.eval_step(x, y)
    logits = net.logits.clone()
    r = ref_metrics(logits, y, len(x), net.num_classes)
    for k in ref:
      ref[k] += r[k]
    if tv_forward is not None:
      err = _rel_l2(logits[:len(x), :net.num_classes], tv_forward(x))
      assert err <= 4e-2, err
  got = net.eval_end()
  assert got["count"] == ref["count"]
  assert round(got["top1"] * got["count"]) == ref["top1"]
  assert round(got["top5"] * got["count"]) == ref["top5"]
  assert abs(got["loss"] * got["count"] - ref["loss"]) <= 1e-5 * abs(ref["loss"])
  return got


def _torchvision_resnet50(net):
  import torchvision
  from tensorflowonspark_b200.ops import igemm
  tv = torchvision.models.resnet50(weights=None, num_classes=net.num_classes).cuda().float().eval()
  st = net.store
  cv = lambda w: w.permute(0, 3, 1, 2).contiguous()  # noqa: E731

  def put_bn(bn, m):
    m.weight.copy_(st.f32(bn.sg)), m.bias.copy_(st.f32(bn.sb))
    m.running_mean.copy_(bn.running_mean), m.running_var.copy_(bn.running_var)

  with torch.no_grad():
    tv.conv1.weight.copy_(cv(igemm.unpack_stem_weight(st.w(net.stem_w).float())))
    put_bn(net.stem_bn, tv.bn1)
    for blk in net.blocks:
      si, bi = int(blk.name[5]) - 1, int(blk.name.split(".")[1])
      t = getattr(tv, "layer{}".format(si + 1))[bi]
      for u, c, m in ((blk.u1, t.conv1, t.bn1), (blk.u2, t.conv2, t.bn2), (blk.u3, t.conv3, t.bn3)):
        c.weight.copy_(cv(st.w(u.conv.sw).float()))
        put_bn(u.bn, m)
      if blk.ds is not None:
        t.downsample[0].weight.copy_(cv(st.w(blk.ds.conv.sw).float()))
        put_bn(blk.ds.bn, t.downsample[1])
    tv.fc.weight.copy_(st.w(net.fc.sw).float()), tv.fc.bias.copy_(st.f32(net.fc.sbias))
  mean = torch.tensor(net.mean, device="cuda").view(1, 3, 1, 1)
  std = torch.tensor(net.std, device="cuda").view(1, 3, 1, 1)

  def fwd(x):
    with torch.no_grad():
      return tv((x.permute(0, 3, 1, 2).float() / 255.0 - mean) / std)
  return fwd


def test_resnet50_eval_logits_and_totals():
  from tensorflowonspark_b200.models import resnet
  B = 16
  net = resnet.ResNetTrainer(depth=50, batch=B, image=224, device="cuda:0", seed=11, lr=0.01)
  _perturb(net, 5)
  x, y = net.synthetic_batch(seed=0)
  for _ in range(2):
    net.train_step(x, y)
  batches = _eval_batches(net, (B, B, B - 3), seed=100)
  _check_totals(net, batches, _torchvision_resnet50(net))
  # the training buffers still hold the staged training batch
  assert torch.equal(net.in_u8, x) and torch.equal(net.labels, y)


def _cifar_reference(net):
  """fp32 basic-block ResNet from the trainer's bf16 filters, fp32 scale / offset and running
  statistics."""
  st = net.store

  def cbn(x, u, relu=True, res=None):
    w = st.w(u.conv.sw).float().permute(0, 3, 1, 2)
    y = F.conv2d(x, w, stride=u.conv.stride, padding=u.conv.pad)
    y = F.batch_norm(y, u.bn.running_mean, u.bn.running_var, st.f32(u.bn.sg), st.f32(u.bn.sb),
                     False, 0.0, u.bn.eps)
    if res is not None:
      y = y + res
    return F.relu(y) if relu else y

  mean = torch.tensor(net.mean, device="cuda").view(1, 3, 1, 1)
  std = torch.tensor(net.std, device="cuda").view(1, 3, 1, 1)

  def fwd(x):
    with torch.no_grad():
      h = (x.permute(0, 3, 1, 2).float() / 255.0 - mean) / std
      h = F.pad(h, (0, 0, 0, 0, 0, 5))            # 8 input channels, 5 of them zero
      h = cbn(h, net.stem)
      for b in net.blocks:
        idn = cbn(h, b.ds, relu=False) if b.ds is not None else h
        h = cbn(cbn(h, b.u1), b.u2, res=idn)
      h = h.mean((2, 3))
      return (h @ st.w(net.fc.sw).float().t() + st.f32(net.fc.sbias))[:, :net.num_classes]
  return fwd


def test_cifar_resnet20_eval_logits_and_totals():
  from tensorflowonspark_b200.models import resnet
  B = 64
  net = resnet.CifarResNetTrainer(depth=20, batch=B, device="cuda:0", seed=7, lr=0.01)
  _perturb(net, 9)
  x, y = net.synthetic_batch(seed=0)
  for _ in range(2):
    net.train_step(x, y)
  _check_totals(net, _eval_batches(net, (B, B, 17), seed=200), _cifar_reference(net))


def _state(net):
  sd = {"master": net.store.master, "weights": net.store.weights, "aux32": net.store.aux32,
        "running": net.running.tensor(), "in_u8": net.in_u8, "labels": net.labels}
  for k, v in net.optim.state_dict().items():
    if isinstance(v, torch.Tensor):
      sd["optim." + k] = v
  return {k: v.detach().clone() for k, v in sd.items()}


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("model", ["resnet50", "cifar20"])
def test_evaluation_leaves_training_untouched(model, graph):
  """Trainer A: 3 steps, evaluate, 3 steps; trainer B (same seed): 6 steps.  Evaluation must not
  change one bit of A's training state (parameters, running statistics, optimizer state, staged
  batch).  The two trainers' later steps are compared within the run-to-run spread of training,
  whose fp32 atomics make two runs differ in the last bits."""
  from tensorflowonspark_b200.models import resnet

  def make():
    if model == "resnet50":
      return resnet.ResNetTrainer(depth=50, batch=16, image=64, device="cuda:0", seed=3, lr=0.01)
    return resnet.CifarResNetTrainer(depth=20, batch=32, device="cuda:0", seed=3, lr=0.01)

  a, b = make(), make()
  losses = {}
  for net in (a, b):
    x, y = net.synthetic_batch(seed=1)
    net.set_input(x, y)           # one batch staged once, as the drivers do
    if graph:
      net.capture()
    losses[id(net)] = []
  for net, evaluate in ((a, True), (b, False)):
    for i in range(6):
      if i == 3 and evaluate:
        torch.cuda.synchronize()
        before = _state(net)
        net.evaluate(_eval_batches(net, (net.B, 5), seed=50))
        after = _state(net)
        for k in before:
          assert torch.equal(before[k], after[k]), k
      losses[id(net)].append(float(net.train_step()))
  la, lb = losses[id(a)], losses[id(b)]
  assert all(v == v for v in la + lb)
  for u, v in zip(la, lb):
    assert abs(u - v) <= 1e-3 * abs(v), (la, lb)
  assert _rel_l2(a.store.master, b.store.master) <= 1e-4


def test_totals_do_not_depend_on_batching():
  from tensorflowonspark_b200.models import resnet
  B = 32
  net = resnet.CifarResNetTrainer(depth=20, batch=B, device="cuda:0", seed=5)
  _perturb(net, 4)
  xs, ys = zip(*_eval_batches(net, (B,) * 4, seed=300))
  X, Y = torch.cat(xs)[:3 * B + 5], torch.cat(ys)[:3 * B + 5]
  one = net.evaluate([(X[i:i + B], Y[i:i + B]) for i in range(0, len(X), B)])
  cuts = [0, 5, 5 + B, 5 + 2 * B, len(X)]
  two = net.evaluate([(X[c0:c1].cpu().numpy(), Y[c0:c1].cpu().numpy())   # host path
                      for c0, c1 in zip(cuts, cuts[1:])])
  assert one["count"] == two["count"] == 3 * B + 5
  assert (one["top1"], one["top5"]) == (two["top1"], two["top5"])


def _free_port():
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    return str(s.getsockname()[1])


def test_eval_totals_two_ranks():
  """Peer-to-peer, NVLS (when available), HierComm (1 host x 2 GPUs, 2 one-GPU hosts) and
  GroupComm: identical totals on every rank, computed with rank 0's running statistics."""
  if torch.cuda.device_count() < 2:
    pytest.skip("needs 2 GPUs")
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node",
                      "2", "--master-addr", "127.0.0.1", "--master-port", _free_port(),
                      os.path.join(root, "tools", "gpu_check_eval.py")],
                     capture_output=True, text=True, timeout=900, cwd=root)
  print(p.stdout[-4000:], p.stderr[-2000:])
  assert p.returncode == 0 and "EVAL CHECK PASSED" in p.stdout

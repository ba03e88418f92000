"""GPU tier: held-out evaluation of the segmentation U-Net - the seg_eval_metrics kernel against a
float64 reference and against pixel_xent's arg-max, its bitwise reproducibility, the evaluation
logits against an fp32 PyTorch U-Net, that evaluation (and predict) leave training untouched,
that the totals do not depend on batching or mask dtype, the checkpoint round trip, and (2+ GPUs)
the totals across ranks through tools/gpu_check_seg_eval.py."""
import os
import socket
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SLOTS = 72


def ref_seg(logits, labels, n, V):
  """float64 totals with the kernel's rules: images >= n and channels >= V are never read; the
  prediction is the lowest index among the maximal logits (pixel_xent); labels outside [0, V)
  are counted as invalid and not scored."""
  L = logits[:n].double().reshape(-1, 8)[:, :V].cpu()
  y = labels[:n].reshape(-1).long().cpu()
  valid = (y >= 0) & (y < V)
  L, y = L[valid], y[valid]
  pred = L.argmax(1)   # first maximal index
  cm = torch.zeros(8, 8, dtype=torch.float64)
  cm.index_put_((y, pred), torch.ones(len(y), dtype=torch.float64), accumulate=True)
  loss = float((torch.logsumexp(L, 1) - L.gather(1, y[:, None])[:, 0]).sum())
  return {"count": int(valid.sum()), "correct": int((pred == y).sum()),
          "invalid": int((~valid).sum()), "loss": loss, "cm": cm}


def unpack(acc):
  a = acc.double().cpu()
  return {"count": int(a[0]), "correct": int(a[1]), "invalid": int(a[2]), "loss": float(a[3]),
          "cm": a[4:68].reshape(8, 8)}


class _Metric(object):
  def __init__(self, logits):
    from tensorflowonspark_b200 import ops
    self.ops = ops
    self.partial = torch.zeros(ops.C().seg_eval_scratch(logits.numel() // 8), dtype=torch.float64,
                               device="cuda")
    self.counter = torch.zeros(1, dtype=torch.int32, device="cuda")

  def __call__(self, logits, labels, n, V, acc=None, nv=None):
    acc = torch.zeros(SLOTS, dtype=torch.float64, device="cuda") if acc is None else acc
    nv = torch.tensor([n], dtype=torch.int32, device="cuda") if nv is None else nv
    self.ops.K.seg_eval_metrics(logits, labels, nv, acc, self.partial, self.counter, V)
    return acc


def _case(B, HW, V, seed):
  g = torch.Generator().manual_seed(seed)
  logits = torch.randn(B, HW, HW, 8, generator=g) * 3
  logits[..., V:] = 1e4                    # padded channels hold large values: never read
  labels = torch.randint(0, V, (B, HW, HW), generator=g, dtype=torch.int32)
  flat_l, flat_y = logits.view(-1, 8), labels.view(-1)
  P = flat_y.numel()
  idx = torch.randperm(P, generator=g)
  for k, p in enumerate(idx[:600].tolist()):   # planted ties on both sides of the label
    y = int(flat_y[p]) if V == 2 else min(max(int(flat_y[p]), 1), V - 2)
    flat_y[p] = y
    top = float(flat_l[p, :V].max()) + 1.0
    flat_l[p, y] = top
    other = y - 1 if (k % 2 == 0 and y > 0) else (y + 1 if y + 1 < V else y - 1)
    flat_l[p, other] = top               # the lower index wins the tie
  bad = idx[600:660]
  flat_y[bad[:20]], flat_y[bad[20:40]], flat_y[bad[40:]] = -1, V, 255
  return logits.to(torch.bfloat16).cuda(), labels.cuda()


def _assert_same(got, ref, ctx):
  for k in ("count", "correct", "invalid"):
    assert got[k] == ref[k], (ctx, k, got[k], ref[k])
  assert torch.equal(got["cm"], ref["cm"]), ctx
  assert abs(got["loss"] - ref["loss"]) <= 1e-5 * max(1.0, abs(ref["loss"])), (ctx, got, ref)


@pytest.mark.parametrize("V", [2, 3, 8])
def test_seg_eval_metrics_against_float64(V):
  B, HW = 6, 48
  logits, labels = _case(B, HW, V, seed=V)
  run = _Metric(logits)
  for n in (0, 1, B - 1, B):
    got, ref = unpack(run(logits, labels, n, V)), ref_seg(logits, labels, n, V)
    _assert_same(got, ref, n)
  ref = ref_seg(logits, labels, B, V)
  assert ref["invalid"] > 0 and ref["correct"] < ref["count"]
  # the planted ties count: scoring with the higher index would differ
  L = logits.double().reshape(-1, 8)[:, :V].cpu()
  assert int((L.flip(1).argmax(1) != V - 1 - L.argmax(1)).sum()) > 0


def test_seg_eval_correct_matches_pixel_xent():
  from tensorflowonspark_b200 import ops
  B, HW, V = 4, 64, 3
  logits, labels = _case(B, HW, V, seed=11)
  labels = labels.clamp(0, V - 1)          # pixel_xent scores every pixel
  got = unpack(_Metric(logits)(logits, labels, B, V))
  loss = torch.zeros(1, dtype=torch.float32, device="cuda")
  correct = torch.zeros(1, dtype=torch.float32, device="cuda")
  ops.K.pixel_xent(logits, labels, None, loss, correct, V, 1.0)
  assert got["count"] == B * HW * HW and got["correct"] == int(correct.item())


def test_seg_eval_metrics_bitwise_across_runs_and_graph_replay():
  from tensorflowonspark_b200 import ops
  B, HW, V = 64, 128, 3                    # the trainer's shape: 1,056 CTAs, the last ones empty
  logits, labels = _case(B, HW, V, seed=3)
  run = _Metric(logits)
  a = run(logits, labels, B - 1, V)
  b = run(logits, labels, B - 1, V)
  acc = torch.zeros(SLOTS, dtype=torch.float64, device="cuda")
  nv = torch.tensor([B - 1], dtype=torch.int32, device="cuda")
  run(logits, labels, 0, V, acc, nv)       # warm-up outside the capture
  acc.zero_()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    ops.K.seg_eval_metrics(logits, labels, nv, acc, run.partial, run.counter, V)
  g.replay()
  torch.cuda.synchronize()
  first = acc.clone()
  acc.zero_()
  g.replay()                               # the counter was reset inside the kernel
  torch.cuda.synchronize()
  assert torch.equal(a, b) and torch.equal(a, first) and torch.equal(a, acc)
  assert int(run.counter.item()) == 0
  _assert_same(unpack(a), ref_seg(logits, labels, B - 1, V), "B-1")


# --------------------------------------------------------------------------- the network
def _perturb(net, seed):
  """Non-trivial decoder batch-norm parameters and running statistics."""
  gen = torch.Generator().manual_seed(seed)
  sd = net.state_dict()
  for k in list(sd):
    if k.endswith(".gamma"):
      sd[k] = 0.5 + 0.5 * torch.rand(sd[k].shape, generator=gen)
    elif k.endswith(".beta"):
      sd[k] = 0.1 * torch.randn(sd[k].shape, generator=gen)
  sd["__running__"] = 0.05 * torch.randn(sd["__running__"].shape, generator=gen)
  net.load_state_dict(sd)
  for up in net.ups:
    up.bn.running_var.copy_(0.5 + torch.rand(up.bn.C, generator=gen).cuda())


def _rel_l2(a, b):
  return float((a.double() - b.double()).norm() / b.double().norm())


def _torch_unet(net):
  """fp32 PyTorch U-Net from the trainer's bf16 filters, fp32 biases / scale / offset and running
  statistics: MobileNetV2 encoder (ReLU6, depthwise 3x3), decoder conv_transpose2d + batch norm +
  ReLU, concatenation, last transposed convolution."""
  from tensorflowonspark_b200.models import unet
  st = net.store
  enc = net.encoder

  def fwd(x_u8):
    with torch.no_grad():
      h = (x_u8.permute(0, 3, 1, 2).float() / 255.0 - 0.5) / 0.5
      bufs = {enc.x.data_ptr(): F.pad(h, (0, 0, 0, 0, 0, 5))}
      for layer in enc.layers:
        if isinstance(layer, unet._FrozenConv):
          w = layer.w.float().permute(0, 3, 1, 2)
          y = F.conv2d(bufs[layer.x.data_ptr()], w, layer.bias, layer.stride, layer.k // 2)
          y = y.clamp(0, 6) if layer.act == 2 else (y.clamp(min=0) if layer.act == 1 else y)
        elif isinstance(layer, unet._FrozenDepthwise):
          C = layer.w.shape[1]
          w = layer.w.float().t().reshape(C, 1, 3, 3)
          y = F.conv2d(bufs[layer.x.data_ptr()], w, layer.bias, layer.stride, 1, groups=C)
          y = y.clamp(0, 6)
        else:
          y = bufs[layer.y.data_ptr()] + bufs[layer.x.data_ptr()]
        bufs[layer.y.data_ptr()] = y
      skips = [bufs[s.data_ptr()] for s in enc.skips]
      h = skips[-1]
      for i, up in enumerate(net.ups):
        w = st.w(up.sw).float().permute(0, 3, 1, 2)
        h = F.conv_transpose2d(h, w, None, 2, 1, 1)
        h = F.batch_norm(h, up.bn.running_mean, up.bn.running_var, st.f32(up.bn.sg),
                         st.f32(up.bn.sb), False, 0.0, up.bn.eps).clamp(min=0)
        h = torch.cat([h, skips[-2 - i]], 1)
      w = st.w(net.s_last).float().permute(0, 3, 1, 2)
      out = F.conv_transpose2d(h, w, st.f32(net.s_last_b), 2, 1, 1)
      return out.permute(0, 2, 3, 1)[..., :net.classes]
  return fwd


def _masks(x):
  return ((x[..., 0] > 127).int() + (x[..., 1] > 200).int()).to(torch.int32)


def _eval_batches(net, sizes, seed):
  out = []
  for i, n in enumerate(sizes):
    x, _ = net.synthetic_batch(seed=seed + i)
    out.append((x[:n], _masks(x[:n])))
  return out


def test_unet_eval_logits_and_totals():
  from tensorflowonspark_b200.models import unet
  B = 8
  net = unet.UNetTrainer(batch=B, image=128, classes=3, device="cuda:0", seed=11)
  x, y = net.synthetic_batch(seed=0)
  for _ in range(2):
    net.train_step(x, _masks(x))
  _perturb(net, 5)
  ref_net = _torch_unet(net)
  net.eval_begin()
  tot = {"count": 0, "correct": 0, "invalid": 0, "loss": 0.0, "cm": torch.zeros(8, 8, dtype=torch.float64)}
  errs = []
  for bx, by in _eval_batches(net, (B, B, B - 3), seed=100):   # eager, capture, replay
    net.eval_step(bx, by)
    logits = net.logits.clone()
    r = ref_seg(logits, by, len(bx), 3)
    for k in tot:
      tot[k] = tot[k] + r[k]
    errs.append(_rel_l2(logits[:len(bx), ..., :3], ref_net(bx)))
  print("U-Net eval logits vs fp32 PyTorch, relative L2:", errs)
  assert max(errs) <= 4e-2, errs
  res = net.eval_end()
  got = unpack(torch.tensor(net._evaluator.acc.tolist()))
  _assert_same(got, tot, "totals")
  assert res["count"] == tot["count"] == (3 * B - 3) * 128 * 128 and res["images"] == 3 * B - 3
  assert res["accuracy"] == tot["correct"] / tot["count"]
  cm = tot["cm"][:3, :3]
  iou = (cm.diag() / (cm.sum(0) + cm.sum(1) - cm.diag())).tolist()
  assert res["iou"] == pytest.approx(iou, rel=1e-12)
  # the training buffers still hold the staged training batch
  assert torch.equal(net.in_u8, x) and torch.equal(net.labels, _masks(x))


def _state(net):
  sd = {"master": net.store.master, "weights": net.store.weights, "aux32": net.store.aux32,
        "running": net.running.tensor(), "in_u8": net.in_u8, "labels": net.labels}
  for i, up in enumerate(net.ups):
    sd["up{}.sum".format(i)], sd["up{}.sumsq".format(i)] = up.bn.sum, up.bn.sumsq
  for k, v in net.optim.state_dict().items():
    if isinstance(v, torch.Tensor):
      sd["optim." + k] = v
  return {k: v.detach().clone() for k, v in sd.items()}


@pytest.mark.parametrize("graph", [False, True])
def test_evaluation_leaves_training_untouched(graph):
  """Trainer A: 3 steps, evaluate, 3 steps; trainer B (same seed): 6 steps.  Evaluation must not
  change one bit of A's training state.  The later losses are compared within the run-to-run
  spread of training (fp32 atomics).  The parameters are not compared across the two trainers:
  Adam turns the last-bit differences of near-zero gradients into whole steps of lr."""
  from tensorflowonspark_b200.models import unet

  def make():
    return unet.UNetTrainer(batch=8, image=128, classes=3, device="cuda:0", seed=3)

  a, b = make(), make()
  losses = {}
  for net in (a, b):
    x, _ = net.synthetic_batch(seed=1)
    net.set_input(x, _masks(x))           # one batch staged once, as the drivers do
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


def test_predict_accumulates_no_batch_statistics():
  from tensorflowonspark_b200.models import unet
  net = unet.UNetTrainer(batch=4, image=128, classes=3, device="cuda:0", seed=2)
  x, _ = net.synthetic_batch(seed=1)
  net.train_step(x, _masks(x))
  out = net.predict(x)
  torch.cuda.synchronize()
  assert out.shape == (4, 128, 128, 3)
  for up in net.ups:
    assert not bool(up.bn.sum.any()) and not bool(up.bn.sumsq.any()), up.bn.name


def test_totals_do_not_depend_on_batching_or_mask_dtype():
  from tensorflowonspark_b200.models import unet
  B = 8
  net = unet.UNetTrainer(batch=B, image=128, classes=3, device="cuda:0", seed=5)
  _perturb(net, 4)
  xs, ys = zip(*_eval_batches(net, (B,) * 3, seed=300))
  X, Y = torch.cat(xs)[:2 * B + 5], torch.cat(ys)[:2 * B + 5]
  one = net.evaluate([(X[i:i + B], Y[i:i + B]) for i in range(0, len(X), B)])   # device int32
  acc_one = net._evaluator.acc.clone()
  cuts = [0, 5, 5 + B, len(X)]
  two = net.evaluate([(X[c0:c1].cpu().numpy(), Y[c0:c1].to(torch.uint8).cpu().numpy())   # host uint8
                      for c0, c1 in zip(cuts, cuts[1:])])
  acc_two = net._evaluator.acc.clone()
  assert one["count"] == two["count"] == (2 * B + 5) * 128 * 128
  assert one["images"] == two["images"] == 2 * B + 5
  assert torch.equal(acc_one[:3], acc_two[:3]) and torch.equal(acc_one[4:68], acc_two[4:68])
  # out-of-range mask values are never narrowed into range: 256 as int32 and -1 stay invalid
  bad = Y[:B].clone()
  bad[0, 0, 0], bad[1, 5, 5] = 256, -1
  with pytest.raises(ValueError):
    net.evaluate([(X[:B], bad)])
  with pytest.raises(ValueError):
    net.evaluate([(X[:B].cpu().numpy(), bad.cpu().numpy())])


def test_checkpoint_round_trip_keeps_evaluation():
  from tensorflowonspark_b200.models import unet
  net = unet.UNetTrainer(batch=8, image=128, classes=3, device="cuda:0", seed=6)
  x, _ = net.synthetic_batch(seed=1)
  for _ in range(3):
    net.train_step(x, _masks(x))
  batches = _eval_batches(net, (8, 3), seed=70)
  a = net.evaluate(batches)
  acc_a = net._evaluator.acc.clone()
  fresh = unet.UNetTrainer(batch=8, image=128, classes=3, device="cuda:0", seed=99)
  fresh.load_state_dict(net.state_dict())
  b = fresh.evaluate(batches)
  assert torch.equal(acc_a, fresh._evaluator.acc)
  assert a["count"] == b["count"] and a["loss"] == b["loss"] and a["iou"] == b["iou"]
  # a parameters-only checkpoint (no "__running__") still loads
  sd = net.state_dict()
  sd.pop("__running__")
  fresh.load_state_dict(sd)


def _free_port():
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    return str(s.getsockname()[1])


def test_seg_eval_totals_two_ranks():
  """Peer-to-peer, NVLS (when available), HierComm and GroupComm: identical totals on every
  rank, equal to rank 0's model scored alone on the union of the ranks' shards."""
  if torch.cuda.device_count() < 2:
    pytest.skip("needs 2 GPUs")
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node",
                      "2", "--master-addr", "127.0.0.1", "--master-port", _free_port(),
                      os.path.join(root, "tools", "gpu_check_seg_eval.py")],
                     capture_output=True, text=True, timeout=900, cwd=root)
  print(p.stdout[-4000:], p.stderr[-2000:])
  assert p.returncode == 0 and "SEG EVAL CHECK PASSED" in p.stdout

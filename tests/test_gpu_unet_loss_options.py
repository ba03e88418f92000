"""The U-Net's loss options (``ignore_index``, ``class_weights``) on the GPU: the optioned
pixel_xent against a float64 F.cross_entropy(weight, ignore_index), the label pre-pass
seg_label_norm (exact and bitwise reproducible), the equivalences with the default path, the
optioned seg_eval_metrics against numpy, and a 21-class trainer with void pixels end to end."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_gpu_unet_classes as gc  # noqa: E402


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

CASES = [(3, 8), (8, 8), (9, 16), (21, 24), (150, 152), (256, 256)]   # (V, VP)


def _C():
  return gc._C()


def _weights(V, VP, seed, zero=(1,)):
  """Dyadic weights (multiples of 1/4, exact in any sum of a few million), some zero."""
  g = torch.Generator().manual_seed(seed)
  w = torch.randint(1, 12, (V,), generator=g).double() / 4
  for c in zero:
    if c < V:
      w[c] = 0.0
  wd = torch.zeros(VP, dtype=torch.float32)
  wd[:V] = w.float()
  return w, wd.cuda()


def _norm_buffers(V):
  norm = torch.zeros(3, dtype=torch.float64, device="cuda")
  scratch = torch.zeros(_C().seg_label_norm_scratch(V), dtype=torch.int64, device="cuda")
  return norm, scratch


def _ref_weights(y64, V, w, ignore):
  """Per pixel: w[y] (1 without weights or outside [0, V)), 0 when ignored; and the ignore mask."""
  ok = (y64 >= 0) & (y64 < V)
  wy = torch.ones(len(y64), dtype=torch.float64)
  if w is not None:
    wy = torch.where(ok, w[y64.clamp(0, V - 1).long()], wy)
  ign = (y64 == ignore) if ignore is not None else torch.zeros(len(y64), dtype=torch.bool)
  wy[ign] = 0.0
  return wy, ign


def _run(l, y, V, ignore, wd):
  norm, scratch = _norm_buffers(V)
  C = _C()
  C.seg_label_norm(y, norm, scratch, V, ignore, wd)
  d = torch.full_like(l, float("nan"))
  loss, hits = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
  C.pixel_xent(l, y, d, loss, hits, V, 1.0, ignore, wd, norm)
  torch.cuda.synchronize()
  assert not scratch.any(), "pre-pass scratch left at zero"
  return norm.cpu(), d, float(loss), float(hits)


@pytest.mark.parametrize("V,VP", CASES)
@pytest.mark.parametrize("ignore,weighted", [(255, True), (0, True), (255, False), (None, True),
                                             (-1, False)])
def test_optioned_pixel_xent_against_float64(V, VP, ignore, weighted):
  shape = (3, 7, 11)
  P = 3 * 7 * 11
  l = gc._logits(V, VP, shape, seed=V)
  y = gc._labels(V, shape, seed=V)     # includes V - 1, V, 255 and -1
  y.view(-1)[40:60] = 255
  w, wd = _weights(V, VP, seed=V) if weighted else (None, None)
  norm, d, loss, hits = _run(l, y, V, ignore, wd)
  l64, y64 = l.double().cpu().view(P, VP), y.cpu().view(P)
  wy, ign = _ref_weights(y64, V, w, ignore)
  sw = float(wy.sum())
  assert norm[0].item() == sw and norm[1].item() == float((~ign).sum())
  assert norm[2].item() == float(np.float32(1.0 / sw))
  # float64 F.cross_entropy on the bf16 logits, for the labels it accepts
  term, p, ok = gc._ref_terms(l64, y64, V)
  if VP == 8:   # the 8-channel kernel's rule for a label in [V, 8): l_y is that padding channel
    pad = (y64 >= V) & (y64 < 8)
    term[pad] -= l64[pad, y64[pad].long()]
  assert loss == pytest.approx(float((wy * term).sum()) / sw, rel=1e-4)
  sel = ok & ~ign
  if sel.any():
    xl = l64[sel, :V].clone().requires_grad_(True)
    wt = w if w is not None else torch.ones(V, dtype=torch.float64)
    ref = F.cross_entropy(xl, y64[sel].long(), weight=wt, reduction="sum") / sw
    ref.backward()
    got = d.double().cpu().view(P, VP)
    assert torch.allclose(got[sel, :V], xl.grad, rtol=1e-2, atol=1e-3 * float(wt.max()) / sw)
  onehot = torch.zeros(P, V, dtype=torch.float64)
  onehot[sel, y64[sel].long()] = 1.0
  want = wy[:, None] * (p - onehot) / sw
  got = d.double().cpu().view(P, VP)
  assert torch.allclose(got[:, :V], want, rtol=1e-2, atol=1e-3 * float(wy.max()) / sw)
  assert torch.equal(got[:, V:], torch.zeros(P, VP - V, dtype=torch.float64)), "padding"
  assert torch.equal(got[ign], torch.zeros(int(ign.sum()), VP, dtype=torch.float64)), "ignored"
  am = gc._ref_argmax(l64, V)
  assert hits == float(((am == y64) & ~ign).sum())
  # NaN logits: hits follow the arg-max rule over S
  ln = gc._logits(V, VP, shape, seed=V + 1, nan=True)
  _, _, _, hits = _run(ln, y, V, ignore, wd)
  assert hits == float(((gc._ref_argmax(ln.double().cpu().view(P, VP), V) == y64) & ~ign).sum())


@pytest.mark.parametrize("V,VP", CASES)
def test_empty_denominator_gives_zero_loss_and_gradient(V, VP):
  shape = (2, 9, 13)
  l = gc._logits(V, VP, shape, seed=2 * V, nan=True)
  # every pixel ignored
  y = torch.full(shape, 7, dtype=torch.int32, device="cuda")
  norm, d, loss, hits = _run(l, y, V, 7, None)
  assert norm.tolist() == [0.0, 0.0, 0.0] and loss == 0.0 and hits == 0.0
  assert not d.any() and not d.isnan().any()
  # only classes of weight zero present
  y = torch.randint(0, 2, shape, dtype=torch.int32).cuda() * (V - 1)
  _, wd = _weights(V, VP, seed=1, zero=(0, V - 1))
  norm, d, loss, hits = _run(l, y, V, None, wd)
  assert norm.tolist() == [0.0, float(y.numel()), 0.0] and loss == 0.0
  assert not d.any() and not d.isnan().any()


def test_label_prepass_is_exact_and_bitwise_reproducible():
  V = 150
  g = torch.Generator().manual_seed(3)
  y = torch.randint(0, V, (64, 128, 128), generator=g, dtype=torch.int32)
  y[:, 60:70] = 255
  y[0, 0, :5] = -3
  y = y.cuda()
  w, wd = _weights(V, 152, seed=4)
  C = _C()
  norm, scratch = _norm_buffers(V)
  C.seg_label_norm(y, norm, scratch, V, 255, wd)
  first = norm.clone()
  y64 = y.cpu().view(-1)
  wy, ign = _ref_weights(y64, V, w, 255)
  assert first[1].item() == float((~ign).sum()) == 64 * 118 * 128
  assert first[0].item() == float(wy.sum())
  for _ in range(2):
    C.seg_label_norm(y, norm, scratch, V, 255, wd)
    assert torch.equal(norm, first)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    C.seg_label_norm(y, norm, scratch, V, 255, wd)
  for _ in range(2):
    norm.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(norm, first)
  # a graph replay reads the labels present at replay time
  y[:, :64] = 255
  graph.replay()
  torch.cuda.synchronize()
  wy2, ign2 = _ref_weights(y.cpu().view(-1), V, w, 255)
  assert norm[0].item() == float(wy2.sum()) and norm[1].item() == float((~ign2).sum())
  assert not scratch.any()


@pytest.mark.parametrize("V,VP", CASES)
def test_absent_ignore_value_is_bitwise_the_default_path(V, VP):
  C = _C()
  G = 1 if VP == 8 else max(2, 1 << (VP // 8 - 1).bit_length())   # lanes per pixel
  for shape in [(4, 32, 32), (1, 1, 32 // G)]:   # the second: one warp holds every pixel
    P = int(np.prod(shape))
    l = gc._logits(V, VP, shape, seed=11)
    y = torch.randint(0, V, shape, dtype=torch.int32).cuda()
    d0 = torch.zeros_like(l)
    loss0, hits0 = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    C.pixel_xent(l, y, d0, loss0, hits0, V, 1.0 / P)
    norm, d, loss, hits = _run(l, y, V, 100000, None)
    assert norm.tolist() == [P, P, 1.0 / P]
    assert torch.equal(d, d0), "dlogits"
    assert hits == float(hits0)
    if P <= 32:
      assert loss == float(loss0), "loss"
    else:
      # the same per-warp partials (sums of pixel losses >= 0, so the total bounds their
      # magnitudes), one float atomic per warp in any order: each total is within
      # gamma_prob(warps - 1) of the exact sum, so two totals within twice that
      warps = -(-P * G // 32)
      bound = 2 * pc.gamma_prob(warps - 1) * abs(float(loss0)) * (1 + 2.0 ** -20)
      assert abs(loss - float(loss0)) <= bound, (loss, float(loss0), bound)


def _bf16_ulp(x):
  m = x.abs().float().clamp_min(torch.finfo(torch.float32).tiny)
  return torch.pow(2.0, torch.floor(torch.log2(m)) - 7)


@pytest.mark.parametrize("V,VP", CASES)
def test_uniform_weights_match_unweighted_within_one_ulp(V, VP):
  shape = (2, 33, 17)
  l = gc._logits(V, VP, shape, seed=21)
  y = torch.randint(0, V, shape, dtype=torch.int32).cuda()
  wd = torch.zeros(VP, dtype=torch.float32, device="cuda")
  wd[:V] = 3.0
  _, d1, loss1, _ = _run(l, y, V, None, None)
  _, d3, loss3, _ = _run(l, y, V, None, wd)
  a, b = d1.float(), d3.float()
  assert bool(((a - b).abs() <= _bf16_ulp(torch.maximum(a.abs(), b.abs()))).all())
  assert loss3 == pytest.approx(loss1, rel=1e-5)


# ----------------------------------------------------------------------------- evaluation
def _ref_eval(l, y, n, V, w, ignore):
  P = l.numel() // l.shape[-1]
  ppi = P // l.shape[0]
  l64 = l.double().cpu().view(P, l.shape[-1])[:n * ppi]
  y64 = y.cpu().view(P)[:n * ppi]
  ign = y64 == ignore
  ok = (y64 >= 0) & (y64 < V) & ~ign
  term, _, _ = gc._ref_terms(l64, y64, V)
  wy = w[y64.clamp(0, V - 1).long()] if w is not None else torch.ones(len(y64), dtype=torch.float64)
  am = gc._ref_argmax(l64, V)
  cm = torch.zeros(V * V, dtype=torch.float64)
  cm.index_add_(0, (y64[ok].long() * V + am[ok]), torch.ones(int(ok.sum()), dtype=torch.float64))
  return {"count": int(ok.sum()), "correct": int((am[ok] == y64[ok]).sum()),
          "invalid": int((~ok & ~ign).sum()), "loss": float((wy * term)[ok].sum()), "cm": cm}


@pytest.mark.parametrize("V,VP", [(3, 8), (8, 8), (21, 24), (150, 152), (256, 256)])
@pytest.mark.parametrize("ignore", [255, 1])
def test_optioned_seg_eval_metrics_against_numpy(V, VP, ignore):
  from tensorflowonspark_b200.models import unet
  shape = (7, 9, 23)
  l = gc._logits(V, VP, shape, seed=5 * V)
  y = gc._labels(V, shape, seed=5 * V)
  y.view(-1)[100:160] = 255
  w, wd = _weights(V, VP, seed=V)
  acc, scratch, counter = gc._eval_tensors(V, l)
  n_valid = torch.tensor([5], dtype=torch.int32, device="cuda")
  _C().seg_eval_metrics(l, y, n_valid, acc, scratch, counter, V, ignore, wd)
  torch.cuda.synchronize()
  ref = _ref_eval(l, y, 5, V, w, ignore)
  _, conf, ld, _ = unet.seg_eval_layout(V)
  a = acc.cpu()
  assert [int(a[i]) for i in range(3)] == [ref["count"], ref["correct"], ref["invalid"]]
  assert float(a[3]) == pytest.approx(ref["loss"], rel=1e-5)
  cm = a[conf:conf + ld * ld].view(ld, ld)[:V, :V].reshape(-1)
  assert torch.equal(cm, ref["cm"])
  assert int(counter) == 0


@pytest.mark.parametrize("V,VP", [(3, 8), (21, 24), (256, 256)])
def test_optioned_seg_eval_metrics_is_bitwise_reproducible(V, VP):
  shape = (8, 64, 64)
  l = gc._logits(V, VP, shape, seed=9)
  y = gc._labels(V, shape, seed=9)
  y[:, 20:30] = 255
  _, wd = _weights(V, VP, seed=2)
  acc, scratch, counter = gc._eval_tensors(V, l)
  n_valid = torch.tensor([8], dtype=torch.int32, device="cuda")
  C = _C()
  one = torch.zeros_like(acc)
  C.seg_eval_metrics(l, y, n_valid, one, scratch, counter, V, 255, wd)
  want = torch.zeros_like(acc)
  for _ in range(2):
    C.seg_eval_metrics(l, y, n_valid, acc, scratch, counter, V, 255, wd)
    want = want + one
    assert torch.equal(acc, want), "eager launches differ"
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    C.seg_eval_metrics(l, y, n_valid, acc, scratch, counter, V, 255, wd)
  for _ in range(2):
    g.replay()
    want = want + one
    torch.cuda.synchronize()
    assert torch.equal(acc, want), "graph replay differs from the eager launches"
  a4 = torch.zeros_like(acc)
  n_valid.fill_(4)
  C.seg_eval_metrics(l[:4].contiguous(), y[:4].contiguous(), n_valid, a4, scratch, counter, V,
                     255, wd)
  C.seg_eval_metrics(l[4:].contiguous(), y[4:].contiguous(), n_valid, a4, scratch, counter, V,
                     255, wd)
  torch.cuda.synchronize()
  ints = [0, 1, 2] + list(range(4, acc.numel()))   # every slot but the loss is an integer count
  assert torch.equal(a4[ints], one[ints])
  assert float(a4[3]) == pytest.approx(float(one[3]), rel=1e-12)


# ----------------------------------------------------------------------------- the 21-class U-Net
V21 = 21


def _void_labels(x, rows):
  from tensorflowonspark_b200.models import unet
  y = unet.synthetic_labels(x, V21)
  y[:, rows[0]:rows[1]] = 255
  return y


def _class_weights():
  return [0.5 + (c % 4) * 0.5 for c in range(V21)]   # 0.5 .. 2.0


def test_21_class_void_loss_and_last_layer_gradients():
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.models import unet
  B, cw = 8, _class_weights()
  net = unet.UNetTrainer(batch=B, image=128, classes=V21, seed=3, ignore_index=255,
                         class_weights=cw)
  x, _ = net.synthetic_batch(seed=1)
  y = _void_labels(x, (50, 70))
  net.train_step(x, y)
  net.set_input(x, y)
  net._forward(True)
  st, K = net.store, ops.K
  net.loss_sum.zero_()
  net.correct.zero_()
  K.seg_label_norm(net.labels, net.loss_norm, net._norm_scratch, V21, 255, net.weights)
  K.pixel_xent(net.logits, net.labels, net.dlogits, net.loss_sum, net.correct, V21, 1.0,
               255, net.weights, net.loss_norm)
  net.optim.zero_grads()
  net.p_last_wgrad.run()
  K.colsum(net.dlogits, st.g(net.s_last_b))
  torch.cuda.synchronize()
  # fp32 autograd with the same F.cross_entropy options, on the trainer's logits
  lg = net.logits[..., :V21].float().permute(0, 3, 1, 2).clone().requires_grad_(True)
  wt = torch.tensor(cw, dtype=torch.float32, device="cuda")
  ref = F.cross_entropy(lg, y.long(), weight=wt, ignore_index=255)
  ref.backward()
  assert float(net.loss_sum) == pytest.approx(ref.item(), rel=1e-4)
  keep = y != 255
  assert float(net.loss_norm[0]) == float((wt[y.clamp(0, V21 - 1).long()] * keep).sum())
  assert int(net.loss_norm[1]) == int(keep.sum())
  d = net.dlogits.float()
  assert not d[~keep].any() and not d[..., V21:].any()
  g_ref = lg.grad.permute(0, 2, 3, 1)
  se = gc._load("seg_eval_ref_loss_opts", os.path.join("tests", "test_gpu_seg_eval.py"))
  assert se._rel_l2(d[..., :V21], g_ref) <= 1e-2
  h = net.cats[-1][0].float().permute(0, 3, 1, 2)
  w = st.w(net.s_last).float().permute(0, 3, 1, 2).clone().requires_grad_(True)
  b = st.f32(net.s_last_b).clone().requires_grad_(True)
  out = F.conv_transpose2d(h, w, b, 2, 1, 1)
  g_full = torch.zeros_like(out)
  g_full[:, :V21] = lg.grad
  out.backward(g_full)
  assert se._rel_l2(st.g(net.s_last).permute(0, 3, 1, 2), w.grad) <= 1e-2
  assert se._rel_l2(st.g(net.s_last_b), b.grad) <= 1e-2


def test_21_class_void_captured_step_uses_each_batch_denominator():
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.models import unet
  B, cw = 8, _class_weights()
  net = unet.UNetTrainer(batch=B, image=128, classes=V21, seed=4, ignore_index=255,
                         class_weights=cw)
  x, _ = net.synthetic_batch(seed=2)
  net.set_input(x, _void_labels(x, (60, 64)))
  net.train_step()
  net.capture()
  wt = torch.tensor(cw, dtype=torch.float64)
  for rows in ((60, 64), (10, 100)):   # different void fractions, one graph
    y = _void_labels(x, rows)
    net.set_input(x, y)
    net.train_step()
    torch.cuda.synchronize()
    keep = (y != 255).cpu()
    yc = y.cpu().clamp(0, V21 - 1).long()
    assert net.loss_norm[0].item() == float((wt[yc] * keep).sum())
    assert net.loss_norm[1].item() == float(keep.sum())
    lg = net.logits[..., :V21].float().permute(0, 3, 1, 2)
    ref = F.cross_entropy(lg, y.long(), weight=wt.float().cuda(), ignore_index=255)
    assert float(net.loss_sum) == pytest.approx(float(ref), rel=1e-4), rows
    # the captured loss kernels equal an eager launch on the same logits and labels, bit for bit
    d_graph, norm_graph = net.dlogits.clone(), net.loss_norm.clone()
    norm, scratch = _norm_buffers(V21)
    d = torch.zeros_like(net.dlogits)
    loss, hits = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    ops.K.seg_label_norm(net.labels, norm, scratch, V21, 255, net.weights)
    ops.K.pixel_xent(net.logits, net.labels, d, loss, hits, V21, 1.0, 255, net.weights, norm)
    torch.cuda.synchronize()
    assert torch.equal(norm, norm_graph) and torch.equal(d, d_graph)
    assert float(hits) == float(net.correct)


def test_21_class_void_trainer_learns_and_evaluates():
  from tensorflowonspark_b200.models import unet
  B = 16
  net = unet.UNetTrainer(batch=B, image=128, classes=V21, seed=5, lr=2e-3, ignore_index=255,
                         class_weights=_class_weights())
  held = []
  for i in range(2):
    hx, _ = net.synthetic_batch(seed=500 + i)
    held.append((hx, _void_labels(hx, (0, 16))))
  before = net.evaluate(held)
  xs = [net.synthetic_batch(seed=i)[0] for i in range(4)]
  net.set_input(xs[0], _void_labels(xs[0], (40, 56)))
  net.train_step()
  net.capture()
  first = float(net.loss_sum)
  for i in range(600):
    x = xs[i % 4]
    net.set_input(x, _void_labels(x, (40 + i % 7, 56 + i % 5)))
    loss = net.train_step()
  last = float(loss)
  after = net.evaluate(held)
  print("21 classes with void pixels: loss {:.3f} -> {:.3f}, mean IoU {:.3f} -> {:.3f}".format(
      first, last, before["mean_iou"], after["mean_iou"]))
  assert last < 0.85 * first
  assert after["mean_iou"] > 1.3 * before["mean_iou"]
  void = 2 * B * 16 * 128
  assert after["count"] == 2 * B * 128 * 128 - void and after["ignored"] == void
  # the same masks as uint8 host arrays, evaluated twice: identical totals
  host = [(x.cpu(), y.to(torch.uint8).cpu()) for x, y in held]
  np.testing.assert_equal(net.evaluate(host), after)
  # a default trainer still rejects the void label
  plain = unet.UNetTrainer(batch=B, image=128, classes=V21, seed=5, training=False)
  with pytest.raises(ValueError, match="outside"):
    plain.evaluate(held)
  # an inference-only trainer with the options scores the void masks
  served = unet.UNetTrainer(batch=B, image=128, classes=V21, seed=5, training=False,
                            ignore_index=255)
  res = served.evaluate(held)
  assert res["ignored"] == void and res["count"] == 2 * B * 128 * 128 - void

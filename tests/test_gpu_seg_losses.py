"""The U-Net's focal and Dice losses on the GPU: seg_loss_grad and seg_dice_stats against the float64
references of tools/seg_loss_reference.py, focal at gamma = 0 bitwise pixel_xent, the Dice
statistics bitwise reproducible under graph replay, and a 21-class trainer with void pixels for
each loss: last-layer gradients against fp32 autograd, captured against eager, launch sequences,
accumulation, learning, checkpoints and serving."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_gpu_unet_classes as gc  # noqa: E402
import test_gpu_unet_loss_options as lo  # noqa: E402
import test_seg_losses_host as host  # noqa: E402

pytestmark = pytest.mark.gpu

R = host.R
CASES = lo.CASES
GAMMAS = host.GAMMAS
OPTIONS = [(None, False), (255, True)]   # (ignore_index, class weights)


def _C():
  return gc._C()


def _inputs(V, VP, seed, ignore, weighted, shape=(3, 7, 11)):
  """bf16 logits, labels (V - 1, V, 255 and -1 among them, a void band with ignore) and a few
  pixels whose logit gap makes p_y exactly 1 in fp32."""
  P = int(np.prod(shape))
  l = gc._logits(V, VP, shape, seed=seed)
  y = gc._labels(V, shape, seed=seed)
  if ignore is not None:
    y.view(-1)[40:60] = ignore
  lf = l.view(P, VP)
  for i in range(60, 70):   # p_y = 1: e_j = exp(-120) underflows
    yi = int(y.view(-1)[i]) % V
    y.view(-1)[i] = yi
    lf[i, :V] = -60.0
    lf[i, yi] = 60.0
  w, wd = lo._weights(V, VP, seed=V) if weighted else (None, None)
  return l, y, w, wd


def _grad(l, y, V, ignore, wd, norm, **terms):
  d = torch.full_like(l, float("nan"))
  loss, hits = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
  _C().seg_loss_grad(l, y, d, loss, hits, V, 1.0 / y.numel(), ignore, wd, norm, **terms)
  return d, loss, hits


def _norm(y, V, ignore, wd):
  if ignore is None and wd is None:
    return None
  norm, scratch = lo._norm_buffers(V)
  _C().seg_label_norm(y, norm, scratch, V, ignore, wd)
  return norm


def _dice_buffers(VP):
  coef = torch.full((2, VP), float("nan"), device="cuda")
  scratch = torch.zeros(_C().seg_dice_scratch(VP), dtype=torch.float32, device="cuda")
  return coef, scratch


def _pad_term(l64, y64, V, VP, s):
  """The 8-channel kernels read a label in [V, 8) from its padding channel (pixel_xent's rule)."""
  if VP != 8:
    return 0.0
  pad = (y64 >= V) & (y64 < 8)
  return float((s[pad] * l64[pad, y64[pad].long()]).sum())


def _check_grad(got, want, V, VP, atol):
  P = want.shape[0]
  g = got.double().cpu().view(P, VP)
  assert torch.allclose(g[:, :V], want, rtol=1e-2, atol=atol)
  assert torch.equal(g[:, V:], torch.zeros(P, VP - V, dtype=torch.float64)), "padding"


@pytest.mark.parametrize("V,VP", CASES)
@pytest.mark.parametrize("ignore,weighted", OPTIONS)
@pytest.mark.parametrize("gamma", GAMMAS)
def test_focal_against_float64(V, VP, ignore, weighted, gamma):
  l, y, w, wd = _inputs(V, VP, V, ignore, weighted)
  norm = _norm(y, V, ignore, wd)
  d, loss, hits = _grad(l, y, V, ignore, wd, norm, focal_gamma=gamma)
  torch.cuda.synchronize()
  P = y.numel()
  l64, y64 = l.double().cpu().view(P, VP), y.cpu().view(P).long()
  s = R.pixel_scale(y64, V, w, ignore)
  ref_loss, ref = R.focal(l64, y64, V, gamma, w, ignore)
  ref_loss -= _pad_term(l64, y64, V, VP, s)
  assert float(loss) == pytest.approx(ref_loss, rel=1e-4, abs=1e-6)
  _check_grad(d, ref, V, VP, atol=1e-3 * float(s.max()))   # 1e-3 max w / sum w, or 1e-3 / P
  assert bool(torch.isfinite(d.float()).all())
  if ignore is not None:
    assert not d.view(P, VP)[(y64 == ignore).cuda()].any(), "ignored pixels"
  gap = d.view(P, VP)[60:70].float()   # p_y = 1 exactly: q = 0
  if gamma > 0:
    assert not gap.any()
  am = gc._ref_argmax(l64, V)
  keep = y64 != ignore if ignore is not None else torch.ones(P, dtype=torch.bool)
  assert float(hits) == float(((am == y64) & keep).sum())


@pytest.mark.parametrize("V,VP", CASES)
@pytest.mark.parametrize("ignore,weighted", OPTIONS)
def test_focal_at_gamma_zero_is_bitwise_pixel_xent(V, VP, ignore, weighted):
  for shape in [(3, 7, 11), (4, 32, 32)]:
    l, y, w, wd = _inputs(V, VP, V + 5, ignore, weighted, shape)
    norm = _norm(y, V, ignore, wd)
    d, loss, hits = _grad(l, y, V, ignore, wd, norm, focal_gamma=0.0)
    d0 = torch.full_like(l, float("nan"))
    loss0, hits0 = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    _C().pixel_xent(l, y, d0, loss0, hits0, V, 1.0 / y.numel(), ignore, wd, norm)
    torch.cuda.synchronize()
    assert torch.equal(d.view(torch.int16), d0.view(torch.int16)), "dlogits bits"
    assert float(hits) == float(hits0)
    assert float(loss) == pytest.approx(float(loss0), rel=1e-6)


@pytest.mark.parametrize("V,VP", CASES)
@pytest.mark.parametrize("ignore,weighted", OPTIONS)
@pytest.mark.parametrize("with_ce", [False, True], ids=["dice", "dice_ce"])
def test_dice_against_float64(V, VP, ignore, weighted, with_ce):
  smooth = 1e-5
  l, y, w, wd = _inputs(V, VP, 2 * V, ignore, weighted)
  norm = _norm(y, V, ignore, wd)
  coef, scratch = _dice_buffers(VP)
  C = _C()
  d = torch.full_like(l, float("nan"))
  loss, hits = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
  C.seg_dice_stats(l, y, coef, loss, scratch, V, smooth, ignore, wd)
  C.seg_loss_grad(l, y, d, loss, hits, V, 1.0 / y.numel(), ignore, wd, norm,
                  cross_entropy=with_ce, dice_coef=coef)
  torch.cuda.synchronize()
  assert not scratch[-1:].any(), "ticket left at zero"
  P = y.numel()
  l64, y64 = l.double().cpu().view(P, VP), y.cpu().view(P).long()
  ref_loss, ref, A, B = R.dice(l64, y64, V, smooth, w, ignore)
  c = coef.double().cpu()
  assert torch.allclose(c[0, :V], A, rtol=1e-4, atol=0) and torch.allclose(c[1, :V], B, rtol=1e-4)
  assert not c[:, V:].any()
  if with_ce:
    s = R.pixel_scale(y64, V, w, ignore)
    ce_loss, ce = R.focal(l64, y64, V, 0.0, w, ignore)
    ref_loss += ce_loss - _pad_term(l64, y64, V, VP, s)
    ref = ref + ce
  assert float(loss) == pytest.approx(ref_loss, rel=1e-4, abs=1e-6)
  _check_grad(d, ref, V, VP, atol=1e-3 * float(ref.abs().max()))
  if ignore is not None:
    assert not d.view(P, VP)[(y64 == ignore).cuda()].any(), "ignored pixels"


@pytest.mark.parametrize("V,VP", [(3, 8), (21, 24), (150, 152), (256, 256)])
def test_dice_stats_bitwise_reproducible_and_graph_replayable(V, VP):
  shape = (16, 64, 64)
  l = gc._logits(V, VP, shape, seed=9)
  y = gc._labels(V, shape, seed=9)
  y[:, 20:30] = 255
  _, wd = lo._weights(V, VP, seed=2)
  C = _C()
  coef, scratch = _dice_buffers(VP)
  loss = torch.zeros(1, device="cuda")
  norm = _norm(y, V, 255, wd)

  def run():
    loss.zero_()
    C.seg_dice_stats(l, y, coef, loss, scratch, V, 1e-5, 255, wd)
    d, _, _ = _grad(l, y, V, 255, wd, norm, cross_entropy=False, dice_coef=coef)
    return coef.clone(), loss.clone(), d
  first = run()
  second = run()
  for a, b in zip(first, second):
    assert torch.equal(a, b), "eager launches differ"
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    loss.zero_()
    C.seg_dice_stats(l, y, coef, loss, scratch, V, 1e-5, 255, wd)
  for _ in range(2):
    coef.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(coef, first[0]) and torch.equal(loss, first[1]), "graph replay differs"
  assert not scratch[-1:].any(), "ticket left at zero"


@pytest.mark.parametrize("V,VP", CASES)
def test_all_ignored_batch_gives_zero_dice_loss_and_gradient(V, VP):
  shape = (2, 9, 13)
  l = gc._logits(V, VP, shape, seed=2 * V)
  y = torch.full(shape, 7, dtype=torch.int32, device="cuda")
  norm = _norm(y, V, 7, None)
  coef, scratch = _dice_buffers(VP)
  for with_ce in (False, True):
    d = torch.full_like(l, float("nan"))
    loss, hits = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    _C().seg_dice_stats(l, y, coef, loss, scratch, V, 1e-5, 7, None)
    _C().seg_loss_grad(l, y, d, loss, hits, V, 1.0, 7, None, norm, cross_entropy=with_ce,
                       dice_coef=coef)
    torch.cuda.synchronize()
    assert float(loss) == 0.0 and float(hits) == 0.0
    assert not d.any() and not d.isnan().any()


def test_loss_entry_points_reject_bad_arguments():
  C = _C()
  l = gc._logits(21, 24, (1, 4, 4), seed=1)
  y = torch.zeros(1, 4, 4, dtype=torch.int32, device="cuda")
  d, loss = torch.zeros_like(l), torch.zeros(1, device="cuda")
  coef, scratch = _dice_buffers(24)
  with pytest.raises(RuntimeError):
    C.seg_loss_grad(l, y, d, loss, None, 25, 1.0)                     # VP does not match V
  with pytest.raises(RuntimeError):
    C.seg_loss_grad(l, y, d, loss, None, 21, 1.0, cross_entropy=False)    # no term
  with pytest.raises(RuntimeError):
    C.seg_loss_grad(l, y, d, loss, None, 21, 1.0, focal_gamma=-1.0)
  with pytest.raises(RuntimeError):
    C.seg_loss_grad(l, y, d, loss, None, 21, 1.0, dice_coef=coef[:, :16].contiguous())
  with pytest.raises(RuntimeError):
    C.seg_dice_stats(l, y, coef, loss, scratch[:100], 21, 1e-5)
  with pytest.raises(RuntimeError):
    C.seg_dice_stats(l, y, coef, loss, scratch, 21, 0.0)
  with pytest.raises(RuntimeError):
    C.seg_dice_stats(l, y, coef, loss, scratch, 25, 1e-5)


# ----------------------------------------------------------------------------- the 21-class U-Net
V21 = 21
LOSSES = ["focal", "dice", "dice_ce"]


def _trainer(loss, **kw):
  from tensorflowonspark_b200.models import unet
  kw.setdefault("seed", 3)
  return unet.UNetTrainer(batch=kw.pop("batch", 8), image=128, classes=V21, ignore_index=255,
                          class_weights=lo._class_weights(), loss=loss, **kw)


def _torch_loss(loss, lg, y, cw, gamma=2.0, smooth=1e-5):
  """fp32 PyTorch loss of the trainer's options on logits lg [B, V, H, W]."""
  wt = torch.tensor(cw, dtype=torch.float32, device="cuda")
  keep = y != 255
  yl = y.clamp(0, V21 - 1).long()
  out = 0.0
  if loss in ("focal",):
    logp = torch.log_softmax(lg, 1).gather(1, yl[:, None])[:, 0]
    fl = -(1 - logp.exp()) ** gamma * logp
    wy = wt[yl] * keep
    out = out + (wy * fl).sum() / wy.sum()
  if loss == "dice_ce":
    out = out + F.cross_entropy(lg, y.long(), weight=wt, ignore_index=255)
  if loss in ("dice", "dice_ce"):
    p = torch.softmax(lg, 1).permute(0, 2, 3, 1)[keep]
    oh = F.one_hot(yl[keep], V21).float()
    I, P, Y = (p * oh).sum(0), p.sum(0), oh.sum(0)
    out = out + (wt / wt.sum() * (1 - (2 * I + smooth) / (P + Y + smooth))).sum()
  return out


@pytest.mark.parametrize("loss", LOSSES)
def test_21_class_void_last_layer_gradients_match_autograd(loss):
  net = _trainer(loss)
  x, _ = net.synthetic_batch(seed=1)
  y = lo._void_labels(x, (50, 70))
  net.train_step(x, y)
  net.set_input(x, y)
  net._forward(True)
  st = net.store
  net.loss_sum.zero_()
  net.correct.zero_()
  net._loss()
  net.optim.zero_grads()
  net.p_last_wgrad.run()
  from tensorflowonspark_b200 import ops
  ops.K.colsum(net.dlogits, st.g(net.s_last_b))
  torch.cuda.synchronize()
  lg = net.logits[..., :V21].float().permute(0, 3, 1, 2).clone().requires_grad_(True)
  ref = _torch_loss(loss, lg, y, lo._class_weights())
  ref.backward()
  assert float(net.loss_sum) == pytest.approx(ref.item(), rel=1e-4)
  keep = y != 255
  d = net.dlogits.float()
  assert not d[~keep].any() and not d[..., V21:].any()
  se = gc._load("seg_eval_ref_loss_opts", os.path.join("tests", "test_gpu_seg_eval.py"))
  g_ref = lg.grad.permute(0, 2, 3, 1)
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


@pytest.mark.parametrize("loss", LOSSES)
def test_21_class_captured_step_equals_eager(loss):
  net = _trainer(loss, seed=4)
  x, _ = net.synthetic_batch(seed=2)
  net.set_input(x, lo._void_labels(x, (60, 64)))
  net.train_step()
  net.capture()
  for rows in ((60, 64), (10, 100)):
    net.set_input(x, lo._void_labels(x, rows))
    net.train_step()
    torch.cuda.synchronize()
    d_graph, loss_graph = net.dlogits.clone(), float(net.loss_sum)
    coef_graph = net.dice_coef.clone() if net.dice_coef is not None else None
    hits_graph = float(net.correct)
    net.dlogits.fill_(float("nan"))
    net.loss_sum.zero_()
    net.correct.zero_()
    net._loss()   # eager, on the logits the graph's forward left
    torch.cuda.synchronize()
    assert torch.equal(net.dlogits, d_graph), rows
    if coef_graph is not None:
      assert torch.equal(net.dice_coef, coef_graph)
    assert float(net.correct) == hits_graph
    # (the gradient kernel's warps add their loss partials with float atomics in any order)
    assert float(net.loss_sum) == pytest.approx(loss_graph, rel=1e-5)


class _Recorder(object):
  """ops.K stand-in recording the name of every launch."""

  def __init__(self, k):
    self.k, self.names = k, []

  def __getattr__(self, name):
    fn = getattr(self.k, name)

    def call(*a, **kw):
      self.names.append(name)
      return fn(*a, **kw)
    return call


def _step_names(net, monkeypatch):
  from tensorflowonspark_b200 import ops
  rec = _Recorder(ops.K)
  monkeypatch.setattr(ops, "K", rec)
  before = ops.launch_count()
  net.step_kernels()
  torch.cuda.synchronize()
  n = ops.launch_count() - before
  monkeypatch.undo()
  return rec.names, n


@pytest.mark.parametrize("options", [{}, {"ignore_index": 255, "class_weights": [1.0] * V21}],
                         ids=["plain", "options"])
def test_launch_sequences(options, monkeypatch):
  from tensorflowonspark_b200.models import unet
  seqs = {}
  for loss in ["cross_entropy"] + LOSSES:
    net = unet.UNetTrainer(batch=2, image=128, classes=V21, seed=3, loss=loss, **options)
    x, y = net.synthetic_batch(seed=1)
    net.set_input(x, y)
    seqs[loss] = _step_names(net, monkeypatch)
    del net
  default = unet.UNetTrainer(batch=2, image=128, classes=V21, seed=3, **options)
  x, y = default.synthetic_batch(seed=1)
  default.set_input(x, y)
  names, n = _step_names(default, monkeypatch)
  ce, n_ce = seqs["cross_entropy"]
  assert (names, n) == (ce, n_ce), "a default trainer launches the cross-entropy step"
  assert ce.count("pixel_xent") == 1 and "seg_loss_grad" not in ce and "seg_dice_stats" not in ce
  i = ce.index("pixel_xent")
  focal, n_focal = seqs["focal"]
  assert n_focal == n_ce and focal == ce[:i] + ["seg_loss_grad"] + ce[i + 1:]
  for loss in ("dice", "dice_ce"):
    names, n = seqs[loss]
    assert n == n_ce + 1 and names == ce[:i] + ["seg_dice_stats", "seg_loss_grad"] + ce[i + 1:]


def test_dice_ce_accumulation_of_one_batch_is_one_step():
  import test_gpu_grad_accum as ga
  from tensorflowonspark_b200.models import unet

  def make(k):
    return unet.UNetTrainer(batch=4, image=128, classes=V21, seed=9, lr=2e-3, ignore_index=255,
                            class_weights=lo._class_weights(), loss="dice_ce",
                            gradient_accumulation_steps=k)
  net = make(1)
  x, _ = net.synthetic_batch(seed=1)
  batch = (x, lo._void_labels(x, (40, 56)))
  del net
  ga._same_batch_k_times(make, batch, k=2, frac=ga.FRAC["adam"])


@pytest.mark.parametrize("loss", LOSSES)
def test_21_class_void_trainer_learns_checkpoints_and_serves(loss):
  from tensorflowonspark_b200.models import unet
  B = 16
  net = _trainer(loss, batch=B, seed=5, lr=2e-3)
  held = []
  for i in range(2):
    hx, _ = net.synthetic_batch(seed=500 + i)
    held.append((hx, lo._void_labels(hx, (0, 16))))
  before = net.evaluate(held)
  assert set(before) == {"count", "images", "loss", "accuracy", "mean_iou", "iou", "ignored"}
  xs = [net.synthetic_batch(seed=i)[0] for i in range(4)]
  net.set_input(xs[0], lo._void_labels(xs[0], (40, 56)))
  net.train_step()
  net.capture()
  first = float(net.loss_sum)
  for i in range(600):
    x = xs[i % 4]
    net.set_input(x, lo._void_labels(x, (40 + i % 7, 56 + i % 5)))
    last = net.train_step()
  last = float(last)
  after = net.evaluate(held)
  print("{}: loss {:.3f} -> {:.3f}, mean IoU {:.3f} -> {:.3f}".format(
      loss, first, last, before["mean_iou"], after["mean_iou"]))
  assert np.isfinite(last) and last < first
  if loss == "dice":
    assert last < 0.85 * first
  else:
    # soft Dice alone lowers its loss here but leaves the held-out mean IoU near chance within
    # 600 steps (a softmax spread over neighbouring bands already has D_c ~ 1/3 with an arg-max
    # close to chance); with the cross-entropy term or the focal loss the arg-max is learnt
    assert after["mean_iou"] > 1.3 * before["mean_iou"]
  # checkpoint round trip into a trainer with the same loss, and an inference-only replica
  x, y = held[0]
  ref = net.predict(x).clone()
  net2 = _trainer(loss, batch=B, seed=6)
  net2.load_state_dict(net.state_dict())
  assert torch.equal(net2.predict(x), ref)
  served = unet.UNetTrainer(batch=B, image=128, classes=V21, seed=7, training=False,
                            ignore_index=255)
  served.load_state_dict(net.state_dict())
  assert torch.equal(served.predict(x), ref)
  assert served.evaluate(held)["mean_iou"] == after["mean_iou"]
  replica = unet.build_served(net.state_dict(), image=128, classes=V21, batch=B)
  replica.select_outputs(["mask"])
  for _ in range(2):   # eager, then captured
    out = replica(image=x.cpu().numpy())
  assert torch.equal(torch.from_numpy(out["mask"]).cuda().long(), gc._ref_argmax(
      ref.double().cpu().reshape(-1, V21), V21).view(B, 128, 128).cuda())

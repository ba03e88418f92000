"""CPU tier of the step conformance suite (tools/step_conformance.py): the float64 layer
references against torch autograd, the checkers against planted faults in stored values, and the
launch claiming and snapshot logic on synthetic launches."""
import importlib.util
import os

import pytest
import torch
import torch.nn.functional as F

_spec = importlib.util.spec_from_file_location(
    "step_conformance", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                     "tools", "step_conformance.py"))
sc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(sc)
pc = sc.pc

D = torch.float64


def _g(seed):
  return torch.Generator().manual_seed(seed)


def _rand(shape, g, scale=1.0, shift=0.0):
  return torch.randn(shape, generator=g, dtype=D) * scale + shift


def _bn_train(x, gam, bet, eps=1e-5):
  """Batch norm in training mode over NHWC x, as torch computes it (biased variance)."""
  m = x.mean((0, 1, 2))
  v = x.var((0, 1, 2), unbiased=False)
  return (x - m) / torch.sqrt(v + eps) * gam + bet


def _bn_fwd_ref(x, gam, bet, eps=1e-5):
  """The step suite's forward chain: finalize from the column sums, then the apply."""
  xx = sc.col(x)
  refs = pc.bn_finalize_refs(xx.sum(0), (xx * xx).sum(0), gam, bet, torch.zeros_like(gam),
                             torch.ones_like(gam), float(xx.shape[0]), eps, 0.1)
  return refs["scale"][0], refs["shift"][0], refs["mean"][0], refs["invstd"][0]


def _bn_bwd_ref(dy, x, keep, gam, mean, invstd):
  """dgamma, dbeta, dx of the step suite's backward chain for one batch norm."""
  g = sc.col(dy) * sc.col(keep)
  xm = sc.col(x) - mean
  (dg, _), (db, _) = pc.bn_bwd_reduce_refs(g, xm, invstd, 10)
  dx, _ = pc.bn_bwd_dx_ref(g, sc.col(x), gam, mean, invstd, dg, db)
  return dg, db, dx.reshape(x.shape)


@pytest.mark.parametrize("stride", [1, 2])
def test_bottleneck_block_references_match_autograd(stride):
  """conv1 1x1 -> bn -> relu -> conv2 3x3/s -> bn -> relu -> conv3 1x1 -> bn (+ shortcut) -> relu,
  with a projection shortcut at stride 2, forward and backward through the layer references."""
  g = _g(stride)
  N, H, Cin, w = 2, 6, 16, 4
  x = _rand((N, H, H, Cin), g)
  ws = [_rand((w, 1, 1, Cin), g, 0.3), _rand((w, 3, 3, w), g, 0.3), _rand((4 * w, 1, 1, w), g, 0.3)]
  wd = _rand((4 * w, 1, 1, Cin), g, 0.3)
  gams = [_rand((c,), g, 0.2, 1.0) for c in (w, w, 4 * w, 4 * w)]
  bets = [_rand((c,), g, 0.2) for c in (w, w, 4 * w, 4 * w)]
  G = _rand((N, (H - 1) // stride + 1, (H - 1) // stride + 1, 4 * w), g)
  # autograd
  leaves = [t.clone().requires_grad_() for t in [x] + ws + [wd] + gams + bets]
  tx, t1, t2, t3, td = leaves[:5]
  tg, tb = leaves[5:9], leaves[9:]
  conv = lambda a, k, s, p: F.conv2d(a.permute(0, 3, 1, 2), k.permute(0, 3, 1, 2), stride=s,  # noqa
                                     padding=p).permute(0, 2, 3, 1)
  a1 = torch.relu(_bn_train(conv(tx, t1, 1, 0), tg[0], tb[0]))
  a2 = torch.relu(_bn_train(conv(a1, t2, stride, 1), tg[1], tb[1]))
  sh = _bn_train(conv(tx, td, stride, 0), tg[3], tb[3]) if stride == 2 else tx
  out = torch.relu(_bn_train(conv(a2, t3, 1, 0), tg[2], tb[2]) + sh)
  (out * G).sum().backward()
  # the layer references
  r1, _ = sc.conv_ref(x, ws[0], 1, 0)
  s1, h1, m1, i1 = _bn_fwd_ref(r1, gams[0], bets[0])
  ra1, _, pre1, _ = pc.bn_apply_ref(sc.col(r1), s1, h1)
  ra1 = ra1.reshape(r1.shape)
  r2, _ = sc.conv_ref(ra1, ws[1], stride, 1)
  s2, h2, m2, i2 = _bn_fwd_ref(r2, gams[1], bets[1])
  ra2, _, pre2, _ = pc.bn_apply_ref(sc.col(r2), s2, h2)
  ra2 = ra2.reshape(r2.shape)
  r3, _ = sc.conv_ref(ra2, ws[2], 1, 0)
  s3, h3, m3, i3 = _bn_fwd_ref(r3, gams[2], bets[2])
  if stride == 2:
    rd, _ = sc.conv_ref(x, wd, stride, 0)
    sd, hd, md, idd = _bn_fwd_ref(rd, gams[3], bets[3])
    idn = pc.bn_apply_ref(sc.col(rd), sd, hd, act=0)[0].reshape(rd.shape)
  else:
    idn = x
  y, _, pre3, _ = pc.bn_apply_ref(sc.col(r3), s3, h3, sc.col(idn))
  assert torch.allclose(y.reshape(out.shape), out.detach(), rtol=1e-12, atol=1e-12)
  keep3 = (pre3 > 0).reshape(out.shape)
  dg3, db3, g_r3 = _bn_bwd_ref(G, r3, keep3, gams[2], m3, i3)
  dw3, _ = sc.wgrad_ref(g_r3, ra2, ws[2].shape, 1, 0)
  g_a2, _ = sc.dgrad_ref(g_r3, ws[2], ra2.shape, 1, 0)
  dg2, db2, g_r2 = _bn_bwd_ref(g_a2, r2, (pre2 > 0).reshape(r2.shape), gams[1], m2, i2)
  dw2, _ = sc.wgrad_ref(g_r2, ra1, ws[1].shape, stride, 1)
  g_a1, _ = sc.dgrad_ref(g_r2, ws[1], ra1.shape, stride, 1)
  dg1, db1, g_r1 = _bn_bwd_ref(g_a1, r1, (pre1 > 0).reshape(r1.shape), gams[0], m1, i1)
  dw1, _ = sc.wgrad_ref(g_r1, x, ws[0].shape, 1, 0)
  g_x, _ = sc.dgrad_ref(g_r1, ws[0], x.shape, 1, 0)
  if stride == 2:
    dgd, dbd, g_rd = _bn_bwd_ref(G, rd, keep3, gams[3], md, idd)
    dwd, _ = sc.wgrad_ref(g_rd, x, wd.shape, stride, 0)
    g_x = g_x + sc.dgrad_ref(g_rd, wd, x.shape, stride, 0)[0]
    assert torch.allclose(dwd, td.grad, rtol=1e-9, atol=1e-11)
    assert torch.allclose(dgd, tg[3].grad, rtol=1e-9, atol=1e-11)
    assert torch.allclose(dbd, tb[3].grad, rtol=1e-9, atol=1e-11)
  else:
    g_x = g_x + G * keep3   # the identity shortcut: mask * g_out accumulated into conv1's dgrad
  for got, want in ((g_x, tx.grad), (dw1, t1.grad), (dw2, t2.grad), (dw3, t3.grad),
                    (dg1, tg[0].grad), (dg2, tg[1].grad), (dg3, tg[2].grad), (db1, tb[0].grad),
                    (db2, tb[1].grad), (db3, tb[2].grad)):
    assert torch.allclose(got, want, rtol=1e-9, atol=1e-11), float((got - want).abs().max())


def test_fused_dgamma_reference_matches_the_direct_sum():
  g = _g(3)
  x, dy = _rand((50, 8), g, 1.0, 2.0), _rand((50, 8), g)
  mean, invstd = x.mean(0), 1.0 / x.std(0)
  ref, bnd = pc.bn_bwd_fused_dgamma_ref(dy.sum(0), (dy * x).sum(0), mean, invstd)
  (direct, _), _ = pc.bn_bwd_reduce_refs(dy, x - mean, invstd, 10)
  assert bool(((ref - direct).abs() <= bnd).all())


def test_stem_references_match_the_unpacked_convolution():
  from tensorflowonspark_b200.ops import igemm
  g = _g(4)
  N, H, Co = 2, 17, 8
  OH, OW, Wp = igemm.stem_geometry(H, H)
  img = _rand((N, H, H, 3), g)
  xp = torch.zeros(N, H, Wp, 8, dtype=D)
  xp[:, :, igemm.STEM_PAD:igemm.STEM_PAD + H, :3] = img
  w7 = _rand((Co, 7, 7, 3), g, 0.2)
  wp = igemm.pack_stem_weight(w7)
  y, _ = sc.stem_ref(xp, wp, OW)
  want = F.conv2d(img.permute(0, 3, 1, 2), w7.permute(0, 3, 1, 2), stride=2, padding=3)
  assert torch.allclose(y, want.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
  dy = _rand((N, OH, OW, Co), g)
  dw, _ = sc.stem_wgrad_ref(dy, xp)
  tw = w7.clone().requires_grad_()
  (F.conv2d(img.permute(0, 3, 1, 2), tw.permute(0, 3, 1, 2), stride=2, padding=3) *
   dy.permute(0, 3, 1, 2)).sum().backward()
  assert torch.allclose(igemm.unpack_stem_weight(dw), tw.grad, rtol=1e-10, atol=1e-12)


def test_momentum_reference_matches_torch_sgd():
  g = _g(5)
  w, gr = _rand((64,), g), _rand((64,), g)
  decay = torch.arange(64) < 40
  s0 = _rand((64,), g)
  s, w1, _, _ = sc.momentum_ref(w, s0, gr, decay, 0.1, 0.9, 1e-4)
  for sel, wd in ((decay, 1e-4), (~decay, 0.0)):
    p = torch.nn.Parameter(w[sel].clone())
    opt = torch.optim.SGD([p], lr=0.1, momentum=0.9, weight_decay=wd)
    opt.state[p]["momentum_buffer"] = s0[sel].clone()
    p.grad = gr[sel].clone()
    opt.step()
    assert torch.allclose(p.detach(), w1[sel], rtol=1e-12, atol=1e-14)
    assert torch.allclose(opt.state[p]["momentum_buffer"], s[sel], rtol=1e-12, atol=1e-14)


# ----------------------------------------------------------------------------- planted faults
def _bn_apply_case(seed):
  g = _g(seed)
  x, res = _rand((400, 16), g, 1.5, 0.2), _rand((400, 16), g)
  scale, shift = _rand((16,), g, 0.3, 1.0), _rand((16,), g, 0.3)
  return x, res, scale, shift


def test_dropped_residual_term_is_caught():
  x, res, scale, shift = _bn_apply_case(6)
  ref, bound, _, _ = pc.bn_apply_ref(x, scale, shift, res)
  good = pc.bf16_rne(ref)
  rep = sc.Report()
  assert rep.close("blk.u3.bn", "bn fwd y", 7, good, ref, bound) <= 1.0
  stored = pc.bf16_rne(pc.bn_apply_ref(x, scale, shift, None)[0])
  assert rep.close("blk.u3.bn", "bn fwd y", 7, stored, ref, bound) > 10.0
  assert rep.failing_layers() == ["blk.u3.bn"]
  assert "launch #7" in rep.failures[0][2]


def test_wrong_mask_is_caught():
  g = _g(7)
  x, dy = _rand((512, 16), g, 1.0, 0.3), _rand((512, 16), g)
  gam, mean = _rand((16,), g, 0.2, 1.0), x.mean(0)
  invstd = 1.0 / x.std(0)
  keep = torch.rand((512, 16), generator=g) < 0.5
  other = torch.rand((512, 16), generator=g) < 0.5
  dg, db, dx = _bn_bwd_ref(dy, x, keep, gam, mean, invstd)
  ref, bound = pc.bn_bwd_dx_ref(dy * keep, x, gam, mean, invstd, dg, db)
  rep = sc.Report()
  assert rep.close("b.u2.bn", "bn bwd dx", 3, pc.bf16_rne(dx), ref, bound) <= 1.0
  _, _, wrong = _bn_bwd_ref(dy, x, other, gam, mean, invstd)
  rep.close("b.u2.bn", "bn bwd dx", 3, pc.bf16_rne(wrong), ref, bound)
  assert rep.failing_layers() == ["b.u2.bn"]


def test_stale_accumulator_is_caught():
  """An accumulating data gradient whose stored result was built on another value of the buffer
  than the one the layer feeding it left (e.g. the previous step's)."""
  g = _g(8)
  dy, w = _rand((2, 5, 5, 8), g), _rand((8, 3, 3, 4), g, 0.2)
  prev, stale = _rand((2, 5, 5, 4), g), _rand((2, 5, 5, 4), g)
  part, M = sc.dgrad_ref(dy, w, (2, 5, 5, 4), 1, 1)
  ref = part + prev
  bound = pc.elem_bound(ref, M, 9 * 8 + 1, partial=part, prev=prev)
  rep = sc.Report()
  assert rep.close("b.u1.conv", "conv dgrad", 11, pc.bf16_rne(ref), ref, bound) <= 1.0
  rep.close("b.u1.conv", "conv dgrad", 11, pc.bf16_rne(part + stale), ref, bound)
  assert rep.failing_layers() == ["b.u1.conv"]


def test_one_channel_offset_in_a_fused_sum_is_caught():
  g = _g(9)
  y = pc.bf16_rne(_rand((300, 24), g, 1.0, 0.5))
  gp = pc.gamma_prob(64)
  rep = sc.Report()
  s = y.sum(0)
  assert rep.close("c", "conv fwd stats", 0, s, s, gp * y.abs().sum(0)) <= 1.0
  rep.close("c", "conv fwd stats", 0, torch.roll(s, 1), s, gp * y.abs().sum(0))
  assert rep.failing_layers() == ["c"]


def test_nan_fails_and_zero_bound_needs_exact():
  rep = sc.Report()
  ref = torch.zeros(4, dtype=D)
  assert rep.close("a", "k", 0, torch.zeros(4), ref, torch.zeros(4, dtype=D)) == 0.0
  rep.close("b", "k", 1, torch.tensor([0.0, float("nan"), 0.0, 0.0]), ref, torch.ones(4, dtype=D))
  rep.close("c", "k", 2, torch.tensor([0.0, 1e-30, 0.0, 0.0]), ref, torch.zeros(4, dtype=D))
  assert rep.failing_layers() == ["b", "c"]


# ----------------------------------------------------------------------------- claims, snapshots
def _launches(spec):
  return [sc.Launch(i, k, n, p) for i, (k, n, p) in enumerate(spec)]


def test_every_launch_is_claimed_exactly_once():
  p1, p2 = object(), object()
  ls = _launches([("host", "StatsArena.zero", None), ("plan", "igemm_run", p1),
                  ("k", "bn_apply_finalize", None), ("plan", "igemm_run", p2)])
  cl = sc.Claims(ls)
  assert cl.take("arena", "host", "StatsArena.zero") == 0
  assert cl.take("c1", "plan", plan=p1) == 1
  assert cl.take("bn1", "k", "bn_apply_finalize") == 2
  with pytest.raises(AssertionError, match="claimed by no layer check"):
    cl.finish()
  assert cl.take("c2", "plan", plan=p2) == 3
  assert cl.finish() == 4
  assert cl.owner == {0: "arena", 1: "c1", 2: "bn1", 3: "c2"}


def test_a_launch_of_another_kind_fails_naming_the_layer():
  p1, p2 = object(), object()
  cl = sc.Claims(_launches([("plan", "igemm_run", p1), ("k", "bn_bwd_apply", None)]))
  with pytest.raises(AssertionError, match="layer3.0.u1.conv"):
    cl.take("layer3.0.u1.conv", "plan", plan=p2)     # another plan than the layer's
  cl.take("layer3.0.u1.conv", "plan", plan=p1)
  with pytest.raises(AssertionError, match="layer3.0.u1.bn: expected a k launch"):
    cl.take("layer3.0.u1.bn", "k", "bn_bwd_reduce")  # an unfused reduction that never ran
  cl.take("layer3.0.u1.bn", "k", "bn_bwd_apply")
  with pytest.raises(AssertionError, match="the step ended"):
    cl.take("fc", "k", "colsum")


def test_snapshots_keep_values_overwritten_in_place():
  flat = torch.zeros(32)
  stage = torch.zeros(2, 4, dtype=torch.bfloat16)
  s = sc.Snapshots([("master", flat), ("p.w", flat[8:16]), ("blk1.g_out", stage),
                    ("blk1.g_x", stage), ("blk0.g_out", stage)])
  assert s.update(0) == []
  stage.fill_(1.0)                 # launch 1 writes g_out
  assert s.update(1) == [1]
  stage.add_(2.0)                  # launch 2 accumulates g_x in place
  flat[8:16] = 5.0                 # ... and launch 2 also writes a parameter
  assert s.update(2) == [0, 1]
  assert float(s.before("blk1.g_x", 2)[0, 0]) == 1.0
  assert float(s.after("blk1.g_x", 2)[0, 0]) == 3.0
  assert float(s.before("blk0.g_out", 1)[1, 3]) == 0.0
  assert float(s.before("p.w", 2)[0]) == 0.0 and float(s.after("p.w", 2)[0]) == 5.0
  assert s.writers("blk1.g_out") == [1, 2]
  # NaN payloads compare by their bits: rewriting the same NaN is no write, another one is
  stage.view(torch.int16).fill_(0x7FC1)
  assert s.update(3) == [1]
  assert s.update(4) == []
  stage.view(torch.int16).fill_(0x7FA5)
  assert s.update(5) == [1]


def test_mask_bits_follow_the_kernels_layout():
  m = torch.tensor([0b00000101, 0b10000000], dtype=torch.uint8)
  bits = sc.mask_bits(m, (2, 8))
  assert bits[0].tolist() == [True, False, True] + [False] * 5
  assert bits[1].tolist() == [False] * 7 + [True]


# ----------------------------------------------------------------------------- real layer checks
class _Obj(object):
  def __init__(self, **kw):
    self.__dict__.update(kw)


def _run_launches(buffers, writes):
  """Snapshots over ``buffers`` and one launch per entry of ``writes`` ((kind, name, plan,
  fn): fn changes the buffers in place as the launch would)."""
  snaps = sc.Snapshots(list(buffers.items()))
  launches = []
  for i, (kind, name, plan, fn) in enumerate(writes):
    fn()
    la = sc.Launch(i, kind, name, plan)
    la.wrote = snaps.update(i)
    launches.append(la)
  return sc._Ctx(None, launches, snaps), launches


def _dgrad_case(fault):
  """An identity block's conv1 data gradient, g_x = mask * g_out + dgrad(g_r1), in place over the
  stage buffer, checked by the suite's own ``_dgrad``; ``fault`` plants a wiring error."""
  g = _g(10)
  N, H, Ci, Co = 2, 4, 16, 8
  dy = pc.bf16_rne(_rand((N, H, H, Co), g)).float()
  w = pc.bf16_rne(_rand((Co, 1, 1, Ci), g, 0.3)).float()
  g_out = pc.bf16_rne(_rand((N, H, H, Ci), g)).float()
  stale = pc.bf16_rne(_rand((N, H, H, Ci), g)).float()
  mask = torch.randint(0, 256, (N * H * H * Ci // 8,), generator=g, dtype=torch.uint8)
  x = _rand((N, H, H, Ci), g).float()
  buf = {"weights:c.w": w, "g_r1": dy, "g_x": g_out.clone(), "mask": mask, "x": x,
         "stats_arena": torch.zeros(8)}
  part = sc.dgrad_ref(dy.double(), w.double(), (N, H, H, Ci), 1, 0)[0]
  keep = sc.mask_bits(mask, (N, H, H, Ci))
  prev = {"stale": stale.double(), "unmasked": g_out.double()}.get(fault, g_out.double() * keep)
  if fault == "writes":
    prev = torch.zeros_like(prev)
  plan = object()

  def launch():
    buf["g_x"].copy_(pc.bf16_rne(part + prev))
    if fault == "clobbers_x":
      buf["x"].zero_()
  c, _ = _run_launches(buf, [("plan", "igemm_run", plan, launch)])
  conv = _Obj(dgrad=plan, sw={"name": "c.w", "shape": (Co, 1, 1, Ci)}, stride=1, pad=0, k=1,
              cin=Ci, cout=Co)
  sc._dgrad(c, "layer1.1.u1.conv", conv, "g_r1", "g_x", (N, H, H, Ci), accumulate=True,
            maskname="mask")
  assert c.claims.finish() == 1
  return c.rep


def test_dgrad_checker_passes_the_right_wiring():
  rep = _dgrad_case(None)
  assert not rep.failures, rep.failures


@pytest.mark.parametrize("fault", ["stale", "unmasked", "writes", "clobbers_x"])
def test_dgrad_checker_catches_planted_wiring_faults(fault):
  """A stale accumulator (the launch added another value than the buffer held), the mask not
  applied, a write instead of an accumulate, and a launch that also clobbers another buffer."""
  rep = _dgrad_case(fault)
  assert rep.failing_layers() == ["layer1.1.u1.conv"]
  if fault == "clobbers_x":
    assert "wrote x it does not own" in rep.failures[0][2]


def _bn_bwd_case(fault):
  """An unfused batch-norm backward (reduce, then apply) checked by the suite's own ``_bn_bwd``."""
  g = _g(11)
  P, C = 256, 16
  shape = (2, 8, 16, C)
  x = pc.bf16_rne(_rand(shape, g, 1.0, 0.5)).float()
  dy = pc.bf16_rne(_rand(shape, g)).float()
  mask = torch.randint(0, 256, (P * C // 8,), generator=g, dtype=torch.uint8)
  other = torch.randint(0, 256, (P * C // 8,), generator=g, dtype=torch.uint8)
  mean = sc.col(x.double()).mean(0).float()
  invstd = (1.0 / sc.col(x.double()).std(0)).float()
  gam = _rand((C,), g, 0.2, 1.0).float()
  grads, dx = torch.zeros(2 * C), torch.zeros(shape, dtype=torch.bfloat16)
  buf = {"grads": grads, "grads:gamma": grads[:C], "grads:beta": grads[C:], "master:gamma": gam,
         "g_a2": dy, "r2": x, "b.u2.bn.mask": mask, "b.u2.bn.mean": mean,
         "b.u2.bn.invstd": invstd, "g_r2": dx}
  used = other if fault == "wrong_mask" else mask
  keep = sc.col(sc.mask_bits(used, shape))
  gg = sc.col(dy.double()) * keep
  xm = sc.col(x.double()) - mean.double()
  (dg, _), (db, _) = pc.bn_bwd_reduce_refs(gg, xm, invstd.double(), 10)

  def reduce():
    grads[:C], grads[C:] = dg.float(), db.float()

  def apply():
    r, _ = pc.bn_bwd_dx_ref(gg, sc.col(x.double()), gam.double(), mean.double(), invstd.double(),
                            grads[:C].double(), grads[C:].double())
    dx.copy_(r.reshape(shape).to(torch.bfloat16))
  c, _ = _run_launches(buf, [("k", "bn_bwd_reduce", None, reduce),
                             ("k", "bn_bwd_apply", None, apply)])
  bn = _Obj(acc=None, fused_reduce=False, mask=mask, sg={"name": "gamma"}, sb={"name": "beta"})
  sc._bn_bwd(c, "b.u2.bn", bn, "b.u2.bn", "g_a2", "r2", "b.u2.bn.mask", "g_r2", None)
  assert c.claims.finish() == 2
  return c.rep


def test_bn_backward_checker_passes_the_right_wiring():
  rep = _bn_bwd_case(None)
  assert not rep.failures, rep.failures


def test_bn_backward_checker_catches_another_mask():
  assert _bn_bwd_case("wrong_mask").failing_layers()[0] == "b.u2.bn"

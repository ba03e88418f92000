"""Gradient accumulation (``gradient_accumulation_steps``) on the GPU: the accumulating batch-norm,
fused-stem and depthwise backward kernels against their writing variants, and the three trainers
against k = 1 training.

The module's name sorts it after tests/test_gpu_cluster.py: the cluster tests need a GPU that no
process holds, and a CUDA context created earlier in the same pytest process would occupy it.
"""
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BN_WIDTHS = (16, 32, 64, 128, 256, 512, 1024, 2048)   # every batch-norm width the models launch


@pytest.fixture(scope="module", autouse=True)
def _ext():
  from tensorflowonspark_b200 import _build
  _build.load(required=True)
  torch.cuda.set_device(0)


def _C():
  from tensorflowonspark_b200 import ops
  return ops.C()


def _gen(seed):
  g = torch.Generator(device="cpu")
  g.manual_seed(seed)
  return g


def _rand(shape, g, dtype=torch.float32, scale=1.0):
  return (torch.randn(shape, generator=g) * scale).to("cuda", dtype)


def _bits(t):
  return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _same_bits(a, b, what):
  diff = _bits(a) != _bits(b)
  assert not diff.any(), "{}: {} of {} elements differ, max |a - b| {}".format(
      what, int(diff.sum()), diff.numel(), float((a.float() - b.float()).abs().max()))


# ------------------------------------------------------------------ batch-norm backward
def _one_rounding_apart(a, b, dy, x, gamma, mean, invstd, dg, db):
  """dx of the accumulating unfused apply against the writing one.  Both compute
  dx = A g + B x + K (A = gamma invstd, B = -A invstd dgamma / M, K = -A dbeta / M - B mean) from the
  same source and the same dgamma / dbeta, but the coefficients' multiplies and adds are
  contractible, and ptxas fuses the product with 1 / M into an FFMA once in the writing kernel's
  SASS and twice in the accumulating one's (sm_90a, the project's flags).  K, and so dx before
  rounding, can then differ by a few fp32 ulps of the terms; where the terms cancel that is more
  than one bf16 step of dx.  So: each element within one bf16 step (2^-7 relative) plus 2^-20 of
  |A dy| + |B x| + |K|, and at most 1 in 10^4 elements different at all."""
  M = x.shape[0]
  f = lambda t: t.double()  # noqa: E731
  A = f(gamma) * f(invstd)
  B = -A * f(invstd) * f(dg) / M
  K = -A * f(db) / M - B * f(mean)
  scale = (A * f(dy)).abs() + (B * f(x)).abs() + K.abs()
  da, dw = f(a), f(b)
  bound = 2.0 ** -7 * torch.maximum(da.abs(), dw.abs()) + 2.0 ** -20 * scale
  assert bool(((da - dw).abs() <= bound).all()), float(((da - dw).abs() - bound).max())
  differ = int((_bits(a) != _bits(b)).sum())
  assert differ <= max(1, a.numel() // 10000), differ


def _bn_case(C, P, relu, seed):
  g = _gen(seed)
  dy, x = _rand((P, C), g, torch.bfloat16), _rand((P, C), g, torch.bfloat16)
  y = torch.relu(_rand((P, C), g)).to(torch.bfloat16)
  mask = torch.randint(0, 256, (P * C // 8,), generator=g, dtype=torch.uint8).cuda()
  ysrc = {0: None, 1: y, 2: None, 3: mask}[relu]
  mean, invstd = _rand((C,), g, scale=0.1), (torch.rand(C, generator=g) + 0.5).cuda()
  gamma, sc, sh = _rand((C,), g), _rand((C,), g), _rand((C,), g)
  return dy, x, ysrc, mean, invstd, gamma, sc, sh


@pytest.mark.parametrize("rev", [False, True], ids=["forward_rows", "reversed_rows"])
@pytest.mark.parametrize("relu", [0, 1, 2, 3])
@pytest.mark.parametrize("C", BN_WIDTHS)
def test_bn_backward_accumulate_variant(C, relu, rev):
  """The same reduction result through the writing and the accumulating apply: dx equal up to one
  bf16 step on a few elements (_one_rounding_apart), and the parameter gradient prefilled with A
  ends as fl(A + v) (exactly one add per channel)."""
  C_ = _C()
  P = 1237 + C // 8   # ragged: not a multiple of any block's row count
  dy, x, ysrc, mean, invstd, gamma, sc, sh = _bn_case(C, P, relu, seed=C + relu)
  dg, db = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
  C_.bn_set_row_reverse(rev)
  try:
    C_.bn_bwd_reduce(dy, x, ysrc, mean, invstd, dg, db, relu, sc, sh)
    dx_w = torch.empty_like(x)
    C_.bn_bwd_apply(dy, x, ysrc, gamma, mean, invstd, dg, db, dx_w, None, relu, sc, sh)
    g = _gen(99)
    A_g, A_b = _rand((C,), g), _rand((C,), g)
    acc_g, acc_b = A_g.clone(), A_b.clone()
    dx_a = torch.empty_like(x)
    C_.bn_bwd_apply(dy, x, ysrc, gamma, mean, invstd, dg, db, dx_a, None, relu, sc, sh,
                    acc_dgamma=acc_g, acc_dbeta=acc_b)
  finally:
    C_.bn_set_row_reverse(False)
  torch.cuda.synchronize()
  _one_rounding_apart(dx_a, dx_w, dy, x, gamma, mean, invstd, dg, db)
  _same_bits(acc_g, A_g + dg, "dgamma")
  _same_bits(acc_b, A_b + db, "dbeta")


@pytest.mark.parametrize("rev", [False, True], ids=["forward_rows", "reversed_rows"])
@pytest.mark.parametrize("C", BN_WIDTHS)
def test_bn_fused_reduce_apply_accumulate_variant(C, rev):
  """Fused-reduce apply (sum(g), sum(g x) from a dgrad epilogue): the writing variant publishes
  v = (dgamma, dbeta); the accumulating one adds v to A bit for bit and forms the same dx."""
  C_ = _C()
  P = 999 + C // 8
  dy, x, ysrc, mean, invstd, gamma, sc, sh = _bn_case(C, P, 3, seed=7 * C)
  g = _gen(C)
  sum_g, sum_gx = _rand((C,), g, scale=30.0), _rand((C,), g, scale=30.0)
  v_g, v_b = torch.full((C,), float("nan"), device="cuda"), torch.full((C,), float("nan"), device="cuda")
  C_.bn_set_row_reverse(rev)
  try:
    dx_w = torch.empty_like(x)
    C_.bn_bwd_apply(dy, x, ysrc, gamma, mean, invstd, v_g, v_b, dx_w, None, 3, sc, sh, sum_g, sum_gx)
    A_g, A_b = _rand((C,), g), _rand((C,), g)
    acc_g, acc_b = A_g.clone(), A_b.clone()
    dx_a = torch.empty_like(x)
    C_.bn_bwd_apply(dy, x, ysrc, gamma, mean, invstd, acc_g, acc_b, dx_a, None, 3, sc, sh, sum_g,
                    sum_gx, acc_dgamma=acc_g, acc_dbeta=acc_b)
  finally:
    C_.bn_set_row_reverse(False)
  torch.cuda.synchronize()
  _same_bits(dx_a, dx_w, "dx")
  _same_bits(acc_g, A_g + v_g, "dgamma")
  _same_bits(acc_b, A_b + v_b, "dbeta")


def test_bn_apply_rejects_half_an_accumulator():
  C_ = _C()
  dy, x, _, mean, invstd, gamma, sc, sh = _bn_case(64, 64, 2, seed=1)
  z = torch.zeros(64, device="cuda")
  with pytest.raises(RuntimeError, match="go together"):
    C_.bn_bwd_apply(dy, x, None, gamma, mean, invstd, z, z, torch.empty_like(x), None, 2, sc, sh,
                    acc_dgamma=z)


# ------------------------------------------------------------------ fused stem backward
@pytest.mark.parametrize("shape", [(4, 32, 32, 64), (3, 27, 31, 64), (2, 17, 9, 16)])
def test_stem_pool_bn_backward_accumulate_variant(shape):
  """Reduce into scratch, the apply adds it to A: the parameter gradient is fl(A + scratch) bit for
  bit, the scratch matches the writing variant's value (atomic-order rounding apart) and so does
  dx."""
  C_ = _C()
  N, H, W, C = shape
  OH, OW = (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1
  g = _gen(N * H + W)
  x = _rand(shape, g, torch.bfloat16)
  y = torch.empty((N, OH, OW, C), dtype=torch.bfloat16, device="cuda")
  idx = torch.empty((N, OH, OW, C), dtype=torch.uint8, device="cuda")
  # the forward writes idx the backward reads (the argmax tap of each window)
  z = lambda: torch.zeros(C, device="cuda")  # noqa: E731
  s, ss = x.float().sum((0, 1, 2)), (x.float() ** 2).sum((0, 1, 2))
  gamma, beta = _rand((C,), g), _rand((C,), g)
  mean, invstd, sc, sh = z(), z(), z(), z()
  C_.stem_bn_relu_pool_fwd(x, y, idx, s, ss, gamma, beta, z(), z() + 1, mean, invstd, sc, sh,
                           float(N * H * W), 1e-5, 0.1)
  dy = _rand((N, OH, OW, C), g, torch.bfloat16)
  v_g, v_b, dx_w = z(), z(), torch.empty_like(x)
  C_.stem_pool_bn_bwd(dy, idx, x, gamma, mean, invstd, sc, sh, v_g, v_b, dx_w)
  A_g, A_b = _rand((C,), g), _rand((C,), g)
  acc_g, acc_b, s_g, s_b, dx_a = A_g.clone(), A_b.clone(), z(), z(), torch.empty_like(x)
  C_.stem_pool_bn_bwd(dy, idx, x, gamma, mean, invstd, sc, sh, s_g, s_b, dx_a, acc_dgamma=acc_g,
                      acc_dbeta=acc_b)
  torch.cuda.synchronize()
  _same_bits(acc_g, A_g + s_g, "dgamma")
  _same_bits(acc_b, A_b + s_b, "dbeta")
  torch.testing.assert_close(s_g, v_g, rtol=1e-4, atol=1e-3)
  torch.testing.assert_close(s_b, v_b, rtol=1e-4, atol=1e-3)
  torch.testing.assert_close(dx_a.float(), dx_w.float(), rtol=2e-2, atol=2e-2)


# ------------------------------------------------------------------ depthwise backward
@pytest.mark.parametrize("with_add", [False, True], ids=["no_add", "add"])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("shape", [(2, 16, 16, 96), (3, 9, 13, 144), (1, 8, 8, 40)])
def test_depthwise_backward_accumulate_variant(shape, stride, with_add):
  """Deterministic kernel: dx bitwise equal, dw / dbias / dbias_in end as fl(A + v) bit for bit."""
  C_ = _C()
  N, H, W, C = shape
  OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
  g = _gen(H * C + stride)
  relu6 = lambda t: t.clamp(0, 6).to(torch.bfloat16)  # noqa: E731
  x = relu6(_rand(shape, g, scale=3.0))
  w = _rand((9, C), g, torch.bfloat16)
  y = relu6(_rand((N, OH, OW, C), g, scale=3.0))
  dy = _rand((N, OH, OW, C), g, torch.bfloat16)
  add = _rand((N, H, W, C + 16), g, torch.bfloat16) if with_add else None
  off = 8 if with_add else 0
  scratch = torch.zeros(C_.depthwise3x3_bwd_scratch(N, H, C, stride), device="cuda")
  outs = {}
  for acc in (False, True):
    A = [_rand((9, C), _gen(5)), _rand((C,), _gen(6)), _rand((C,), _gen(7))]
    bufs = [a.clone() for a in A] if acc else [torch.full_like(a, float("nan")) for a in A]
    dx = torch.empty_like(x)
    C_.depthwise3x3_bwd(x, w, y, dy, add, off, dx, *bufs, scratch, stride, accumulate=acc)
    outs[acc] = (dx, bufs, A)
  torch.cuda.synchronize()
  _same_bits(outs[True][0], outs[False][0], "dx")
  for name, a, v, got in zip(("dw", "dbias", "dbias_in"), outs[True][2], outs[False][1],
                             outs[True][1]):
    _same_bits(got, a + v, name)


# ------------------------------------------------------------------ trainers
OPTS = {"sgd": dict(lr=0.05, momentum=0.0), "momentum": dict(lr=0.05),
        "adam": dict(lr=1e-3), "adamw": dict(lr=1e-3, weight_decay=0.01),
        "lars": dict(lr=0.1), "lamb": dict(lr=5e-3, weight_decay=0.01)}
# elements of any tensor that may miss a comparison: one run's noise can exceed the noise a single
# repeat shows on a handful of elements, while a producer that overwrites instead of adding, or a
# micro-batch dropped or counted twice, moves most elements of its tensors
FEW = 4
# Adam's first update is sign-like: an element whose gradient is at the rounding level may step
# either way, so a larger share of elements may differ by up to 2 lr
FRAC = {"adam": 0.05, "adamw": 0.05, "lamb": 0.05}


def _masters(net):
  torch.cuda.synchronize()
  return net.store.state_dict()


def _compare(a, b, what, rtol=5e-2, atol_rel=1e-2, frac=0.01):
  """Per parameter name, so that a producer that overwrites instead of adding is named (it is off
  by a factor of k on most elements of its tensor).  The backward is not bitwise reproducible:
  float atomics reorder sums, and a last-bit change can round a bf16 activation gradient the other
  way, which moves the gradients by up to a few 1e-3 relative.  So each element must match to
  ``rtol`` or to ``atol_rel`` of the tensor's largest magnitude, and a share ``frac`` of a tensor's
  elements may miss (Adam's first update is sign-like: an element whose gradient is at the
  rounding level may step either way)."""
  assert a.keys() == b.keys()
  bad = {}
  for n in a:
    atol = atol_rel * float(b[n].abs().max()) + 1e-12
    off = int((~torch.isclose(a[n], b[n], rtol=rtol, atol=atol)).sum())
    if off > max(frac * a[n].numel(), FEW):
      bad[n] = (off, a[n].numel(), float((a[n] - b[n]).abs().max()), float(b[n].abs().max()))
  assert not bad, "{}: {} of {} parameters differ (elements off, of, max diff, max): {}".format(
      what, len(bad), len(a), dict(list(bad.items())[:8]))


def _grads(net, scale=1.0):
  torch.cuda.synchronize()
  st = net.store
  return {s["name"]: st._view(st.grads, s).cpu() * scale for s in st.order}


def _against_noise(ref, ref2, got, what, frac=0.0, margin=4.0, floor=0.02):
  """``got`` against ``ref`` per parameter name, so that a producer that overwrites instead of
  adding is named (it is off by (k - 1) / k of the gradient on most elements of its tensor).  The
  backward is not bitwise reproducible: float atomics reorder sums, and a last-bit change can round
  a bf16 activation gradient the other way.  ``ref2`` repeats ``ref``'s run, so ``|ref2 - ref|``
  measures that noise: each element must be within ``margin`` times the tensor's largest noise or
  ``floor`` of its largest magnitude, and a share ``frac`` of the elements may miss (Adam's first
  update is sign-like: an element whose gradient is at the rounding level may step either way)."""
  bad = {}
  for n in ref:
    noise = float((ref2[n] - ref[n]).abs().max())
    tol = max(margin * noise, floor * float(ref[n].abs().max())) + 1e-12
    err = (got[n] - ref[n]).abs()
    off = int((err > tol).sum())
    if off > max(frac * err.numel(), FEW):
      bad[n] = (off, err.numel(), float(err.max()), tol)
  assert not bad, "{}: {} of {} parameters differ (elements off, of, max error, tolerance): {}".format(
      what, len(bad), len(ref), dict(list(bad.items())[:8]))


def _same_batch_k_times(make, batch, k=3, frac=0.0, floor=0.02):
  """Two k = 1 trainers: one step each; a k trainer: k micro-steps of the same batch.  The
  gradient buffers (the optimizer leaves them as they are) hold g and k g, per parameter, and the
  updates (master - initial master) must match."""
  one, one2, acc = make(1), make(1), make(k)
  w0 = _masters(one)
  for net in (one, one2):
    net.train_step(*batch)
  for i in range(k):
    assert acc.micro_step == i
    acc.train_step(*batch)
  assert acc.micro_step == 0
  _against_noise(_grads(one), _grads(one2), _grads(acc, 1.0 / k), "gradient buffer",
                 frac=min(frac, 0.01), floor=floor)
  d = [{n: m[n] - w0[n] for n in w0} for m in (_masters(one), _masters(one2), _masters(acc))]
  _against_noise(*d, "update", frac=frac, floor=floor)


def _resnet50(k, **kw):
  from tensorflowonspark_b200.models import resnet
  return resnet.ResNetTrainer(depth=50, batch=8, image=64, num_classes=37, device="cuda:0",
                              gradient_accumulation_steps=k, **kw)


def _cifar(k, **kw):
  from tensorflowonspark_b200.models import resnet
  return resnet.CifarResNetTrainer(depth=20, batch=32, device="cuda:0",
                                   gradient_accumulation_steps=k, **kw)


def _unet(k, **kw):
  from tensorflowonspark_b200.models import unet
  return unet.UNetTrainer(batch=4, image=128, classes=21, seed=9, lr=2e-3,
                          gradient_accumulation_steps=k, **kw)


def _unet_batch(net, seed=1):
  from tensorflowonspark_b200.models import unet
  x, _ = net.synthetic_batch(seed=seed)
  return x, unet.synthetic_labels(x, net.classes)


@pytest.mark.parametrize("extras", [{}, {"clip_norm": 0.5, "ema_decay": 0.9}],
                         ids=["plain", "clip_ema"])
@pytest.mark.parametrize("opt", sorted(OPTS))
def test_resnet50_same_micro_batch_k_times_is_one_step(opt, extras):
  kw = dict(OPTS[opt], optimizer=opt, **extras)
  batch = _resnet50(1).synthetic_batch(seed=3)
  # (at 64 x 64 the last stage's maps are 2 x 2: its batch norms average 32 values, and a rounding
  # change upstream moves their gradients by up to ~15 % of the tensor's largest; a producer that
  # overwrites instead of adding is off by 2/3 on most elements)
  _same_batch_k_times(lambda k: _resnet50(k, **kw), batch, frac=max(FRAC.get(opt, 0.0), 0.01),
                      floor=0.2)


@pytest.mark.parametrize("extras", [{}, {"clip_norm": 0.5, "ema_decay": 0.9}],
                         ids=["plain", "clip_ema"])
@pytest.mark.parametrize("opt", sorted(OPTS))
def test_cifar_same_micro_batch_k_times_is_one_step(opt, extras):
  kw = dict(OPTS[opt], optimizer=opt, **extras)
  batch = _cifar(1).synthetic_batch(seed=4)
  _same_batch_k_times(lambda k: _cifar(k, **kw), batch, frac=FRAC.get(opt, 0.0))


@pytest.mark.parametrize("kw", [{}, {"encoder_trainable_from": 13},
                                {"ignore_index": 0, "class_weights": [1.0 + 0.1 * i for i in range(21)]},
                                {"encoder_trainable_from": 13, "optimizer": "lamb",
                                 "clip_norm": 0.5, "ema_decay": 0.9}],
                         ids=["frozen", "finetune13", "ignore_weights", "finetune_lamb_clip_ema"])
def test_unet_same_micro_batch_k_times_is_one_step(kw):
  net = _unet(1, **kw)
  batch = _unet_batch(net)
  del net
  _same_batch_k_times(lambda k: _unet(k, **kw), batch, frac=FRAC["adam"])   # (Adam family)


def _window_vs_mean(make, batches):
  """SGD without momentum or decay: the k-window update is the mean of the k single updates."""
  acc = make(len(batches))
  w0 = _masters(acc)
  for bt in batches:
    acc.train_step(*bt)
  got = _masters(acc)
  singles = []
  for bt in batches:
    net = make(1)
    net.train_step(*bt)
    singles.append(_masters(net))
  want = {n: sum(s[n] - w0[n] for s in singles) / len(batches) for n in w0}
  return {n: got[n] - w0[n] for n in w0}, want


def test_cifar_window_is_the_mean_of_single_updates():
  make = lambda k: _cifar(k, optimizer="sgd", lr=0.05, momentum=0.0, weight_decay=0.0)  # noqa: E731
  net = make(1)
  got, want = _window_vs_mean(make, [net.synthetic_batch(seed=s) for s in (11, 12, 13)])
  _compare(got, want, "cifar window")


def test_unet_finetune_window_sums_the_micro_batch_gradients():
  """(The U-Net trains with the Adam family, whose first update is sign-like, so the window is
  checked on its gradient buffer: the sum of the micro-batches' gradients, producer by producer.)"""
  kw = dict(encoder_trainable_from=13, ignore_index=0)
  acc = _unet(2, **kw)
  b1, b2 = _unet_batch(acc, 1), _unet_batch(acc, 2)
  acc.train_step(*b1)
  acc.train_step(*b2)
  singles = []
  for bt in (b1, b2):
    net = _unet(1, **kw)
    net.train_step(*bt)
    torch.cuda.synchronize()
    singles.append(net.store.grads.clone())
  torch.cuda.synchronize()
  st = acc.store
  got = {s["name"]: st._view(st.grads, s).cpu() for s in st.order}
  want = {s["name"]: st._view(singles[0] + singles[1], s).cpu() for s in st.order}
  _compare(got, want, "unet window gradients")


def test_resnet50_window_is_the_mean_of_single_updates():
  make = lambda k: _resnet50(k, optimizer="sgd", lr=0.05, momentum=0.0, weight_decay=0.0)  # noqa: E731
  net = make(1)
  got, want = _window_vs_mean(make, [net.synthetic_batch(seed=s) for s in (21, 22)])
  _compare(got, want, "resnet50 window", atol_rel=0.05)


# ------------------------------------------------------------------ graphs and launches
class _Spy(object):
  def __init__(self, optim):
    self.calls = []
    for name in ("launch", "finish", "step", "after_replay"):
      real = getattr(optim, name)
      setattr(optim, name, self._wrap(name, real))

  def _wrap(self, name, real):
    def call(*a, **k):
      self.calls.append(name)
      return real(*a, **k)
    return call


OPT_KERNELS = {"allreduce_opt", "lars_norms", "grad_sumsq", "clip_finalize"}


def _spy_kernels(monkeypatch, record):
  """Route every ``ops.K`` launch through ``record(name)`` (the optimizer and communication
  kernels all launch through ``ops.K``)."""
  from tensorflowonspark_b200 import ops

  class Spy(object):
    def __getattr__(self, name):
      fn = getattr(ops.C(), name)

      def call(*a, **kw):
        record(name)
        ops.count()
        return fn(*a, **kw)
      setattr(self, name, call)
      return call
  monkeypatch.setattr(ops, "K", Spy())


@pytest.mark.parametrize("make", [_resnet50, _cifar, _unet], ids=["resnet50", "cifar", "unet"])
def test_captured_window_matches_eager(make, monkeypatch):
  """The first / middle / last graphs: the kernels captured into the first and middle ones
  include no optimizer or communication kernel, the last one's do; from the same state, the
  gradient buffers after captured micro-steps 0 and 1 and the update after the captured window
  match eager ones (within the noise a second eager run shows), and only the last micro-step
  calls the optimizer."""
  k = 3
  graph, eager, eager2 = make(k), make(k), make(k)
  batch = _unet_batch(graph) if make is _unet else graph.synthetic_batch(seed=5)
  for net in (graph, eager, eager2):
    net.set_input(*batch)
  captured = []   # (window position being captured, kernel)
  _spy_kernels(monkeypatch, lambda name: captured.append((graph.micro_step, name))
               if torch.cuda.is_current_stream_capturing() else None)
  graph.capture()   # warm-up: one eager window
  assert set(graph.graphs) == {(True, False), (False, False), (False, True)}
  phases = {i: {n for at, n in captured if at == i} for i in range(k)}
  for i in range(k - 1):
    assert "bn_bwd_apply" in phases[i] and not OPT_KERNELS & phases[i], (i, phases[i])
  assert "allreduce_opt" in phases[k - 1], phases[k - 1]
  assert graph.micro_step == 0
  sd, osd = graph.state_dict(), graph.optim.state_dict()
  for net in (graph, eager, eager2):   # the same weights and optimizer state in all three
    net.load_state_dict(sd)
    net.optim.load_state_dict(osd)
  w0 = _masters(graph)
  floor = 0.2 if make is _resnet50 else 0.02   # (see test_resnet50_same_micro_batch_k_times...)
  spy = _Spy(graph.optim)
  for i in range(k):
    assert graph.micro_step == eager.micro_step == i
    for net in (graph, eager, eager2):
      net.train_step()
    if i < k - 1:
      _against_noise(_grads(eager), _grads(eager2), _grads(graph),
                     "micro-step {}: graph vs eager gradients".format(i), floor=floor, frac=1e-4)
      assert not spy.calls, (i, spy.calls)   # no optimizer / communication on micro-steps 1..k-1
    else:
      assert spy.calls == ["after_replay"], spy.calls
  d = [{n: m[n] - w0[n] for n in w0} for m in (_masters(eager), _masters(eager2), _masters(graph))]
  _against_noise(*d, "update: graph vs eager", floor=floor,
                 frac=FRAC["adam"] if make is _unet else 0.01)


@pytest.mark.parametrize("make", [_resnet50, _cifar, _unet], ids=["resnet50", "cifar", "unet"])
def test_micro_steps_launch_no_optimizer_kernel(make, monkeypatch):
  k = 2
  net = make(k)
  batch = _unet_batch(net) if make is _unet else net.synthetic_batch(seed=5)
  names = []
  _spy_kernels(monkeypatch, names.append)
  net.train_step(*batch)
  assert not OPT_KERNELS & set(names), names
  names.clear()
  net.train_step(*batch)
  assert OPT_KERNELS & set(names), names


def test_resnet101_and_152_train():
  """Their batch-norm arenas are sized from the model (the default capacity holds ResNet-50's)."""
  from tensorflowonspark_b200.models import resnet
  for depth in (101, 152):
    net = resnet.ResNetTrainer(depth=depth, batch=2, image=64, num_classes=10, device="cuda:0",
                               gradient_accumulation_steps=2)
    batch = net.synthetic_batch(seed=1)
    losses = [float(net.train_step(*batch)) for _ in range(4)]
    assert all(math.isfinite(v) for v in losses), (depth, losses)
    assert net.stats_arena.used <= net.stats_arena.buf.numel()
    del net


# ------------------------------------------------------------------ checkpoints and evaluation
def test_mid_window_evaluation_leaves_the_update_unchanged():
  a, b = _cifar(2), _cifar(2)
  b1, b2 = a.synthetic_batch(seed=1), a.synthetic_batch(seed=2)
  held = [a.synthetic_batch(seed=s) for s in (30, 31)]
  a.train_step(*b1)
  a.evaluate(held)
  a.train_step(*b2)
  b.train_step(*b1)
  b.train_step(*b2)
  _compare(_masters(a), _masters(b), "evaluation mid-window")


def test_mid_window_evaluation_unet_and_average():
  make = lambda: _unet(2, encoder_trainable_from=13, ema_decay=0.9)  # noqa: E731
  a, b, c = make(), make(), make()
  b1, b2 = _unet_batch(a, 1), _unet_batch(a, 2)
  w0 = _masters(a)
  for net, evaluate in ((a, True), (b, False), (c, False)):
    net.train_step(*b1)
    if evaluate:
      net.evaluate([b1], averaged=False)
      net.averaged()
    net.train_step(*b2)
  # the window's gradient sums (kept by the optimizer) and the update; c measures the noise
  _against_noise(_grads(b), _grads(c), _grads(a), "unet gradients, evaluation mid-window")
  d = [{n: m[n] - w0[n] for n in w0} for m in (_masters(b), _masters(c), _masters(a))]
  _against_noise(*d, "unet update, evaluation mid-window", frac=FRAC["adam"])


def test_checkpoint_of_k4_loads_into_k1_with_scale_one_over_world():
  a = _cifar(4)
  batch = a.synthetic_batch(seed=1)
  assert float(a.optim.hyper[3]) == float(torch.tensor(0.25))
  for _ in range(6):
    a.train_step(*batch)   # mid-window: micro_step 2
  assert a.micro_step == 2
  params, optim = a.state_dict(), a.optim.state_dict()
  assert float(optim["hyper"][3]) == 1.0          # k-free
  assert float(a.optim.hyper[3]) == 0.25          # the live scale is untouched
  one = _cifar(1)
  one.load_state_dict(params)
  one.optim.load_state_dict(optim)
  assert float(one.optim.hyper[3]) == 1.0
  four = _cifar(4)
  four.train_step(*batch)
  four.load_state_dict(params)
  four.optim.load_state_dict(optim)
  assert four.micro_step == 0 and float(four.optim.hyper[3]) == 0.25
  assert not four.store.grads.any()
  # both continue: k = 1 with one step, k = 4 with four steps of the same batch
  one.train_step(*batch)
  for _ in range(4):
    four.train_step(*batch)
  _compare(_masters(one), _masters(four), "continued from a checkpoint")


def test_loading_mid_window_restarts_the_window():
  net = _unet(3, encoder_trainable_from=13)
  sd = net.state_dict()
  batch = _unet_batch(net)
  net.train_step(*batch)
  assert net.micro_step == 1 and net.store.grads.any()
  net.load_state_dict(sd)
  torch.cuda.synchronize()
  assert net.micro_step == 0 and not net.store.grads.any()
  assert float(net.optim.hyper[3]) == float(torch.tensor(1.0 / 3))
  r = _resnet50(2)
  sd = r.state_dict()
  r.train_step(*r.synthetic_batch(seed=1))
  r.load_backbone(sd)
  torch.cuda.synchronize()
  assert r.micro_step == 0 and not r.store.grads.any()


def test_losses_are_per_micro_batch_and_finite():
  net = _cifar(2)
  net.capture()
  losses = []
  for s in range(8):
    losses.append(float(net.train_step(*net.synthetic_batch(seed=s % 2))))
  assert all(math.isfinite(v) for v in losses), losses


# ------------------------------------------------------------------ two or more GPUs
def _free_port():
  import socket
  with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as sk:
    sk.bind(("127.0.0.1", 0))
    return str(sk.getsockname()[1])


def test_grad_accum_two_ranks():
  """P2P, NVLS (when available), HierComm, GroupComm and first_step_fused_broadcast with k = 2:
  replicas bitwise identical, results equal to one rank on the summed micro-batches."""
  if torch.cuda.device_count() < 2:
    pytest.skip("needs 2 GPUs")
  p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node",
                      "2", "--master-addr", "127.0.0.1", "--master-port", _free_port(),
                      os.path.join(ROOT, "tools", "gpu_check_grad_accum.py")],
                     capture_output=True, text=True, timeout=900, cwd=ROOT)
  print(p.stdout[-4000:], p.stderr[-2000:])
  assert p.returncode == 0 and "GRAD ACCUM CHECK PASSED" in p.stdout

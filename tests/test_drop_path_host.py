"""Stochastic depth (``drop_path_rate``) for the ResNet trainers, host side (no GPU): the option
check, timm's linear-decay rates, the per-step draw (engine.DropPathDraws), the trainers' structure
(no state at rate 0, no fused bn3 reduction in a dropping block, one draw per ``train_step``), the
float64 references of the scaled batch-norm kernels that tests/test_gpu_drop_path.py compares
against, the bindings' refusals of bad ``sample_scale`` vectors, ptxas on csrc/bn_bwd.cu and the
examples' ``--drop_path_rate`` flag."""
import importlib
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tensorflowonspark_b200.models import engine, resnet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_example_drivers_dryrun as dry  # noqa: E402
import test_unet_classes_host as uc  # noqa: E402
from test_example_drivers_dryrun import fake_gpu  # noqa: E402,F401  (fixture)
from test_mixup_host import _Allocated, cpu_plans, no_alloc  # noqa: E402,F401  (fixtures)

NAN = float("nan")
TRAINERS = ["ResNetTrainer", "CifarResNetTrainer"]


# ------------------------------------------------------------------ float64 references
def sample_of_rows(N, HW):
  """Sample index of each of the N * HW rows of an NHWC tensor."""
  return torch.arange(N).repeat_interleave(HW)


def ref_scaled_apply(x, residual, scale, shift, s, act=1):
  """(y, pre) of the scaled forward apply in float64: pre = s[n] (x scale + shift) (+ residual),
  y = relu(pre) (act 1) or pre (act 0); x, residual NHWC, scale / shift [C], s [N]."""
  x = x.double().cpu()
  N, C = x.shape[0], x.shape[-1]
  sv = s.double().cpu().view(N, *([1] * (x.dim() - 1)))
  pre = sv * (x * scale.double().cpu().view(1, 1, 1, C) + shift.double().cpu().view(1, 1, 1, C))
  if residual is not None:
    pre = pre + residual.double().cpu()
  return (pre.clamp(min=0) if act == 1 else pre), pre


def ref_scaled_bwd(dy, x, keep, gamma, mean, invstd, s):
  """(dgamma, dbeta, dx, dres) in float64 of a batch norm whose output is scaled per sample by s
  and followed by a ReLU (``keep``: the mask, True where the pre-activation was > 0):
  g = keep dy (the shortcut's gradient, dres), gs = s[n] g, dgamma = sum gs xhat, dbeta = sum gs,
  dx = gamma invstd (gs - dbeta / M - xhat dgamma / M), xhat = (x - mean) invstd, M = N H W."""
  N, C = x.shape[0], x.shape[-1]
  x, dy = x.double().cpu().reshape(-1, C), dy.double().cpu().reshape(-1, C)
  keep = keep.cpu().reshape(-1, C)
  g = torch.where(keep, dy, torch.zeros_like(dy))
  gs = s.double().cpu()[sample_of_rows(N, x.shape[0] // N)].view(-1, 1) * g
  mean, invstd, gamma = (t.double().cpu().view(1, C) for t in (mean, invstd, gamma))
  xhat = (x - mean) * invstd
  M = x.shape[0]
  dgamma, dbeta = (gs * xhat).sum(0), gs.sum(0)
  dx = gamma * invstd * (gs - dbeta / M - xhat * dgamma / M)
  return dgamma, dbeta, dx, g


def _bn_stats(x, eps):
  """float64 batch mean and 1 / sqrt(biased var + eps) per channel of an NHWC tensor."""
  xf = x.double().reshape(-1, x.shape[-1])
  mean = xf.mean(0)
  return mean, 1.0 / torch.sqrt(((xf - mean) ** 2).mean(0) + eps)


@pytest.mark.parametrize("with_res", [False, True])
@pytest.mark.parametrize("s", [[1.0, 1.0, 1.0], [0.0, 1.25, 1.25], [0.0, 0.0, 2.0]])
def test_scaled_references_match_torch_autograd(with_res, s):
  g = torch.Generator().manual_seed(len(s) + 10 * with_res)
  N, H, W, C = 3, 4, 5, 8
  eps = 1e-5
  x = torch.randn(N, H, W, C, generator=g, dtype=torch.float64)
  res = torch.randn(N, H, W, C, generator=g, dtype=torch.float64) if with_res else None
  gamma = 0.5 + torch.rand(C, generator=g, dtype=torch.float64)
  beta = 0.1 * torch.randn(C, generator=g, dtype=torch.float64)
  dy = torch.randn(N, H, W, C, generator=g, dtype=torch.float64)
  sv = torch.tensor(s, dtype=torch.float64)
  # torch: out = relu(s_b * BN(x) + res), BN over the whole batch in training mode
  xt = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
  gt, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
  rt = res.permute(0, 3, 1, 2).clone().requires_grad_(True) if with_res else None
  bn = F.batch_norm(xt, None, None, gt, bt, training=True, eps=eps)
  pre = sv.view(N, 1, 1, 1) * bn + (rt if with_res else 0)
  out = pre.clamp(min=0)
  out.backward(dy.permute(0, 3, 1, 2))
  mean, invstd = _bn_stats(x, eps)
  scale, shift = gamma * invstd, beta - mean * gamma * invstd
  y, pre_ref = ref_scaled_apply(x, res, scale, shift, sv, act=1)
  nhwc = lambda t: t.permute(0, 2, 3, 1)  # noqa: E731
  torch.testing.assert_close(y, nhwc(out.detach()), rtol=1e-10, atol=1e-12)
  dgamma, dbeta, dx, dres = ref_scaled_bwd(dy, x, pre_ref > 0, gamma, mean, invstd, sv)
  torch.testing.assert_close(dx.view(N, H, W, C), nhwc(xt.grad), rtol=1e-9, atol=1e-12)
  torch.testing.assert_close(dgamma, gt.grad, rtol=1e-9, atol=1e-12)
  torch.testing.assert_close(dbeta, bt.grad, rtol=1e-9, atol=1e-12)
  if with_res:   # the shortcut gets the unscaled masked gradient
    torch.testing.assert_close(dres.view(N, H, W, C), nhwc(rt.grad), rtol=1e-12, atol=1e-12)
  if s[0] == 0.0:   # a dropped sample still gets a gradient through the batch statistics
    assert float(xt.grad[0].abs().sum()) > 0


# ------------------------------------------------------------------ option checks
@pytest.mark.parametrize("trainer", TRAINERS)
@pytest.mark.parametrize("r", [-0.1, 1, 1.0, 1.5, NAN, math.inf, -math.inf, "0.1", None, True,
                               False, [0.1]])
def test_bad_drop_path_rate_raises_before_allocation(no_alloc, trainer, r):
  with pytest.raises(ValueError, match="drop_path_rate must be a real number in"):
    getattr(resnet, trainer)(device="cpu", num_classes=5, drop_path_rate=r)


def test_drop_path_is_refused_on_an_inference_trainer(no_alloc):
  with pytest.raises(ValueError, match="drop_path_rate needs training=True"):
    resnet.ResNetTrainer(device="cpu", num_classes=5, training=False, drop_path_rate=0.05)
  with pytest.raises(_Allocated):   # 0 is the default, fine without training
    resnet.ResNetTrainer(device="cpu", num_classes=5, training=False, drop_path_rate=0)


@pytest.mark.parametrize("trainer", TRAINERS)
@pytest.mark.parametrize("r", [0, 0.0, 0.05, 0.1, 0.999, np.float32(0.2), np.float64(0.5)])
def test_good_drop_path_rates_pass_the_check(no_alloc, trainer, r):
  with pytest.raises(_Allocated):
    getattr(resnet, trainer)(device="cpu", num_classes=5, drop_path_rate=r)


def test_check_drop_path_rate_returns_a_float():
  for r in (0, 0.1, np.float32(0.25)):
    got = engine.check_drop_path_rate(r)
    assert type(got) is float and got == float(r)
  assert engine.check_drop_path_rate() == 0.0


# ------------------------------------------------------------------ rates
@pytest.mark.parametrize("r", [0.0, 0.05, 0.1, 0.3])
@pytest.mark.parametrize("n", [2, 9, 16, 27])
def test_rates_decay_linearly_from_zero_to_r(r, n):
  rates = engine.drop_path_rates(r, n)
  assert len(rates) == n and rates[0] == 0.0 and rates[-1] == r
  assert list(rates) == [r * i / (n - 1) for i in range(n)]
  # timm's resnet: drop_path_rate * net_block_idx / (net_num_blocks - 1)
  assert all(a <= b for a, b in zip(rates, rates[1:]))


def test_trainers_expose_their_rates(cpu_plans):
  net = resnet.CifarResNetTrainer(depth=20, batch=2, device="cpu", drop_path_rate=0.1)
  assert net.drop_path_rate == 0.1 and len(net.drop_path_rates) == 9
  assert net.drop_path_rates == engine.drop_path_rates(0.1, 9)
  net = resnet.ResNetTrainer(depth=50, batch=2, image=64, device="cpu", drop_path_rate=0.05)
  assert net.drop_path_rate == 0.05 and net.drop_path_rates == engine.drop_path_rates(0.05, 16)
  assert resnet.ResNetTrainer(depth=50, batch=2, image=64, device="cpu",
                              training=False).drop_path_rates == (0.0,) * 16


# ------------------------------------------------------------------ the draw
def test_draws_repeat_per_seed_and_rank_and_differ_across_ranks():
  rates = engine.drop_path_rates(0.3, 8)
  draw = lambda seed, rank: [engine.DropPathDraws(rates, 16, seed, rank).draw()  # noqa: E731
                             for _ in range(1)][0]
  a = engine.DropPathDraws(rates, 16, seed=5, rank=0)
  b = engine.DropPathDraws(rates, 16, seed=5, rank=0)
  for _ in range(20):
    assert np.array_equal(a.draw(), b.draw())
  assert not np.array_equal(draw(5, 0), draw(5, 1))
  assert not np.array_equal(draw(5, 0), draw(6, 0))


def test_draw_values_and_keep_frequencies():
  rates = (0.0, 0.05, 0.3, 0.5, 0.9)
  B, n = 64, 400
  d = engine.DropPathDraws(rates, B, seed=3)
  draws = np.stack([d.draw() for _ in range(n)])           # [n, blocks, B]
  assert draws.dtype == np.float32 and draws.shape == (n, len(rates), B)
  assert (draws[:, 0] == 1.0).all()                           # p = 0: all ones
  for i, p in enumerate(rates[1:], 1):
    kept = np.float32(1.0 / (1.0 - p))
    assert set(np.unique(draws[:, i]).tolist()) <= {0.0, float(kept)}
    k, m = int((draws[:, i] != 0).sum()), n * B
    assert abs(k - m * (1 - p)) <= 5 * math.sqrt(m * p * (1 - p)) + 1, (p, k, m)


def test_drop_path_does_not_change_the_mix_draws(cpu_plans):
  kw = {"depth": 20, "batch": 4, "device": "cpu", "mixup_alpha": 0.2, "cutmix_alpha": 1.0,
        "seed": 9}
  a = resnet.CifarResNetTrainer(**kw)
  b = resnet.CifarResNetTrainer(drop_path_rate=0.2, **kw)
  for _ in range(8):
    a._stage_draws()
    b._stage_draws()
    assert a.last_mix == b.last_mix
    assert torch.equal(a.mix, b.mix)
  assert a.last_drop_path is None and b.last_drop_path is not None


# ------------------------------------------------------------------ trainer structure
def _fused(net):
  return [bn.name for bn in net._batch_norms() if bn.fused_reduce]


def test_rate_zero_trainers_have_no_drop_path_state(cpu_plans):
  for make in (lambda **k: resnet.CifarResNetTrainer(depth=20, batch=2, device="cpu", **k),
               lambda **k: resnet.ResNetTrainer(depth=50, batch=2, image=64, device="cpu", **k)):
    for net in (make(), make(drop_path_rate=0.0)):
      assert net.dropper is None and net.drop_scale is None and net.last_drop_path is None
      assert all(net._drop_arg(i) == {} for i in range(len(net.blocks)))
      net._stage_draws()
      assert net.last_drop_path is None
  plain = resnet.ResNetTrainer(depth=50, batch=2, image=64, device="cpu")
  zero = resnet.ResNetTrainer(depth=50, batch=2, image=64, device="cpu", drop_path_rate=0.0)
  assert _fused(plain) == _fused(zero)
  # every identity block's conv1 finishes the previous block's bn3 reduction (12 of 16 blocks)
  assert len([n for n in _fused(plain) if n.endswith(".u3.bn")]) == 12


@pytest.mark.parametrize("r", [0.05, 0.1])
def test_dropping_blocks_take_the_unfused_bn3_reduction(cpu_plans, r):
  plain = resnet.ResNetTrainer(depth=50, batch=2, image=64, device="cpu")
  net = resnet.ResNetTrainer(depth=50, batch=2, image=64, device="cpu", drop_path_rate=r)
  for b, p in zip(net.blocks, net.drop_path_rates):
    if p > 0:
      assert not b.u3.bn.fused_reduce, b.name
  # only those reductions moved: bn1 / bn2 and block 0's bn3 are fused as before
  want = [n for n in _fused(plain) if not n.endswith(".u3.bn") or n.startswith("layer1.0.")]
  assert _fused(net) == want
  assert "layer1.0.u3.bn" in _fused(net)
  assert net.drop_scale.shape == (16, 2) and net.drop_scale.dtype == torch.float32
  assert net._drop_arg(0) == {} and net._drop_arg(1)["sample_scale"].shape == (2,)


@pytest.mark.parametrize("trainer", TRAINERS)
def test_one_draw_is_staged_per_train_step(cpu_plans, monkeypatch, trainer):
  kw = {"batch": 3, "device": "cpu", "drop_path_rate": 0.5, "seed": 11}
  net = (resnet.CifarResNetTrainer(depth=20, **kw) if trainer == "CifarResNetTrainer" else
         resnet.ResNetTrainer(depth=50, image=64, **kw))
  calls = []
  real = net.dropper.draw
  monkeypatch.setattr(net.dropper, "draw", lambda: calls.append(1) or real())
  monkeypatch.setattr(net.accum, "run", lambda *a, **k: None)
  twin = engine.DropPathDraws(net.drop_path_rates, 3, seed=11, rank=0)
  for i in range(5):
    net.train_step()
    assert len(calls) == i + 1
    want = twin.draw()
    assert np.array_equal(net.last_drop_path, want)
    assert torch.equal(net.drop_scale, torch.from_numpy(want))


# ------------------------------------------------------------------ binding refusals
def _C():
  from tensorflowonspark_b200 import ops
  return ops.C()


X4 = (2, 4, 4, 8)
BAD_SCALE = [
    (torch.zeros(X4), torch.zeros(2, dtype=torch.float64), "sample_scale must be float32"),
    (torch.zeros(X4), torch.zeros(2, dtype=torch.bfloat16), "sample_scale must be float32"),
    (torch.zeros(X4), torch.zeros(4)[::2], "sample_scale must be contiguous"),
    (torch.zeros(X4), torch.zeros(3), "one value per sample"),
    (torch.zeros(X4), torch.zeros(1, 2), "one value per sample"),
    (torch.zeros(8, 8), torch.zeros(8), "needs a 4-D NHWC x"),
    (torch.zeros(2, 16, 8), torch.zeros(2), "needs a 4-D NHWC x"),
    (torch.zeros(X4), torch.zeros(2), "sample_scale must be on the CUDA device of x"),
]


def _calls(x, ss):
  C = x.shape[-1]
  v = torch.zeros(C)
  return {
      "bn_apply": lambda: _C().bn_apply(x, None, v, v, x, 1, None, sample_scale=ss),
      "bn_apply_finalize": lambda: _C().bn_apply_finalize(
          x, None, x, 1, None, v, v, v, v, None, None, v, v, v, v, 8.0, 1e-5, 0.1,
          sample_scale=ss),
      "bn_bwd_reduce": lambda: _C().bn_bwd_reduce(x, x, None, v, v, v, v, 3, None, None,
                                                  sample_scale=ss),
      "bn_bwd_apply": lambda: _C().bn_bwd_apply(x, x, None, v, v, v, v, v, x, None, 3, None, None,
                                                sample_scale=ss),
  }


@pytest.mark.parametrize("entry", ["bn_apply", "bn_apply_finalize", "bn_bwd_reduce",
                                   "bn_bwd_apply"])
@pytest.mark.parametrize("x,ss,match", BAD_SCALE)
def test_bad_sample_scale_is_refused_before_the_launch(entry, x, ss, match):
  with pytest.raises(ValueError, match=match):
    _calls(x, ss)[entry]()


def test_sample_scale_is_refused_with_a_fused_reduction():
  x, v = torch.zeros(X4), torch.zeros(8)
  for kw in ({"sum_g": v, "sum_gx": v}, {"sum_g": v}, {"sum_gx": v}):
    with pytest.raises(ValueError, match="cannot be used with a fused reduction"):
      _C().bn_bwd_apply(x, x, None, v, v, v, v, v, x, None, 3, None, None,
                        sample_scale=torch.zeros(2), **kw)


def test_sample_scale_is_refused_with_the_recomputed_mask():
  x, v = torch.zeros(X4), torch.zeros(8)
  with pytest.raises(ValueError, match="needs relu 0, 1 or 3"):
    _C().bn_bwd_apply(x, x, None, v, v, v, v, v, x, None, 2, v, v, sample_scale=torch.zeros(2))
  with pytest.raises(ValueError, match="needs relu 0, 1 or 3"):
    _C().bn_bwd_reduce(x, x, None, v, v, v, v, 2, v, v, sample_scale=torch.zeros(2))


def test_entry_points_keep_their_positional_form():
  x, v = torch.zeros(X4, dtype=torch.bfloat16), torch.zeros(8)
  for call in (lambda: _C().bn_apply(x, None, v, v, x, 1, None),
               lambda: _C().bn_apply(x, None, v, v, x, 1, None, None),
               lambda: _C().bn_apply_finalize(x, None, x, 1, None, v, v, v, v, None, None, v, v, v,
                                              v, 8.0, 1e-5, 0.1),
               lambda: _C().bn_bwd_reduce(x, x, None, v, v, v, v, 3, None, None)):
    with pytest.raises(RuntimeError, match="CUDA tensor"):
      call()
  with pytest.raises(RuntimeError, match="acc_dgamma and acc_dbeta go together"):
    _C().bn_bwd_apply(x, x, None, v, v, v, v, v, x, None, 3, None, None, None, None, v, None)


def test_engine_refuses_a_scale_on_a_fused_reduction():
  st = engine.ParamStore()
  bn = engine.BatchNorm(st, "blk.u3.bn", 8)
  bn.fused_reduce, bn.acc, bn.dgamma, bn.dbeta = True, None, torch.zeros(8), torch.zeros(8)
  with pytest.raises(ValueError, match="blk.u3.bn: sample_scale needs the unfused"):
    bn.backward(None, None, None, None, sample_scale=torch.ones(2))


# ------------------------------------------------------------------ ptxas
SCALED_KERNELS = {"bn_fwd_apply_scaled_kernel": 2, "bn_bwd_reduce_scaled_kernel": 1,
                  "bn_bwd_apply_scaled_kernel": 1, "bn_bwd_apply_acc_scaled_kernel": 1}


@pytest.mark.skipif(not os.path.exists(uc.NVCC), reason="nvcc not found")
def test_scaled_batch_norm_kernels_have_no_stack_frame_or_spills(tmp_path):
  kernels = uc._ptxas("bn_bwd.cu", tmp_path)
  new = {}
  for name, n in SCALED_KERNELS.items():
    mangled = "{}{}".format(len(name), name)     # the length-prefixed name: an exact match
    got = {k: v for k, v in kernels.items() if mangled in k}
    assert len(got) == n, (name, sorted(kernels))
    new.update(got)
  assert len(kernels) == len(new) + 5, sorted(kernels)   # the five kernels that were there before
  bad = {k: v for k, v in new.items() if v != (0, 0, 0)}
  assert not bad, "stack frame / spill stores / spill loads (bytes): {}".format(bad)


# ------------------------------------------------------------------ example flags
def _spark(argv):
  mod = importlib.import_module("resnet_spark")
  mod.main_fun(["resnet_spark.py", "--batch_size", "4", "--image", "64"] + argv, dry._Ctx(1))
  return dry._Trainer.made[-1]


def test_resnet_spark_drop_path_flag(fake_gpu):
  assert importlib.import_module("resnet_spark").parse([]).drop_path_rate == 0.0
  assert "drop_path_rate" not in _spark(["--train_steps", "2"]).kw
  assert _spark(["--train_steps", "2", "--drop_path_rate", "0.05"]).kw["drop_path_rate"] == 0.05
  net = _spark(["--train_steps", "2", "--model", "resnet56", "--drop_path_rate", "0.1"])
  assert net.kw["drop_path_rate"] == 0.1


def test_resnet_cifar_drop_path_flag(fake_gpu):
  mod = importlib.import_module("resnet_cifar_main")
  assert mod.define_flags().parse_args([]).drop_path_rate == 0.0
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "2"], mod.LocalContext())
  assert "drop_path_rate" not in dry._Trainer.made[-1].kw
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "2", "--drop_path_rate", "0.1"],
               mod.LocalContext())
  assert dry._Trainer.made[-1].kw["drop_path_rate"] == 0.1

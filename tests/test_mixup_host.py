"""Mixup and CutMix for the ResNet trainers, host side (no GPU): option checks, the per-step draw
(engine.MixDraws), the float64 references of the mixed decode and the two mixed-target losses that
tests/test_gpu_mixup.py compares the kernels against, the bindings' refusals of bad mix vectors,
ptxas on csrc/mix.cu and the examples' mixing flags."""
import importlib
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tensorflowonspark_b200.models import engine, resnet
from tensorflowonspark_b200.ops import igemm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_example_drivers_dryrun as dry  # noqa: E402
import test_unet_classes_host as uc  # noqa: E402
from test_example_drivers_dryrun import fake_gpu  # noqa: E402,F401  (fixture)

NAN = float("nan")
MIX_KW = ("mixup_alpha", "cutmix_alpha", "mix_prob", "mix_switch_prob")


class _Plan(object):
  def set_reverse(self, flag):
    pass


@pytest.fixture
def cpu_plans(monkeypatch):
  """Trainers built on the CPU: every igemm plan builder returns a placeholder."""
  for name in ("conv_fprop", "conv_dgrad", "conv_wgrad", "stem_fprop", "stem_wgrad", "gemm",
               "gemm_wgrad"):
    monkeypatch.setattr(igemm, name, lambda *a, **k: _Plan())


class _Allocated(Exception):
  pass


@pytest.fixture
def no_alloc(monkeypatch):
  """Building a parameter store is the first allocation of both trainers: make it fail loudly."""
  def boom(*a, **k):
    raise _Allocated()
  monkeypatch.setattr(resnet, "ParamStore", boom)


# ------------------------------------------------------------------ float64 references
def partner(B):
  """Row i's partner p(i) = B - 1 - i (timm's batch mode: the batch flipped)."""
  return torch.arange(B - 1, -1, -1)


def f32(v):
  """v as the kernels hold it (fp32), as a Python float."""
  return float(torch.tensor(v, dtype=torch.float32))


def ref_decode(img, Wp, wofs, mean, std):
  """(out, mag): uint8 RGB [N, H, W, 3] normalised with the fp32 constants the kernel holds (mean,
  1 / std) into float64 [N, H, Wp, 8]; channels 3..7 and the columns outside [wofs, wofs + W) are 0.
  ``mag`` bounds the terms: (x / 255 + |mean|) / std."""
  N, H, W, _ = img.shape
  m = torch.tensor([f32(mean[c % len(mean)]) for c in range(3)], dtype=torch.float64)
  si = torch.tensor([f32(1.0 / std[c % len(std)]) for c in range(3)], dtype=torch.float64)
  v = img.double().cpu() / 255.0
  out = torch.zeros(N, H, Wp, 8, dtype=torch.float64)
  mag = torch.zeros_like(out)
  out[:, :, wofs:wofs + W, :3] = (v - m) * si
  mag[:, :, wofs:wofs + W, :3] = (v + m.abs()) * si.abs()
  return out, mag


def ref_mix_decode(img, Wp, wofs, mean, std, draw):
  """(out, mag) of the mixed decode of ``draw`` = (mode, lam, box) with lam rounded to fp32:
  mixup lam n(u_i) + (1 - lam) n(u_p), cutmix n(u_p) inside the box (rows [y0, y1), columns
  [x0, x1) of the image, clamped to it) and n(u_i) elsewhere."""
  mode, lam, (y0, y1, x0, x1) = draw
  out, mag = ref_decode(img, Wp, wofs, mean, std)
  p = partner(img.shape[0])
  if mode == "mixup":
    lam = f32(lam)
    return lam * out + (1 - lam) * out[p], lam * mag + (1 - lam) * mag[p]
  if mode == "cutmix":
    H, W = img.shape[1:3]
    y0, y1 = min(max(y0, 0), H), min(max(y1, 0), H)
    x0, x1 = min(max(x0, 0), W), min(max(x1, 0), W)
    out, mag = out.clone(), mag.clone()
    if y1 > y0 and x1 > x0:
      out[:, y0:y1, wofs + x0:wofs + x1] = out[p][:, y0:y1, wofs + x0:wofs + x1]
      mag[:, y0:y1, wofs + x0:wofs + x1] = mag[p][:, y0:y1, wofs + x0:wofs + x1]
  return out, mag


def mixed_onehot(labels, V, eps, lam):
  """float64 [B, V] targets lam s(y_i) + (1 - lam) s(y_p), s(y) = (1 - eps) onehot(y) + eps / V."""
  s = F.one_hot(labels.long().cpu(), V).double() * (1 - eps) + eps / V
  return lam * s + (1 - lam) * s[partner(len(labels))]


def ref_mixed_xent(logits, labels, V, eps, lam):
  """float64 per-row loss -sum_j t_j log softmax(l)_j and its gradient softmax(l) - t over the
  first V columns, t = mixed_onehot(labels, V, eps, lam)."""
  l = logits[:, :V].double().cpu()
  t = mixed_onehot(labels, V, eps, lam)
  logp = torch.log_softmax(l, 1)
  return -(t * logp).sum(1), logp.exp() - t


def mixed_multihot(targets, V, eps, lam):
  """float64 [B, V] targets lam s(y_i) + (1 - lam) s(y_p), s(y) = y (1 - eps) + eps / 2, y the
  nonzero bytes."""
  s = (targets[:, :V].cpu() != 0).double() * (1 - eps) + eps / 2
  return lam * s + (1 - lam) * s[partner(len(targets))]


def softplus(x):
  return x.clamp(min=0) + torch.log1p(torch.exp(-x.abs()))


def ref_mixed_bce(logits, targets, V, eps, lam, pos_weight=None):
  """float64 per-element loss p t softplus(-l) + (1 - t) softplus(l) and its gradient
  sigmoid(l) (p t + 1 - t) - p t, t = mixed_multihot(targets, V, eps, lam)."""
  l = logits[:, :V].double().cpu()
  t = mixed_multihot(targets, V, eps, lam)
  p = torch.ones(V, dtype=torch.float64) if pos_weight is None else \
      torch.as_tensor(pos_weight, dtype=torch.float64).cpu()
  pt = p * t
  return pt * softplus(-l) + (1 - t) * softplus(l), torch.sigmoid(l) * (pt + 1 - t) - pt


def dominant_rows(B, lam):
  """The row whose label each row's hit is scored against: its own when lam >= 0.5."""
  return torch.arange(B) if lam >= 0.5 else partner(B)


def ref_hits(logits, labels, V, lam):
  """Rows whose lowest-index arg-max is the dominant label."""
  amax = logits[:, :V].double().cpu().argmax(1)
  return int((amax == labels.long().cpu()[dominant_rows(len(labels), lam)]).sum())


def ref_exact_rows(logits, targets, V, lam):
  """Rows whose prediction (l > 0) equals the dominant row's multi-hot target everywhere."""
  want = (targets[:, :V].cpu() != 0)[dominant_rows(len(targets), lam)]
  return int(((logits[:, :V].cpu() > 0) == want).all(1).sum())


# ------------------------------------------------------------------ option checks
@pytest.mark.parametrize("trainer", ["ResNetTrainer", "CifarResNetTrainer"])
@pytest.mark.parametrize("kw,match", [
    ({"mixup_alpha": -0.1}, "mixup_alpha must be a real number finite and >= 0"),
    ({"mixup_alpha": NAN}, "mixup_alpha"),
    ({"mixup_alpha": math.inf}, "mixup_alpha"),
    ({"mixup_alpha": "0.2"}, "mixup_alpha"),
    ({"mixup_alpha": None}, "mixup_alpha"),
    ({"mixup_alpha": True}, "mixup_alpha"),
    ({"cutmix_alpha": -1}, "cutmix_alpha"),
    ({"cutmix_alpha": math.inf}, "cutmix_alpha"),
    ({"cutmix_alpha": NAN}, "cutmix_alpha"),
    ({"mix_prob": -0.01}, r"mix_prob must be a real number in \[0, 1\]"),
    ({"mix_prob": 1.01}, "mix_prob"),
    ({"mix_prob": NAN}, "mix_prob"),
    ({"mix_prob": None}, "mix_prob"),
    ({"mix_switch_prob": 2}, "mix_switch_prob"),
    ({"mix_switch_prob": -math.inf}, "mix_switch_prob"),
    ({"mix_switch_prob": False}, "mix_switch_prob"),
])
def test_bad_mixing_options_raise_before_allocation(no_alloc, trainer, kw, match):
  with pytest.raises(ValueError, match=match):
    getattr(resnet, trainer)(device="cpu", num_classes=5, **kw)


@pytest.mark.parametrize("kw", [{"mixup_alpha": 0.2}, {"cutmix_alpha": 1.0}, {"mix_prob": 0.5},
                                {"mix_switch_prob": 0.0}])
def test_mixing_options_are_refused_on_an_inference_trainer(no_alloc, kw):
  with pytest.raises(ValueError, match="training=True"):
    resnet.ResNetTrainer(device="cpu", num_classes=5, training=False, **kw)


@pytest.mark.parametrize("trainer", ["ResNetTrainer", "CifarResNetTrainer"])
@pytest.mark.parametrize("kw", [{}, {"mixup_alpha": 0.2}, {"cutmix_alpha": 1},
                                {"mixup_alpha": 0.8, "cutmix_alpha": 1.0, "mix_prob": 0,
                                 "mix_switch_prob": 1},
                                {"mixup_alpha": np.float32(0.1), "mix_prob": 1.0}])
def test_good_mixing_options_pass_the_checks(no_alloc, trainer, kw):
  with pytest.raises(_Allocated):
    getattr(resnet, trainer)(device="cpu", num_classes=5, **kw)


def test_defaults_pass_on_an_inference_trainer(no_alloc):
  with pytest.raises(_Allocated):
    resnet.ResNetTrainer(device="cpu", num_classes=5, training=False, mixup_alpha=0, mix_prob=1,
                         mix_switch_prob=0.5)


def test_check_mix_args_returns_floats():
  got = engine.check_mix_args(1, 0, 1, 0)
  assert got == (1.0, 0.0, 1.0, 0.0) and all(type(v) is float for v in got)
  assert engine.check_mix_args() == (0.0, 0.0, 1.0, 0.5)


def test_default_trainer_has_no_mixing_state(cpu_plans):
  for net in (resnet.CifarResNetTrainer(depth=20, batch=2, device="cpu"),
              resnet.CifarResNetTrainer(depth=20, batch=2, device="cpu", mix_prob=0.3)):
    assert (net.mixup_alpha, net.cutmix_alpha) == (0.0, 0.0)
    assert net.mixer is None and net.mix is None and net.last_mix is None
    assert net._mix_arg() == {}     # the decode and loss get the arguments they always got
    net._stage_mix()                # draws nothing
    assert net.last_mix is None


def test_mixing_trainer_stages_each_draw(cpu_plans):
  net = resnet.CifarResNetTrainer(depth=20, batch=3, device="cpu", mixup_alpha=0.2,
                                  cutmix_alpha=1.0, seed=77)
  assert (net.mixup_alpha, net.cutmix_alpha, net.mix_prob, net.mix_switch_prob) == \
      (0.2, 1.0, 1.0, 0.5)
  assert net.mix.dtype == torch.float32 and net.mix.shape == (engine.MIX_SLOTS,)
  assert net._mix_arg()["mix"] is net.mix
  twin = engine.MixDraws(0.2, 1.0, seed=77, rank=0)
  for _ in range(6):
    net._stage_mix()
    want = twin.draw(32, 32)
    assert net.last_mix == want
    assert net.mix.tolist() == [f32(v) for v in engine.MixDraws.vector(want)]


# ------------------------------------------------------------------ the draw
def _draws(n, H=224, W=224, **kw):
  m = engine.MixDraws(**dict({"mixup_alpha": 0.0, "cutmix_alpha": 0.0, "seed": 1, "rank": 0},
                             **kw))
  return [m.draw(H, W) for _ in range(n)]


def test_draws_repeat_per_seed_and_rank_and_differ_across_ranks():
  kw = {"mixup_alpha": 0.2, "cutmix_alpha": 1.0, "mix_prob": 0.8}
  a = _draws(200, seed=5, rank=0, **kw)
  assert a == _draws(200, seed=5, rank=0, **kw)
  assert a != _draws(200, seed=5, rank=1, **kw)
  assert a != _draws(200, seed=6, rank=0, **kw)


def _binomial_ok(k, n, p, z=5.0):
  return abs(k - n * p) <= z * math.sqrt(n * p * (1 - p)) + 1


@pytest.mark.parametrize("mix_prob,switch", [(1.0, 0.5), (0.7, 0.3), (0.25, 0.9), (0.0, 0.5)])
def test_mode_frequencies(mix_prob, switch):
  n = 4000
  d = _draws(n, mixup_alpha=0.4, cutmix_alpha=1.0, mix_prob=mix_prob, mix_switch_prob=switch)
  modes = [m for m, _, _ in d]
  mixed = n - modes.count("none")
  assert _binomial_ok(mixed, n, mix_prob)
  if mixed:
    assert _binomial_ok(modes.count("cutmix"), mixed, switch)
  assert all(lam == 1.0 and box == (0, 0, 0, 0) for m, lam, box in d if m == "none")
  # only one alpha > 0: that mode, whatever mix_switch_prob says
  assert {m for m, _, _ in _draws(300, mixup_alpha=0.4, mix_switch_prob=1.0)} == {"mixup"}
  assert {m for m, _, _ in _draws(300, cutmix_alpha=0.4, mix_switch_prob=0.0)} == {"cutmix"}


@pytest.mark.parametrize("alpha", [0.2, 1.0])
def test_lambda_is_beta_distributed(alpha):
  from scipy import stats
  lams = [lam for _, lam, _ in _draws(5000, mixup_alpha=alpha, seed=11)]
  assert all(0.0 <= v <= 1.0 for v in lams)
  assert stats.kstest(lams, stats.beta(alpha, alpha).cdf).pvalue > 1e-3


@pytest.mark.parametrize("H,W", [(224, 224), (32, 32), (7, 5), (2, 2)])
def test_cutmix_boxes_stay_inside_and_correct_lambda(H, W):
  d = _draws(3000, H, W, cutmix_alpha=1.0, seed=H * W)
  for mode, lam, (y0, y1, x0, x1) in d:
    assert mode == "cutmix"
    assert 0 <= y0 <= y1 <= H and 0 <= x0 <= x1 <= W
    assert lam == 1.0 - (y1 - y0) * (x1 - x0) / float(H * W)


def test_empty_box_and_full_image_are_reached():
  # alpha 0.01 puts lam at 0 or 1 to double precision often: full boxes need lam == 0 and the
  # centre pixel in the middle of an even side
  d = _draws(2000, 2, 2, cutmix_alpha=0.01, seed=3)
  areas = {(y1 - y0) * (x1 - x0) for _, _, (y0, y1, x0, x1) in d}
  assert 0 in areas and 4 in areas
  assert {lam for _, lam, _ in d} >= {0.0, 1.0}


def test_vector_layout():
  assert engine.MixDraws.vector(("none", 1.0, (0, 0, 0, 0))) == [0, 1, 0, 0, 0, 0, 0, 0]
  assert engine.MixDraws.vector(("mixup", 0.25, (0, 0, 0, 0)))[:2] == [1, 0.25]
  assert engine.MixDraws.vector(("cutmix", 0.5, (1, 3, 2, 4))) == [2, 0.5, 1, 3, 2, 4, 0, 0]


# ------------------------------------------------------------------ references against torch
@pytest.mark.parametrize("B", [4, 5])
@pytest.mark.parametrize("draw", [("none", 1.0, (0, 0, 0, 0)), ("mixup", 0.3, (0, 0, 0, 0)),
                                  ("mixup", 0.0, (0, 0, 0, 0)), ("cutmix", 0.6, (1, 4, 0, 3)),
                                  ("cutmix", 1.0, (2, 2, 0, 5)), ("cutmix", 0.0, (0, 6, 0, 5))])
def test_mix_decode_reference_matches_torch(B, draw):
  g = torch.Generator().manual_seed(B)
  img = torch.randint(0, 256, (B, 6, 5, 3), dtype=torch.uint8, generator=g)
  mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
  out, mag = ref_mix_decode(img, 9, 3, mean, std, draw)
  m = torch.tensor([f32(v) for v in mean], dtype=torch.float64)
  si = torch.tensor([f32(1 / v) for v in std], dtype=torch.float64)
  x = (img.double() / 255 - m) * si
  mode, lam, (y0, y1, x0, x1) = draw
  if mode == "mixup":
    x = f32(lam) * x + (1 - f32(lam)) * x.flip(0)
  elif mode == "cutmix":
    x[:, y0:y1, x0:x1] = x.flip(0)[:, y0:y1, x0:x1]
  torch.testing.assert_close(out[:, :, 3:8, :3], x, rtol=1e-12, atol=1e-12)
  assert not out[:, :, :3].any() and not out[:, :, 8:].any() and not out[..., 3:].any()
  assert bool((mag >= out.abs()).all())


@pytest.mark.parametrize("V", [1, 10, 37])
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("lam", [1.0, 0.3, 0.0])
def test_mixed_xent_reference_matches_torch(V, eps, lam):
  g = torch.Generator().manual_seed(V)
  B = 7
  logits = torch.randn(B, V + 3, generator=g, dtype=torch.float64) * 3
  labels = torch.randint(0, V, (B,), generator=g, dtype=torch.int32)
  loss, grad = ref_mixed_xent(logits, labels, V, eps, lam)
  x = logits[:, :V].clone().requires_grad_(True)
  t = mixed_onehot(labels, V, eps, lam)
  want = -(t * F.log_softmax(x, 1)).sum(1)
  want.sum().backward()
  torch.testing.assert_close(loss, want.detach(), rtol=1e-12, atol=1e-12)
  torch.testing.assert_close(grad, x.grad, rtol=1e-12, atol=1e-12)
  # timm's form: lam CE(x, y) + (1 - lam) CE(x, y.flip(0)) with the smoothing of F.cross_entropy
  y = labels.long()
  timm = lam * F.cross_entropy(x.detach(), y, label_smoothing=eps, reduction="none") + \
      (1 - lam) * F.cross_entropy(x.detach(), y.flip(0), label_smoothing=eps, reduction="none")
  torch.testing.assert_close(loss, timm, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("V", [1, 7, 20])
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("lam", [1.0, 0.7, 0.2])
def test_mixed_bce_reference_matches_torch(V, eps, weighted, lam):
  g = torch.Generator().manual_seed(V + 10 * weighted)
  B = 5
  logits = torch.randn(B, V + 3, generator=g, dtype=torch.float64) * 4
  logits[0, :V] = 1e4
  y = torch.randint(0, 2, (B, V), generator=g, dtype=torch.uint8)
  y[1] *= 3                       # any nonzero byte is a positive
  pw = torch.rand(V, generator=g, dtype=torch.float64) * 3 if weighted else None
  loss, grad = ref_mixed_bce(logits, y, V, eps, lam, pw)
  x = logits[:, :V].clone().requires_grad_(True)
  t = mixed_multihot(y, V, eps, lam)
  want = F.binary_cross_entropy_with_logits(x, t, pos_weight=pw, reduction="none")
  want.sum().backward()
  assert bool(torch.isfinite(loss).all() and torch.isfinite(grad).all())
  torch.testing.assert_close(loss, want.detach(), rtol=1e-12, atol=1e-12)
  torch.testing.assert_close(grad, x.grad, rtol=1e-12, atol=1e-12)


def test_dominant_sample_rule():
  labels = torch.tensor([0, 1, 2, 3], dtype=torch.int32)
  logits = F.one_hot(labels.long(), 4).double()
  assert ref_hits(logits, labels, 4, 0.5) == 4 and ref_hits(logits, labels, 4, 0.49) == 0
  flipped = logits.flip(0)
  assert ref_hits(flipped, labels, 4, 0.3) == 4 and ref_hits(flipped, labels, 4, 0.7) == 0
  y = torch.tensor([[1, 0], [0, 1], [1, 1]], dtype=torch.uint8)
  l = torch.tensor([[1.0, -1.0], [-1.0, 1.0], [1.0, 1.0]])
  assert ref_exact_rows(l, y, 2, 1.0) == 3 and ref_exact_rows(l, y, 2, 0.0) == 1


# ------------------------------------------------------------------ binding refusals
def _C():
  from tensorflowonspark_b200 import ops
  return ops.C()


BAD_MIX = [
    (torch.zeros(8, dtype=torch.float64), "mix must be float32"),
    (torch.zeros(8, dtype=torch.int32), "mix must be float32"),
    (torch.zeros(7), "vector of 8 values"),
    (torch.zeros(9), "vector of 8 values"),
    (torch.zeros(16)[::2], "vector of 8 values"),
    (torch.zeros(8), "mix must be on the CUDA device"),
]


@pytest.mark.parametrize("mix,match", BAD_MIX)
def test_softmax_xent_refuses_bad_mix_before_the_launch(mix, match):
  a = (torch.zeros(4, 16), torch.zeros(4, dtype=torch.int32), None, torch.zeros(1), None, 10, 0.25)
  with pytest.raises(ValueError, match=match):
    _C().softmax_xent(*a, mix=mix)


def test_softmax_xent_mix_needs_fp32_logits_and_one_label_per_row():
  a = (torch.zeros(4, dtype=torch.int32), None, torch.zeros(1), None, 10, 0.25)
  with pytest.raises(ValueError, match="mix needs fp32 logits"):
    _C().softmax_xent(torch.zeros(4, 16, dtype=torch.bfloat16), *a, mix=torch.zeros(8))
  with pytest.raises(ValueError, match="one label per row"):
    _C().softmax_xent(torch.zeros(4, 16), torch.zeros(5, dtype=torch.int32), *a[1:],
                      mix=torch.zeros(8))
  with pytest.raises(RuntimeError, match="logits"):   # without mix: the old checks
    _C().softmax_xent(torch.zeros(4, 16), *a, mix=None)


@pytest.mark.parametrize("mix,match", BAD_MIX)
def test_sigmoid_bce_refuses_bad_mix_before_the_launch(mix, match):
  a = {"logits": torch.zeros(4, 16), "targets": torch.zeros(4, 10, dtype=torch.uint8),
       "dlogits": None, "loss_sum": torch.zeros(1), "correct": None, "V": 10, "scale": 0.025}
  with pytest.raises(ValueError, match=match):
    _C().sigmoid_bce(**a, mix=mix)
  with pytest.raises(RuntimeError, match="CUDA tensor"):
    _C().sigmoid_bce(**a, mix=None)


@pytest.mark.parametrize("mix,match", BAD_MIX)
def test_decode_normalize_refuses_bad_mix_before_the_launch(mix, match):
  img, out = torch.zeros(2, 4, 6, 3, dtype=torch.uint8), torch.zeros(2, 4, 8, 8,
                                                                      dtype=torch.bfloat16)
  with pytest.raises(ValueError, match=match):
    _C().decode_normalize(img, out, 1, [0.5], [0.5], mix=mix)


@pytest.mark.parametrize("ishape,oshape", [((2, 4, 6, 3), (2, 4, 8, 16)), ((2, 4, 6, 1), (2, 4, 8, 8)),
                                           ((2, 4, 6, 3), (2, 4, 8, 3))])
def test_decode_normalize_mix_needs_rgb_into_8_channels(ishape, oshape):
  img, out = torch.zeros(ishape, dtype=torch.uint8), torch.zeros(oshape, dtype=torch.bfloat16)
  with pytest.raises(ValueError, match="RGB into 8 channels"):
    _C().decode_normalize(img, out, 1, [0.5], [0.5], mix=torch.zeros(8))


def test_decode_normalize_keeps_its_positional_form():
  img, out = torch.zeros(2, 4, 6, 3, dtype=torch.uint8), torch.zeros(2, 4, 8, 8,
                                                                      dtype=torch.bfloat16)
  with pytest.raises(RuntimeError, match="CUDA tensor"):
    _C().decode_normalize(img, out, 1, [0.5], [0.5])
  with pytest.raises(RuntimeError, match="CUDA tensor"):
    _C().decode_normalize(img, out, 1, [0.5], [0.5], None)


# ------------------------------------------------------------------ ptxas
@pytest.mark.skipif(not os.path.exists(uc.NVCC), reason="nvcc not found")
def test_mix_kernels_have_no_stack_frame_or_spills(tmp_path):
  kernels = uc._ptxas("mix.cu", tmp_path)
  names = {"pair_mix_rgb8_kernel": 1, "mixed_target_xent_kernel": 2, "mixed_target_bce_kernel": 4}
  for name, n in names.items():
    assert len([k for k in kernels if name in k]) == n, (name, sorted(kernels))
  assert len(kernels) == sum(names.values()), sorted(kernels)
  bad = {k: v for k, v in kernels.items() if v != (0, 0, 0)}
  assert not bad, "stack frame / spill stores / spill loads (bytes): {}".format(bad)


def test_new_kernel_names_contain_no_existing_kernel_name():
  import re
  csrc = os.path.join(ROOT, "csrc")
  old = set()
  for f in os.listdir(csrc):
    if f.endswith((".cu", ".cuh")) and f != "mix.cu":
      with open(os.path.join(csrc, f)) as fh:
        old |= set(re.findall(r"\b(\w+_kernel)\b", fh.read()))
  for new in ("pair_mix_rgb8_kernel", "mixed_target_xent_kernel", "mixed_target_bce_kernel"):
    assert not [o for o in old if o in new], new


# ------------------------------------------------------------------ example flags
def _spark(argv):
  mod = importlib.import_module("resnet_spark")
  mod.main_fun(["resnet_spark.py", "--batch_size", "4", "--image", "64"] + argv, dry._Ctx(1))
  return dry._Trainer.made[-1]


def test_resnet_spark_mixing_flags(fake_gpu):
  args = importlib.import_module("resnet_spark").parse([])
  assert (args.mixup_alpha, args.cutmix_alpha, args.mix_prob, args.mix_switch_prob) == \
      (0.0, 0.0, 1.0, 0.5)
  net = _spark(["--train_steps", "2"])
  assert not set(MIX_KW) & set(net.kw)
  net = _spark(["--train_steps", "2", "--mixup_alpha", "0.2", "--cutmix_alpha", "1.0",
                "--mix_prob", "0.8", "--mix_switch_prob", "0.3"])
  assert [net.kw[k] for k in MIX_KW] == [0.2, 1.0, 0.8, 0.3]
  net = _spark(["--train_steps", "2", "--model", "resnet56", "--cutmix_alpha", "1.0"])
  assert net.kw["cutmix_alpha"] == 1.0 and "mixup_alpha" not in net.kw


def test_resnet_cifar_mixing_flags(fake_gpu):
  mod = importlib.import_module("resnet_cifar_main")
  args = mod.define_flags().parse_args([])
  assert (args.mixup_alpha, args.cutmix_alpha, args.mix_prob, args.mix_switch_prob) == \
      (0.0, 0.0, 1.0, 0.5)
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "2"], mod.LocalContext())
  assert not set(MIX_KW) & set(dry._Trainer.made[-1].kw)
  mod.main_fun(["x", "--use_synthetic_data", "--train_steps", "2", "--mixup_alpha", "0.2",
                "--mix_prob", "0.5"], mod.LocalContext())
  kw = dry._Trainer.made[-1].kw
  assert kw["mixup_alpha"] == 0.2 and kw["mix_prob"] == 0.5 and "cutmix_alpha" not in kw

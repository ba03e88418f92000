"""One real training step of the ResNet-50 trainer, checked layer by layer against float64 on the
values its kernels pass to one another (tools/step_conformance.py holds the recorder, the
references and the claiming rules).

The kernel suites replay each launch's signature on fresh tensors; this one checks the wiring
between launches: which buffer a launch reads, whether it writes or accumulates, which mask and
statistics it is given and what the previous step left behind.  The checked step is the third
``train_step`` of a fresh trainer: the two before it use other batches and lr > 0, so anything a
step leaves behind has had the chance to leak into it.

The mutation tests change one piece of a trainer's host-side wiring - only flags and plan choices,
or a buffer swapped for one of the same shape, so that every launch stays inside its buffers - and
require the checker to fail at the layer the change breaks.
"""
import gc
import importlib.util
import os
import time

import pytest

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location(
    "step_conformance", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                     "tools", "step_conformance.py"))
sc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(sc)

LR, MOMENTUM, WD = 0.1, 0.9, 1e-4


def _free():
  import torch
  torch.cuda.synchronize()
  gc.collect()
  torch.cuda.empty_cache()


def _resnet50(batch, image, **kw):
  from tensorflowonspark_b200.models import resnet
  return resnet.ResNetTrainer(50, batch=batch, image=image, lr=LR, momentum=MOMENTUM,
                              weight_decay=WD, **kw)


def _check_step(net, seed):
  phase = net.accum.phase()
  launches, snaps = sc.record_step(net, net.synthetic_batch(seed=seed), sc.resnet_buffers(net))
  rep, claimed = sc.check_resnet_step(net, launches, snaps, LR, MOMENTUM, WD, phase)
  return rep, claimed, launches, snaps


def _check_third_step(net, mutate=None):
  """Two steps on other batches, ``mutate(net)``, then the recorded and checked third step."""
  for seed in (1, 2):
    net.train_step(*net.synthetic_batch(seed=seed))
  if mutate is not None:
    mutate(net)
  return _check_step(net, 3)


def _report(what, rep, claimed, launches, snaps, t0):
  import torch
  print("\n{}: {} launches, {} claimed; snapshots {:.2f} GB; peak allocated {:.2f} GB; {:.1f} s"
        .format(what, len(launches), claimed, snaps.nbytes() / 1e9,
                torch.cuda.max_memory_allocated() / 1e9, time.time() - t0))
  print(rep.table())
  print(rep.layer_table())
  assert claimed == len(launches)
  assert not rep.failures, "\n".join(m for _, _, m in sorted(rep.failures)[:10])


@pytest.mark.parametrize("batch,image", [(8, 64), (16, 224)])
def test_resnet50_step_matches_float64_layer_by_layer(batch, image):
  import torch
  _free()
  torch.cuda.reset_peak_memory_stats()
  t0 = time.time()
  net = _resnet50(batch, image)
  rep, claimed, launches, snaps = _check_third_step(net)
  _report("ResNet-50 {} x {}^2".format(batch, image), rep, claimed, launches, snaps, t0)
  # every layer class of the step was compared
  assert {"conv fwd", "conv fwd stats", "bn fwd y", "bn fwd mask", "bn fwd stats", "conv dgrad",
          "conv wgrad", "bn bwd dx", "bn bwd dgamma/dbeta", "optimizer", "loss",
          "stem pool"} <= set(rep.classes)
  del net, snaps, launches
  _free()


def _forced_draw(net):
  """Drops samples in every block that can drop: [n_blocks, B] fp32."""
  import numpy as np
  s = np.ones((len(net.blocks), net.B), dtype=np.float32)
  for i, p in enumerate(net.drop_path_rates):
    if p > 0:
      for b in range(net.B):
        s[i, b] = 0.0 if (i + b) % 3 == 0 else np.float32(1.0 / (1.0 - p))
  return s


def test_resnet50_drop_path_step_matches_float64_layer_by_layer():
  """drop_path_rate=0.3 under a forced draw: the scaled bn3 apply and backward, and the unfused
  bn3 reductions of every dropping block."""
  import torch
  _free()
  torch.cuda.reset_peak_memory_stats()
  t0 = time.time()
  net = _resnet50(8, 64, drop_path_rate=0.3)
  for seed in (1, 2):
    net.train_step(*net.synthetic_batch(seed=seed))
  forced = _forced_draw(net)
  net.dropper.draw = lambda: forced.copy()
  rep, claimed, launches, snaps = _check_step(net, 3)
  _report("ResNet-50 drop path 0.3", rep, claimed, launches, snaps, t0)
  assert (net.last_drop_path == forced).all()
  assert {"bn fwd y (drop path)", "bn bwd dx (drop path)",
          "bn bwd dgamma/dbeta (drop path)"} <= set(rep.classes)
  del net, snaps, launches
  _free()


def test_resnet50_accumulation_window_matches_float64_layer_by_layer():
  """gradient_accumulation_steps=2: steps 1-2 are one window; step 3 (zeroes the gradients, no
  update) and step 4 (adds to them and updates with their mean) are both checked, each
  accumulator as (after) = (before) + this micro-batch's contribution."""
  import torch
  _free()
  torch.cuda.reset_peak_memory_stats()
  t0 = time.time()
  net = _resnet50(8, 64, gradient_accumulation_steps=2)
  for seed in (1, 2):
    net.train_step(*net.synthetic_batch(seed=seed))
  for seed, phase in ((3, (True, False)), (4, (False, True))):
    assert net.accum.phase() == phase
    rep, claimed, launches, snaps = _check_step(net, seed)
    _report("ResNet-50 accumulation, micro-step {}".format(int(phase[1])), rep, claimed,
            launches, snaps, t0)
    assert "bn bwd accumulate" in rep.classes
    assert ("optimizer" in rep.classes) == phase[1]
    del snaps, launches
  del net
  _free()


# ----------------------------------------------------------------------------- mutants
def _identity_conv1_writes(net):
  """layer1.1's conv1 data gradient writes g_x instead of accumulating mask * g_out into it."""
  from tensorflowonspark_b200.ops import igemm
  b, prev = net.blocks[1], net.blocks[0]
  conv = b.u1.conv
  red = (prev.r3, prev.u3.bn.mask, prev.u3.bn.red_g, prev.u3.bn.red_gx)
  conv.dgrad = igemm.conv_dgrad(b.g_r1, net.store.w(conv.sw), b.g_x, conv.stride, conv.pad,
                                bn_reduce=red)


def _bn3_reduction_dropped(net):
  """layer1.2's conv1 data gradient no longer accumulates layer1.1's bn3 sums, which still counts
  on them (neither fused nor run unfused)."""
  from tensorflowonspark_b200.ops import igemm
  b = net.blocks[2]
  conv = b.u1.conv
  conv.dgrad = igemm.conv_dgrad(b.g_r1, net.store.w(conv.sw), b.g_x, conv.stride, conv.pad,
                                accumulate=True, acc_mask=b.u3.bn.mask)


def _bn2_gets_bn1_mask(net):
  """layer1.1's bn2 backward is handed bn1's ReLU mask (same shape in an identity block)."""
  b = net.blocks[1]
  bn2, bn1 = b.u2.bn, b.u1.bn
  orig = bn2.backward
  bn2.backward = lambda *a, **k: orig(*a, **dict(k, mask=bn1.mask))


def _arena_not_zeroed(net):
  """The statistics arena's per-step clear covers nothing: the fused sums start from the last
  step's."""
  net.stats_arena.used = 0


def _dgrad_clobbers_a1(net):
  """layer1.1's conv3 data gradient writes over a1 (same shape) instead of g_a2: a1 is clobbered
  before conv2's weight gradient reads it."""
  from tensorflowonspark_b200.ops import igemm
  b = net.blocks[1]
  conv, bn2 = b.u3.conv, b.u2.bn
  conv.dgrad = igemm.conv_dgrad(b.g_r3, net.store.w(conv.sw), b.a1, conv.stride, conv.pad,
                                bn_reduce=(b.r2, bn2.mask, bn2.red_g, bn2.red_gx))


MUTANTS = {
    "conv3_dgrad_clobbers_a1": (_dgrad_clobbers_a1, "layer1.1.u3.conv"),
    "identity_conv1_dgrad_writes": (_identity_conv1_writes, "layer1.1.u1.conv"),
    "bn3_reduction_dropped": (_bn3_reduction_dropped, "layer1.1.u3.bn"),
    "bn2_backward_with_bn1_mask": (_bn2_gets_bn1_mask, "layer1.1.u2.bn"),
    "stats_arena_not_zeroed": (_arena_not_zeroed, "stats_arena"),
}


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_wiring_mutant_is_caught_at_its_layer(name):
  mutate, layer = MUTANTS[name]
  _free()
  net = _resnet50(8, 64)
  rep, _, _, _ = _check_third_step(net, mutate)
  failing = rep.failing_layers()
  print("\n{}: first failures {}".format(name, failing[:4]))
  assert failing, name + ": the step checker passed a miswired trainer"
  assert failing[0] == layer, "{}: first failure at {}, expected {}:\n{}".format(
      name, failing[0], layer, "\n".join(m for _, _, m in sorted(rep.failures)[:4]))
  del net
  _free()

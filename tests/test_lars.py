"""LARS optimizer, host side: the norm pass's work tables, bucket validation, the warm-up
schedule and the optimizer state round trip (no GPU needed)."""
import numpy as np
import pytest
import torch

from tensorflowonspark_b200.models import engine, resnet
from tensorflowonspark_b200.parallel import fused_optim
from tensorflowonspark_b200.parallel.fused_optim import FusedOptimizer, lars_tables

AWKWARD = (1, 7, 8, 9, 4096, 1_000_003)


def _store(sizes=AWKWARD, tail=(64, 64, 10, 3)):
  st = engine.ParamStore()
  for i, n in enumerate(sizes):
    st.register("w%d" % i, (n,), True, engine.constant(0.5))
  for i, n in enumerate(tail):
    st.register("bn%d" % i, (n,), False, engine.constant(1.0))
  st.finalize("cpu")
  return st


def _bounds(st):
  return [s["offset"] for s in st.order if s["decay"]] + [st.decay_end]


def _bucket_layouts(st):
  """Bucket lists covering [0, total): cuts only at tensor starts inside the decayed head,
  anywhere (multiples of 8) inside the tail, and buckets that span head and tail."""
  b = _bounds(st)
  n, de = st.total, st.decay_end
  mid_tail = de + ((n - de) // 3) // 8 * 8
  return [
      [(0, n, None)],
      [(0, de, "a"), (de, n, "b")],
      [(b[4], n, 0), (0, b[2], 1), (b[2], b[4], 2)],
      [(0, b[5], 0), (b[5], mid_tail, 1), (mid_tail, n, 2)],
      [(b[1], b[3], 0), (mid_tail, n, 1), (0, b[1], 2), (b[3], mid_tail, 3)],
  ]


@pytest.mark.parametrize("layout", range(5))
@pytest.mark.parametrize("world", range(1, 9))
def test_segments_cover_every_adapted_element_once(layout, world):
  st = _store()
  bounds = _bounds(st)
  buckets = _bucket_layouts(st)[layout]
  tabs = lars_tables(bounds, buckets, world, seg_len=4096)
  covered = np.zeros(st.decay_end, dtype=np.int32)
  for (b, e, _), per_rank in zip(buckets, tabs):
    assert len(per_rank) == world
    for r, tab in enumerate(per_rank):
      lo, hi = fused_optim._shard(b, e, world, r)
      assert len(tab["tseg"]) == tab["nt"] + 1 and tab["tseg"][0] == 0
      assert tab["tseg"][-1] == len(tab["seg"])
      for j in range(tab["nt"]):
        t = tab["t0"] + j
        for s0, s1 in tab["seg"][tab["tseg"][j]:tab["tseg"][j + 1]]:
          assert lo <= s0 < s1 <= hi, "segment outside the shard"
          assert bounds[t] <= s0 and s1 <= bounds[t + 1], "segment outside its tensor"
          assert s0 % 8 == 0 and s1 % 8 == 0 and s1 - s0 <= 4096
          assert s1 <= st.decay_end, "the non-adapted tail is not covered"
          covered[s0:s1] += 1
      # the tensors listed are exactly the ones the shard intersects
      inter = [t for t in range(len(bounds) - 1)
               if max(bounds[t], lo) < min(bounds[t + 1], hi, st.decay_end)]
      assert inter == list(range(tab["t0"], tab["t0"] + tab["nt"]))
  assert covered.min() == 1 and covered.max() == 1


def test_bucket_bound_inside_an_adapted_tensor_raises():
  st = _store()
  b = _bounds(st)
  cut = b[4] + 8          # inside the 4096-element tensor
  with pytest.raises(ValueError, match="inside an adapted tensor"):
    FusedOptimizer(st, opt="lars", buckets=[(0, cut, 0), (cut, st.total, 1)])
  # the same cut is fine for momentum (no per-tensor norms) and in the tail for LARS
  FusedOptimizer(st, opt="momentum", buckets=[(0, cut, 0), (cut, st.total, 1)])
  tail_cut = st.decay_end + 64
  FusedOptimizer(st, opt="lars", buckets=[(0, tail_cut, 0), (tail_cut, st.total, 1)])


def test_shard_with_too_many_tensors_raises():
  st = _store(sizes=(8,) * (fused_optim.LARS_MAX_TENSORS + 1), tail=(8,))
  with pytest.raises(ValueError, match="adapted tensors"):
    FusedOptimizer(st, opt="lars")
  # two buckets split the tensors below the limit
  half = _bounds(st)[fused_optim.LARS_MAX_TENSORS // 2]
  FusedOptimizer(st, opt="lars", buckets=[(0, half, 0), (half, st.total, 1)])


def _resnet_registrations(depth):
  """A ParamStore with ResNetTrainer's registrations (CPU), wrapped so that
  ResNetTrainer._comm_buckets can run on it."""
  st = engine.ParamStore()
  t = resnet.ResNetTrainer.__new__(resnet.ResNetTrainer)
  t.store = st
  st.register("stem.conv.w", (64, 7, 64), True, engine.constant(0.1))
  engine.BatchNorm(st, "stem.bn", 64)
  t.blocks = []
  cin = 64
  for si, nblocks in enumerate(resnet.ResNetTrainer.CFG[depth]):
    width = 64 * (2 ** si)
    for bi in range(nblocks):
      stride = 2 if (bi == 0 and si > 0) else 1
      b = resnet._Block()
      b.name = "layer{}.{}".format(si + 1, bi)
      resnet._Unit(st, b.name + ".u1", cin, width, 1, 1)
      resnet._Unit(st, b.name + ".u2", width, width, 3, stride)
      resnet._Unit(st, b.name + ".u3", width, width * 4, 1, 1, zero_gamma=True)
      if bi == 0:
        resnet._Unit(st, b.name + ".ds", cin, width * 4, 1, stride)
      t.blocks.append(b)
      cin = width * 4
  engine.Dense(st, "fc", cin, 1000, bias=True, init=engine.constant(0.0))
  st.finalize("cpu")
  return t


def test_resnet50_buckets_are_accepted():
  t = _resnet_registrations(50)
  st = t.store
  assert sum(1 for s in st.order if s["decay"]) == 54
  buckets = t._comm_buckets()
  opt = FusedOptimizer(st, opt="lars", buckets=buckets)
  assert opt.lars and len(opt._lars_args) == len(buckets)
  for world in range(1, 9):
    tabs = lars_tables(_bounds(st), buckets, world)
    assert max(tab["nt"] for per_rank in tabs for tab in per_rank) <= 54


def test_resnet152_fits_one_bucket():
  t = _resnet_registrations(152)
  bounds = _bounds(t.store)
  assert len(bounds) - 1 == 156 <= fused_optim.LARS_MAX_TENSORS
  lars_tables(bounds, [(0, t.store.total, None)], 1)


def test_poly_warmup_lr():
  f = resnet.poly_warmup_lr
  base, total, warm = 8.0, 1000, 100
  assert f(0, total, base, warm) == pytest.approx(base / warm)        # warm-up starts near 0
  assert f(warm - 1, total, base, warm) == pytest.approx(base)         # ... and ends at base
  assert f(warm, total, base, warm) == pytest.approx(base)             # decay starts at base
  mid = warm + (total - warm) // 2
  assert f(mid, total, base, warm) == pytest.approx(base * 0.25)       # (1 - 1/2) ** 2
  assert f(mid, total, base, warm, end_lr=1.0, power=1.0) == pytest.approx(1.0 + 7.0 * 0.5)
  last = f(total - 1, total, base, warm)
  assert 0.0 < last < base * 1e-4                                      # last step: nearly end_lr
  assert f(total, total, base, warm, end_lr=0.5) == pytest.approx(0.5)
  assert all(f(s + 1, total, base, warm) <= f(s, total, base, warm) for s in range(warm, total))


def test_state_dict_round_trip_keeps_trust_coefficient():
  st = _store()
  opt = FusedOptimizer(st, opt="lars", lr=0.3, trust_coefficient=0.02, weight_decay=5e-5)
  assert opt.state1 is not None and opt.state2 is None
  assert float(opt.hyper[4]) == pytest.approx(0.02)
  opt.state1.fill_(0.25)
  sd = opt.state_dict()
  other = FusedOptimizer(_store(), opt="lars")
  assert float(other.hyper[4]) == pytest.approx(0.001)
  other.load_state_dict(sd)
  assert float(other.hyper[4]) == pytest.approx(0.02)
  assert float(other.hyper[0]) == pytest.approx(0.3)
  assert torch.equal(other.state1, opt.state1)


def test_existing_optimizer_codes_unchanged():
  assert fused_optim.OPTS == {"sgd": 0, "momentum": 1, "adam": 2, "lars": 3}

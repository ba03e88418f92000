"""CPU tier of the parameter-server kernel checks (tests/test_gpu_ps_kernels.py): the host plan
that splits a row-sparse push between the sparse and dense kernels, the numpy twin of ps_apply at
unaligned ``ema_begin`` / ``decay_end``, the refusals ``PSClient`` makes before any launch, and the
registry that ties every kernel-launching entry point of the extension to a float64 test."""
import importlib.util
import itertools
import os
import re

import numpy as np
import pytest

from tensorflowonspark_b200.parallel import ps

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ----------------------------------------------------------------------- row-sparse push plan
def _coverage(numel, num_ps, base, width, rows):
  """cover[r, e]: how often the plans of all servers write flat element e for table row r."""
  cover = np.zeros((rows, numel), np.int64)
  for lo, hi in ps._slices(numel, num_ps):
    r0, r1, cuts = ps._sparse_plan(lo, hi, base, width)
    for r in range(r0, min(r1, rows)):
      s = base + r * width
      assert lo <= s and s + width <= hi, (lo, hi, r)
      cover[r, s:s + width] += 1
    seen = set()
    for r, a, b in cuts:
      assert r not in seen, ("row cut twice", lo, hi, r)
      assert not r0 <= r < r1, ("cut row also sent whole", lo, hi, r)
      seen.add(r)
      s = base + r * width
      assert lo <= a < b <= hi and s <= a and b <= s + width, (lo, hi, r, a, b)
      if r < rows:
        cover[r, a:b] += 1
  return cover


NUMELS = (1, 5, 8, 23, 40, 96, 97, 150, 200)


@pytest.mark.parametrize("numel", NUMELS)
def test_sparse_plan_covers_every_owned_element_once(numel):
  """Every element of every table row is written exactly once over all servers, whatever the slice
  layout, row width (rows wider than a slice included) and table offset."""
  for num_ps, width, base in itertools.product(range(1, 6), range(1, 51), range(8)):
    rows = (numel - base) // width
    if rows < 1:
      continue
    cover = _coverage(numel, num_ps, base, width, rows)
    want = np.zeros_like(cover)
    for r in range(rows):
      want[r, base + r * width:base + (r + 1) * width] = 1
    assert np.array_equal(cover, want), (numel, num_ps, width, base,
                                         np.argwhere(cover != want)[:4].tolist())


def _apply_plans(numel, num_ps, base, width, idx, grad_rows, lr):
  """The GPU branch of PSClient.push_sparse in float64: the plan of every server applied with the
  kernels' arithmetic (w += -lr g row by row, duplicates adding up)."""
  w = np.zeros(numel)
  for lo, hi in ps._slices(numel, num_ps):
    r0, r1, cuts = ps._sparse_plan(lo, hi, base, width)
    for k, r in enumerate(idx):
      if r0 <= r < r1:
        s = base + r * width
        w[s:s + width] -= lr * grad_rows[k]
    for r, a, b in cuts:
      s = base + r * width
      for k in np.nonzero(idx == r)[0]:
        w[a:b] -= lr * grad_rows[k][a - s:b - s]
  return w


def _local_cluster(tag, num_ps):
  from tensorflowonspark_b200 import reservation
  srv = reservation.Server(1)
  addr = srv.start()

  class Ctx(object):
    def __init__(self, job, i):
      self.job_name, self.task_index = job, i
      self.cluster_spec = {"ps": ["h:%d" % j for j in range(num_ps)], "worker": ["w:9"]}
      self.cluster_id, self.server_addr, self.gpus = tag, addr, []
  return srv, Ctx


@pytest.mark.parametrize("numel,num_ps,base,width,idx", [
    (96, 4, 3, 40, [0, 1]),               # a row wider than a slice holds the whole of one
    (96, 4, 3, 40, [1, 1, 0]),
    (200, 5, 7, 50, [0, 2, 2, 1]),
    (200, 3, 0, 1, list(range(0, 200, 7)) + [5, 5, 5]),
    (97, 2, 5, 23, [3, 0, 3, 2, 1]),
    (40, 2, 3, 5, [4, 0, 6]),
])
def test_sparse_plan_matches_the_numpy_push(numel, num_ps, base, width, idx):
  """The plan applied as the GPU branch applies it gives the shared-memory path's result, with
  duplicate indices; at the parent commit the GPU branch applied the wide row's segment twice."""
  srv, Ctx = _local_cluster("plan-%d-%d-%d-%d" % (numel, num_ps, base, width), num_ps)
  servers = [ps.PSServer(Ctx("ps", i), numel) for i in range(num_ps)]
  client = ps.PSClient(Ctx("worker", 0))
  try:
    idx = np.array(idx)
    rng = np.random.RandomState(numel + width)
    rows = (rng.randint(-64, 64, (len(idx), width)) / 8.0).astype(np.float32)   # exact sums
    client.push_sparse(rows, idx, width=width, base=base, lr=0.5)
    got = client.pull()
    want = _apply_plans(numel, num_ps, base, width, idx, rows.astype(np.float64), 0.5)
    assert np.array_equal(got.astype(np.float64), want), np.nonzero(got != want)
  finally:
    client.close()
    for s in servers:
      s.close()
    srv.stop()


def test_wide_row_case_of_the_issue():
  """numel 96 over 4 servers (slices of 24), a 40-wide table at base 3, rows 0 and 1 pushed once:
  every covered element moves by exactly -1."""
  w = _apply_plans(96, 4, 3, 40, np.array([0, 1]), np.ones((2, 40)), 1.0)
  want = np.zeros(96)
  want[3:83] = -1.0
  assert np.array_equal(w, want), np.nonzero(w != want)
  r0, r1, cuts = ps._sparse_plan(48, 72, 3, 40)       # row 1 = [43, 83) holds the whole slice
  assert r0 == r1 and cuts == [(1, 48, 72)]


# ----------------------------------------------------------------------------- apply twin
def test_apply_numpy_tail_and_decay_per_element_at_unaligned_bounds():
  """SGD by hand: numel 48, decay_end 41, ema_begin 42 - neither is a multiple of 4 or 8, so a
  kernel that decides per group of elements gets elements 40..43 wrong."""
  n, lr, wd, scale = 48, 0.5, 0.25, 2.0
  master = np.arange(n, dtype=np.float32) / 8
  g = np.full(n, 0.125, np.float32)
  hyper = np.array([lr, 0.9, wd, scale, 0.9, 0.999, 1e-7, 0.0], np.float32)
  s1, s2 = np.zeros(n, np.float32), np.zeros(n, np.float32)
  want = master.astype(np.float64).copy()
  for i in range(n):
    if i >= 42:
      want[i] -= 0.125                                       # running-statistics delta
    else:
      want[i] -= lr * (0.125 * scale + (wd * want[i] if i < 41 else 0.0))
  ps.apply_numpy(master, s1, s2, hyper, g, 0, 41, 42, 0)
  assert np.array_equal(master.astype(np.float64), want.astype(np.float32).astype(np.float64))
  assert master[40] == np.float32(5.0 - 0.5 * (0.25 + 0.25 * 5.0))   # decayed, trainable
  assert master[41] == np.float32(5.125 - 0.5 * 0.25)               # trainable, no decay
  assert master[42] == np.float32(5.25 - 0.125)                     # tail


def test_apply_numpy_momentum_state_untouched_in_the_tail_of_a_second_slice():
  n, lo = 16, 32                                             # global [32, 48), ema_begin 42
  master = np.ones(n, np.float32)
  s1 = np.full(n, 2.0, np.float32)
  hyper = np.array([1.0, 0.5, 0.0, 1.0, 0.9, 0.999, 1e-7, 0.0], np.float32)
  ps.apply_numpy(master, s1, np.zeros(n, np.float32), hyper, np.ones(n, np.float32), lo, 48, 42, 1)
  assert np.array_equal(s1[:10], np.full(10, 2.0 * 0.5 + 1.0, np.float32))
  assert np.array_equal(s1[10:], np.full(6, 2.0, np.float32))
  assert np.array_equal(master, np.r_[np.full(10, -1.0), np.zeros(6)].astype(np.float32))


# ----------------------------------------------------------------------- PSClient refusals
class _T(object):
  """Stands in for a tensor: only its length matters to the checks."""

  def __init__(self, n):
    self.n = n

  def numel(self):
    return self.n


@pytest.mark.parametrize("case,kw", [
    ("no running past total", dict(running=None)),
    ("short running", dict(running=_T(7))),
    ("no aux32", dict(aux32=None)),
    ("short aux32", dict(aux32=_T(15))),
    ("short weights", dict(weights=_T(47))),
    ("no weights", dict(weights=None)),
    ("decay_end past total", dict(decay_end=56)),
    ("total past numel", dict(total=72)),
])
def test_pull_model_refusals(case, kw):
  args = dict(numel=64, total=48, decay_end=32, weights=_T(48), aux32=_T(16), running=_T(16))
  ps._check_pull_model(**args)                  # the complete set is accepted
  args.update(kw)
  with pytest.raises(ValueError):
    ps._check_pull_model(**args)


def test_pull_model_needs_no_running_or_aux32_when_there_is_no_tail():
  ps._check_pull_model(48, 48, 48, _T(48), None, None)


@pytest.mark.parametrize("case,kw", [
    ("no running past total", dict(running=None)),
    ("short running", dict(running=_T(8))),
    ("never pulled", dict(running_pulled=None)),
    ("short gradients", dict(grads=_T(40))),
    ("total past numel", dict(total=72)),
])
def test_push_grads_refusals(case, kw):
  args = dict(numel=64, total=48, grads=_T(48), running=_T(16), running_pulled=_T(16))
  ps._check_push_grads(**args)
  args.update(kw)
  with pytest.raises(ValueError):
    ps._check_push_grads(**args)


def test_refused_push_grads_does_not_advance_the_sequence():
  """A refused push must leave the client's sequence numbers alone: the next push would otherwise
  wait for a slot the server never saw filled."""
  client = object.__new__(ps.PSClient)
  client.cuda, client.numel, client.pushes, client._running_pulled = True, 64, 3, None
  with pytest.raises(ValueError):
    client.push_grads(_T(48), None, total=48)
  assert client.pushes == 3
  with pytest.raises(ValueError):
    client.pull_model(None)


# ----------------------------------------------------------------------------- registry
# m.def entry points of csrc/binding.cpp that launch no kernel, or whose kernels the single-GPU
# suite cannot run: name -> reason
NOT_FLOAT64_CHECKED = {
    "bcast_pull": "two or more GPUs: tools/gpu_check_multi.py",
    "flag_barrier": "two or more GPUs: tools/gpu_check_multi.py",
    "bn_stats": "not launched by the package",
    "cast_f32_bf16": "not launched by the package",
    "igemm_plan_fwd": "plan builder, no kernel",
    "igemm_plan_wgrad": "plan builder, no kernel",
    "igemm_free": "frees a plan",
    "igemm_info": "plan description",
    "igemm_set_reverse": "setter",
    "bn_set_row_reverse": "setter",
    "set_flag_timeout_ms": "setter",
    "multilabel_eval_slots": "scratch sizer",
    "seg_eval_scratch": "scratch sizer",
    "seg_eval_slots": "scratch sizer",
    "seg_label_norm_scratch": "scratch sizer",
    "seg_dice_scratch": "scratch sizer",
    "depthwise3x3_bwd_scratch": "scratch sizer",
    "symm_alloc": "symmetric memory, no kernel",
    "symm_open": "symmetric memory, no kernel",
    "symm_close": "symmetric memory, no kernel",
    "symm_free": "symmetric memory, no kernel",
    "tensor_from_ptr": "wraps a pointer, no kernel",
    "num_sms": "device query",
}


def test_every_kernel_entry_point_has_a_float64_check():
  """Every m.def of csrc/binding.cpp is either checked against float64 by a GPU test or listed
  above with the reason it is not."""
  spec = importlib.util.spec_from_file_location(
      "kernel_conformance_suite", os.path.join(_ROOT, "tests", "test_gpu_kernel_conformance.py"))
  reg = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(reg)                  # (defines its lists without touching a GPU)
  with open(os.path.join(_ROOT, "csrc", "binding.cpp")) as f:
    defs = set(re.findall(r'm\.def\("(\w+)"', f.read()))
  assert defs, "no m.def found in csrc/binding.cpp"
  checked = set(reg.KERNEL_OPS) | set(reg._plans.K_OPS) | \
      {k.split("[")[0] for k in reg.COVERED_ELSEWHERE}
  assert not checked & set(NOT_FLOAT64_CHECKED), checked & set(NOT_FLOAT64_CHECKED)
  missing = sorted(defs - checked - set(NOT_FLOAT64_CHECKED))
  assert not missing, "entry points with neither a float64 test nor a reason: {}".format(missing)
  stale = sorted((checked | set(NOT_FLOAT64_CHECKED)) - defs)
  assert not stale, "listed entry points that csrc/binding.cpp no longer defines: {}".format(stale)
  for op, test in reg.COVERED_ELSEWHERE.items():
    fname, tname = test.split("::")
    with open(os.path.join(_ROOT, "tests", fname)) as f:
      assert re.search(r"^def {}\(".format(tname), f.read(), re.M), (op, test)

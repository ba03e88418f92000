"""GPU tier: weight averaging (``ema_decay``) fused into the gradient all-reduce + optimizer
kernels.  The kernel against the float64 recurrence of test_weight_average_host.py for sgd /
momentum / adam / lars, training bitwise unchanged by the average (eager and graph replay), the
three trainers' averaged views, averaged evaluation, export and serving, the U-Net's swap, and
checkpoints, and the exported average behind pipeline.TFModel.  The multi-rank paths are
tools/gpu_check_weight_average.py (2+ GPUs)."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_weight_average_host import ema_bound, ema_reference  # noqa: E402

SIZES = (1, 7, 8, 9, 4096, 300_003)
OPT_KW = {"sgd": dict(lr=0.05, weight_decay=1e-3), "momentum": dict(lr=0.05, weight_decay=1e-3),
          "adam": dict(lr=1e-3, weight_decay=1e-3),
          "lars": dict(lr=0.8, weight_decay=1e-3, trust_coefficient=0.02)}


@pytest.fixture(scope="module", autouse=True)
def _ext():
  from tensorflowonspark_b200 import _build
  _build.load(required=True)


def _store():
  from tensorflowonspark_b200.models import engine
  st = engine.ParamStore()
  for i, n in enumerate(SIZES):
    st.register("w%d" % i, (n,), True, engine.normal(0.05))
  for i, n in enumerate((64, 10, 3)):
    st.register("bn%d" % i, (n,), False, engine.constant(1.0))
  st.finalize(torch.device("cuda", 0), seed=5)
  return st


def _optimizer(st, opt, ema):
  """Two buckets (the overlapped launch / finish path), cut at a tensor start."""
  from tensorflowonspark_b200.parallel.fused_optim import FusedOptimizer
  cut = st.by_name["w4"]["offset"]
  return FusedOptimizer(st, opt=opt, buckets=[(cut, st.total, "late"), (0, cut, "early")],
                        ema_decay=ema, **OPT_KW[opt])


def _grads(st, steps):
  """Random gradients on every real element, 0 on the padding (as a trainer's)."""
  gen = torch.Generator().manual_seed(42)
  mask = torch.zeros(st.total)
  for s in st.order:
    mask[s["offset"]:s["offset"] + s["numel"]] = 1.0
  return [(torch.randn(st.total, generator=gen) * 0.1 * mask).cuda() for _ in range(steps)]


def _step(opt, st, g):
  opt.zero_grads()
  st.grads.copy_(g)
  opt.finish()


@pytest.mark.parametrize("d", [0.0, 0.9, 0.999])
@pytest.mark.parametrize("opt", ["sgd", "momentum", "adam", "lars"])
def test_kernel_average_matches_float64(opt, d):
  st = _store()
  o = _optimizer(st, opt, d)
  masters = []
  for k, g in enumerate(_grads(st, 20)):
    _step(o, st, g)
    torch.cuda.synchronize()
    masters.append(st.master.detach().cpu().clone())
    ema = o.ema.detach().cpu()
    if k == 0 or d == 0.0:   # update 1 copies; d = 0 keeps copying
      assert torch.equal(ema, masters[-1]), "step %d" % (k + 1)
  assert o.average_count() == 20
  ref = ema_reference(masters, d)[-1]
  err = (o.ema.detach().cpu().double() - ref).abs()
  bound = ema_bound(masters, d)
  assert bool((err <= bound).all()), float((err - bound).max())
  if d > 0:   # and the average really differs from the last master
    assert not torch.equal(o.ema.cpu(), masters[-1])


def _run(opt, ema, capture):
  st = _store()
  o = _optimizer(st, opt, ema)
  grads = _grads(st, 6)
  if capture:
    o.zero_grads()
    st.grads.copy_(grads[0])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      o.finish()
    o.reset_average()          # the capture does not run the kernels; start the count anew
    for gr in grads:
      st.grads.copy_(gr)
      g.replay()
  else:
    for gr in grads:
      _step(o, st, gr)
  torch.cuda.synchronize()
  out = [st.master, st.weights, st.aux32] + [t for t in (o.state1, o.state2) if t is not None]
  return [t.clone() for t in out], (o.ema.clone() if o.ema is not None else None), o.hyper[:8].clone()


@pytest.mark.parametrize("capture", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("opt", ["sgd", "momentum", "adam", "lars"])
def test_training_is_bitwise_unchanged_by_the_average(opt, capture):
  plain, _, h0 = _run(opt, None, capture)
  avg, ema, h1 = _run(opt, 0.9, capture)
  for a, b in zip(plain, avg):
    assert torch.equal(a, b)
  assert torch.equal(h0, h1)
  _, ema_eager, _ = _run(opt, 0.9, False)
  assert torch.equal(ema, ema_eager)          # the replayed graph keeps averaging


def test_launch_count_per_step_is_unchanged_without_the_average():
  from tensorflowonspark_b200 import ops
  counts = []
  for ema in (None, 0.9):
    st = _store()
    o = _optimizer(st, "adam", ema)
    g = _grads(st, 1)[0]
    c0 = ops.launch_count()
    _step(o, st, g)
    counts.append(ops.launch_count() - c0)
  assert counts[0] == counts[1] == 1 + 2     # zero_grads + one fused kernel per bucket


# ------------------------------------------------------------------ trainers
def _train(net, batches, steps, record):
  masters = []
  for k in range(steps):
    x, y = batches[k % len(batches)]
    net.train_step(x, y)
    if record:
      torch.cuda.synchronize()
      masters.append(net.store.master.detach().cpu().clone())
  torch.cuda.synchronize()
  return masters


def _check_view(net, masters, d):
  """averaged().state_dict() against the float64 recurrence over the per-step masters."""
  sd = net.averaged().state_dict()
  ref, bound = ema_reference(masters, d)[-1], ema_bound(masters, d)
  for s in net.store.order:
    sl = slice(s["offset"], s["offset"] + s["numel"])
    err = (sd[s["name"]].reshape(-1).double() - ref[sl]).abs()
    assert bool((err <= bound[sl]).all()), s["name"]
  assert torch.equal(sd["__running__"], net.running.tensor().cpu())
  return sd


def _resnet_batches(net, n, seed):
  return [net.synthetic_batch(seed=seed + i) for i in range(n)]


def test_resnet50_37_classes_average_eval_export_and_serving(tmp_path, monkeypatch):
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.utils import checkpoint
  d, B, V = 0.9, 8, 37
  net = resnet.ResNetTrainer(depth=50, batch=B, image=64, num_classes=V, seed=3, ema_decay=d)
  masters = _train(net, _resnet_batches(net, 2, 0), 5, True)
  sd = _check_view(net, masters, d)
  assert float(sd["fc.w"][V:].abs().max()) == 0.0 and float(sd["fc.b"][V:].abs().max()) == 0.0
  held = _resnet_batches(net, 2, 100)
  live = net.evaluate(held)
  got = net.evaluate(held, averaged=True)
  fresh = resnet.ResNetTrainer(depth=50, batch=B, image=64, num_classes=V, training=False)
  fresh.load_state_dict(sd)
  want = fresh.evaluate(held)
  assert got == want and got != live
  # the export of the average serves what a training=False trainer loading it serves
  d_exp = str(tmp_path / "export")
  checkpoint.export_model(net.averaged(), d_exp)
  monkeypatch.setenv("TFOS_SERVE_BATCH", str(B))
  model, sig = checkpoint.load_model(d_exp, "serve")
  assert isinstance(model, resnet.ServedResNet)
  assert sig["builder_args"] == {"depth": 50, "image": 64, "num_classes": V}
  x = held[0][0].cpu().numpy()
  out = model(image=x)
  ref = resnet.ServedResNet(sd, depth=50, image=64, num_classes=V, batch=B)(image=x)
  assert np.array_equal(out["logits"], ref["logits"])
  assert np.array_equal(out["prediction"], ref["prediction"])
  # and close to the averaged evaluation's own logits (bf16-folded vs fp32-folded filters)
  net.eval_begin(averaged=True)
  net.eval_step(*held[0])
  ev = net.logits[:, :V].float().cpu().numpy()
  net.eval_end()
  assert np.abs(out["logits"] - ev).max() <= 0.05 * np.abs(ev).max() + 1e-3


def test_cifar_resnet20_average_and_evaluation():
  from tensorflowonspark_b200.models import resnet
  d, B = 0.99, 32
  net = resnet.CifarResNetTrainer(depth=20, batch=B, seed=4, ema_decay=d, num_classes=10)
  batches = _resnet_batches(net, 2, 0)
  net.set_input(*batches[0])
  net.capture()                       # averaging keeps running under graph replay
  net.optim.reset_average()           # (the capture's warm-up steps updated the masters)
  masters = _train(net, batches, 6, True)
  sd = _check_view(net, masters, d)
  held = _resnet_batches(net, 2, 50)
  got = net.evaluate(held, averaged=True)
  fresh = resnet.CifarResNetTrainer(depth=20, batch=B, seed=77)
  fresh.load_state_dict(sd)
  assert got == fresh.evaluate(held)


def _same(a, b):
  """Evaluation results equal, NaN IoUs (classes absent from labels and predictions) included."""
  assert set(a) == set(b)
  for key in a:
    assert np.array_equal(np.asarray(a[key], dtype=np.float64), np.asarray(b[key], dtype=np.float64),
                          equal_nan=True), key


def _unet_batches(net, V, n, seed):
  from tensorflowonspark_b200.models import unet
  out = []
  for i in range(n):
    x, _ = net.synthetic_batch(seed=seed + i)
    out.append((x, unet.synthetic_labels(x, V)))
  return out


@pytest.mark.parametrize("k", [None, 13], ids=["frozen", "finetune13"])
def test_unet_21_classes_average_swap_eval_export(k, tmp_path, monkeypatch):
  from tensorflowonspark_b200.models import unet
  from tensorflowonspark_b200.utils import checkpoint
  d, B, V = 0.9, 4, 21
  kw = dict(batch=B, image=128, classes=V, seed=9, lr=2e-3, encoder_trainable_from=k)
  net = unet.UNetTrainer(ema_decay=d, **kw)
  batches = _unet_batches(net, V, 2, 0)
  masters = _train(net, batches, 4, True)
  sd = _check_view(net, masters, d)
  enc = dict(zip([id(c) for c in net._encoder_convs()], sd["__encoder__"]))
  assert len(net.encoder.trainable_units) == (0 if k is None else 12)
  for c in net.encoder.trainable_units:
    w, b = enc[id(c)]
    assert torch.equal(w, sd[c.sw["name"]].to(torch.bfloat16)) and torch.equal(b, sd[c.sb["name"]])
  held = _unet_batches(net, V, 2, 100)
  got = net.evaluate(held, averaged=True)
  fresh = unet.UNetTrainer(batch=B, image=128, classes=V, training=False)
  fresh.load_state_dict(sd)
  _same(got, fresh.evaluate(held))
  # train_step refuses to run on the swapped-in average
  net.eval_begin(averaged=True)
  with pytest.raises(RuntimeError, match="eval_end"):
    net.train_step(*batches[0])
  want = net.predict(held[0][0]).float().cpu().numpy()      # the average's logits
  net.eval_end()
  d_exp = str(tmp_path / "export")
  checkpoint.export_model(net.averaged(), d_exp)
  monkeypatch.setenv("TFOS_SERVE_BATCH", str(B))
  model, _ = checkpoint.load_model(d_exp, "serve")
  model.select_outputs(["mask", "logits"])
  out = model(image=held[0][0].cpu().numpy())
  assert np.array_equal(out["logits"], want)
  assert np.array_equal(out["mask"], want.argmax(-1).astype(np.uint8))


def test_unet_averaged_evaluation_leaves_the_training_state_bitwise_unchanged():
  """Everything the next (captured) step reads is bit for bit what it was before the averaged
  evaluation, so training continues as if it had not happened."""
  from tensorflowonspark_b200.models import unet
  V = 21
  net = unet.UNetTrainer(batch=4, image=128, classes=V, seed=9, ema_decay=0.9,
                         encoder_trainable_from=13)
  batches = _unet_batches(net, V, 2, 0)
  net.set_input(*batches[0])
  net.capture()
  _train(net, batches, 2, False)
  state = lambda: [t.clone() for t in (  # noqa: E731
      net.store.master, net.store.weights, net.store.aux32, net.optim.ema, net.optim.state1,
      net.optim.state2, net.optim.hyper, net.running.tensor(), net.in_u8, net.labels)]
  before = state()
  live = net.evaluate(_unet_batches(net, V, 1, 100))
  avg = net.evaluate(_unet_batches(net, V, 1, 100), averaged=True)
  torch.cuda.synchronize()
  names = ("master", "weights", "aux32", "ema", "state1", "state2", "hyper", "running", "in_u8",
           "labels")
  for name, a, b in zip(names, before, state()):
    assert torch.equal(a, b), name
  assert live["loss"] != avg["loss"]
  n = net.optim.average_count()
  _train(net, batches, 2, False)           # and the captured step still runs
  assert net.optim.average_count() == n + 2


# ------------------------------------------------------------------ checkpoints
def test_optimizer_resumed_from_a_checkpoint_ends_with_the_same_average():
  """Saved at update k, loaded into a new optimizer (and store) and continued to N: bitwise the
  average of an uninterrupted run.  (On the synthetic store, whose updates are deterministic;
  a trainer's steps are not bit-reproducible from run to run - batch-norm gradient sums use
  float atomics - so the trainer test below checks the hand-over itself.)"""
  N, k = 12, 5
  for opt in ("momentum", "adam", "lars"):
    st = _store()
    a = _optimizer(st, opt, 0.9)
    grads = _grads(st, N)
    for g in grads[:k]:
      _step(a, st, g)
    params, optim = st.state_dict(), a.state_dict()
    for g in grads[k:]:
      _step(a, st, g)
    st2 = _store()
    c = _optimizer(st2, opt, 0.9)
    st2.load_state_dict(params)
    c.load_state_dict(optim)
    assert c.average_count() == k
    for g in grads[k:]:
      _step(c, st2, g)
    torch.cuda.synchronize()
    assert torch.equal(c.ema, a.ema) and torch.equal(st2.master, st.master), opt


def test_trainer_checkpoint_carries_the_average_and_loads_reset():
  from tensorflowonspark_b200.models import resnet
  B, k, d = 32, 3, 0.9

  def make():
    return resnet.CifarResNetTrainer(depth=20, batch=B, seed=4, ema_decay=d)
  b = make()
  batches = _resnet_batches(b, 2, 0)
  _train(b, batches, k, False)
  params, optim = b.state_dict(), b.optim.state_dict()
  c = make()
  c.load_state_dict(params)
  c.optim.load_state_dict(optim)
  assert c.optim.average_count() == k and torch.equal(c.optim.ema.cpu(), optim["ema"])
  start = c.optim.ema.detach().cpu().clone()
  masters = _train(c, batches, 3, True)
  # the continued average is the recurrence started from the loaded one
  ref = start.double()
  dd = float(np.float32(d))
  for w in masters:
    ref = dd * ref + (1 - dd) * w.double()
  bound = 2.0 ** -23 * torch.stack([start.abs()] + [w.abs() for w in masters]).amax(0).double() * 3
  assert bool(((c.optim.ema.cpu().double() - ref).abs() <= bound).all())
  # a parameter-only load and load_backbone restart the average from the current parameters
  for load in (c.load_state_dict, c.load_backbone):
    load(params)                     # (load_backbone keeps the current head)
    assert c.optim.average_count() == 0
    view, cur = c.averaged().state_dict(), c.state_dict()
    for s in c.store.order:
      assert torch.equal(view[s["name"]], cur[s["name"]]), s["name"]
    c.train_step(*batches[0])
    torch.cuda.synchronize()
    assert torch.equal(c.optim.ema, c.store.master)


# ------------------------------------------------------------------ TFModel
def transform_check(out_dir):
  """The exported average of a 21-class U-Net behind pipeline.TFModel: its mask and logits cells
  are the average's logits (the trainer's predict() while an averaged evaluation has the average
  in).  Runs in a fresh process: the sparklite executor forks before this process touches CUDA."""
  sys.path.insert(0, ROOT)
  from tensorflowonspark_b200._spark import SparkConf, SparkContext, SparkSession
  from tensorflowonspark_b200.models import unet
  from tensorflowonspark_b200.pipeline import TFModel
  from tensorflowonspark_b200.sparklite.sql import BinaryType, StructField, StructType
  from tensorflowonspark_b200.utils import checkpoint
  os.environ["TFOS_SERVE_BATCH"] = "8"
  V = 21
  sc = SparkContext(conf=SparkConf().setAppName("serve_unet_average")
                    .set("spark.executor.instances", "1")
                    .set("spark.executor.resource.gpu.amount", "1")
                    .set("spark.task.resource.gpu.amount", "1"))
  spark = SparkSession(sc)
  net = unet.UNetTrainer(batch=8, image=128, classes=V, seed=31, lr=2e-3, ema_decay=0.9)
  x, _ = net.synthetic_batch(seed=3)
  for _ in range(3):
    net.train_step(x, unet.synthetic_labels(x, V))
  export = os.path.join(out_dir, "export")
  checkpoint.export_model(net.averaged(), export)
  imgs = x.cpu().numpy()
  live = net.predict(x).float().cpu().numpy()
  net.eval_begin(averaged=True)
  want = net.predict(x).float().cpu().numpy()
  net.eval_end()
  assert not np.array_equal(want, live)
  del net
  df = spark.createDataFrame(sc.parallelize([(r.tobytes(),) for r in imgs], 2),
                             StructType([StructField("image", BinaryType())]))
  rows = TFModel(argparse.Namespace(num_gpus=1)).setExportDir(export).setBatchSize(8) \
      .setInputMapping({"image": "image"}).setOutputMapping({"mask": "m", "logits": "l"}) \
      .transform(df).collect()
  sc.stop()
  masks = np.stack([np.frombuffer(r.m, dtype=np.uint8) for r in rows]).reshape(8, 128, 128)
  logits = np.stack([np.frombuffer(r.l, dtype=np.float32) for r in rows]).reshape(8, 128, 128, V)
  assert np.array_equal(logits, want)
  assert np.array_equal(masks, want.argmax(-1).astype(np.uint8))
  print("AVERAGE TRANSFORM CHECK PASSED")


def test_exported_average_behind_tfmodel(tmp_path):
  p = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, 'tests'); "
                      "import test_gpu_weight_average as t; t.transform_check({!r})".format(
                          str(tmp_path))], capture_output=True, text=True, timeout=900, cwd=ROOT)
  print(p.stdout[-3000:], p.stderr[-3000:])
  assert p.returncode == 0 and "AVERAGE TRANSFORM CHECK PASSED" in p.stdout

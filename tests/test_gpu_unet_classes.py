"""The segmentation U-Net beyond eight classes (9..256): the wide-logit kernels pixel_xent,
seg_eval_metrics and seg_predict (csrc/seg_wide.cuh) against float64, and a 21-class trainer end
to end - its logits, last-layer gradients, learning, checkpoints, serving and fine-tuning (its new
GEMM plans are replayed against float64 by tests/test_gpu_option_conformance.py)."""
import argparse
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [(9, 16), (16, 16), (21, 24), (150, 152), (256, 256)]   # (V, VP)


def _load(name, rel):
  spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, rel))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def _C():
  from tensorflowonspark_b200 import ops
  return ops.C()


def _logits(V, VP, shape, seed, nan=False):
  """bf16 logits [*shape, VP] on a coarse grid (many ties), huge values in the padding channels
  (which must never be read), and - with ``nan`` - NaN in l_0 of some pixels and in other
  channels of others."""
  g = torch.Generator().manual_seed(seed)
  l = torch.randint(-6, 7, tuple(shape) + (VP,), generator=g).float() * 0.5
  l[..., V:] = 1e4
  if nan:
    P = l[..., 0].numel()
    flat = l.view(P, VP)
    idx = torch.randperm(P, generator=g)
    flat[idx[:P // 8], 0] = float("nan")
    rows = idx[P // 8:P // 4]
    flat[rows, torch.randint(1, V, (len(rows),), generator=g)] = float("nan")
    flat[idx[P // 4:P // 4 + 5], :V] = -float("inf")   # an all -inf pixel: class 0
  return l.to(torch.bfloat16).cuda()


def _labels(V, shape, seed):
  g = torch.Generator().manual_seed(seed + 1)
  y = torch.randint(0, V, tuple(shape), generator=g, dtype=torch.int32)
  flat = y.view(-1)
  for i, v in enumerate((V - 1, V, 255, -1)):
    flat[i * 7:(i + 1) * 7] = v
  return y.cuda()


def _ref_argmax(l64, V):
  """0 when l_0 is NaN, else the lowest index of the maximum of the non-NaN l_j, j < V."""
  v = l64[:, :V].clone()
  nan0 = torch.isnan(v[:, 0])
  v[torch.isnan(v)] = -float("inf")
  am = torch.argmax(v, dim=1)   # first maximal index
  am[nan0] = 0
  return am


def _ref_terms(l64, y, V):
  """Per pixel: log-sum-exp over j < V minus l_y (l_y = 0 for a label outside [0, V)), softmax."""
  v = l64[:, :V]
  lse = torch.logsumexp(v, dim=1)
  ok = (y >= 0) & (y < V)
  ly = torch.where(ok, v.gather(1, y.clamp(0, V - 1).long()[:, None])[:, 0], torch.zeros_like(lse))
  return lse - ly, torch.softmax(v, dim=1), ok


@pytest.mark.parametrize("V,VP", CASES)
def test_pixel_xent_wide_against_float64(V, VP):
  shape = (3, 7, 11)   # 231 pixels: odd, not a multiple of any warp tile
  P = 3 * 7 * 11
  l = _logits(V, VP, shape, seed=V)
  y = _labels(V, shape, seed=V)
  d = torch.full_like(l, float("nan"))
  loss, hits = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
  scale = 1.0 / P
  _C().pixel_xent(l, y, d, loss, hits, V, scale)
  torch.cuda.synchronize()
  l64, y64 = l.double().cpu().view(P, VP), y.cpu().view(P)
  term, p, ok = _ref_terms(l64, y64, V)
  assert float(loss) == pytest.approx(float(term.sum()) * scale, rel=1e-4)
  am = _ref_argmax(l64, V)
  assert float(hits) == float((am == y64).sum())
  onehot = torch.zeros(P, V, dtype=torch.float64)
  onehot[ok, y64[ok].long()] = 1.0
  ref = (p - onehot) * scale
  got = d.double().cpu().view(P, VP)
  assert torch.equal(got[:, V:], torch.zeros(P, VP - V, dtype=torch.float64)), "padding gradient"
  assert torch.allclose(got[:, :V], ref, rtol=1e-2, atol=1e-3 * scale)
  # NaN logits: the hits follow the arg-max rule
  ln = _logits(V, VP, shape, seed=V + 1, nan=True)
  hits.zero_()
  _C().pixel_xent(ln, y, None, loss, hits, V, scale)
  torch.cuda.synchronize()
  assert float(hits) == float((_ref_argmax(ln.double().cpu().view(P, VP), V) == y64).sum())


@pytest.mark.parametrize("V,VP", CASES)
def test_seg_predict_wide_against_float64(V, VP):
  shape = (5, 13, 17)
  P = 5 * 13 * 17
  l = _logits(V, VP, shape, seed=3 * V, nan=True)
  mask = torch.full(shape, 77, dtype=torch.uint8, device="cuda")
  out = torch.full(shape + (V,), 123.0, device="cuda")
  _C().seg_predict(l, mask, out, V)
  _C().seg_predict(l, mask2 := torch.zeros_like(mask), None, V)
  torch.cuda.synchronize()
  l64 = l.double().cpu().view(P, VP)
  am = _ref_argmax(l64, V)
  assert torch.equal(mask.cpu().view(P).long(), am)
  assert torch.equal(mask2, mask)
  assert torch.allclose(out.cpu().view(P, V), l.float().cpu().view(P, VP)[:, :V], rtol=0, atol=0,
                        equal_nan=True)


def _ref_eval(l, y, n, V):
  P = l.shape[0] * int(np.prod(l.shape[1:-1]))
  ppi = P // l.shape[0]
  l64 = l.double().cpu().view(P, l.shape[-1])[:n * ppi]
  y64 = y.cpu().view(P)[:n * ppi]
  ok = (y64 >= 0) & (y64 < V)
  term, _, _ = _ref_terms(l64, y64, V)
  am = _ref_argmax(l64, V)
  cm = torch.zeros(V * V, dtype=torch.float64)
  cm.index_add_(0, (y64[ok].long() * V + am[ok]), torch.ones(int(ok.sum()), dtype=torch.float64))
  return {"count": int(ok.sum()), "correct": int((am[ok] == y64[ok]).sum()),
          "invalid": int((~ok).sum()), "loss": float(term[ok].sum()), "cm": cm}


def _eval_tensors(V, l):
  P = l.numel() // l.shape[-1]
  acc = torch.zeros(_C().seg_eval_slots(V), dtype=torch.float64, device="cuda")
  scratch = torch.zeros(_C().seg_eval_scratch(P, V), dtype=torch.float64, device="cuda")
  counter = torch.zeros(1, dtype=torch.int32, device="cuda")
  return acc, scratch, counter


@pytest.mark.parametrize("V,VP", CASES)
def test_seg_eval_metrics_wide_against_float64(V, VP):
  from tensorflowonspark_b200.models import unet
  shape = (7, 9, 23)
  l = _logits(V, VP, shape, seed=5 * V)
  y = _labels(V, shape, seed=5 * V)
  acc, scratch, counter = _eval_tensors(V, l)
  assert acc.numel() == unet.seg_eval_layout(V)[3]
  n_valid = torch.tensor([5], dtype=torch.int32, device="cuda")
  _C().seg_eval_metrics(l, y, n_valid, acc, scratch, counter, V)
  torch.cuda.synchronize()
  ref = _ref_eval(l, y, 5, V)
  a = acc.cpu()
  assert [int(a[i]) for i in range(3)] == [ref["count"], ref["correct"], ref["invalid"]]
  assert float(a[3]) == pytest.approx(ref["loss"], rel=1e-5)
  assert float(a[4]) == 0.0
  assert torch.equal(a[5:], ref["cm"])
  assert int(counter) == 0 and not scratch[:V * V].any(), "table and counter left at zero"
  # NaN logits: the confusion counts follow the arg-max rule
  ln = _logits(V, VP, shape, seed=5 * V + 1, nan=True)
  acc.zero_()
  _C().seg_eval_metrics(ln, y, n_valid, acc, scratch, counter, V)
  torch.cuda.synchronize()
  ref = _ref_eval(ln, y, 5, V)
  assert torch.equal(acc.cpu()[5:], ref["cm"])
  assert int(acc[1]) == ref["correct"]


@pytest.mark.parametrize("V,VP", [(21, 24), (256, 256)])
def test_seg_eval_metrics_wide_is_bitwise_reproducible(V, VP):
  shape = (8, 64, 64)
  l = _logits(V, VP, shape, seed=9)
  y = _labels(V, shape, seed=9)
  acc, scratch, counter = _eval_tensors(V, l)
  n_valid = torch.tensor([8], dtype=torch.int32, device="cuda")
  C = _C()
  one = torch.zeros_like(acc)
  C.seg_eval_metrics(l, y, n_valid, one, scratch, counter, V)
  # each launch adds the same totals: acc_k = acc_(k-1) + one, bit for bit (same fp64 addition)
  want = torch.zeros_like(acc)
  for _ in range(2):   # two eager launches, no host reset
    C.seg_eval_metrics(l, y, n_valid, acc, scratch, counter, V)
    want = want + one
    assert torch.equal(acc, want), "eager launches differ"
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    C.seg_eval_metrics(l, y, n_valid, acc, scratch, counter, V)
  for _ in range(2):
    g.replay()
    want = want + one
    torch.cuda.synchronize()
    assert torch.equal(acc, want), "graph replay differs from the eager launches"
  acc0 = one
  # the integer totals of one 8-image call equal those of two 4-image calls
  a4 = torch.zeros_like(acc)
  n_valid.fill_(4)
  C.seg_eval_metrics(l[:4].contiguous(), y[:4].contiguous(), n_valid, a4, scratch, counter, V)
  C.seg_eval_metrics(l[4:].contiguous(), y[4:].contiguous(), n_valid, a4, scratch, counter, V)
  torch.cuda.synchronize()
  ints = [0, 1, 2] + list(range(5, acc.numel()))
  assert torch.equal(a4[ints], acc0[ints])
  assert float(a4[3]) == pytest.approx(float(acc0[3]), rel=1e-12)


def test_wide_kernels_reject_mismatched_channels():
  C = _C()
  l = torch.zeros(2, 4, 4, 24, dtype=torch.bfloat16, device="cuda")
  mask = torch.zeros(2, 4, 4, dtype=torch.uint8, device="cuda")
  for V in (16, 8, 25, 257):
    with pytest.raises(RuntimeError):
      C.seg_predict(l, mask, None, V)


# ----------------------------------------------------------------------------- the 21-class U-Net
def _labels_of(x, V):
  from tensorflowonspark_b200.models import unet
  return unet.synthetic_labels(x, V)


def test_21_class_logits_and_last_layer_gradients():
  from tensorflowonspark_b200.models import unet
  se = _load("seg_eval_ref", os.path.join("tests", "test_gpu_seg_eval.py"))
  V, B = 21, 8
  net = unet.UNetTrainer(batch=B, image=128, classes=V, seed=3)
  assert net.VP == 24 and net.logits.shape[-1] == 24
  x, _ = net.synthetic_batch(seed=1)
  y = _labels_of(x, V)
  for _ in range(2):
    net.train_step(x, y)
  se._perturb(net, 7)
  ref = se._torch_unet(net)
  net.eval_begin()
  net.eval_step(x, y)
  err = se._rel_l2(net.logits[..., :V], ref(x))
  print("21-class eval logits vs fp32 PyTorch, relative L2: {:.4f}".format(err))
  assert err <= 4e-2
  net.eval_end()
  # the last layer's gradients of one training forward against autograd on its own input
  from tensorflowonspark_b200 import ops
  net.set_input(x, y)
  net._forward(True)
  st = net.store
  net.loss_sum.zero_()
  ops.K.pixel_xent(net.logits, net.labels, net.dlogits, net.loss_sum, net.correct, V,
                   1.0 / net.labels.numel())
  net.optim.zero_grads()
  net.p_last_wgrad.run()
  ops.K.colsum(net.dlogits, st.g(net.s_last_b))
  torch.cuda.synchronize()
  h = net.cats[-1][0].float().permute(0, 3, 1, 2)
  w = st.w(net.s_last).float().permute(0, 3, 1, 2).clone().requires_grad_(True)
  b = st.f32(net.s_last_b).clone().requires_grad_(True)
  out = F.conv_transpose2d(h, w, b, 2, 1, 1)
  out.backward(net.dlogits.float().permute(0, 3, 1, 2))
  gw = st.g(net.s_last).permute(0, 3, 1, 2)
  assert se._rel_l2(gw, w.grad) <= 1e-2
  assert se._rel_l2(st.g(net.s_last_b), b.grad) <= 1e-2
  assert not st.g(net.s_last)[..., V:].any() and not st.g(net.s_last_b)[V:].any()


def test_21_class_trainer_learns_the_synthetic_labels():
  from tensorflowonspark_b200.models import unet
  V, B = 21, 16
  net = unet.UNetTrainer(batch=B, image=128, classes=V, seed=5, lr=2e-3)
  held = []
  for i in range(2):
    hx, _ = net.synthetic_batch(seed=500 + i)
    held.append((hx, _labels_of(hx, V)))
  before = net.evaluate(held)
  xs = [net.synthetic_batch(seed=i)[0] for i in range(4)]
  net.set_input(xs[0], _labels_of(xs[0], V))
  net.train_step()
  net.capture()
  first = float(net.loss_sum)
  for i in range(300):
    x = xs[i % 4]
    net.set_input(x, _labels_of(x, V))
    loss = net.train_step()
  last = float(loss)
  after = net.evaluate(held)
  print("21 classes: loss {:.3f} -> {:.3f}, mean IoU {:.3f} -> {:.3f}".format(
      first, last, before["mean_iou"], after["mean_iou"]))
  assert last < 0.85 * first
  assert after["mean_iou"] > 1.3 * before["mean_iou"]
  assert len(after["iou"]) == V and after["count"] == 2 * B * 128 * 128


def test_21_class_checkpoint_serving_and_fine_tuning():
  from tensorflowonspark_b200.models import unet
  V, B = 21, 8
  net = unet.UNetTrainer(batch=B, image=128, classes=V, seed=9)
  x, _ = net.synthetic_batch(seed=2)
  y = _labels_of(x, V)
  for _ in range(3):
    net.train_step(x, y)
  ref = net.predict(x).clone()
  res = net.evaluate([(x, y)])
  # checkpoint round trip
  net2 = unet.UNetTrainer(batch=B, image=128, classes=V, seed=10)
  net2.load_state_dict(net.state_dict())
  assert torch.equal(net2.predict(x), ref)
  # served: the mask is exactly the prediction evaluation scores
  served = unet.build_served(net.state_dict(), image=128, classes=V, batch=B)
  assert served.logits is None, "logits buffer allocated before it is asked for"
  served.select_outputs(["mask"])
  for _ in range(2):   # eager, then captured
    out = served(image=x.cpu().numpy())
  assert served.logits is None and set(out) == {"mask"}
  mask = torch.from_numpy(out["mask"]).cuda()
  assert float((mask.int() == y).double().mean()) == pytest.approx(res["accuracy"], abs=0)
  served.select_outputs(["mask", "logits"])
  for _ in range(2):
    out = served(image=x.cpu().numpy())
  assert out["logits"].shape == (B, 128, 128, V) and out["logits"].dtype == np.float32
  assert torch.equal(torch.from_numpy(out["logits"]).cuda(), ref.float())
  assert torch.equal(torch.from_numpy(out["mask"]).cuda(), mask)
  # one fine-tuning step from block 13 on
  tuned = unet.UNetTrainer(batch=B, image=128, classes=V, seed=9, encoder_trainable_from=13)
  loss = float(tuned.train_step(x, y))
  assert np.isfinite(loss)


def transform_check(out_dir):
  """A 21-class export behind pipeline.TFModel, mask and logits cells.  Runs in a fresh process:
  the sparklite executor forks before this process touches CUDA."""
  sys.path.insert(0, ROOT)
  from tensorflowonspark_b200._spark import SparkConf, SparkContext, SparkSession
  from tensorflowonspark_b200.models import unet
  from tensorflowonspark_b200.pipeline import TFModel
  from tensorflowonspark_b200.sparklite.sql import BinaryType, StructField, StructType
  from tensorflowonspark_b200.utils import checkpoint
  os.environ["TFOS_SERVE_BATCH"] = "8"
  V = 21
  sc = SparkContext(conf=SparkConf().setAppName("serve_unet_21").set("spark.executor.instances", "1")
                    .set("spark.executor.resource.gpu.amount", "1")
                    .set("spark.task.resource.gpu.amount", "1"))
  spark = SparkSession(sc)
  net = unet.UNetTrainer(batch=8, image=128, classes=V, seed=31)
  x, _ = net.synthetic_batch(seed=3)
  net.train_step(x, unet.synthetic_labels(x, V))
  export = os.path.join(out_dir, "export")
  checkpoint.export_model(net, export)
  imgs = x.cpu().numpy()
  want = net.predict(x).float().cpu().numpy()
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
  assert np.array_equal(masks, want.argmax(-1).astype(np.uint8))   # no NaN / ties in practice
  print("TRANSFORM CHECK PASSED")


def test_21_class_export_behind_tfmodel(tmp_path):
  p = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, 'tests'); "
                      "import test_gpu_unet_classes as t; t.transform_check({!r})".format(
                          str(tmp_path))], capture_output=True, text=True, timeout=900, cwd=ROOT)
  print(p.stdout[-3000:], p.stderr[-3000:])
  assert p.returncode == 0 and "TRANSFORM CHECK PASSED" in p.stdout

"""GPU tier: serving the segmentation U-Net - the seg_predict kernel against a host reference of
the prediction rule and against evaluation, trainer -> export -> ServedUNet bitwise against the
trainer's own forward, against an fp32 PyTorch U-Net, the encoder in the exported state, the
inference-only trainer, and TFModel / the inference CLI / the inference example end to end."""
import base64
import gc
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HW = 128


def ref_predict(logits, V):
  """Host reference of the rule: strict > over channels j < V starting from channel 0."""
  l = logits.float().reshape(-1, 8).cpu().numpy()
  mx, am = l[:, 0].copy(), np.zeros(len(l), dtype=np.uint8)
  for j in range(1, V):
    up = l[:, j] > mx
    mx = np.where(up, l[:, j], mx)
    am[up] = j
  return am


def _logits_case(n, hw, V, seed):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(n, hw, hw, 8, generator=g) * 3
  x[..., V:] = 1e4                       # padded channels: never read
  flat = x.view(-1, 8)
  P = flat.shape[0]
  idx = torch.randperm(P, generator=g)
  for k, p in enumerate(idx[:400].tolist()):   # ties between two valid channels, both orders
    a, b = (k % V, (k + 1) % V) if V > 1 else (0, 0)
    top = float(flat[p, :V].max()) + 1.0
    flat[p, a] = flat[p, b] = top
  nan = float("nan")
  flat[idx[400:440], 0] = nan            # NaN in channel 0: the scan keeps channel 0
  flat[idx[440:480], V - 1] = nan        # NaN elsewhere: never picked
  flat[idx[480:500]] = nan
  return x.to(torch.bfloat16).cuda()


@pytest.mark.parametrize("V", [2, 3, 8])
def test_seg_predict_against_host_reference(V):
  from tensorflowonspark_b200 import ops
  for n, hw in ((5, 37), (3, 128)):      # 6845 pixels: not a multiple of 16, 512 or 2048
    logits = _logits_case(n, hw, V, seed=V + n)
    P = n * hw * hw
    want = ref_predict(logits, V)
    if V < 8:                            # the padded channels hold the maxima: reading them fails
      assert (ref_predict(logits, 8) != want).any()
    guard = torch.full((P + 4096,), 0xAB, dtype=torch.uint8, device="cuda")
    mask = guard[:P]
    ops.K.seg_predict(logits, mask, None, V)
    torch.cuda.synchronize()
    assert np.array_equal(mask.cpu().numpy(), want), (n, hw, V)
    assert bool((guard[P:] == 0xAB).all()), "seg_predict wrote past the mask"
    # with the fp32 logits: bit-exact widenings of channels < V, nothing past either buffer
    out_guard = torch.full((P * V + 4096,), -7.0, dtype=torch.float32, device="cuda")
    out = out_guard[:P * V]
    mask.fill_(0xCD)
    ops.K.seg_predict(logits, mask, out, V)
    torch.cuda.synchronize()
    assert np.array_equal(mask.cpu().numpy(), want)
    widened = logits.reshape(-1, 8)[:, :V].float().contiguous()
    assert torch.equal(out.view(P, V).view(torch.int32), widened.view(torch.int32))
    assert bool((out_guard[P * V:] == -7.0).all()) and bool((guard[P:] == 0xAB).all())


def test_seg_predict_is_the_prediction_evaluation_scores():
  from tensorflowonspark_b200 import ops
  B, hw, V = 6, 64, 3
  g = torch.Generator().manual_seed(1)
  logits = (torch.randn(B, hw, hw, 8, generator=g) * 3)
  logits[..., V:] = 1e4
  flat = logits.view(-1, 8)
  for p in torch.randperm(flat.shape[0], generator=g)[:300].tolist():
    flat[p, 1] = flat[p, 2] = float(flat[p, :V].max()) + 1.0
  logits = logits.to(torch.bfloat16).cuda()
  labels = torch.randint(0, V, (B, hw, hw), generator=g, dtype=torch.int32).cuda()
  mask = torch.empty(B, hw, hw, dtype=torch.uint8, device="cuda")
  ops.K.seg_predict(logits, mask, None, V)
  acc = torch.zeros(72, dtype=torch.float64, device="cuda")
  partial = torch.zeros(ops.C().seg_eval_scratch(B * hw * hw), dtype=torch.float64, device="cuda")
  counter = torch.zeros(1, dtype=torch.int32, device="cuda")
  nv = torch.tensor([B], dtype=torch.int32, device="cuda")
  ops.K.seg_eval_metrics(logits, labels, nv, acc, partial, counter, V)
  torch.cuda.synchronize()
  cm = acc[4:68].cpu().view(8, 8)
  y, m = labels.long().cpu().view(-1), mask.long().cpu().view(-1)
  mine = torch.zeros(8, 8, dtype=torch.float64)
  mine.index_put_((y, m), torch.ones(len(y), dtype=torch.float64), accumulate=True)
  assert torch.equal(cm, mine)
  for c in range(V):
    assert int(((m == y) & (y == c)).sum()) == int(cm[c, c])
  assert int(acc[1]) == int((m == y).sum())


# --------------------------------------------------------------------------- the network
def _masks(x):
  return ((x[..., 0] > 127).int() + (x[..., 1] > 200).int()).to(torch.int32)


def _perturb(net, seed):
  """Non-trivial decoder batch-norm parameters and running statistics."""
  gen = torch.Generator().manual_seed(seed)
  sd = net.state_dict()
  for k in list(sd):
    if k.endswith(".gamma"):
      sd[k] = 0.5 + 0.5 * torch.rand(sd[k].shape, generator=gen)
    elif k.endswith(".beta"):
      sd[k] = 0.1 * torch.randn(sd[k].shape, generator=gen)
  sd["__running__"] = 0.05 * torch.randn(sd["__running__"].shape, generator=gen)
  net.load_state_dict(sd)
  for up in net.ups:
    up.bn.running_var.copy_(0.5 + torch.rand(up.bn.C, generator=gen).cuda())


def _trained(B, seed=11, steps=3):
  from tensorflowonspark_b200.models import unet
  net = unet.UNetTrainer(batch=B, image=HW, classes=3, device="cuda:0", seed=seed)
  x, _ = net.synthetic_batch(seed=0)
  for _ in range(steps):
    net.train_step(x, _masks(x))
  _perturb(net, seed + 1)
  return net


def _images(n, seed):
  g = torch.Generator().manual_seed(seed)
  return torch.randint(0, 256, (n, HW, HW, 3), dtype=torch.uint8, generator=g)


def _predict(net, x):
  """The trainer's predict() logits of n <= B images (padded to its batch)."""
  n = len(x)
  pad = torch.zeros((net.B,) + tuple(x.shape[1:]), dtype=torch.uint8)
  pad[:n] = x
  return net.predict(pad.cuda())[:n].float().cpu()


def _export_and_load(net, tmp_path, monkeypatch, batch, name="export"):
  from tensorflowonspark_b200.utils import checkpoint
  d = str(tmp_path / name)
  checkpoint.export_model(net, d)
  monkeypatch.setenv("TFOS_SERVE_BATCH", str(batch))
  model, sig = checkpoint.load_model(d, "serve")
  return model, sig, d


def test_export_serves_the_trainers_forward_bitwise(tmp_path, monkeypatch):
  from tensorflowonspark_b200.models import unet
  B = 8
  net = _trained(B)
  model, sig, _ = _export_and_load(net, tmp_path, monkeypatch, B)
  assert isinstance(model, unet.ServedUNet) and model.B == B and model.net.optim is None
  assert sig["builder"] == "tensorflowonspark_b200.models.unet:build_served"
  assert sig["builder_args"] == {"image": HW, "classes": 3}
  for i, n in enumerate((B, B, B, 3)):       # eager, capture, replay, ragged tail
    x = _images(n, seed=20 + i)
    out = model(image=x.numpy())
    assert out["mask"].shape == (n, HW, HW) and out["mask"].dtype == np.uint8
    assert out["logits"].shape == (n, HW, HW, 3) and out["logits"].dtype == np.float32
    want = _predict(net, x)
    assert np.array_equal(out["logits"].view(np.int32), want.numpy().view(np.int32)), i
    full = torch.zeros(n, HW, HW, 8, dtype=torch.bfloat16)
    full[..., :3] = want.to(torch.bfloat16)
    assert np.array_equal(out["mask"].reshape(-1), ref_predict(full, 3)), i
  assert model.graph is not None
  # row cells (the TFModel path) give the same results; malformed input is refused
  x = _images(5, seed=40)
  model.submit_rows({"image": [r.numpy().tobytes() for r in x]})
  rows = model.collect()
  direct = model(image=x.numpy())
  assert np.array_equal(rows["mask"], direct["mask"]) and np.array_equal(rows["logits"], direct["logits"])
  with pytest.raises(ValueError, match="49152"):
    model.submit_rows({"image": [b"\0" * 100]})
  with pytest.raises(ValueError, match="exceeds the served batch size 8"):
    model(image=_images(B + 1, seed=1).numpy())
  with pytest.raises(ValueError, match="mask"):
    model.select_outputs(["prediction"])


def test_mask_only_selection_and_fp32_reference(tmp_path, monkeypatch):
  """Served at 16 rows per batch from a trainer at 8: the logits against an fp32 PyTorch U-Net,
  and a mask-only selection gives the same masks without the logits."""
  B = 8
  net = _trained(B, seed=13)
  model, _, _ = _export_and_load(net, tmp_path, monkeypatch, 16)
  ref = _torch_unet(net)
  x = _images(16, seed=50)
  both = model(image=x.numpy())
  want = ref(x.cuda()).cpu()
  err = float((torch.from_numpy(both["logits"]).double() - want.double()).norm() / want.double().norm())
  print("served U-Net logits vs fp32 PyTorch, relative L2:", err)
  assert err < 1e-2, err
  model.select_outputs(["mask"])
  for _ in range(3):                          # eager, capture, replay of the mask-only graph
    got = model(image=x.numpy())
    assert set(got) == {"mask"} and np.array_equal(got["mask"], both["mask"])
  model.select_outputs(["mask", "logits"])
  again = model(image=x.numpy())
  assert np.array_equal(again["logits"], both["logits"])


def test_export_carries_the_encoder(tmp_path, monkeypatch):
  from tensorflowonspark_b200.models import unet
  B = 4
  net = _trained(B, seed=17, steps=1)
  g = torch.Generator().manual_seed(3)
  for layer in net.encoder.layers:
    if hasattr(layer, "w"):
      layer.w.mul_((1.0 + 0.2 * torch.rand(layer.w.shape, generator=g)).to(layer.w))
      layer.bias.add_(0.05 * torch.randn(layer.bias.shape, generator=g).cuda())
  model, _, d = _export_and_load(net, tmp_path, monkeypatch, B)
  x = _images(B, seed=60)
  served = model(image=x.numpy())["logits"]
  assert np.array_equal(served.view(np.int32), _predict(net, x).numpy().view(np.int32))
  # a state without __encoder__ (an older checkpoint) serves the seeded encoder
  state = torch.load(os.path.join(d, "weights.pt"), weights_only=False)
  enc = state.pop("__encoder__")
  assert len(enc) == len([c for c in net.encoder.layers if not isinstance(c, unet._Residual)])
  seeded = unet.build_served(state, image=HW, classes=3, batch=B)(image=x.numpy())["logits"]
  plain = unet.UNetTrainer(batch=B, image=HW, classes=3, device="cuda:0", training=False)
  plain.load_state_dict(state)
  assert np.array_equal(seeded.view(np.int32), _predict(plain, x).numpy().view(np.int32))
  assert not np.array_equal(seeded, served)


def test_inference_only_trainer():
  from tensorflowonspark_b200.models import unet
  B = 8

  def allocated():
    gc.collect()               # earlier tests' trainers must not be freed inside a measurement
    torch.cuda.synchronize()
    return torch.cuda.memory_allocated()
  base = allocated()
  tr = unet.UNetTrainer(batch=B, image=HW, classes=3, device="cuda:0", seed=21)
  m_train = allocated() - base
  base = allocated()
  inf = unet.UNetTrainer(batch=B, image=HW, classes=3, device="cuda:0", seed=5, training=False)
  m_inf = allocated() - base
  print("UNetTrainer bytes, training / inference-only:", m_train, m_inf)
  assert inf.optim is None and inf.store.grads is None and m_inf < m_train
  assert all(up.fwd is None and up.wgrad is None and up.dgrad is None for up in inf.ups)
  x, _ = tr.synthetic_batch(seed=2)
  tr.train_step(x, _masks(x))
  _perturb(tr, 8)
  inf.load_state_dict(tr.state_dict())
  assert torch.equal(inf.predict(x).view(torch.int16), tr.predict(x).view(torch.int16))
  batches = [(x, _masks(x)), (x[:3], _masks(x[:3]))]
  a, b = inf.evaluate(batches), tr.evaluate(batches)
  assert a["count"] == b["count"] == (B + 3) * HW * HW and a["accuracy"] == b["accuracy"]
  with pytest.raises(RuntimeError, match="training=False"):
    inf.train_step(x, _masks(x))


def _torch_unet(net):
  """fp32 PyTorch U-Net from the trainer's bf16 filters, fp32 biases / scale / offset and running
  statistics: MobileNetV2 encoder (ReLU6, depthwise 3x3), decoder conv_transpose2d + batch norm +
  ReLU, concatenation, last transposed convolution."""
  from tensorflowonspark_b200.models import unet
  st = net.store
  enc = net.encoder

  def fwd(x_u8):
    with torch.no_grad():
      h = (x_u8.permute(0, 3, 1, 2).float() / 255.0 - 0.5) / 0.5
      bufs = {enc.x.data_ptr(): F.pad(h, (0, 0, 0, 0, 0, 5))}
      for layer in enc.layers:
        if isinstance(layer, unet._FrozenConv):
          w = layer.w.float().permute(0, 3, 1, 2)
          y = F.conv2d(bufs[layer.x.data_ptr()], w, layer.bias, layer.stride, layer.k // 2)
          y = y.clamp(0, 6) if layer.act == 2 else (y.clamp(min=0) if layer.act == 1 else y)
        elif isinstance(layer, unet._FrozenDepthwise):
          C = layer.w.shape[1]
          w = layer.w.float().t().reshape(C, 1, 3, 3)
          y = F.conv2d(bufs[layer.x.data_ptr()], w, layer.bias, layer.stride, 1, groups=C)
          y = y.clamp(0, 6)
        else:
          y = bufs[layer.y.data_ptr()] + bufs[layer.x.data_ptr()]
        bufs[layer.y.data_ptr()] = y
      skips = [bufs[s.data_ptr()] for s in enc.skips]
      h = skips[-1]
      for i, up in enumerate(net.ups):
        w = st.w(up.sw).float().permute(0, 3, 1, 2)
        h = F.conv_transpose2d(h, w, None, 2, 1, 1)
        h = F.batch_norm(h, up.bn.running_mean, up.bn.running_var, st.f32(up.bn.sg),
                         st.f32(up.bn.sb), False, 0.0, up.bn.eps).clamp(min=0)
        h = torch.cat([h, skips[-2 - i]], 1)
      w = st.w(net.s_last).float().permute(0, 3, 1, 2)
      out = F.conv_transpose2d(h, w, st.f32(net.s_last_b), 2, 1, 1)
      return out.permute(0, 2, 3, 1)[..., :net.classes]
  return fwd


# --------------------------------------------------------------- TFModel, the CLI, the example
def _subprocess(args, env=None, timeout=900):
  p = subprocess.run([sys.executable] + args, capture_output=True, text=True, timeout=timeout,
                     cwd=ROOT, env=dict(os.environ, **(env or {})))
  print(p.stdout[-3000:], p.stderr[-3000:])
  assert p.returncode == 0
  return p.stdout


def transform_check(out_dir):
  """Run in a fresh process: the sparklite executor forks before this process touches CUDA."""
  sys.path.insert(0, ROOT)
  from tensorflowonspark_b200._spark import SparkConf, SparkContext, SparkSession
  from tensorflowonspark_b200.pipeline import TFModel
  from tensorflowonspark_b200.sparklite.sql import BinaryType, StructField, StructType
  import argparse
  os.environ["TFOS_SERVE_BATCH"] = "8"
  sc = SparkContext(conf=SparkConf().setAppName("serve_unet").set("spark.executor.instances", "1")
                    .set("spark.executor.resource.gpu.amount", "1")
                    .set("spark.task.resource.gpu.amount", "1"))
  spark = SparkSession(sc)
  from tensorflowonspark_b200.models import unet
  from tensorflowonspark_b200.utils import checkpoint
  net = _trained(8, seed=31, steps=2)
  export = os.path.join(out_dir, "export")
  checkpoint.export_model(net, export)
  x = _images(21, seed=70).numpy()
  df = spark.createDataFrame(sc.parallelize([(r.tobytes(),) for r in x], 2),
                             StructType([StructField("image", BinaryType())]))

  def model(outputs):
    return TFModel(argparse.Namespace(num_gpus=1)).setExportDir(export).setBatchSize(8) \
        .setInputMapping({"image": "image"}).setOutputMapping(outputs)
  rows = model({"mask": "mask"}).transform(df).collect()
  assert set(rows[0].asDict()) == {"mask"}, rows[0]
  masks = np.stack([np.frombuffer(r.mask, dtype=np.uint8) for r in rows]).reshape(-1, HW, HW)
  both = model({"mask": "m", "logits": "l"}).transform(df).collect()
  logits = np.stack([np.frombuffer(r.l, dtype=np.float32) for r in both]).reshape(-1, HW, HW, 3)
  sc.stop()
  state = torch.load(os.path.join(export, "weights.pt"), weights_only=False)
  direct = unet.build_served(state, image=HW, classes=3, batch=8)
  want = {"mask": [], "logits": []}
  for i in range(0, len(x), 8):
    o = direct(image=x[i:i + 8])
    want["mask"].append(o["mask"])
    want["logits"].append(o["logits"])
  assert np.array_equal(masks, np.concatenate(want["mask"]))
  assert np.array_equal(logits, np.concatenate(want["logits"]))
  print("TRANSFORM CHECK PASSED")


def test_tfmodel_transform_binary_column(tmp_path):
  out = _subprocess(["-c", "import sys; sys.path.insert(0, 'tests'); import test_gpu_serve_unet as t; "
                     "t.transform_check({!r})".format(str(tmp_path))])
  assert "TRANSFORM CHECK PASSED" in out


def _export(tmp_path, monkeypatch, B=8):
  net = _trained(B, seed=41, steps=2)
  model, _, d = _export_and_load(net, tmp_path, monkeypatch, B)
  return model, d


def test_inference_cli_writes_base64_masks(tmp_path, monkeypatch):
  from tensorflowonspark_b200 import tfrecord
  model, export = _export(tmp_path, monkeypatch)
  x = _images(11, seed=80).numpy()
  tfr = tmp_path / "tfr"
  tfr.mkdir()
  tfrecord.write_records(str(tfr / "part-00000"),
                         [tfrecord.encode_example({"image": ("bytes", [r.tobytes()])}) for r in x])
  out = str(tmp_path / "pred")
  argv = ["--export_dir", export, "--input", str(tfr), "--schema_hint", "struct<image:binary>",
          "--input_mapping", json.dumps({"image": "image"}), "--output_mapping",
          json.dumps({"mask": "mask"}), "--output", out, "--batch_size", "8", "--cluster_size", "1"]
  # the CLI's main() on a context that gives its executor GPU 0 through the resource API: this
  # process holds the GPU, so the CLI's own "free GPU" rule would find none on a one-GPU host
  _subprocess(["-c", "import sys; sys.path.insert(0, '.'); "
               "from tensorflowonspark_b200._spark import SparkConf, SparkContext; "
               "SparkContext(conf=SparkConf().setAppName('cli').set('spark.executor.instances', '1')"
               ".set('spark.executor.resource.gpu.amount', '1').set('spark.task.resource.gpu.amount', '1')); "
               "from tensorflowonspark_b200 import inference; sys.exit(inference.main({!r}))".format(argv)],
              env={"TFOS_SERVE_BATCH": "8"})
  recs = [json.loads(line) for f in sorted(glob.glob(out + "/part-*")) for line in open(f)]
  got = np.stack([np.frombuffer(base64.b64decode(r["mask"]), dtype=np.uint8) for r in recs])
  want = np.concatenate([model(image=x[i:i + 8])["mask"] for i in range(0, len(x), 8)])
  assert len(recs) == len(x) and set(recs[0]) == {"mask"}
  assert np.array_equal(got, want.reshape(len(x), -1))


def test_segmentation_inference_example(tmp_path, monkeypatch):
  _, export = _export(tmp_path, monkeypatch)
  out = _subprocess(["examples/segmentation/segmentation_inference.py", "--export_dir", export,
                     "--num_images", "20", "--partitions", "2", "--batch_size", "8", "--output",
                     str(tmp_path / "pred")], env={"TFOS_SERVE_BATCH": "8"})
  assert "20 images, pixel accuracy" in out
  assert glob.glob(str(tmp_path / "pred" / "part-*"))

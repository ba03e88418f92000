"""Serving throughput of the segmentation U-Net on one GPU, in one process, as one JSON record.

  python tools/bench_serve_unet.py [--batches 64 256] [--image 128] [--classes 3] [--out f]

Reports, with the card's name, power limit and SM clock read in the same run:
  * seg_predict time per launch (CUDA events over --launches launches) at every batch, mask only
    and mask + fp32 logits, with the bytes it must move (16 B of bf16 logits read and 1 B of mask
    written per pixel, + 4 B per valid channel with the logits) and its share of the HBM bound
    at 3.35 TB/s.  At batch 64 the 16.8 MB of logits fit in the 50 MB L2, so that share can
    exceed what HBM alone would allow;
  * ServedUNet images/s at every batch and selection, measured the way
    bench/inference_resnet50.py probes ServedResNet: fed with row cells (staging copy + H2D +
    forward + seg_predict + read-back) and with the staging buffer left as it is (H2D + forward +
    seg_predict + read-back), alternated with the ceiling - the inference trainer's forward
    (``predict``'s path) captured as a graph and replayed on a device-resident batch;
  * ``TFModel.transform(...).collect()`` over a binary DataFrame on one executor = one GPU,
    mask only, timed on the second call (the first one loads the replica).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12   # H100 SXM5 80 GB HBM3 peak


def gpu_info():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    return out.stdout.strip().splitlines()[0]
  except Exception as e:   # pragma: no cover - depends on the host
    return "unknown ({})".format(e)


def events_ms(fn, iters):
  import torch
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(iters):
    fn()
  e1.record()
  e1.synchronize()
  return e0.elapsed_time(e1) / iters


def kernel_times(B, HW, V, launches):
  import torch
  from tensorflowonspark_b200 import ops
  P = B * HW * HW
  logits = torch.randn(B, HW, HW, 8, device="cuda").to(torch.bfloat16)
  mask = torch.empty(B, HW, HW, dtype=torch.uint8, device="cuda")
  out = torch.empty(B, HW, HW, V, dtype=torch.float32, device="cuda")
  res = {}
  for name, o in (("mask", None), ("mask+logits", out)):
    fn = lambda: ops.K.seg_predict(logits, mask, o, V)   # noqa: E731
    events_ms(fn, 50)
    ms = events_ms(fn, launches)
    nbytes = P * 16 + P + (P * V * 4 if o is not None else 0)
    res[name] = {"us": ms * 1e3, "bytes": nbytes, "hbm_share": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S,
                 "launches": launches}
  return res


def replica_rates(export_dir, B, HW, V, iters, rounds):
  """Replica images/s (rows / gpu_only, per selection) alternated with the forward-graph ceiling."""
  import numpy as np
  import torch
  from tensorflowonspark_b200.models import unet
  state = torch.load(os.path.join(export_dir, "weights.pt"), map_location="cpu", weights_only=False)
  m = unet.ServedUNet(state, image=HW, classes=V, batch=B)
  rng = np.random.RandomState(7)
  pool = [rng.randint(0, 256, size=HW * HW * 3, dtype=np.uint8).tobytes() for _ in range(32)]
  rows = [pool[i % 32] for i in range(B)]
  ceil_net = unet.UNetTrainer(batch=B, image=HW, classes=V, device="cuda:0", training=False)
  ceil_net.load_state_dict(state)
  x, _ = ceil_net.synthetic_batch(seed=1)
  ceil_net.set_input(x)
  ceil_net.predict()
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    ceil_net.predict()
  out = {}

  def probe(how, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
      if how == "rows":
        m.submit_rows({"image": rows})
      else:
        m.feeder.acquire_host()
        m.feeder.push_host()
        m._enqueue(B)
      if m.pending() > 1:
        m.collect()
    while m.pending():
      m.collect()
    torch.cuda.synchronize()
    return B * n / (time.perf_counter() - t0)

  for r in range(rounds):
    for sel in (("mask",), ("mask", "logits")):
      m.select_outputs(sel)
      for how in ("rows", "gpu_only"):
        probe(how, 4)                      # eager batch + capture of this selection, warm-up
        key = "{} {}".format("+".join(sel), how)
        out.setdefault(key, []).append(probe(how, iters))
      events_ms(g.replay, 3)
      out.setdefault("forward_graph_ceiling", []).append(B * 1e3 / events_ms(g.replay, iters))
  del m, ceil_net
  torch.cuda.empty_cache()
  return {k: {"best": max(v), "rounds": v} for k, v in out.items()}


def gen_rows(n, seed, HW):
  import numpy as np
  rng = np.random.RandomState(seed)
  pool = [rng.randint(0, 256, size=HW * HW * 3, dtype=np.uint8).tobytes() for _ in range(32)]
  return [(pool[i % 32],) for i in range(n)]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batches", type=int, nargs="+", default=[64, 256])
  ap.add_argument("--image", type=int, default=128)
  ap.add_argument("--classes", type=int, default=3)
  ap.add_argument("--launches", type=int, default=1000)
  ap.add_argument("--iters", type=int, default=20)
  ap.add_argument("--rounds", type=int, default=2)
  ap.add_argument("--transform_batches", type=int, default=20)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  HW, V = args.image, args.classes
  # the Spark executor forks before this process touches CUDA
  from tensorflowonspark_b200._spark import SparkConf, SparkContext, SparkSession
  Bt = args.batches[0]
  os.environ["TFOS_SERVE_BATCH"] = str(Bt)
  sc = SparkContext(conf=SparkConf().setAppName("bench_serve_unet").set("spark.executor.instances", "1")
                    .set("spark.executor.resource.gpu.amount", "1")
                    .set("spark.task.resource.gpu.amount", "1"))
  import torch
  if not torch.cuda.is_available():
    sys.exit("bench_serve_unet: no CUDA device")
  from tensorflowonspark_b200.models import unet
  from tensorflowonspark_b200.utils import checkpoint
  torch.cuda.set_device(0)
  info = gpu_info()
  tmp = tempfile.mkdtemp(prefix="tfos_serve_unet_")
  export_dir = os.path.join(tmp, "export")
  net = unet.UNetTrainer(batch=8, image=HW, classes=V, device="cuda:0", training=False)
  checkpoint.export_model(net, export_dir)
  del net
  rec = {"gpu (name, power limit, sm clock, max sm clock)": info, "image": HW, "classes": V,
         "seg_predict": {}, "replica_images_per_s": {}}
  for B in args.batches:
    rec["seg_predict"]["batch {}".format(B)] = kernel_times(B, HW, V, args.launches)
    rec["replica_images_per_s"]["batch {}".format(B)] = replica_rates(export_dir, B, HW, V,
                                                                      args.iters, args.rounds)

  from tensorflowonspark_b200.pipeline import TFModel
  from tensorflowonspark_b200.sparklite.sql import BinaryType, StructField, StructType
  spark = SparkSession(sc)
  n = Bt * args.transform_batches
  schema = StructType([StructField("image", BinaryType())])
  model = TFModel(argparse.Namespace(num_gpus=1)).setExportDir(export_dir).setBatchSize(Bt) \
      .setInputMapping({"image": "image"}).setOutputMapping({"mask": "mask"})
  frame = lambda k: spark.createDataFrame(sc.parallelize([0], 1).flatMap(   # noqa: E731
      lambda _: gen_rows(k, 3, HW)), schema)
  model.transform(frame(Bt * 4)).collect()
  t0 = time.perf_counter()
  rows = model.transform(frame(n)).collect()
  dt = time.perf_counter() - t0
  assert len(rows) == n and len(rows[0].mask) == HW * HW
  sc.stop()
  rec["tfmodel_transform_collect"] = {"images_per_s": n / dt, "images": n, "batch": Bt,
                                      "outputs": ["mask"], "executors": 1,
                                      "note": "second transform(...).collect(), wall clock"}
  rec["gpu_after"] = gpu_info()
  print(json.dumps(rec))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
      json.dump(rec, f, indent=1)


if __name__ == "__main__":
  main()

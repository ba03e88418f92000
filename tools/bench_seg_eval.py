"""Held-out evaluation throughput of the segmentation U-Net training trainer on one GPU.

  python tools/bench_seg_eval.py [--batch 64] [--image 128] [--classes 3] [--iters 20] [--out f]

Reports, with the card's name, power limit and SM clock read in the same run:
  * seg_eval_metrics time per launch and its share of the HBM bound for the bytes it must read
    (8 bf16 logits + one int32 label per pixel), at 3.35 TB/s;
  * eval images/s: the captured eval_step graph replayed on device-resident batches (device events
    after warm-up), timed alternately with ``predict()``'s forward captured as a graph - the
    same inference network without the metric;
  * the same through ``evaluate()`` from host (numpy, uint8 masks) batches, end to end.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM5 80 GB HBM3 peak


def gpu_info():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    return out.stdout.strip().splitlines()[0]
  except Exception as e:   # pragma: no cover - depends on the host
    return "unknown ({})".format(e)


def events_ms(fn, iters):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(iters):
    fn()
  e1.record()
  e1.synchronize()
  return e0.elapsed_time(e1) / iters


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, default=64)
  ap.add_argument("--image", type=int, default=128)
  ap.add_argument("--classes", type=int, default=3)
  ap.add_argument("--iters", type=int, default=20)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit("bench_seg_eval: no CUDA device")
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.models import unet
  torch.cuda.set_device(0)
  B, HW = args.batch, args.image
  net = unet.UNetTrainer(batch=B, image=HW, classes=args.classes, device="cuda:0")
  x, y = net.synthetic_batch(seed=0)
  net.train_step(x, y)
  net.capture()
  for _ in range(3):
    net.train_step()

  ex, ey = net.synthetic_batch(seed=1)
  net.eval_begin()
  for _ in range(3):            # eager, capture, replay
    net.eval_step(ex, ey)
  ev = net._evaluator
  torch.cuda.synchronize()
  pg = torch.cuda.CUDAGraph()   # predict()'s forward (in_u8 holds the training batch)
  net.predict()
  torch.cuda.synchronize()
  with torch.cuda.graph(pg):
    net.predict()
  rates = {"eval_replay": [], "predict": []}
  for _ in range(args.rounds):  # alternate the two in one process
    rates["eval_replay"].append(B * 1e3 / events_ms(ev.graph.replay, args.iters))
    rates["predict"].append(B * 1e3 / events_ms(pg.replay, args.iters))
  net.eval_end()

  acc0 = ev.acc.clone()
  metric_ms = events_ms(lambda: ops.K.seg_eval_metrics(net.logits, ev.labels, ev.n_valid, ev.acc,
                                                       ev.partial, ev.counter, net.classes),
                        args.iters * 10)
  ev.acc.copy_(acc0)
  nbytes = net.logits.numel() * 2 + ev.labels.numel() * 4

  host = [(ex.cpu().numpy(), ey.to(torch.uint8).cpu().numpy()) for _ in range(4)]
  net.evaluate(host[:2])
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  res = net.evaluate(host * 4)
  e2e = 16 * B / (time.perf_counter() - t0)

  out = {"gpu": gpu_info(), "batch": B, "image": HW, "classes": net.classes,
         "seg_eval_metrics_us": metric_ms * 1e3, "seg_eval_metrics_bytes": nbytes,
         "seg_eval_metrics_hbm_share": nbytes / (metric_ms * 1e-3) / HBM_BYTES_PER_S,
         "eval_images_per_s": max(rates["eval_replay"]),
         "eval_images_per_s_rounds": rates["eval_replay"],
         "predict_images_per_s": max(rates["predict"]),
         "predict_images_per_s_rounds": rates["predict"],
         "evaluate_host_e2e_images_per_s": e2e,
         "eval_pixels": res["count"], "eval_images": res["images"]}
  print(json.dumps(out))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
      json.dump(out, f, indent=1)


if __name__ == "__main__":
  main()

"""Cost of the segmentation U-Net's class count on one GPU, at V = 3, 21 and 150 classes.

  python tools/bench_unet_classes.py [--batch 64] [--image 128] [--steps 50] [--out f]

Prints one JSON document with the card's name, power limit and SM clock read in the same run:
  * the captured training step: milliseconds per step from device events over ``--steps``
    graph replays after warm-up;
  * the per-pixel kernels on the trainer's logits [B, H, W, VP] (the wide kernels above 8
    classes): pixel_xent, seg_eval_metrics, seg_predict mask only and mask + fp32 logits, time
    per launch over 50 launches, the bytes the algorithm needs (computed from the shapes below,
    each tensor once) and that traffic as a share of the 3.35 TB/s data-sheet HBM figure;
  * evaluation images/s (``UNetTrainer.evaluate`` over device batches, captured after the first);
  * mask-only serving images/s (``ServedUNet``, host uint8 images in, masks out).
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from bench_unet_finetune import HBM_BYTES_PER_S, events_ms, gpu_info  # noqa: E402


def kernel_bytes(P, V, VP):
  """Bytes each kernel must move at least: bf16 logits / dlogits [P, VP], int32 labels, uint8
  mask, fp32 compact logits [P, V]."""
  logits = 2 * P * VP
  return {"pixel_xent": logits + 4 * P + logits,
          "seg_eval_metrics": logits + 4 * P,
          "seg_predict_mask": logits + P,
          "seg_predict_mask_logits": logits + P + 4 * P * V}


def bench_classes(V, args):
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.models import unet
  B, H = args.batch, args.image
  net = unet.UNetTrainer(batch=B, image=H, classes=V, device="cuda:0")
  x, _ = net.synthetic_batch(seed=0)
  y = unet.synthetic_labels(x, V)
  net.set_input(x, y)
  net.train_step()
  net.capture()
  for _ in range(5):
    net.train_step()
  step_ms = events_ms(net.train_step, args.steps)
  rec = {"classes": V, "padded": net.VP, "step_ms": round(step_ms, 3)}

  P = net.labels.numel()
  C = ops.C()
  dev = net.device
  loss = torch.zeros(1, device=dev)
  hits = torch.zeros(1, device=dev)
  acc = torch.zeros(C.seg_eval_slots(V), dtype=torch.float64, device=dev)
  scratch = torch.zeros(C.seg_eval_scratch(P, V), dtype=torch.float64, device=dev)
  counter = torch.zeros(1, dtype=torch.int32, device=dev)
  n_valid = torch.tensor([B], dtype=torch.int32, device=dev)
  mask = torch.zeros(net.labels.shape, dtype=torch.uint8, device=dev)
  out = torch.zeros(net.labels.shape + (V,), dtype=torch.float32, device=dev)
  calls = {
      "pixel_xent": lambda: C.pixel_xent(net.logits, net.labels, net.dlogits, loss, hits, V,
                                         1.0 / P),
      "seg_eval_metrics": lambda: C.seg_eval_metrics(net.logits, net.labels, n_valid, acc, scratch,
                                                     counter, V),
      "seg_predict_mask": lambda: C.seg_predict(net.logits, mask, None, V),
      "seg_predict_mask_logits": lambda: C.seg_predict(net.logits, mask, out, V),
  }
  nbytes = kernel_bytes(P, V, net.VP)
  kern = {}
  for name, fn in calls.items():
    for _ in range(5):
      fn()
    ms = events_ms(fn, 50)
    kern[name] = {"us": round(1e3 * ms, 2), "bytes": nbytes[name],
                  "hbm_share": round(nbytes[name] / (ms * 1e-3) / HBM_BYTES_PER_S, 3)}
  rec["kernels"] = kern
  del out, scratch

  batches = []
  for i in range(4):
    ex, _ = net.synthetic_batch(seed=100 + i)
    batches.append((ex, unet.synthetic_labels(ex, V)))
  net.evaluate(batches)   # eager + capture
  torch.cuda.synchronize()
  t0 = time.time()
  reps = 5
  for _ in range(reps):
    net.evaluate(batches)
  torch.cuda.synchronize()
  rec["eval_images_per_s"] = round(reps * len(batches) * B / (time.time() - t0), 1)

  state = net.state_dict()
  del net, batches
  torch.cuda.empty_cache()
  served = unet.ServedUNet(state, image=H, classes=V, batch=B)
  served.select_outputs(["mask"])
  imgs = [torch.randint(0, 256, (B, H, H, 3), dtype=torch.uint8).numpy() for _ in range(4)]
  for i in range(3):
    served(image=imgs[i % 4])
  n = 40
  t0 = time.time()
  served.submit(imgs[0])
  for i in range(1, n):
    served.submit(imgs[i % 4])
    served.collect()
  served.collect()
  rec["serve_mask_images_per_s"] = round(n * B / (time.time() - t0), 1)
  del served
  torch.cuda.empty_cache()
  return rec


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--batch", type=int, default=64)
  p.add_argument("--image", type=int, default=128)
  p.add_argument("--steps", type=int, default=50)
  p.add_argument("--classes", type=int, nargs="+", default=[3, 21, 150])
  p.add_argument("--out", default=None)
  args = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_unet_classes needs a GPU")
  torch.cuda.set_device(0)
  doc = {"gpu": gpu_info(), "batch": args.batch, "image": args.image,
         "results": [bench_classes(V, args) for V in args.classes]}
  doc["gpu_after"] = gpu_info()
  text = json.dumps(doc, indent=1)
  print(text)
  if args.out:
    with open(args.out, "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()

"""Cost of the segmentation U-Net's loss options (``ignore_index`` + ``class_weights``) on one GPU,
at V = 3, 21 and 150 classes.

  python tools/bench_seg_loss.py [--batch 64] [--image 128] [--steps 50] [--rounds 5] [--out f]

Prints one JSON document with the card's name, power limit and SM clock read in the same run:
  * the captured training step, milliseconds per step from device events over ``--steps`` graph
    replays, a default trainer and one with ignore_index=255 and class weights alternated for
    ``--rounds`` rounds (median and all rounds);
  * the label pre-pass seg_label_norm and pixel_xent (default and optioned) on the trainer's
    logits, time per launch over 50 launches, the bytes the algorithm needs (int32 labels once;
    bf16 logits read and dlogits written once) and that traffic as a share of the 3.35 TB/s
    data-sheet HBM figure.
Both trainers see the same images and masks: synthetic labels with a void band (255) over an
eighth of the rows, which the default trainer trains towards no class.
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from bench_unet_finetune import HBM_BYTES_PER_S, events_ms, gpu_info  # noqa: E402


def kernel_bytes(P, VP):
  logits = 2 * P * VP
  return {"seg_label_norm": 4 * P, "pixel_xent": logits + 4 * P + logits,
          "pixel_xent_options": logits + 4 * P + logits}


def bench_classes(V, args):
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.models import unet
  B, H = args.batch, args.image
  weights = [1.0 + (c % 5) * 0.25 for c in range(V)]
  nets = {"default": unet.UNetTrainer(batch=B, image=H, classes=V, device="cuda:0"),
          "options": unet.UNetTrainer(batch=B, image=H, classes=V, device="cuda:0",
                                      ignore_index=255, class_weights=weights)}
  x, _ = nets["default"].synthetic_batch(seed=0)
  y = unet.synthetic_labels(x, V)
  y[:, :H // 8] = 255
  for net in nets.values():
    net.set_input(x, y)
    net.train_step()
    net.capture()
    for _ in range(5):
      net.train_step()
  rounds = {k: [] for k in nets}
  for _ in range(args.rounds):
    for k, net in nets.items():
      rounds[k].append(round(events_ms(net.train_step, args.steps), 4))
  rec = {"classes": V, "padded": nets["default"].VP,
         "step_ms": {k: statistics.median(v) for k, v in rounds.items()}, "step_ms_rounds": rounds}

  net = nets["options"]
  P = net.labels.numel()
  C = ops.C()
  dev = net.device
  loss = torch.zeros(1, device=dev)
  hits = torch.zeros(1, device=dev)
  norm = torch.zeros(3, dtype=torch.float64, device=dev)
  scratch = torch.zeros(C.seg_label_norm_scratch(V), dtype=torch.int64, device=dev)
  C.seg_label_norm(net.labels, norm, scratch, V, 255, net.weights)
  calls = {
      "seg_label_norm": lambda: C.seg_label_norm(net.labels, norm, scratch, V, 255, net.weights),
      "pixel_xent": lambda: C.pixel_xent(net.logits, net.labels, net.dlogits, loss, hits, V,
                                         1.0 / P),
      "pixel_xent_options": lambda: C.pixel_xent(net.logits, net.labels, net.dlogits, loss, hits,
                                                 V, 1.0, 255, net.weights, norm),
  }
  nbytes = kernel_bytes(P, net.VP)
  kern = {}
  for name, fn in calls.items():
    for _ in range(5):
      fn()
    ms = events_ms(fn, 50)
    kern[name] = {"us": round(1e3 * ms, 2), "bytes": nbytes[name],
                  "hbm_share": round(nbytes[name] / (ms * 1e-3) / HBM_BYTES_PER_S, 3)}
  rec["kernels"] = kern
  del nets, net
  torch.cuda.empty_cache()
  return rec


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--batch", type=int, default=64)
  p.add_argument("--image", type=int, default=128)
  p.add_argument("--steps", type=int, default=50)
  p.add_argument("--rounds", type=int, default=5)
  p.add_argument("--classes", type=int, nargs="+", default=[3, 21, 150])
  p.add_argument("--out", default=None)
  args = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_seg_loss needs a GPU")
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

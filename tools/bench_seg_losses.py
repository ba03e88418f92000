"""Cost of the segmentation U-Net's focal and Dice losses on one GPU, at V = 3, 21 and 150 classes.

  python tools/bench_seg_losses.py [--batch 64] [--image 128] [--steps 50] [--rounds 3] [--out f]

Prints one JSON document with the card's name, power limit and SM clock read in the same run:
  * per launch, on the logits of a trained step (ignore_index=255 and class weights): pixel_xent,
    seg_dice_stats and seg_loss_grad for focal, dice and dice_ce; microseconds from device events
    over 100 launches after 10 warm-up launches, the bytes each needs (bf16 logits read once,
    int32 labels read once, dlogits written once by the gradient kernels) and that traffic over
    the kernel time as a rate and as a share of the 3.35 TB/s data-sheet HBM figure;
  * the captured training step for each loss, milliseconds per step from device events over
    ``--steps`` graph replays, the losses alternated for ``--rounds`` rounds (median and all).
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

LOSSES = ("cross_entropy", "focal", "dice", "dice_ce")


def kernel_bytes(P, VP):
  logits, labels = 2 * P * VP, 4 * P
  grad = logits + labels + logits
  return {"pixel_xent": grad, "seg_dice_stats": logits + labels, "seg_loss_grad_focal": grad,
          "seg_loss_grad_dice": grad, "seg_loss_grad_dice_ce": grad}


def bench_kernels(V, args):
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.models import unet
  B, H = args.batch, args.image
  weights = [1.0 + (c % 5) * 0.25 for c in range(V)]
  net = unet.UNetTrainer(batch=B, image=H, classes=V, device="cuda:0", ignore_index=255,
                         class_weights=weights, loss="dice_ce")
  x, _ = net.synthetic_batch(seed=0)
  y = unet.synthetic_labels(x, V)
  y[:, :H // 8] = 255
  net.train_step(x, y)
  torch.cuda.synchronize()
  C, P, dev = ops.C(), net.labels.numel(), net.device
  loss, hits = torch.zeros(1, device=dev), torch.zeros(1, device=dev)
  lg, lb, d, w, norm, coef = net.logits, net.labels, net.dlogits, net.weights, net.loss_norm, \
      net.dice_coef
  calls = {
      "pixel_xent": lambda: C.pixel_xent(lg, lb, d, loss, hits, V, 1.0, 255, w, norm),
      "seg_dice_stats": lambda: C.seg_dice_stats(lg, lb, coef, loss, net._dice_scratch, V, 1e-5,
                                                 255, w),
      "seg_loss_grad_focal": lambda: C.seg_loss_grad(lg, lb, d, loss, hits, V, 1.0, 255, w, norm,
                                                     focal_gamma=2.0),
      "seg_loss_grad_dice": lambda: C.seg_loss_grad(lg, lb, d, loss, hits, V, 1.0, 255, w, norm,
                                                    cross_entropy=False, dice_coef=coef),
      "seg_loss_grad_dice_ce": lambda: C.seg_loss_grad(lg, lb, d, loss, hits, V, 1.0, 255, w,
                                                       norm, dice_coef=coef),
  }
  nbytes = kernel_bytes(P, net.VP)
  rows = {}
  for name, fn in calls.items():
    for _ in range(10):
      fn()
    ms = events_ms(fn, 100)
    rate = nbytes[name] / (ms * 1e-3)
    rows[name] = {"us": round(1e3 * ms, 2), "bytes": nbytes[name], "GB_per_s": round(rate / 1e9, 1),
                  "hbm_share": round(rate / HBM_BYTES_PER_S, 3)}
  del net
  torch.cuda.empty_cache()
  return rows


def bench_steps(V, args):
  from tensorflowonspark_b200.models import unet
  B, H = args.batch, args.image
  nets = {}
  for loss in LOSSES:
    nets[loss] = unet.UNetTrainer(batch=B, image=H, classes=V, device="cuda:0", loss=loss)
  x, _ = nets["cross_entropy"].synthetic_batch(seed=0)
  y = unet.synthetic_labels(x, V)
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
  del nets
  torch.cuda.empty_cache()
  return {"step_ms": {k: statistics.median(v) for k, v in rounds.items()}, "step_ms_rounds": rounds}


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--batch", type=int, default=64)
  p.add_argument("--image", type=int, default=128)
  p.add_argument("--steps", type=int, default=50)
  p.add_argument("--rounds", type=int, default=3)
  p.add_argument("--classes", type=int, nargs="+", default=[3, 21, 150])
  p.add_argument("--out", default=None)
  args = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_seg_losses needs a GPU")
  torch.cuda.set_device(0)
  doc = {"gpu": gpu_info(), "batch": args.batch, "image": args.image, "results": []}
  for V in args.classes:
    rec = {"classes": V, "kernels": bench_kernels(V, args)}
    rec.update(bench_steps(V, args))
    doc["results"].append(rec)
  doc["gpu_after"] = gpu_info()
  text = json.dumps(doc, indent=1)
  print(text)
  if args.out:
    with open(args.out, "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()

"""Cost of the weight average (``ema_decay``) on one GPU: the captured training step of the
ResNet-50 trainer (batch 256, 224 x 224, momentum) and of the U-Net trainer (batch 64, 128 x 128,
Adam), each built with and without ``ema_decay=0.999``.

  python tools/bench_weight_average.py [--batch 256] [--unet_batch 64] [--steps 20] [--rounds 5]
                                       [--out f]

The two configurations of a model live in one process and are alternated for ``--rounds`` rounds;
each round times ``--steps`` graph replays with device events.  Prints one JSON document with the
card's name, power limit and SM clock read in the same run, ms/step (median and every round) and
the overhead of averaging in percent.
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from bench_unet_finetune import events_ms, gpu_info  # noqa: E402

DECAY = 0.999


def _alternate(nets, args):
  rounds = {k: [] for k in nets}
  for _ in range(args.rounds):
    for k, net in nets.items():
      rounds[k].append(round(events_ms(net.train_step, args.steps), 3))
  med = {k: statistics.median(v) for k, v in rounds.items()}
  return {"step_ms": med, "step_ms_rounds": rounds,
          "overhead_pct": round(100.0 * (med["ema"] / med["plain"] - 1.0), 3)}


def _warm(net):
  net.set_input(*net.synthetic_batch(seed=0))
  net.train_step()
  net.capture()
  for _ in range(3):
    net.train_step()
  return net


def bench_resnet(args):
  from tensorflowonspark_b200.models import resnet
  nets = {k: _warm(resnet.ResNetTrainer(depth=50, batch=args.batch, image=224, device="cuda:0",
                                        ema_decay=d))
          for k, d in (("plain", None), ("ema", DECAY))}
  out = _alternate(nets, args)
  del nets
  torch.cuda.synchronize()
  torch.cuda.empty_cache()
  return out


def bench_unet(args):
  from tensorflowonspark_b200.models import unet
  nets = {}
  for k, d in (("plain", None), ("ema", DECAY)):
    net = unet.UNetTrainer(batch=args.unet_batch, image=128, classes=3, device="cuda:0",
                           ema_decay=d)
    x, _ = net.synthetic_batch(seed=0)
    net.set_input(x, unet.synthetic_labels(x, 3))
    net.train_step()
    net.capture()
    nets[k] = net
  out = _alternate(nets, args)
  del nets
  torch.cuda.synchronize()
  torch.cuda.empty_cache()
  return out


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--batch", type=int, default=256)
  p.add_argument("--unet_batch", type=int, default=64)
  p.add_argument("--steps", type=int, default=20)
  p.add_argument("--rounds", type=int, default=5)
  p.add_argument("--out", default=None)
  args = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_weight_average needs a GPU")
  torch.cuda.set_device(0)
  doc = {"gpu": gpu_info(), "decay": DECAY, "resnet50_batch": args.batch,
         "unet_batch": args.unet_batch}
  doc["resnet50"] = bench_resnet(args)
  print(json.dumps(doc["resnet50"]), flush=True)
  doc["unet"] = bench_unet(args)
  doc["gpu_after"] = gpu_info()
  text = json.dumps(doc, indent=1)
  print(text)
  if args.out:
    with open(args.out, "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()

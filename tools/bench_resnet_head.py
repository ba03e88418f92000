"""Cost of the ResNet classifier options on one GPU: label smoothing and a head padded to a multiple
of 8 classes.

  python tools/bench_resnet_head.py [--batch 256] [--image 224] [--steps 20] [--rounds 3] [--out f]

Prints one JSON document with the card's name, power limit and SM clock read in the same run:
  * softmax_xent at B = 256 and V = 1000 / 1001 (ld 1000 / 1008), with and without smoothing
    (eps 0.1): time per launch from device events over 200 launches, the bytes the algorithm needs
    (fp32 logits read once, int32 labels, bf16 dlogits written once) and that traffic as a share
    of the 3.35 TB/s data-sheet HBM figure;
  * the captured ResNet-50 training step at num_classes 1000 / 1001 and eps 0 / 0.1, milliseconds
    per step from device events over ``--steps`` graph replays, the four trainers alternated for
    ``--rounds`` rounds (median and all rounds).
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

CASES = [(1000, 0.0), (1000, 0.1), (1001, 0.0), (1001, 0.1)]


def bench_kernel(B):
  from tensorflowonspark_b200 import ops
  C = ops.C()
  out = {}
  for V, eps in CASES:
    VP = (V + 7) // 8 * 8
    g = torch.Generator(device="cuda").manual_seed(V)
    logits = torch.randn(B, VP, device="cuda", generator=g) * 3
    labels = torch.randint(0, V, (B,), dtype=torch.int32, device="cuda", generator=g)
    dl = torch.zeros(B, VP, dtype=torch.bfloat16, device="cuda")
    loss, hits = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")

    def fn():
      C.softmax_xent(logits, labels, dl, loss, hits, V, 1.0 / B, label_smoothing=eps)
    for _ in range(10):
      fn()
    ms = events_ms(fn, 200)
    nbytes = 4 * B * V + 4 * B + 2 * B * VP
    out["V{}_eps{}".format(V, eps)] = {"us": round(1e3 * ms, 2), "bytes": nbytes,
                                       "hbm_share": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3)}
  return out


def bench_steps(args):
  """Two trainers at a time (eps 0 and 0.1 of one class count), alternated: four ResNet-50
  trainers at batch 256 do not fit in 80 GB together."""
  from tensorflowonspark_b200.models import resnet
  rounds = {}
  for V in sorted({V for V, _ in CASES}):
    nets = {}
    for eps in sorted({e for v, e in CASES if v == V}):
      net = resnet.ResNetTrainer(depth=50, batch=args.batch, image=args.image, num_classes=V,
                                 device="cuda:0", label_smoothing=eps)
      net.set_input(*net.synthetic_batch(seed=0))
      net.train_step()
      net.capture()
      for _ in range(3):
        net.train_step()
      nets["V{}_eps{}".format(V, eps)] = net
      rounds["V{}_eps{}".format(V, eps)] = []
    for _ in range(args.rounds):
      for k, net in nets.items():
        rounds[k].append(round(events_ms(net.train_step, args.steps), 3))
    del nets, net
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
  return {"step_ms": {k: statistics.median(v) for k, v in rounds.items()},
          "step_ms_rounds": rounds}


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--batch", type=int, default=256)
  p.add_argument("--image", type=int, default=224)
  p.add_argument("--steps", type=int, default=20)
  p.add_argument("--rounds", type=int, default=3)
  p.add_argument("--out", default=None)
  args = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_resnet_head needs a GPU")
  torch.cuda.set_device(0)
  doc = {"gpu": gpu_info(), "batch": args.batch, "image": args.image,
         "softmax_xent": bench_kernel(args.batch)}
  print(json.dumps(doc["softmax_xent"]), flush=True)
  doc.update(bench_steps(args))
  doc["gpu_after"] = gpu_info()
  text = json.dumps(doc, indent=1)
  print(text)
  if args.out:
    with open(args.out, "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()

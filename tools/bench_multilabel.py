"""Cost of the multi-label head on one GPU: its loss and evaluation kernels next to the softmax
ones, and the captured ResNet-50 step with and without ``multi_label``.

  python tools/bench_multilabel.py [--batch 256] [--image 224] [--steps 30] [--rounds 3] [--out f]

Prints one JSON document with the card's name, power limit and SM clock read in the same run:
  * per launch at B = --batch rows and V = 20 and 1000 classes (fp32 logits padded to a multiple
    of 8, random uint8 multi-hot targets, a pos_weight vector, label smoothing 0.1):
    sigmoid_bce (plain and with both options) against softmax_xent (plain and smoothed), and
    multilabel_eval_metrics against eval_metrics; microseconds per launch from device events
    around replays of a CUDA graph of 100 launches (so host launch overhead is not timed), after
    one warm-up replay;
  * the captured ResNet-50 training step at --batch x --image, default against multi_label=True
    (V = 1000 both), milliseconds per step from device events over --steps graph replays, the two
    trainers alternated for --rounds rounds (median and all).
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


def bench_kernels(B, V):
  from tensorflowonspark_b200 import ops
  C, dev = ops.C(), "cuda:0"
  VP = (V + 7) // 8 * 8
  g = torch.Generator(device="cpu").manual_seed(V)
  logits = (torch.randn(B, VP, generator=g) * 3).to(dev)
  targets = torch.randint(0, 2, (B, V), generator=g, dtype=torch.uint8).to(dev)
  labels = torch.randint(0, V, (B,), generator=g, dtype=torch.int32).to(dev)
  pw = (0.5 + torch.rand(V, generator=g)).to(dev)
  dl = torch.zeros(B, VP, dtype=torch.bfloat16, device=dev)
  loss, hits = torch.zeros(1, device=dev), torch.zeros(1, device=dev)
  nv = torch.tensor([B], dtype=torch.int32, device=dev)
  acc = torch.zeros(8 + 3 * V, dtype=torch.float64, device=dev)
  calls = {
      "softmax_xent": lambda: C.softmax_xent(logits, labels, dl, loss, hits, V, 1.0 / B),
      "softmax_xent_smooth": lambda: C.softmax_xent(logits, labels, dl, loss, hits, V, 1.0 / B,
                                                    label_smoothing=0.1),
      "sigmoid_bce": lambda: C.sigmoid_bce(logits, targets, dl, loss, hits, V, 1.0 / (B * V)),
      "sigmoid_bce_smooth_pos_weight": lambda: C.sigmoid_bce(
          logits, targets, dl, loss, hits, V, 1.0 / (B * V), label_smoothing=0.1, pos_weight=pw),
      "eval_metrics": lambda: C.eval_metrics(logits, labels, nv, acc, V),
      "multilabel_eval_metrics": lambda: C.multilabel_eval_metrics(logits, targets, nv, acc, V),
  }
  rows = {}
  for name, fn in calls.items():
    fn()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      for _ in range(100):
        fn()
    g.replay()
    rows[name] = round(1e3 * events_ms(g.replay, 10) / 100, 2)
  return rows


def bench_steps(args):
  from tensorflowonspark_b200.models import resnet
  nets = {}
  for name, ml in (("default", False), ("multi_label", True)):
    net = resnet.ResNetTrainer(depth=50, batch=args.batch, image=args.image, device="cuda:0",
                               multi_label=ml)
    x, y = net.synthetic_batch(seed=0)
    net.set_input(x, y)
    net.train_step()
    net.capture()
    for _ in range(5):
      net.train_step()
    nets[name] = net
  rounds = {k: [] for k in nets}
  for _ in range(args.rounds):
    for k, net in nets.items():
      rounds[k].append(round(events_ms(net.train_step, args.steps), 4))
  del nets
  torch.cuda.empty_cache()
  return {"step_ms": {k: statistics.median(v) for k, v in rounds.items()}, "step_ms_rounds": rounds}


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--batch", type=int, default=256)
  p.add_argument("--image", type=int, default=224)
  p.add_argument("--steps", type=int, default=30)
  p.add_argument("--rounds", type=int, default=3)
  p.add_argument("--classes", type=int, nargs="+", default=[20, 1000])
  p.add_argument("--out", default=None)
  args = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_multilabel needs a GPU")
  torch.cuda.set_device(0)
  doc = {"gpu": gpu_info(), "batch": args.batch, "image": args.image,
         "kernels_us": {V: bench_kernels(args.batch, V) for V in args.classes}}
  doc.update(bench_steps(args))
  doc["gpu_after"] = gpu_info()
  text = json.dumps(doc, indent=1)
  print(text)
  if args.out:
    with open(args.out, "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()

"""Held-out evaluation throughput of a ResNet-50 training trainer on one GPU.

  python tools/bench_eval.py [--batch 256] [--image 224] [--iters 20] [--out bench_eval.json]

Reports, with the card's name, power limit and SM clock read in the same run:
  * eval images/s: the captured eval_step graph replayed on device-resident batches (device events
    after warm-up);
  * the same through ``evaluate()`` from host (numpy) batches, end to end;
  * bn_fold and eval_metrics time per launch;
  * ServedResNet's ``forward_folded`` images/s at the same batch (a training=False trainer with the
    same parameters), timed alternately with the eval replay, as the yardstick: both run the same
    folded plans, the eval graph adds the metric kernel.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


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
  ap.add_argument("--batch", type=int, default=256)
  ap.add_argument("--image", type=int, default=224)
  ap.add_argument("--iters", type=int, default=20)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit("bench_eval: no CUDA device")
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.models import resnet
  torch.cuda.set_device(0)
  B, HW = args.batch, args.image
  net = resnet.ResNetTrainer(depth=50, batch=B, image=HW, device="cuda:0")
  x, y = net.synthetic_batch(seed=0)
  net.train_step(x, y)
  net.capture()
  for _ in range(3):
    net.train_step()
  served = resnet.ResNetTrainer(depth=50, batch=B, image=HW, device="cuda:0", training=False)
  served.load_state_dict(net.state_dict())
  served.build_folded_inference()
  served.set_input(x)
  sg = torch.cuda.CUDAGraph()
  served.forward_folded()
  torch.cuda.synchronize()
  with torch.cuda.graph(sg):
    served.forward_folded()

  ex, ey = net.synthetic_batch(seed=1)
  net.eval_begin()
  for _ in range(3):            # eager, capture, replay
    net.eval_step(ex, ey)
  ev = net._evaluator
  torch.cuda.synchronize()
  rates = {"eval_replay": [], "forward_folded": []}
  for _ in range(args.rounds):  # alternate the two in one process
    rates["eval_replay"].append(B * 1e3 / events_ms(ev.graph.replay, args.iters))
    rates["forward_folded"].append(B * 1e3 / events_ms(sg.replay, args.iters))
  net.eval_end()

  fold_ms = events_ms(ev.begin, args.iters)   # zero + bn_fold (comm=None: no broadcast)
  acc0 = ev.acc.clone()
  metric_ms = events_ms(lambda: ops.K.eval_metrics(net.logits, ev.labels, ev.n_valid, ev.acc,
                                                   net.num_classes), args.iters * 10)
  zero_ms = events_ms(lambda: ev.acc.zero_(), args.iters * 10)
  ev.acc.copy_(acc0)

  host = [(ex.cpu().numpy(), ey.cpu().numpy()) for _ in range(4)]
  net.evaluate(host[:2])
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  res = net.evaluate(host * 4)
  e2e = 16 * B / (time.perf_counter() - t0)

  out = {"gpu": gpu_info(), "batch": B, "image": HW,
         "eval_images_per_s": max(rates["eval_replay"]),
         "eval_images_per_s_rounds": rates["eval_replay"],
         "forward_folded_images_per_s": max(rates["forward_folded"]),
         "forward_folded_images_per_s_rounds": rates["forward_folded"],
         "evaluate_host_e2e_images_per_s": e2e,
         "bn_fold_ms": fold_ms - zero_ms, "eval_begin_ms": fold_ms, "eval_metrics_ms": metric_ms,
         "eval_count": res["count"]}
  print(json.dumps(out))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
      json.dump(out, f, indent=1)


if __name__ == "__main__":
  main()

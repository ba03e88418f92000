"""Cost of AdamW and LAMB against Adam and momentum (CUDA events, after warm-up).

  python tools/bench_adamw_lamb.py [--batch 256] [--rounds 5] [--steps 20]

1. the optimizer step alone over ResNet-50's parameter layout (25.6 M elements, one bucket, as the
   trainer builds it without peers): adam, adamw, lamb, and lamb's two kernels (norm pass, update)
   separately; microseconds and the bytes each has to move over 3.35 TB/s;
2. the ResNet-50 training step (captured graph) with optimizer="momentum", "adamw" and "lamb",
   three trainers in one process, timed alternately round after round: median and spread of each.
Prints one JSON line; the card name and power limit are part of it.  (tools/bench_optim.py: LARS.)
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from bench_optim import HBM_BPS, card, spread, timed_ms  # noqa: E402


def optimizer_only(dev, rounds):
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.parallel.fused_optim import FusedOptimizer
  net = resnet.ResNetTrainer(depth=50, batch=8, image=64, device=dev, training=False)
  st = net.store
  st.grads.copy_(torch.randn(st.total, device=dev) * 1e-3)
  n, head = st.total, st.decay_end
  opts = {name: FusedOptimizer(st, opt=name, lr=1e-4, weight_decay=1e-4)
          for name in ("adam", "adamw", "lamb")}
  lamb = opts["lamb"]
  calls = {"adam": opts["adam"].step, "adamw": opts["adamw"].step, "lamb": lamb.step,
           "lamb_norm_pass": lambda: ops.K.lars_norms(lamb._lars_args[0]),
           "lamb_update": lambda: ops.K.allreduce_opt(lamb._args[0])}
  # bytes each must move: grads 4 + master 8 + m 8 + v 8 + bf16 weights 2 (+ fp32 tail replica 4);
  # the norm pass reads g, w, m and v of the adapted head once
  update = 30 * n + 4 * (n - head)
  need = {"adam": update, "adamw": update, "lamb": update + 16 * head,
          "lamb_norm_pass": 16 * head, "lamb_update": update}
  for f in calls.values():
    timed_ms(f, 20)
  res = {k: [] for k in calls}
  for _ in range(rounds):
    for k, f in calls.items():
      res[k].append(timed_ms(f, 100) * 1e3)
  out = {"params": n, "adapted": head}
  for k, v in res.items():
    us = statistics.median(v)
    out[k] = {"us": spread(v), "bytes": need[k], "hbm_bound_us": need[k] / HBM_BPS * 1e6,
              "share_of_hbm_peak": need[k] / HBM_BPS * 1e6 / us}
  return out


def training_step(dev, batch, rounds, steps):
  from tensorflowonspark_b200.models import resnet
  lrs = {"momentum": 0.1 * batch / 256.0, "adamw": 1e-3, "lamb": 5e-3}
  nets = {name: resnet.ResNetTrainer(depth=50, batch=batch, image=224, device=dev, lr=lr,
                                     weight_decay=1e-4, optimizer=name)
          for name, lr in lrs.items()}
  x, y = nets["momentum"].synthetic_batch()
  for net in nets.values():
    net.set_input(x, y)
    net.train_step()
    net.capture()
    for _ in range(3):
      net.train_step()
  torch.cuda.synchronize()
  res = {k: [] for k in nets}
  for _ in range(rounds):
    for name, net in nets.items():
      res[name].append(timed_ms(net.train_step, steps))
  med = {k: statistics.median(v) for k, v in res.items()}
  return {"batch": batch, "steps_per_round": steps,
          "ms_per_step": {k: spread(v) for k, v in res.items()},
          "adamw_vs_momentum_pct": 100.0 * (med["adamw"] / med["momentum"] - 1.0),
          "lamb_vs_momentum_pct": 100.0 * (med["lamb"] / med["momentum"] - 1.0),
          "lamb_vs_adamw_pct": 100.0 * (med["lamb"] / med["adamw"] - 1.0)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, default=256)
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--steps", type=int, default=20)
  ap.add_argument("--skip_step", action="store_true", help="optimizer-only numbers")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit("bench_adamw_lamb: no CUDA device")
  dev = torch.device("cuda", 0)
  torch.cuda.set_device(dev)
  from tensorflowonspark_b200 import _build
  _build.load(required=True)
  out = {"card": card(dev), "optimizer_step_resnet50_layout": optimizer_only(dev, args.rounds)}
  if not args.skip_step:
    out["resnet50_train_step"] = training_step(dev, args.batch, args.rounds, args.steps)
  print(json.dumps(out), flush=True)


if __name__ == "__main__":
  main()

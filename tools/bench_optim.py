"""Cost of the LARS optimizer against momentum (CUDA events, after warm-up).

  python tools/bench_optim.py [--batch 256] [--rounds 5] [--steps 20]
  python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 tools/bench_optim.py

1. one GPU: the optimizer step alone over ResNet-50's parameter layout (25.6 M elements, one
   bucket, as the trainer builds it without peers): momentum, LARS, and LARS's two kernels
   (norm pass, update) separately; microseconds and the bytes each has to move over 3.35 TB/s;
2. the ResNet-50 training step (captured graph) with optimizer="momentum" and "lars", two trainers
   in one process, timed alternately round after round: median and spread of each;
3. under torch.distributed.run (2+ GPUs): the same step on the one-host communicator (max over
   ranks) plus the exposed all-reduce time per step measured like bench.py (eager steps).
Prints one JSON line; the card name and power limit are part of it.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

HBM_BPS = 3.35e12   # H100 SXM data sheet


def card(dev):
  out = {"name": torch.cuda.get_device_name(dev)}
  try:
    q = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0),
                        "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30).stdout.strip().split(",")
    out["power_limit_w"], out["max_sm_mhz"] = float(q[0]), float(q[1])
  except Exception as e:   # (the figure is then reported as unknown, never guessed)
    out["power_limit_w"] = None
    out["nvidia_smi"] = str(e)
  return out


def timed_ms(fn, iters):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(iters):
    fn()
  e1.record()
  e1.synchronize()
  return e0.elapsed_time(e1) / iters


def spread(v):
  return {"median": statistics.median(v), "min": min(v), "max": max(v)}


def optimizer_only(dev, rounds):
  """The fused optimizer step over ResNet-50's parameter vector, world 1, one bucket."""
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.parallel.fused_optim import FusedOptimizer
  net = resnet.ResNetTrainer(depth=50, batch=8, image=64, device=dev, training=False)
  st = net.store
  st.grads.copy_(torch.randn(st.total, device=dev) * 1e-3)
  n, head = st.total, st.decay_end
  opts = {name: FusedOptimizer(st, opt=name, lr=1e-3, momentum=0.9, weight_decay=1e-4)
          for name in ("momentum", "lars")}
  lars = opts["lars"]
  calls = {"momentum": opts["momentum"].step, "lars": lars.step,
           "lars_norm_pass": lambda: ops.K.lars_norms(lars._lars_args[0]),
           "lars_update": lambda: ops.K.allreduce_opt(lars._args[0])}
  # bytes each must move: grads 4 + master 8 + state1 8 + bf16 weights 2 (+ fp32 tail replica 4)
  update = 22 * n + 4 * (n - head)
  need = {"momentum": update, "lars": update + 8 * head, "lars_norm_pass": 8 * head,
          "lars_update": update}
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


def training_step(dev, batch, rounds, steps, comm_factory, world):
  from tensorflowonspark_b200.models import resnet
  nets = {}
  for name in ("momentum", "lars"):
    comm = comm_factory()
    nets[name] = resnet.ResNetTrainer(depth=50, batch=batch, image=224, device=dev, comm=comm,
                                      lr=0.1 * batch * world / 256.0, momentum=0.9,
                                      weight_decay=1e-4, optimizer=name)
  x, y = nets["momentum"].synthetic_batch()
  exposed = {}
  for name, net in nets.items():
    net.set_input(x, y)
    if world > 1 and net.optim.overlap:    # eager steps: timed events cannot be captured
      vals = []
      for _ in range(5):
        net.step_kernels()
        vals.append(net.optim.exposed_ms())
      t = torch.tensor([sum(vals[1:]) / len(vals[1:])], device=dev)
      torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
      exposed[name] = float(t)
    net.train_step()
    net.capture()
    for _ in range(3):
      net.train_step()
  torch.cuda.synchronize()
  res = {k: [] for k in nets}
  for _ in range(rounds):
    for name, net in nets.items():
      if world > 1:
        torch.distributed.barrier()
      ms = timed_ms(net.train_step, steps)
      t = torch.tensor([ms], device=dev)
      if world > 1:
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
      res[name].append(float(t))
  out = {"batch_per_gpu": batch, "world": world, "steps_per_round": steps,
         "ms_per_step": {k: spread(v) for k, v in res.items()},
         "lars_overhead_pct": 100.0 * (statistics.median(res["lars"]) /
                                       statistics.median(res["momentum"]) - 1.0)}
  if exposed:
    out["exposed_allreduce_ms"] = exposed
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, default=256)
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--steps", type=int, default=20)
  ap.add_argument("--skip_step", action="store_true", help="optimizer-only numbers")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit("bench_optim: no CUDA device")
  world = int(os.environ.get("WORLD_SIZE", "1"))
  rank = int(os.environ.get("RANK", "0"))
  local = int(os.environ.get("LOCAL_RANK", "0"))
  torch.cuda.set_device(local)
  dev = torch.device("cuda", local)
  from tensorflowonspark_b200 import _build
  _build.load(required=True)
  out = {"card": card(dev)}
  if world > 1:
    import torch.distributed as dist
    from tensorflowonspark_b200.parallel import symm
    dist.init_process_group("nccl", device_id=dev)

    def comm_factory():
      return symm.from_torch_distributed(dev)
  else:
    out["optimizer_step_resnet50_layout"] = optimizer_only(dev, args.rounds)

    def comm_factory():
      return None
  if not args.skip_step:
    out["resnet50_train_step"] = training_step(dev, args.batch, args.rounds, args.steps,
                                               comm_factory, world)
  if rank == 0:
    print(json.dumps(out), flush=True)
  if world > 1:
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
  main()

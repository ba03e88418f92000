"""Cost of gradient clipping (``clip_norm``) on one GPU, and under ``torch.distributed.run`` on
several.

  python tools/bench_grad_clip.py [--batch 256] [--unet_batch 64] [--steps 20] [--rounds 5]
                                  [--skip_trainers] [--out f]
  python -m torch.distributed.run --nproc-per-node 2 tools/bench_grad_clip.py --batch 256

One GPU:
  * the optimizer step alone on the ResNet-50 parameter layout (one bucket, world 1), momentum
    and Adam, clipping off / ``inf`` / active: a CUDA graph of ``step()`` replayed, us per step,
    the bytes it moves and their share of the HBM data-sheet bandwidth (3.35 TB/s).  Clipping
    adds one fp32 read of the gradient and two small launches;
  * the captured ResNet-50 step (batch 256, 224 x 224, momentum) and U-Net step (batch 64,
    128 x 128, Adam), off against an active threshold, alternated round by round.
With WORLD_SIZE > 1: the ResNet-50 step over the one-host communicator (buckets overlapped with
backward), off against on: step time and ``exposed_ms()`` (with clipping every bucket's update
waits for the last bucket's norm, so the update half no longer overlaps backward).
Prints one JSON document with the card's name, power limit and SM clock read in the same run.
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

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
# fp32 bytes per element of one update (grads, master, state1 [, state2] read; master, state1
# [, state2] written; bf16 weights written); clipping reads the gradient once more
BYTES = {"momentum": 4 * 3 + 4 * 2 + 2, "adam": 4 * 4 + 4 * 3 + 2}


def _median_rounds(fns, args):
  rounds = {k: [] for k in fns}
  for _ in range(args.rounds):
    for k, fn in fns.items():
      rounds[k].append(round(events_ms(fn, args.steps), 4))
  return {k: statistics.median(v) for k, v in rounds.items()}, rounds


def optimizer_only(args):
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.parallel.fused_optim import FusedOptimizer
  net = resnet.ResNetTrainer(depth=50, batch=8, image=64, device="cuda:0", training=False)
  st = net.store
  st.grads = torch.randn(st.total, device="cuda:0") * 1e-3
  out = {"elements": st.total}
  keep = []   # every optimizer outlives its graph (torch.cuda.graph() frees unreferenced memory)
  for opt in ("momentum", "adam"):
    fns = {}
    for k, c in (("off", None), ("inf", float("inf")), ("active", 1e-3)):
      o = FusedOptimizer(st, opt=opt, lr=1e-9, clip_norm=c)
      for _ in range(3):
        o.step()
      torch.cuda.synchronize()
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g):
        o.step()
      keep.append((o, g))
      fns[k] = g.replay
    med, rounds = _median_rounds(fns, args)
    res = {}
    for k, ms in med.items():
      b = st.total * (BYTES[opt] + (4 if k != "off" else 0))
      res[k] = {"us": round(ms * 1e3, 2), "bytes": b,
                "hbm_share": round(b / (ms * 1e-3) / HBM_BYTES_PER_S, 3), "rounds_ms": rounds[k]}
    res["extra_us_active"] = round(res["active"]["us"] - res["off"]["us"], 2)
    out[opt] = res
  return out


def _warm(net, x, y):
  net.set_input(x, y)
  net.train_step()
  net.capture()
  for _ in range(3):
    net.train_step()
  return net


def trainers(args):
  from tensorflowonspark_b200.models import resnet, unet
  out = {}
  nets = {}
  for k, c in (("off", None), ("on", 1.0)):
    net = resnet.ResNetTrainer(depth=50, batch=args.batch, image=224, device="cuda:0", clip_norm=c)
    nets[k] = _warm(net, *net.synthetic_batch(seed=0))
  med, rounds = _median_rounds({k: n.train_step for k, n in nets.items()}, args)
  out["resnet50"] = {"step_ms": med, "step_ms_rounds": rounds,
                     "overhead_pct": round(100.0 * (med["on"] / med["off"] - 1.0), 3),
                     "grad_norm": float(nets["on"].grad_norm)}
  del nets
  torch.cuda.synchronize()
  torch.cuda.empty_cache()
  nets = {}
  for k, c in (("off", None), ("on", 1.0)):
    net = unet.UNetTrainer(batch=args.unet_batch, image=128, classes=3, device="cuda:0", clip_norm=c)
    x, _ = net.synthetic_batch(seed=0)
    nets[k] = _warm(net, x, unet.synthetic_labels(x, 3))
  med, rounds = _median_rounds({k: n.train_step for k, n in nets.items()}, args)
  out["unet"] = {"step_ms": med, "step_ms_rounds": rounds,
                 "overhead_pct": round(100.0 * (med["on"] / med["off"] - 1.0), 3),
                 "grad_norm": float(nets["on"].grad_norm)}
  del nets
  torch.cuda.synchronize()
  torch.cuda.empty_cache()
  return out


def distributed(args):
  import torch.distributed as dist
  from tensorflowonspark_b200.models import resnet
  from tensorflowonspark_b200.parallel import symm
  rank = int(os.environ["RANK"])
  dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
  torch.cuda.set_device(dev)
  dist.init_process_group("nccl", device_id=dev)
  res = {}
  for k, c in (("off", None), ("on", 1.0)):
    net = resnet.ResNetTrainer(depth=50, batch=args.batch, image=224, device=dev,
                               comm=symm.from_torch_distributed(dev), clip_norm=c)
    net.set_input(*net.synthetic_batch(seed=rank))
    for _ in range(3):
      net.train_step()
    ms, exposed = [], []
    for _ in range(args.rounds):     # eager steps: the exposed wait is timed with events
      dist.barrier()
      ms.append(round(events_ms(net.train_step, args.steps), 3))
      exposed.append(round(net.optim.exposed_ms(), 4))
    res[k] = {"step_ms_eager": statistics.median(ms), "step_ms_rounds": ms,
              "exposed_ms": statistics.median(exposed), "exposed_ms_rounds": exposed}
    del net
    torch.cuda.synchronize()
  dist.destroy_process_group()
  return res if rank == 0 else None


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--batch", type=int, default=256)
  p.add_argument("--unet_batch", type=int, default=64)
  p.add_argument("--steps", type=int, default=20)
  p.add_argument("--rounds", type=int, default=5)
  p.add_argument("--skip_trainers", action="store_true")
  p.add_argument("--out", default=None)
  args = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_grad_clip needs a GPU")
  doc = {"gpu": gpu_info()}
  if int(os.environ.get("WORLD_SIZE", "1")) > 1:
    doc["world"] = int(os.environ["WORLD_SIZE"])
    doc["resnet50_distributed"] = distributed(args)
    if doc["resnet50_distributed"] is None:
      return
  else:
    torch.cuda.set_device(0)
    doc["optimizer_step_resnet50_layout"] = optimizer_only(args)
    print(json.dumps(doc["optimizer_step_resnet50_layout"]), flush=True)
    if not args.skip_trainers:
      doc.update(trainers(args))
  doc["gpu_after"] = gpu_info()
  text = json.dumps(doc, indent=1)
  print(text)
  if args.out:
    with open(args.out, "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()

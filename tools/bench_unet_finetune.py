"""Cost of fine-tuning the segmentation U-Net's encoder on one GPU.

  python tools/bench_unet_finetune.py [--batch 64] [--image 128] [--steps 50] [--out f]

Prints one JSON document with the card's name, power limit and SM clock read in the same run:
  * the captured training step for encoder_trainable_from = None (frozen encoder), 13 and 0:
    milliseconds per step from device events after warm-up, over ``--steps`` graph replays,
    the configurations alternated over two rounds (best round reported, both listed), and the
    native launches of one eager step;
  * depthwise3x3_bwd at each of the 17 encoder shapes: time per launch, the bytes the algorithm
    needs (x, y, dy, the skip gradient where the block has one, and dx, each once) and the
    achieved bandwidth as a share of the 3.35 TB/s data-sheet figure.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM5 80 GB HBM3 data-sheet peak


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


def bench_steps(args):
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.models import unet
  nets, launches = {}, {}
  for k in (None, 13, 0):
    net = unet.UNetTrainer(batch=args.batch, image=args.image, classes=3, device="cuda:0",
                           encoder_trainable_from=k)
    x, _ = net.synthetic_batch(seed=0)
    net.set_input(x, (x[..., 0] > 127).int() + (x[..., 1] > 200).int())
    n0 = ops.launch_count()
    net.train_step()
    launches[str(k)] = ops.launch_count() - n0
    net.capture()
    for _ in range(5):
      net.train_step()
    nets[str(k)] = net
  rounds = {k: [] for k in nets}
  for _ in range(2):
    for k, net in nets.items():
      rounds[k].append(events_ms(net.graph.replay, args.steps))
  torch.cuda.synchronize()
  out = {k: {"ms_per_step": min(v), "ms_per_step_rounds": v, "launches_per_eager_step": launches[k]}
         for k, v in rounds.items()}
  nets.clear()
  return out


def bench_kernel(args):
  from tensorflowonspark_b200 import ops
  from tensorflowonspark_b200.models import unet
  rows = []
  for block, H, C, s in unet.encoder_depthwise_shapes(args.image):
    N, OH = args.batch, (H - 1) // s + 1
    x = torch.rand(N, H, H, C, device="cuda").mul(7).sub(0.5).to(torch.bfloat16)
    y = torch.rand(N, OH, OH, C, device="cuda").mul(7).sub(0.5).to(torch.bfloat16)
    dy = torch.randn(N, OH, OH, C, device="cuda").to(torch.bfloat16)
    w = torch.randn(9, C, device="cuda").to(torch.bfloat16)
    skip = block in unet.SKIP_BLOCKS
    add = torch.randn(N, H, H, C + 64, device="cuda").to(torch.bfloat16) if skip else None
    dx = torch.empty_like(x)
    dw = torch.empty(9, C, device="cuda")
    db, dbi = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    scratch = torch.zeros(ops.C().depthwise3x3_bwd_scratch(N, H, C, s), device="cuda")
    run = lambda: ops.C().depthwise3x3_bwd(x, w, y, dy, add, 64 if skip else 0, dx, dw, db,  # noqa
                                           dbi, scratch, s)
    for _ in range(3):
      run()
    ms = min(events_ms(run, args.kernel_iters) for _ in range(3))
    nbytes = 2 * (x.numel() * (3 if skip else 2) + y.numel() * 2)
    rows.append({"block": block, "N": N, "H": H, "C": C, "stride": s, "skip_grad": skip,
                 "us": ms * 1e3, "bytes": nbytes,
                 "hbm_share": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S})
    del x, y, dy, add, dx, scratch
  return rows


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, default=64)
  ap.add_argument("--image", type=int, default=128)
  ap.add_argument("--steps", type=int, default=50)
  ap.add_argument("--kernel_iters", type=int, default=50)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit("bench_unet_finetune: no CUDA device")
  torch.cuda.set_device(0)
  out = {"gpu": gpu_info(), "batch": args.batch, "image": args.image, "classes": 3,
         "steps": args.steps, "train_step": bench_steps(args)}
  torch.cuda.empty_cache()
  out["depthwise3x3_bwd"] = bench_kernel(args)
  out["gpu_after"] = gpu_info()
  print(json.dumps(out))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
      json.dump(out, f, indent=1)


if __name__ == "__main__":
  main()

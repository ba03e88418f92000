"""Cost of stochastic depth (``drop_path_rate``) on one GPU: the captured ResNet-50 step with drop
path off and on, the scaled batch-norm kernels next to the plain ones, and the captured CIFAR
ResNet-56 step.

  python tools/bench_drop_path.py [--batch 256] [--image 224] [--steps 30] [--rounds 3] [--out f]

Prints one JSON document with the card's name, power limit and SM clock read in the same run:
  * the captured ResNet-50 training step at --batch x --image with drop_path_rate 0 (a plain
    trainer), 0.05 and 0.1, milliseconds per step from device events over --steps calls of
    train_step (host draw, staging copy and graph replay), alternated for --rounds rounds (median
    and all).  Rates 0.05 and 0.1 launch the same kernels (every block but the first drops, and
    its bn3 reduction is unfused); they run on one trainer whose graph reads the staged draw, with
    the draws of each rate;
  * bn_bwd_reduce, bn_bwd_apply (relu mode 3, the bit mask) and bn_apply_finalize (residual and
    mask) at ResNet-50's layer1 bn3 shape 256 x 56 x 56 x 256, without and with sample_scale;
    microseconds per launch from device events around replays of a CUDA graph of 20 launches, the
    bytes each moves and their share of the 3.35 TB/s HBM3 bound;
  * the captured CIFAR ResNet-56 step at batch 128 with drop_path_rate 0 and 0.1, alternated.
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


def _graph_us(fn, launches=20):
  fn()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for _ in range(launches):
      fn()
  g.replay()
  return 1e3 * events_ms(g.replay, 10) / launches


def bench_kernels(N=256, H=56, W=56, C=256):
  from tensorflowonspark_b200 import ops
  K, dev = ops.C(), "cuda:0"
  g = torch.Generator(device="cpu").manual_seed(0)
  shape = (N, H, W, C)
  x = torch.randn(shape, generator=g).to(torch.bfloat16).to(dev)
  res = torch.randn(shape, generator=g).to(torch.bfloat16).to(dev)
  dy = torch.randn(shape, generator=g).to(torch.bfloat16).to(dev)
  y = torch.empty_like(x)
  dx = torch.empty_like(x)
  bits = torch.randint(0, 256, (x.numel() // 8,), generator=g, dtype=torch.uint8).to(dev)
  v = lambda val=0.0: torch.full((C,), val, device=dev)  # noqa: E731
  gamma, mean, invstd, dg, db = v(1.0), v(0.0), v(1.0), v(), v()
  ssum, ssq = v(0.0), v(float(N * H * W))
  stats = [v() for _ in range(4)]
  rm, rv = v(), v(1.0)
  keep = torch.rand(N, generator=g) >= 0.1
  scale = torch.where(keep, torch.tensor(1 / 0.9), torch.tensor(0.0)).float().to(dev)
  n = x.numel()
  calls = {
      # dy + x read, the mask's byte per 8 elements
      "bn_bwd_reduce": (lambda **kw: K.bn_bwd_reduce(dy, x, bits, mean, invstd, dg, db, 3, None,
                                                     None, **kw), n * 4 + n // 8),
      # dy + x read, dx written, the mask
      "bn_bwd_apply": (lambda **kw: K.bn_bwd_apply(dy, x, bits, gamma, mean, invstd, dg, db, dx,
                                                   None, 3, None, None, **kw), n * 6 + n // 8),
      # x + residual read, y written, the mask written
      "bn_apply_finalize": (lambda **kw: K.bn_apply_finalize(
          x, res, y, 1, bits, ssum, ssq, gamma, gamma, rm, rv, *stats, float(N * H * W), 1e-5,
          0.1, **kw), n * 6 + n // 8),
  }
  rows = {}
  for name, (fn, nbytes) in calls.items():
    for tag, kw in (("", {}), ("_scaled", {"sample_scale": scale})):
      us = _graph_us(lambda: fn(**kw))
      rows[name + tag] = {"us": round(us, 2), "bytes": nbytes,
                          "hbm_share": round(nbytes / HBM_BYTES_PER_S / (us * 1e-6), 3)}
  return {"shape": list(shape), "kernels": rows}


def _captured(net):
  x, y = net.synthetic_batch(seed=0)
  net.set_input(x, y)
  net.train_step()
  net.capture()
  for _ in range(5):
    net.train_step()
  return net


def bench_resnet50(args):
  from tensorflowonspark_b200.models import engine, resnet
  make = lambda **kw: resnet.ResNetTrainer(depth=50, batch=args.batch,  # noqa: E731
                                           image=args.image, device="cuda:0", **kw)
  nets = {"0": _captured(make()), "drop": _captured(make(drop_path_rate=0.05))}
  n = len(nets["drop"].blocks)
  droppers = {r: engine.DropPathDraws(engine.drop_path_rates(float(r), n), args.batch, seed=1)
              for r in ("0.05", "0.1")}
  rounds = {"0": [], "0.05": [], "0.1": []}
  for _ in range(args.rounds):
    for k in rounds:
      net = nets["0" if k == "0" else "drop"]
      if k != "0":
        net.dropper = droppers[k]
      net.train_step()
      rounds[k].append(round(events_ms(net.train_step, args.steps), 4))
  del nets
  torch.cuda.empty_cache()
  return {"batch": args.batch, "image": args.image,
          "step_ms": {k: statistics.median(v) for k, v in rounds.items()}, "step_ms_rounds": rounds}


def bench_cifar(args):
  from tensorflowonspark_b200.models import resnet
  nets = {r: _captured(resnet.CifarResNetTrainer(depth=56, batch=128, device="cuda:0",
                                                 drop_path_rate=float(r)))
          for r in ("0", "0.1")}
  rounds = {k: [] for k in nets}
  for _ in range(args.rounds):
    for k, net in nets.items():
      net.train_step()
      rounds[k].append(round(events_ms(net.train_step, args.steps), 4))
  del nets
  torch.cuda.empty_cache()
  return {"batch": 128, "step_ms": {k: statistics.median(v) for k, v in rounds.items()},
          "step_ms_rounds": rounds}


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--batch", type=int, default=256)
  p.add_argument("--image", type=int, default=224)
  p.add_argument("--steps", type=int, default=30)
  p.add_argument("--rounds", type=int, default=3)
  p.add_argument("--out", default=None)
  args = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_drop_path needs a GPU")
  torch.cuda.set_device(0)
  doc = {"gpu": gpu_info(), "resnet50": bench_resnet50(args), "bn_kernels": bench_kernels(),
         "cifar_resnet56": bench_cifar(args)}
  doc["gpu_after"] = gpu_info()
  text = json.dumps(doc, indent=1)
  print(text)
  if args.out:
    with open(args.out, "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()

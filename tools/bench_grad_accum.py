"""Gradient accumulation on one GPU (CUDA events; the card, its power limit and max SM clock are
read in the same run):

  * the accumulating batch-norm backward apply against the writing one at the ResNet-50 shapes
    (batch 256), alternated, median of rounds;
  * captured ResNet-50 training throughput (images/s) at micro-batch 64 x k in {1, 4} and
    256 x k in {1, 2}, and the time of an accumulating micro-step against a k = 1 step;
  * the largest ResNet-152 micro-batch (from a descending list) whose whole accumulation window
    trains, eager and then captured, and the effective batch it reaches.

  python tools/bench_grad_accum.py [--out results.json] [--quick]
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

# (rows, channels) of the ResNet-50 batch norms at batch 256
BN_SHAPES = [(256 * 56 * 56, 64), (256 * 56 * 56, 256), (256 * 28 * 28, 128),
             (256 * 28 * 28, 512), (256 * 14 * 14, 256), (256 * 14 * 14, 1024),
             (256 * 7 * 7, 512), (256 * 7 * 7, 2048)]


def card():
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                      "--format=csv,noheader"], capture_output=True, text=True)
  return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def events_ms(fn, iters):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(iters):
    fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b) / iters


def bench_bn(rounds, iters):
  from tensorflowonspark_b200 import ops
  C_ = ops.C()
  out = []
  for P, C in BN_SHAPES:
    g = torch.Generator(device="cpu")
    g.manual_seed(C)
    dy = torch.randn(P, C, generator=g).to("cuda", torch.bfloat16)
    x = torch.randn(P, C, generator=g).to("cuda", torch.bfloat16)
    mask = torch.randint(0, 256, (P * C // 8,), dtype=torch.uint8).cuda()
    v = lambda: torch.rand(C, generator=g).cuda() + 0.5  # noqa: E731
    mean, invstd, gamma, sc, sh, dg, db, ag, ab = (v() for _ in range(9))
    dx = torch.empty_like(x)
    write = lambda: C_.bn_bwd_apply(dy, x, mask, gamma, mean, invstd, dg, db, dx, None, 3, sc, sh)  # noqa: E731
    acc = lambda: C_.bn_bwd_apply(dy, x, mask, gamma, mean, invstd, dg, db, dx, None, 3, sc, sh,  # noqa: E731
                                  acc_dgamma=ag, acc_dbeta=ab)
    for f in (write, acc):
      events_ms(f, 5)
    t = {"write": [], "accumulate": []}
    for _ in range(rounds):
      t["write"].append(events_ms(write, iters))
      t["accumulate"].append(events_ms(acc, iters))
    w, a = statistics.median(t["write"]), statistics.median(t["accumulate"])
    out.append({"rows": P, "C": C, "write_us": 1e3 * w, "accumulate_us": 1e3 * a,
                "accumulate_over_write": a / w,
                "spread_write_us": 1e3 * (max(t["write"]) - min(t["write"]))})
    del dy, x, mask, dx
  return out


def bench_resnet50(B, k, windows):
  from tensorflowonspark_b200.models import resnet
  net = resnet.ResNetTrainer(depth=50, batch=B, image=224, device="cuda:0",
                             gradient_accumulation_steps=k)
  net.set_input(*net.synthetic_batch(seed=0))
  net.capture()
  for _ in range(k):
    net.train_step()
  while net.micro_step:
    net.train_step()
  torch.cuda.synchronize()
  window = lambda: [net.train_step() for _ in range(k)]  # noqa: E731
  ms = [events_ms(window, windows) for _ in range(3)]
  res = {"micro_batch": B, "k": k, "effective_batch": B * k, "window_ms": statistics.median(ms),
         "images_per_s": B * k * 1e3 / statistics.median(ms)}
  if k > 1:   # one accumulating micro-step (no update) alone
    mid = lambda: net.graphs[(True, False)].replay()  # noqa: E731
    res["accumulating_micro_step_ms"] = statistics.median(events_ms(mid, windows) for _ in range(3))
    net.accum.restart(net.optim)   # the replays above only added into the gradients
  del net
  gc.collect()
  torch.cuda.empty_cache()
  return res


def largest_resnet152(candidates, k=8):
  """The largest micro-batch in ``candidates`` (descending) at which a whole ResNet-152 window
  trains: k eager micro-steps, the last one updating.  At that size the trainer is then captured
  (first / middle / last graphs) and one captured window replayed; the peak covers both."""
  from tensorflowonspark_b200.models import resnet
  for B in candidates:
    net = None
    try:
      net = resnet.ResNetTrainer(depth=152, batch=B, image=224, device="cuda:0",
                                 gradient_accumulation_steps=k)
      net.set_input(*net.synthetic_batch(seed=0))
      for _ in range(k):
        net.train_step()
      torch.cuda.synchronize()
    except torch.cuda.OutOfMemoryError:
      del net
      gc.collect()
      torch.cuda.empty_cache()
      torch.cuda.reset_peak_memory_stats()
      continue
    eager_peak = torch.cuda.max_memory_allocated() / 2 ** 30
    net.capture()
    for _ in range(k):
      net.train_step()
    torch.cuda.synchronize()
    res = {"micro_batch": B, "largest_tried": B == candidates[0], "k": k,
           "effective_batch_per_gpu": k * B, "eager_window_peak_gib": eager_peak,
           "captured_window_peak_gib": torch.cuda.max_memory_allocated() / 2 ** 30,
           "loss": float(net.loss_sum)}
    del net
    gc.collect()
    torch.cuda.empty_cache()
    return res
  return None


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--out", default=None)
  p.add_argument("--quick", action="store_true", help="fewer rounds (a smoke run of the tool)")
  a = p.parse_args()
  from tensorflowonspark_b200 import _build
  _build.load(required=True)
  torch.cuda.set_device(0)
  res = {"card": card()}
  res["bn_apply"] = bench_bn(3 if a.quick else 7, 20 if a.quick else 100)
  res["resnet50"] = [bench_resnet50(B, k, 5 if a.quick else 20)
                     for B, k in ((64, 1), (64, 4), (256, 1), (256, 2))]
  one = {r["micro_batch"]: r for r in res["resnet50"] if r["k"] == 1}
  for r in res["resnet50"]:
    if r["k"] > 1:
      r["micro_step_over_k1_step"] = r["accumulating_micro_step_ms"] / one[r["micro_batch"]]["window_ms"]
  res["resnet152_largest_micro_batch"] = largest_resnet152([768, 640, 512, 384, 256, 128])
  print(json.dumps(res, indent=1))
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
      json.dump(res, f, indent=1)


if __name__ == "__main__":
  main()

"""Cost of knowledge distillation on one GPU: the captured ResNet-50 step without a teacher and with
a frozen ResNet-50 or ResNet-152 teacher, the teacher's folded forward pass alone and the loss
kernel alone.

  python tools/bench_distill.py [--batch 256] [--image 224] [--steps 30] [--rounds 3] [--out f]

Prints one JSON document with the card's name, power limit and SM clock read in the same run:
  * for each teacher depth (50, 152): a plain ResNet-50 trainer and a distilling one (alpha 0.5,
    T 2, teacher state of a freshly initialised model of that depth) are built together, captured,
    and their train_step timed alternately for --rounds rounds, milliseconds per step from device
    events over --steps calls (median and all rounds).  The two trainers are freed before the next
    depth, so that the peak memory reported is that of one plain student plus one distilling
    student (``peak_allocated_gb``); ``student_teacher_gb`` is what the distilling student and its
    teacher allocated;
  * the teacher's folded forward pass alone (``teacher.run()``) at the same batch, in ms;
  * distill_xent against softmax_xent at B = --batch, V = 1000, microseconds per launch from a
    CUDA graph of 100 launches.
"""
import argparse
import gc
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from bench_unet_finetune import events_ms, gpu_info  # noqa: E402


def _graph_us(fn, launches=100):
  fn()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for _ in range(launches):
      fn()
  g.replay()
  return 1e3 * events_ms(g.replay, 10) / launches


def _free():
  torch.cuda.synchronize()
  gc.collect()
  torch.cuda.empty_cache()


def bench_loss(B, V):
  from tensorflowonspark_b200 import ops
  C, dev = ops.C(), "cuda:0"
  VP = (V + 7) // 8 * 8
  g = torch.Generator(device="cpu").manual_seed(V)
  s = (torch.randn(B, VP, generator=g) * 3).to(dev)
  z = (torch.randn(B, VP, generator=g) * 3).to(dev)
  y = torch.randint(0, V, (B,), generator=g, dtype=torch.int32).to(dev)
  dl = torch.zeros(B, VP, dtype=torch.bfloat16, device=dev)
  loss, hits = torch.zeros(1, device=dev), torch.zeros(1, device=dev)
  return {"batch": B, "classes": V, "us": {
      "softmax_xent": round(_graph_us(lambda: C.softmax_xent(s, y, dl, loss, hits, V, 1.0 / B)), 2),
      "distill_xent": round(_graph_us(lambda: C.distill_xent(s, z, y, dl, loss, hits, V, 1.0 / B,
                                                             alpha=0.5, temperature=2.0)), 2)}}


def bench_teacher(args, depth):
  from tensorflowonspark_b200.models import resnet
  state = resnet.ResNetTrainer(depth=depth, batch=8, image=64, training=False,
                               device="cuda:0").state_dict()
  _free()
  torch.cuda.reset_peak_memory_stats()
  base = torch.cuda.memory_allocated()
  plain = resnet.ResNetTrainer(depth=50, batch=args.batch, image=args.image, device="cuda:0")
  plain_gb = (torch.cuda.memory_allocated() - base) / 2 ** 30
  base = torch.cuda.memory_allocated()
  dist = resnet.ResNetTrainer(depth=50, batch=args.batch, image=args.image, device="cuda:0",
                              teacher=state, teacher_depth=depth, distill_temperature=2.0)
  dist_gb = (torch.cuda.memory_allocated() - base) / 2 ** 30
  nets = {"plain": plain, "teacher": dist}
  for net in nets.values():
    x, y = net.synthetic_batch(seed=0)
    net.set_input(x, y)
    net.train_step()
    net.capture()
    for _ in range(5):
      net.train_step()
  rounds = {"plain": [], "teacher": []}
  for _ in range(args.rounds):
    for k in rounds:
      nets[k].train_step()
      rounds[k].append(round(events_ms(nets[k].train_step, args.steps), 4))
  t = dist.teacher
  t.run()
  fwd = round(events_ms(t.run, args.steps), 4)
  out = {"teacher_depth": depth, "step_ms": {k: statistics.median(v) for k, v in rounds.items()},
         "step_ms_rounds": rounds, "teacher_forward_ms": fwd,
         "plain_student_gb": round(plain_gb, 2), "student_teacher_gb": round(dist_gb, 2),
         "peak_allocated_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}
  del nets, plain, dist, t
  _free()
  return out


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--batch", type=int, default=256)
  p.add_argument("--image", type=int, default=224)
  p.add_argument("--steps", type=int, default=30)
  p.add_argument("--rounds", type=int, default=3)
  p.add_argument("--out", default=None)
  args = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_distill needs a GPU")
  torch.cuda.set_device(0)
  doc = {"gpu": gpu_info(), "batch": args.batch, "image": args.image,
         "loss": bench_loss(args.batch, 1000),
         "steps": [bench_teacher(args, d) for d in (50, 152)]}
  doc["gpu_after"] = gpu_info()
  text = json.dumps(doc, indent=1)
  print(text)
  if args.out:
    with open(args.out, "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()

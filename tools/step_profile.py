"""Per-kernel split of one eager (un-graphed) ResNet-50 training step.

  python tools/step_profile.py --torch-profiler profiles/step   # torch.profiler, CUDA activities

prints (and writes to DIR/step_kernels.txt) one row per kernel: launches, total device time and
share of the summed kernel time, averaged over --steps profiled steps.  Without --torch-profiler
the step is bracketed by cudaProfilerStart/Stop for an Nsight Compute capture:

  ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv \
      --log-file profiles/step.csv python tools/step_profile.py
  python tools/ncu_summary.py profiles/step.csv

(kernels run back to back without the CUDA graph: the table explains a step, it is not a bench
value)."""
import argparse
import collections
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from tensorflowonspark_b200.models import resnet  # noqa: E402


def kernel_name(name):
  """Template instance without the parameter list: 'igemm_fwd_kernel<256, true, 10>'."""
  name = re.sub(r"^void ", "", name)
  name = re.sub(r"\(anonymous namespace\)::|tfos::", "", name)
  depth, out = 0, []
  for ch in name:
    if ch == "(" and depth == 0:
      break
    depth += ch == "<"
    depth -= ch == ">"
    out.append(ch)
  return "".join(out).strip()


def profile_table(net, steps, out_dir):
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(steps):
      net.step_kernels()
    torch.cuda.synchronize()
  launches, us = collections.Counter(), collections.Counter()
  for ev in prof.events():
    if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time_total > 0:
      k = kernel_name(ev.name)
      launches[k] += 1
      us[k] += ev.device_time_total
  total = sum(us.values())
  lines = ["{} (power limit {}), {} eager steps; kernel time per step {:.1f} us".format(
      torch.cuda.get_device_name(0), _power_limit(), steps, total / steps),
      "{:>8s} {:>12s} {:>7s}  {}".format("launches", "us/step", "share", "kernel")]
  for k, t in us.most_common():
    lines.append("{:8d} {:12.1f} {:6.2f}%  {}".format(
        launches[k] // steps, t / steps, 100.0 * t / total, k))
  text = "\n".join(lines)
  print(text)
  os.makedirs(out_dir, exist_ok=True)
  with open(os.path.join(out_dir, "step_kernels.txt"), "w") as f:
    f.write(text + "\n")


def _power_limit():
  import subprocess
  try:
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit",
                           "--format=csv,noheader"], capture_output=True, text=True,
                          timeout=30).stdout.strip() or "unknown"
  except Exception:
    return "unknown"


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, default=256)
  ap.add_argument("--depth", type=int, default=50)
  ap.add_argument("--image", type=int, default=224)
  ap.add_argument("--torch-profiler", metavar="DIR", default=None,
                  help="time the kernels with torch.profiler and write DIR/step_kernels.txt")
  ap.add_argument("--steps", type=int, default=5, help="profiled steps (--torch-profiler)")
  args = ap.parse_args()
  dev = torch.device("cuda", 0)
  net = resnet.ResNetTrainer(depth=args.depth, batch=args.batch, image=args.image, device=dev)
  x, y = net.synthetic_batch(seed=0)
  net.set_input(x, y)
  for _ in range(2):
    net.step_kernels()
  torch.cuda.synchronize()
  if args.torch_profiler:
    profile_table(net, args.steps, args.torch_profiler)
    return
  torch.cuda.profiler.start()
  net.step_kernels()
  torch.cuda.synchronize()
  torch.cuda.profiler.stop()


if __name__ == "__main__":
  main()

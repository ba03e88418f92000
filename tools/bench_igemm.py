"""Per-layer timing of the wgmma implicit-GEMM kernels on ResNet-50 shapes (batch 256).

  python tools/bench_igemm.py               # table: time, TFLOP/s, GB/s, fraction of measured peaks
  python tools/bench_igemm.py --only l1c3   # one case, few iterations (for an ncu capture)

CUDA-event timing after warm-up; every case cycles through enough distinct buffers to exceed
the 50 MB L2.  Peaks come from MEASURED_PEAKS.json when present, else from the H100 SXM data
sheet (3,350 GB/s HBM3, 989 TFLOP/s dense bf16 at up to 700 W): a ceiling, not a reached rate.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from tensorflowonspark_b200.ops import igemm  # noqa: E402

B = 256
# name, kind, (H, W, Cin, Cout, k, stride)
CASES = [
    ("l1c1", "fprop", (56, 56, 256, 64, 1, 1)),
    ("l1c1b0", "fprop", (56, 56, 64, 64, 1, 1)),      # b0: the first block of the layer
    ("l1c2", "fprop", (56, 56, 64, 64, 3, 1)),
    ("l1c3", "fprop", (56, 56, 64, 256, 1, 1)),
    ("l2c1b0", "fprop", (56, 56, 256, 128, 1, 1)),
    ("l2c1", "fprop", (28, 28, 512, 128, 1, 1)),
    ("l2c2", "fprop", (28, 28, 128, 128, 3, 1)),
    ("l2c3", "fprop", (28, 28, 128, 512, 1, 1)),
    ("l3c1b0", "fprop", (28, 28, 512, 256, 1, 1)),
    ("l3c1", "fprop", (14, 14, 1024, 256, 1, 1)),
    ("l3c2", "fprop", (14, 14, 256, 256, 3, 1)),
    ("l3c3", "fprop", (14, 14, 256, 1024, 1, 1)),
    ("l4c1b0", "fprop", (14, 14, 1024, 512, 1, 1)),
    ("l4c1", "fprop", (7, 7, 2048, 512, 1, 1)),
    ("l4c2", "fprop", (7, 7, 512, 512, 3, 1)),
    ("l4c3", "fprop", (7, 7, 512, 2048, 1, 1)),
    ("l2c2s2", "fprop", (56, 56, 128, 128, 3, 2)),
    ("l1c3_dgrad", "dgrad", (56, 56, 64, 256, 1, 1)),
    ("l1c1_dgrad", "dgrad", (56, 56, 256, 64, 1, 1)),
    ("l3c2_dgrad", "dgrad", (14, 14, 256, 256, 3, 1)),
    # the batch-norm backward epilogues of the data gradients: fused reduction (EPI 8), masked
    # residual accumulate (EPI 2 + acc_mask) and both (EPI 10)
    ("l1c1_dgrad_red", "dgrad_red", (56, 56, 256, 64, 1, 1)),
    ("l1c1_dgrad_acc", "dgrad_acc", (56, 56, 256, 64, 1, 1)),
    ("l1c1_dgrad_accred", "dgrad_accred", (56, 56, 256, 64, 1, 1)),
    ("l2c1_dgrad_red", "dgrad_red", (28, 28, 512, 128, 1, 1)),
    ("l2c1_dgrad_accred", "dgrad_accred", (28, 28, 512, 128, 1, 1)),
    ("l3c1_dgrad_accred", "dgrad_accred", (14, 14, 1024, 256, 1, 1)),
    ("l4c1_dgrad_accred", "dgrad_accred", (7, 7, 2048, 512, 1, 1)),
    ("l1c2_dgrad_red", "dgrad_red", (56, 56, 64, 64, 3, 1)),
    ("l3c2_dgrad_red", "dgrad_red", (14, 14, 256, 256, 3, 1)),
    ("l3c3_dgrad_red", "dgrad_red", (14, 14, 256, 1024, 1, 1)),
    ("l4c3_dgrad_red", "dgrad_red", (7, 7, 512, 2048, 1, 1)),
    ("l1c2_wgrad", "wgrad", (56, 56, 64, 64, 3, 1)),
    ("l1c3_wgrad", "wgrad", (56, 56, 64, 256, 1, 1)),
    ("l1c1_wgrad", "wgrad", (56, 56, 256, 64, 1, 1)),
    ("l2c2_wgrad", "wgrad", (28, 28, 128, 128, 3, 1)),
    ("l2c3_wgrad", "wgrad", (28, 28, 128, 512, 1, 1)),
    ("l3c1_wgrad", "wgrad", (14, 14, 1024, 256, 1, 1)),
    ("l3c3_wgrad", "wgrad", (14, 14, 256, 1024, 1, 1)),
    ("l3c2_wgrad", "wgrad", (14, 14, 256, 256, 3, 1)),
    ("l4c2_wgrad", "wgrad", (7, 7, 512, 512, 3, 1)),
    # the first block of layer2-4: stride 2 in the 3x3 (torchvision v1.5)
    ("l2c2s2_wgrad", "wgrad", (56, 56, 128, 128, 3, 2)),
    ("l3c2s2_wgrad", "wgrad", (28, 28, 256, 256, 3, 2)),
    ("l4c2s2_wgrad", "wgrad", (14, 14, 512, 512, 3, 2)),
    ("l4c3_wgrad", "wgrad", (7, 7, 512, 2048, 1, 1)),
    ("l4c1_wgrad", "wgrad", (7, 7, 2048, 512, 1, 1)),
    ("l4c1b1_wgrad", "wgrad", (14, 14, 1024, 512, 1, 1)),   # first block of layer4
    # projection shortcuts of the first blocks: 1x1, stride 2
    ("l2ds_wgrad", "wgrad", (56, 56, 256, 512, 1, 2)),
    ("l3ds_wgrad", "wgrad", (28, 28, 512, 1024, 1, 2)),
    ("l4ds_wgrad", "wgrad", (14, 14, 1024, 2048, 1, 2)),
]


def peaks():
  p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
  if os.path.exists(p):
    d = json.load(open(p))
    return d["hbm_gbs"], d["bf16_tflops"], "measured"
  return 3350.0, 989.0, "H100 SXM data sheet"


def device_line():
  import subprocess
  q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm",
                      "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
  return "{} ({})".format(torch.cuda.get_device_name(0), q or "power limit / max SM clock unknown")


def build(kind, shape, nbuf, stats=True, epi_prefetch=True):
  H, W, Ci, Co, k, s = shape
  pad = k // 2
  OH, OW = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
  dev = "cuda"
  plans = []
  for _ in range(nbuf):
    x = torch.randn(B, H, W, Ci, device=dev).bfloat16()
    w = (torch.randn(Co, k, k, Ci, device=dev) * 0.05).bfloat16()
    y = torch.zeros(B, OH, OW, Co, device=dev, dtype=torch.bfloat16)
    if kind == "fprop":
      st = (torch.zeros(Co, device=dev), torch.zeros(Co, device=dev)) if stats else None
      plans.append(igemm.conv_fprop(x, w, y, s, pad, stats=st))
    elif kind == "dgrad":
      plans.append(igemm.conv_dgrad(y, w, x, s, pad))
    elif kind.startswith("dgrad_"):
      acc = "acc" in kind
      mask = torch.randint(0, 256, (B * H * W * Ci // 8,), device=dev, dtype=torch.uint8)
      red = None
      if "red" in kind:
        red = (torch.randn(B, H, W, Ci, device=dev).bfloat16(), mask,
               torch.zeros(Ci, device=dev), torch.zeros(Ci, device=dev))
      plans.append(igemm.conv_dgrad(y, w, x, s, pad, accumulate=acc,
                                    acc_mask=mask if acc else None, bn_reduce=red,
                                    epi_prefetch=epi_prefetch))
    else:
      dw = torch.zeros(Co, k, k, Ci, device=dev)
      plans.append(igemm.conv_wgrad(y, x, dw, s, pad))
  flops = 2.0 * B * OH * OW * Co * Ci * k * k
  byts = 2.0 * B * (H * W * Ci + OH * OW * Co) + 2.0 * Co * Ci * k * k
  # the epilogue's reads: the previous dx (accumulate) and red_x, each with its bit mask
  byts += ("acc" in kind) * B * H * W * Ci * (2 + 1 / 8.0)
  byts += ("red" in kind) * B * H * W * Ci * (2 + 1 / 8.0)
  return plans, flops, byts


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--only", default=None)
  ap.add_argument("--iters", type=int, default=20)
  ap.add_argument("--no-stats", action="store_true")
  ap.add_argument("--epi-prefetch", type=int, choices=(0, 1), default=1,
                  help="dgrad_* kinds: prefetch the epilogue operands where the plan can")
  ap.add_argument("--kind", default=None,
                  help="fprop | dgrad | dgrad_red | dgrad_acc | dgrad_accred | wgrad")
  args = ap.parse_args()
  hbm, tf, src = peaks()
  print(device_line())
  print("peaks ({}): HBM {:.0f} GB/s, bf16 {:.0f} TFLOP/s".format(src, hbm, tf))
  print("{:12s} {:6s} {:>9s} {:>9s} {:>9s} {:>7s} {:>7s}".format(
      "case", "kind", "us", "TFLOP/s", "GB/s", "%flops", "%hbm"))
  for name, kind, shape in CASES:
    if (args.only and name != args.only) or (args.kind and kind != args.kind):
      continue
    H, W, Ci, Co, k, s = shape
    per = 2.0 * B * (H * W * Ci + H * W * Co)
    nbuf = 1 if args.only else max(2, int(400e6 // per) + 1)
    plans, flops, byts = build(kind, shape, nbuf, not args.no_stats, bool(args.epi_prefetch))
    iters = 3 if args.only else args.iters
    for p in plans[:2]:
      p.run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
      plans[i % len(plans)].run()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    print("{:12s} {:6s} {:9.1f} {:9.1f} {:9.1f} {:6.1f}% {:6.1f}%  {}".format(
        name, kind, us, flops / us / 1e6, byts / us / 1e3, 100 * flops / us / 1e6 / tf,
        100 * byts / us / 1e3 / hbm, plans[0].desc))
    del plans
    torch.cuda.empty_cache()


if __name__ == "__main__":
  main()

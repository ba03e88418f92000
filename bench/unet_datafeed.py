"""Segmentation U-Net fed through InputMode.SPARK: rows travel RDD -> feeder task -> shared-memory
ring (page-locked by the consumer) -> ``cudaMemcpyAsync`` straight from the ring slot on the copy
stream -> native U-Net step, all through ``TFNode.DataFeed`` (BASELINE.json config "segmentation
U-Net InputMode.SPARK DataFeed queue on 8xH100"; the reference's loop being replaced is
tensorflowonspark/TFSparkNode.py:500-502 feeder side, TFNode.py:278-300 consumer side).

  python bench/unet_datafeed.py --gpus 8 --batch 64 --steps 60
(also reachable as `python bench.py --config unet --gpus 8`)

Every step's inputs come from host memory through the public API, so the number IS end to end;
the on-device synthetic rate of the same trainer (``--input_mode tf``) is reported next to it.
"""
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROW_BYTES = 128 * 128 * 3 + 128 * 128


def _example(gpus, batch, mode, examples=0, steps=0):
  cmd = [sys.executable, os.path.join(ROOT, "examples", "segmentation", "segmentation_spark.py"),
         "--cluster_size", str(gpus), "--batch_size", str(batch), "--input_mode", mode,
         "--epochs", "1"]
  cmd += ["--num_examples", str(examples)] if mode == "spark" else ["--steps", str(steps)]
  out = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, cwd=ROOT)
  rates = [float(m.group(1)) for m in re.finditer(r"(\d+) images/s", out.stdout)]
  if not rates:
    sys.stderr.write(out.stdout[-2000:] + out.stderr[-3000:])
    raise SystemExit(1)
  return rates[-1], out.stdout


def run(gpus, batch=64, steps=60):
  examples = int(gpus * batch * steps / 0.9) + gpus * batch
  rate, log = _example(gpus, batch, "spark", examples=examples)
  direct = re.findall(r"straight from the ring (\d+) / staged (\d+)", log)
  synth, _ = _example(gpus, batch, "tf", steps=steps)
  return {
      "metric": "U-Net training images/s through InputMode.SPARK DataFeed (whole job)",
      "value": rate, "unit": "images/s", "n_gpus": gpus, "steps": steps, "warmup": 1,
      "ms_per_step": 1e3 * batch * gpus / rate, "higher_is_better": True, "scaling": "weak",
      "vs_baseline": None, "dtype": "bf16",
      "data": "synthetic rows (uint8 128x128x3 image + 128x128 mask) generated in Spark tasks",
      "config": {"model": "unet_mobilenetv2 128x128x3, 3 classes", "global_batch": batch * gpus,
                 "per_gpu_batch": batch, "parallelism": "dp{} + InputMode.SPARK feed".format(gpus),
                 "timing": "wall clock on the chief after the CUDA-graph capture step"},
      "e2e": {"value": rate, "unit": "images/s", "h2d_bytes_per_step": batch * ROW_BYTES,
              "d2h_bytes_per_step": 0.4,
              "note": "same measurement: inputs arrive through the feed; the loss is read back every 10 steps"},
      "feed_MB_per_s": rate * ROW_BYTES / 1e6,
      "on_device_synthetic_images_per_s": synth,
      "h2d_tensors_straight_from_ring_vs_staged": [list(map(int, d)) for d in direct],
      "gpu_launches": None,
  }


if __name__ == "__main__":
  import argparse
  p = argparse.ArgumentParser()
  p.add_argument("--gpus", type=int, default=1)
  p.add_argument("--batch", type=int, default=64)
  p.add_argument("--steps", type=int, default=60)
  a = p.parse_args()
  print(json.dumps(run(a.gpus, a.batch, a.steps)))

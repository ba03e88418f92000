"""GPU tier: whole programs through TFCluster on a real device (1 executor = 1 GPU):
MNIST via InputMode.SPARK with the native sm_90a trainer -> export -> TFParallel inference, and
the segmentation U-Net fed through DataFeed -> pinned staging -> async H2D."""
import os
import re
import subprocess
import sys
import tempfile

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, timeout=600):
  p = subprocess.run([sys.executable] + args, capture_output=True, text=True, timeout=timeout,
                     cwd=ROOT)
  print(p.stdout[-3000:], p.stderr[-3000:])
  assert p.returncode == 0
  return p.stdout + p.stderr


def test_mnist_spark_train_export_infer_on_gpu():
  d = tempfile.mkdtemp(prefix="tfos_gpu_mnist_")
  _run(["examples/mnist/mnist_data_setup.py", "--output", d + "/data", "--train_size", "8192",
        "--test_size", "1024", "--num_partitions", "4"])
  out = _run(["examples/mnist/mnist_spark.py", "--cluster_size", "1", "--images_labels",
              d + "/data/csv/train", "--epochs", "3", "--learning_rate", "0.05", "--export_dir",
              d + "/export", "--model_dir", d + "/model"])
  assert "native sm_90a trainer" in out          # not the CPU fallback
  assert os.path.exists(d + "/export/weights.pt")
  out = _run(["examples/mnist/mnist_inference.py", "--cluster_size", "1", "--images_labels",
              d + "/data/tfr/test", "--export_dir", d + "/export", "--output", d + "/pred"])
  acc = float(re.search(r"accuracy: ([\d.]+)", out).group(1))
  assert acc > 0.9, out[-500:]


def test_unet_through_datafeed_on_gpu():
  out = _run(["examples/segmentation/segmentation_spark.py", "--cluster_size", "1", "--batch_size",
              "32", "--input_mode", "spark", "--num_examples", "4096"])
  m = re.search(r"rank 0 ran (\d+) steps \((\d+) rows\)", out)
  assert m and int(m.group(1)) == int(4096 * 0.9 / 32) and int(m.group(2)) == int(m.group(1)) * 32
  losses = [float(x) for x in re.findall(r"loss ([\d.]+)", out)]
  assert len(losses) >= 3 and losses[-1] < losses[0]

"""Test configuration.

Tiers (mirrors the reference's strategy, SURVEY.md section 4):
  * unit tests - no Spark, no GPU;
  * distributed tests on the bundled sparklite engine with 2 executor *processes* on CPU
    (gloo where a collective is needed) - the stand-in for the reference's 2-worker
    Spark Standalone cluster;
  * ``@pytest.mark.gpu`` - native-kernel numerics vs plain PyTorch fp32 and end-to-end
    training on a real H100 (``pytest -m gpu``).
"""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("TFOS_SHUTDOWN_POLL_SECS", "0.2")

import torch  # noqa: E402,F401  (imported before executors fork so they inherit it)


def pytest_configure(config):
  config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 box)")


def pytest_collection_modifyitems(config, items):
  if torch.cuda.is_available():
    return
  skip = pytest.mark.skip(reason="no CUDA device")
  for item in items:
    if "gpu" in item.keywords:
      item.add_marker(skip)


@pytest.fixture(scope="module")
def sc():
  from tensorflowonspark_b200.sparklite import SparkContext
  ctx = SparkContext("local[2]", "tfos-tests")
  yield ctx
  ctx.stop()


@pytest.fixture(scope="module")
def spark(sc):
  from tensorflowonspark_b200.sparklite import SparkSession
  return SparkSession(sc)

"""Import-compatibility alias: ``import tensorflowonspark`` / ``from tensorflowonspark import
TFCluster, TFNode, ...`` resolve to the Hopper-native implementation in ``tensorflowonspark_b200``
so programs written against yahoo/TensorFlowOnSpark only change the body of their ``map_fun``."""
import importlib
import sys

import tensorflowonspark_b200 as _impl
from tensorflowonspark_b200 import __version__  # noqa: F401

_MODULES = ("TFCluster", "TFManager", "TFNode", "TFParallel", "TFSparkNode", "compat", "dfutil",
            "gpu_info", "marker", "pipeline", "reservation", "util")

for _m in _MODULES:
  _mod = importlib.import_module("tensorflowonspark_b200." + _m)
  sys.modules[__name__ + "." + _m] = _mod
  globals()[_m] = _mod

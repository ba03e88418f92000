#!/bin/sh
# Compile every CUDA/C++ source under csrc/ for sm_90a into tensorflowonspark_b200/_ext/ (in-tree).
# Works on a machine without a GPU: nvcc cross-compiles.
set -e
cd "$(dirname "$0")/.."
python -c "import __graft_entry__ as g; g.build()"
ls -la tensorflowonspark_b200/_ext/*.so

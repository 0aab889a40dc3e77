#!/bin/bash
# Node preparation (parity: reference tools/pre_run.sh — conda install of torch/mpi4py/blosc).
# On an H100 image everything is already installed; build the native extension in-tree.
set -e
cd "$(dirname "$0")/.."
python -c "import torch; print('torch', torch.__version__, 'cuda', torch.version.cuda)"
python setup.py build_ext --inplace
python -c "import atomo_b200._C; print('atomo_b200._C ok')"

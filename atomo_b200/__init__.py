"""atomo_b200 — a H100-native gradient-sparsification parameter-server engine.

Capabilities mirror hwang595/ATOMO (synchronous PS data parallelism with
atomic-decomposition gradient coders: spectral-SVD ATOMO, entry-wise ATOMO,
QSGD/TernGrad, QSVD, dense/lossless), re-designed for 8xH100:

* models stay in PyTorch (``atomo_b200.models``);
* the gradient coders have a pure-PyTorch reference implementation (CPU/gloo
  path and test oracle) and hand-written sm_90a CUDA kernels
  (``atomo_b200.ops`` / ``atomo_b200/csrc``);
* the worker->PS push and PS->worker parameter broadcast run over a symmetric
  heap in NVLink peer memory (``atomo_b200.parallel``), fused into the encode /
  decode+SGD kernels, with no NCCL call on those paths.
"""

__version__ = "0.1.0"

from . import codings, optim  # noqa: F401

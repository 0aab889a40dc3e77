"""Gradient codings registry (parity: ``/root/reference/src/codings/__init__.py:1-6``).

``codings.build(name, **kw)`` resolves the launcher's ``--code`` flag:
``sgd``/``dense``/``lossless`` (dense pass-through), ``svd`` (spectral ATOMO),
``entrywise`` (entry-wise ATOMO), ``topk`` (top-k sparsification, the oracle of the bf16 engine's top-k units), ``sign`` (scaled sign, the oracle of the bf16 engine's sign units), ``powersgd`` (warm-started rank-r power iteration, the oracle of the bf16 engine's PowerSGD units), ``fp8`` (e4m3 bytes with stochastic rounding, the oracle of the bf16 engine's fp8 units), ``hadamard`` (randomized-Hadamard rotated 2 / 4 / 8-bit quantization, the oracle of the bf16 engine's hadamard units), ``qsgd``, ``terngrad``, ``qsvd``, ``bsvd`` (block-spectral: the estimator of the sm_90a bf16 engine).
"""
from .coding import Coding, available, build, register
from . import utils, sampling
from .svd import SVD
from .qsgd import QSGD, TernGrad
from .entrywise import EntryWise
from .topk import TopK
from .sign import ScaledSign
from .powersgd import PowerSGD
from .fp8 import FP8
from .hadamard import Hadamard
from .qsvd import QSVD
from .block_svd import BlockSVD
from . import lossless_compress
from .lossless_compress import LosslessCompress
from . import svd, qsgd, entrywise, qsvd  # noqa: F401  (module-style access like the reference)

__all__ = ["Coding", "SVD", "QSGD", "TernGrad", "EntryWise", "TopK", "ScaledSign", "PowerSGD", "FP8", "Hadamard", "QSVD", "BlockSVD", "LosslessCompress",
           "utils", "sampling", "build", "register", "available"]

"""Gradient codings registry (parity: ``/root/reference/src/codings/__init__.py:1-6``).

``codings.build(name, **kw)`` resolves the launcher's ``--code`` flag:
``sgd``/``dense``/``lossless`` (dense pass-through), ``svd`` (spectral ATOMO),
``entrywise`` (entry-wise ATOMO), ``qsgd``, ``terngrad``, ``qsvd``, ``bsvd`` (block-spectral: the estimator of the sm_90a bf16 engine).
"""
from .coding import Coding, available, build, register
from . import utils, sampling
from .svd import SVD
from .qsgd import QSGD, TernGrad
from .entrywise import EntryWise
from .qsvd import QSVD
from .block_svd import BlockSVD
from . import lossless_compress
from .lossless_compress import LosslessCompress
from . import svd, qsgd, entrywise, qsvd  # noqa: F401  (module-style access like the reference)

__all__ = ["Coding", "SVD", "QSGD", "TernGrad", "EntryWise", "QSVD", "BlockSVD", "LosslessCompress",
           "utils", "sampling", "build", "register", "available"]

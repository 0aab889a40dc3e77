"""Distributed Lion (Liu et al., "Communication Efficient Distributed Training with Distributed Lion", NeurIPS 2024):
plain fp32 numpy functions that are the oracle of the bf16 engine's ``code="dlion"`` (``csrc/v2_signum.cu``), bit for
bit.  The bit rule, coin, packing, vote and decay are Signum's (``codings.signum``); only the worker rule and the mean
aggregation are new here.

Not a registered :class:`~atomo_b200.codings.coding.Coding`: only the p2p bf16 engine runs the code.

* **Worker step** (:func:`worker_step`): with ``om1 = 1 - b1`` and ``om2 = 1 - b2`` formed in fp32, the direction
  ``c = b1 m + om1 g`` and then ``m <- b2 m + om2 g``, each operation rounded separately under flush-to-zero, ``m``
  starting at zero.  With ``b1 == 0``, ``c = g`` and no momentum exists.  The pushed bit is Signum's bit of ``c``.
* **Aggregation**: ``vote`` is Signum's (:func:`atomo_b200.codings.signum.vote`); ``mean`` (:func:`mean`) is
  ``(pos - neg) / counted`` with one rounded fp32 division, 0 when nothing is counted, and NaN over a tile when a counted
  worker's tile (or vector value) is not finite.
* **Step** (:func:`step`): ``fmaf(-lr, v, p)`` with one rounding; weights are first scaled by Signum's
  :func:`~atomo_b200.codings.signum.decay_factor` when there is weight decay.
"""
from __future__ import annotations

import numpy as np

from .hadamard import fma32
from .signum import _NAN, ftz, vote

AGGREGATES = ("vote", "mean")


def _mul(a, b) -> np.ndarray:
    return ftz(ftz(a) * ftz(b))


def _add(a, b) -> np.ndarray:
    return ftz(ftz(a) + ftz(b))


def worker_step(m, g, b1: float, b2: float):
    """``(c, m')``: the direction ``b1 m + (1 - b1) g`` and the new momentum ``b2 m + (1 - b2) g``, fp32 with
    flush-to-zero and every operation rounded on its own, as ``lion_direction`` / ``lion_momentum``
    (``csrc/v2_momentum.cuh``) compute them."""
    b1, b2 = np.float32(b1), np.float32(b2)
    om1, om2 = np.float32(1) - b1, np.float32(1) - b2
    m, g = np.asarray(m, dtype=np.float32), np.asarray(g, dtype=np.float32)
    c = _add(_mul(b1, m), _mul(om1, g))
    return c, _add(_mul(b2, m), _mul(om2, g))


def mean(bit_rows, n: int, bad=()) -> np.ndarray:
    """fp32 mean of ``n`` elements' signs over the counted workers (one row of ``n`` bits per counted worker, 1 =
    negative): ``(pos - neg) / counted`` rounded once, 0 with no counted worker; a true entry of ``bad`` makes the whole
    tile NaN."""
    b = np.asarray(bit_rows, dtype=np.int64).reshape(-1, n)
    counted = b.shape[0]
    neg = b.sum(axis=0)
    if counted == 0:
        v = np.zeros(n, np.float32)
    else:
        v = ((counted - 2 * neg).astype(np.float32) / np.float32(counted)).astype(np.float32)
    if any(bad):
        v[:] = _NAN
    return v


def aggregate(kind: str, bit_rows, n: int, bad=()) -> np.ndarray:
    """The owners' aggregate of ``kind`` (``"vote"`` or ``"mean"``)."""
    if kind not in AGGREGATES:
        raise ValueError("dlion aggregate: vote | mean (got %r)" % (kind,))
    return vote(bit_rows, n, bad) if kind == "vote" else mean(bit_rows, n, bad)


def step(p, v, lr: float) -> np.ndarray:
    """``fmaf(-lr, v, p)`` in fp32 with one rounding: ``-lr * v`` is not exact for a mean ``v``."""
    p = np.asarray(p, dtype=np.float32)
    return fma32(np.float32(-lr), np.asarray(v, dtype=np.float32), p).astype(np.float32)

"""Signum with majority vote (Bernstein et al., "signSGD: Compressed Optimisation for Non-Convex Problems", ICML 2018,
and "signSGD with Majority Vote is Communication Efficient and Fault Tolerant", ICLR 2019): plain fp32 numpy functions
that are the oracle of the bf16 engine's Signum (``csrc/v2_signum.cu``), bit for bit.

Not a registered :class:`~atomo_b200.codings.coding.Coding`: only the p2p bf16 engine runs the code.

* **Worker momentum** (heavy-ball form): ``u <- beta * u + g`` in fp32, each operation rounded separately, starting at
  zero (:func:`momentum_step`).  The kernels are built with flush-to-zero, so fp32 subnormal inputs and results read as
  signed zero (:func:`ftz`).  With ``beta == 0`` no buffer exists and ``u = g``.  ``g`` is the bf16 weight gradient or
  the fp32 vector gradient.
* **Bit** (:func:`bits`): 1 when ``u < 0``, 0 when ``u > 0``.  A zero (``+0``, ``-0`` or subnormal) takes a fair coin:
  uniform word ``e & 3`` of Philox(seed ^ ``COIN_KEY_XOR``, (e >> 2, unit, step, worker)), with ``e`` the element index
  inside the unit, is 1 below one half (:func:`coin_uniforms`).  A NaN or Inf takes its sign bit, and makes its tile
  non-finite.
* **Packing** (:func:`pack`): one 4096-element bucket per PS tile, bit ``i`` of uint64 word ``j`` of a tile is its
  element ``64 j + i``; a tile's last word holds only its real elements (padding bits 0).
* **Vote** (:func:`vote`): per element over the counted workers, ``neg`` = number of 1 bits, ``pos = counted - neg``;
  ``+1`` if ``pos > neg``, ``-1`` if ``neg > pos``, ``0`` on a tie.  A counted worker whose tile (weights) or value
  (vectors: anywhere in the 4096-element vector tile) is not finite makes the tile's vote NaN.
* **Step** (:func:`step`): ``p <- fmaf(-lr, vote, p)``; with ``weight_decay`` the owner first scales weights (not
  vectors) by ``fp32(1 - lr * wd)`` (:func:`decay_factor`), the decoupled decay of AdamW.
"""
from __future__ import annotations

import numpy as np

from .powersgd import philox

COIN_KEY_XOR = 0x9E6C63D0676A9A99   # csrc/v2_signum.cu SIGNUM_SEED_XOR
TILE_ELEMS = 4096
_NAN = np.frombuffer(np.uint32(0x7FFFFFFF).tobytes(), dtype=np.float32)[0]


def ftz(x) -> np.ndarray:
    """fp32 with subnormals replaced by zero of the same sign."""
    x = np.asarray(x, dtype=np.float32)
    b = x.view(np.uint32)
    return np.where((b & 0x7F800000) == 0, (b & 0x80000000).view(np.float32), x).astype(np.float32)


def momentum_step(u, g, beta: float) -> np.ndarray:
    """``beta * u + g`` in fp32 with flush-to-zero, as ``mc_step`` (``csrc/v2_momentum.cuh``) computes it."""
    b = np.float32(beta)
    t = ftz(ftz(b) * ftz(u))
    return ftz(t + ftz(g))


def classify(x) -> np.ndarray:
    """0 positive, 1 negative, 2 zero (``+-0`` and subnormals), 3 NaN / Inf, on the fp32 bits."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32)
    ex = b & 0x7F800000
    return np.where(ex == 0x7F800000, 3, np.where(ex == 0, 2, b >> 31)).astype(np.int64)


def coin_uniforms(seed: int, unit: int, elems, step: int, worker: int) -> np.ndarray:
    """The uniform of element ``e`` of unit ``unit`` (fp32 in [0, 1)), as the kernels draw the coin of a zero."""
    e = np.asarray(elems, dtype=np.uint64)
    key = (int(seed) ^ COIN_KEY_XOR) & 0xFFFFFFFFFFFFFFFF
    w = philox(key, e >> np.uint64(2), unit, step, worker)
    sel = (e & np.uint64(3)).astype(np.int64)
    r = np.choose(sel, [w[0], w[1], w[2], w[3]])
    return ((r >> np.uint64(8)).astype(np.float64) / 16777216.0).astype(np.float32)


def bits(u, uniforms) -> np.ndarray:
    """The pushed bit of every element of ``u`` (0 / 1, int64); ``uniforms`` is the coin's uniform per element."""
    u = np.asarray(u, dtype=np.float32)
    cls = classify(u)
    coin = (np.asarray(uniforms, dtype=np.float32) < np.float32(0.5)).astype(np.int64)
    return np.where(cls == 2, coin, (u.view(np.uint32) >> 31).astype(np.int64))


def pack(b) -> np.ndarray:
    """uint64 words of a tile's bits (bit ``i`` of word ``j`` is element ``64 j + i``), ``ceil(n / 64)`` of them."""
    b = np.asarray(b, dtype=np.uint64)
    n = b.size
    pad = np.zeros(-(-n // 64) * 64, dtype=np.uint64)
    pad[:n] = b
    sh = np.arange(64, dtype=np.uint64)
    return np.bitwise_or.reduce(pad.reshape(-1, 64) << sh, axis=1)


def unpack(words, n: int) -> np.ndarray:
    """The first ``n`` bits of uint64 ``words`` (int64), inverse of :func:`pack`."""
    w = np.asarray(words, dtype=np.uint64).reshape(-1, 1)
    return ((w >> np.arange(64, dtype=np.uint64)) & np.uint64(1)).reshape(-1)[:n].astype(np.int64)


def nonfinite(u) -> bool:
    return bool((classify(u) == 3).any())


def vote(bit_rows, n: int, bad=()) -> np.ndarray:
    """fp32 vote of ``n`` elements from the counted workers' bits (one row of ``n`` bits per counted worker); a true
    entry of ``bad`` (one per counted worker) marks a non-finite tile and makes the whole vote NaN.  No counted worker:
    0."""
    b = np.asarray(bit_rows, dtype=np.int64).reshape(-1, n)
    neg = b.sum(axis=0)
    pos = b.shape[0] - neg
    v = np.where(pos > neg, 1.0, np.where(neg > pos, -1.0, 0.0)).astype(np.float32)
    if any(bad):
        v[:] = _NAN
    return v


def step(p, v, lr: float) -> np.ndarray:
    """``fmaf(-lr, v, p)`` in fp32: ``-lr * v`` is exact for ``v`` in {-1, 0, 1}, so one rounded add."""
    p = np.asarray(p, dtype=np.float32)
    return (p + np.float32(-lr) * np.asarray(v, dtype=np.float32)).astype(np.float32)


def decay_factor(lr: float, wd: float) -> np.float32:
    """The owner's decoupled weight decay factor, ``1 - lr * wd`` in double rounded to fp32 once."""
    return np.float32(1.0 - float(lr) * float(wd))

"""PowerSGD: a warm-started rank-``r`` power-iteration code of a whole weight matrix (Vogels et al. 2019).

The low-rank contractive code for error feedback.  A weight gradient is seen as the matrix ``M`` (``[O][C]``) and sent
as two thin factors ``P_hat`` (``[O][r]``, orthonormal or zero columns) and ``Q'`` (``[C][r]``) with
``g_hat = P_hat Q'^T``, the projection of ``M`` onto the span of ``P_hat``.  The projection is contractive:
``||M - P_hat P_hat^T M||^2 = ||M||^2 - ||Q'||^2 <= ||M||^2``, so a residual fed back step after step stays bounded.
Without error feedback the code is biased.

This coder is the oracle of the bf16 engine's PowerSGD units (``csrc/v2_powersgd.cu``), one encode of one worker:

* ``M`` is the bf16 gradient in the PHYSICAL element order of the engine (channels-last ``[O][kh][kw][I]`` for convs):
  row ``o`` is the contiguous slab of ``C = numel / O`` values.  Tensors with ``r (O + C) >= O C`` travel dense;
* the warm state ``Q_w`` (``[C][r]``, fp32) starts as standard normals (:func:`normals`): Philox4x32-10 of
  ``csrc/common.cuh`` keyed by ``(seed, unit, column, draw counter)``, Box-Muller in fp64;
* ``P = M Q_w`` (fp32 sums), ``G = P^T P`` in fp64, a Cholesky factor of ``G`` under a fixed pivot rule
  (:func:`cholesky_rinv`): column ``j`` is *degenerate* if its pivot is ``<= 1e-12 max_j G_jj``, zero or non-finite,
  and a degenerate column of ``P_hat = P R^{-1}`` is zero;
* ``Q' = M^T P_hat``; the pushed estimate is ``g_hat = P_hat Q'^T``;
* the warm state becomes ``Q'``; degenerate columns are re-drawn with the next draw counter, so the subspace cannot
  collapse to zero for good.  A tensor whose ``G`` is non-finite (an Inf or NaN in it) pushes zeros and keeps ``Q_w``.

This is the per-worker-subspace variant, one push per step: every worker pushes its own rank-``r`` pair and the owner
averages ``P_hat_w Q'_w^T`` over the workers (a mean of rank up to ``W r``).  The all-reduce variant of the paper
(two communication rounds and a ``P`` shared by all workers) is not implemented.
"""
from __future__ import annotations

import numpy as np
import torch

from .coding import Coding, register

POWER_MAX_RANK = 4
PIVOT_RTOL = 1e-12
PHILOX_KEY_XOR = 0x70C5D1A3B2E49F17      # the seed of the warm-state draws differs from the other codes'

_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_U32 = np.uint64(0xFFFFFFFF)


def check_rank(rank: int) -> int:
    r = int(rank)
    if not 1 <= r <= POWER_MAX_RANK:
        raise ValueError("powersgd: svd_rank must be in [1, %d] (got %r)" % (POWER_MAX_RANK, rank))
    return r


def coded(shape, rank: int) -> bool:
    """Whether a weight of ``shape`` travels as a rank-``rank`` pair: ``r (O + C) < O C`` (else it travels dense)."""
    if len(shape) < 2:
        return False
    o = int(shape[0])
    c = int(np.prod(shape[1:]))
    return rank * (o + c) < o * c


def philox(seed: int, c0, c1, c2, c3):
    """Philox4x32-10 of ``csrc/common.cuh`` on arrays of counters: the four 32-bit output words."""
    c = [np.asarray(x, dtype=np.uint64) & _U32 for x in np.broadcast_arrays(c0, c1, c2, c3)]
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(_M0) * c[0], np.uint64(_M1) * c[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & _U32, p1 >> np.uint64(32), p1 & _U32
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0, k1 = (k0 + np.uint64(_W0)) & _U32, (k1 + np.uint64(_W1)) & _U32
    return c


def normals(seed: int, unit: int, cols: int, rank: int, draw: int) -> np.ndarray:
    """``[cols][rank]`` standard normals of ``(seed, unit, column, draw)``: normal ``k`` of column ``c`` is Box-Muller
    of words ``2 (k & 1)``, ``2 (k & 1) + 1`` of Philox(seed ^ PHILOX_KEY_XOR, (c, unit, draw, k >> 1)), in fp64
    (``u1 = ((w0 >> 8) + 1) / 2^24``, ``u2 = (w1 >> 8) / 2^24``, ``z = sqrt(-2 ln u1) cos(2 pi u2)``), rounded to fp32."""
    out = np.zeros((cols, rank), dtype=np.float32)
    key = (int(seed) ^ PHILOX_KEY_XOR) & 0xFFFFFFFFFFFFFFFF
    col = np.arange(cols, dtype=np.uint64)
    for k in range(rank):
        w = philox(key, col, unit, draw, k >> 1)
        w0, w1 = w[2 * (k & 1)], w[2 * (k & 1) + 1]
        u1 = ((w0 >> np.uint64(8)).astype(np.float64) + 1.0) / 16777216.0
        u2 = (w1 >> np.uint64(8)).astype(np.float64) / 16777216.0
        out[:, k] = (np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)).astype(np.float32)
    return out


def cholesky_rinv(G: np.ndarray):
    """``(R^{-1}, mask)`` of the fp64 Gram matrix ``G`` (``r x r``) under the fixed pivot rule: columns in order, column
    ``j``'s pivot ``d = G_jj - sum_k L_jk^2`` over the earlier non-degenerate columns; ``j`` is degenerate when
    ``d <= 1e-12 max_j G_jj``, ``d == 0`` or ``d`` is non-finite, and its ``L`` column and ``R^{-1}`` column are zero.
    ``P R^{-1}`` then has orthonormal or zero columns.  A non-finite ``G`` makes every column degenerate."""
    r = G.shape[0]
    L = np.zeros((r, r))
    rinv = np.zeros((r, r))
    mask = 0
    if not np.isfinite(G).all():
        return rinv, 0
    tol = PIVOT_RTOL * max(float(np.max(np.diag(G))), 0.0)
    for j in range(r):
        d = G[j, j]
        for k in range(j):
            d -= L[j, k] * L[j, k]
        if not np.isfinite(d) or d <= tol or d == 0.0:
            continue
        ljj = np.sqrt(d)
        L[j, j] = ljj
        for i in range(j + 1, r):
            s = G[i, j]
            for k in range(j):
                s -= L[i, k] * L[j, k]
            L[i, j] = s / ljj
        for i in range(r):     # R^{-1}[:, j] = (e_j - sum_{k<j} L_jk R^{-1}[:, k]) / L_jj
            s = 1.0 if i == j else 0.0
            for k in range(j):
                s -= L[j, k] * rinv[i, k]
            rinv[i, j] = s / ljj
        mask |= 1 << j
    return rinv, mask


def bf16_matrix(grad: torch.Tensor) -> np.ndarray:
    """``[O][C]`` fp32 values of ``bf16(grad)`` in the engine's physical order (channels-last for 4-D tensors)."""
    g = grad.detach()
    if g.dim() == 4:
        g = g.permute(0, 2, 3, 1)
    return g.reshape(g.shape[0], -1).to(torch.bfloat16).float().cpu().numpy().astype(np.float32)


def power_step(M: np.ndarray, qw: np.ndarray):
    """One encode of the fp32 matrix ``M`` from the warm state ``qw``: a dict with ``p``, ``gram``, ``rinv``, ``mask``,
    ``nonfinite``, ``phat`` and ``qnew`` (fp32 arrays; ``phat`` / ``qnew`` are what is pushed)."""
    rank = qw.shape[1]
    P = (M.astype(np.float64) @ qw.astype(np.float64)).astype(np.float32)
    with np.errstate(all="ignore"):
        G = P.astype(np.float64).T @ P.astype(np.float64)
    nonfinite = not np.isfinite(G).all()
    rinv, mask = cholesky_rinv(G)
    if nonfinite:
        phat = np.zeros_like(P)
        qnew = np.zeros((M.shape[1], rank), dtype=np.float32)
    else:
        phat = (P.astype(np.float64) @ rinv).astype(np.float32)
        qnew = (M.astype(np.float64).T @ phat.astype(np.float64)).astype(np.float32)
    return {"p": P, "gram": G, "rinv": rinv, "mask": mask, "nonfinite": nonfinite, "phat": phat, "qnew": qnew}


def next_warm_state(step: dict, qw: np.ndarray, seed: int, unit: int, draw: int):
    """``(Q_w, draw)`` after an encode: ``Q'`` with its degenerate columns re-drawn under ``draw + 1`` (the counter
    advances only when a column is re-drawn); unchanged after a non-finite tensor."""
    if step["nonfinite"]:
        return qw.copy(), draw
    rank = qw.shape[1]
    deg = [k for k in range(rank) if not (step["mask"] >> k) & 1]
    q = step["qnew"].copy()
    if deg:
        draw += 1
        z = normals(seed, unit, q.shape[0], rank, draw)
        q[:, deg] = z[:, deg]
    return q, draw


@register("powersgd")
class PowerSGD(Coding):
    """One worker's PowerSGD coder with its warm state per tensor (keyed by ``unit``, the engine's unit index)."""

    def __init__(self, svd_rank: int = 1, seed: int = 1, *args, **kwargs):
        super().__init__()
        self.rank = check_rank(svd_rank)
        self.seed = int(seed)
        self.state = {}

    def warm(self, unit: int, cols: int):
        if unit not in self.state:
            self.state[unit] = (normals(self.seed, unit, cols, self.rank, 0), 0)
        return self.state[unit]

    def encode(self, grad: torch.Tensor, unit: int = 0, **kwargs) -> dict:
        M = bf16_matrix(grad)
        qw, draw = self.warm(unit, M.shape[1])
        st = power_step(M, qw)
        self.state[unit] = next_warm_state(st, qw, self.seed, unit, draw)
        return {"phat": torch.from_numpy(st["phat"]), "qnew": torch.from_numpy(st["qnew"]), "mask": st["mask"],
                "shape": list(grad.shape)}

    @staticmethod
    def decode_matrix(code: dict) -> torch.Tensor:
        """``P_hat Q'^T`` in fp64, ``[O][C]`` in the physical order."""
        return code["phat"].double() @ code["qnew"].double().T

    def decode(self, code: dict, cuda: bool = False, **kwargs) -> torch.Tensor:
        shape = code["shape"]
        m = self.decode_matrix(code).float()
        out = m.reshape(shape[0], *shape[2:], shape[1]).permute(0, 3, 1, 2) if len(shape) == 4 else m.reshape(shape)
        out = out.contiguous()
        return out.cuda() if cuda else out

    def error_sq(self, grad: torch.Tensor, unit: int = 0):
        """``(||A||^2 - ||Q'||^2, ||A - g_hat||^2)`` in fp64 of one encode of ``grad`` from the current warm state
        (``A`` = :func:`bf16_matrix`), without advancing the state.  The two agree up to the rounding of the factors."""
        M = bf16_matrix(grad)
        qw, _ = self.warm(unit, M.shape[1])
        st = power_step(M, qw)
        A = M.astype(np.float64)
        q = st["qnew"].astype(np.float64)
        ghat = st["phat"].astype(np.float64) @ q.T
        return float((A * A).sum() - (q * q).sum()), float(((A - ghat) ** 2).sum())

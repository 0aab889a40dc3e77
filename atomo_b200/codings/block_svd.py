"""Block-spectral ATOMO (``--code bsvd``): the estimator of the overlapped bf16 engine, in plain PyTorch.

The reference SVD-codes every tensor whole (``/root/reference/src/codings/svd.py:79-118``).  The sm_90a engine
(``csrc/v2_encode.cu``) never forms an SVD of a wide matrix: it splits a tensor into *units* whose small side has at
most 64 columns and diagonalises each unit's Gram matrix with an in-kernel Jacobi solver —

* a convolution ``(O, I, kh, kw)`` with ``I % 16 == 0`` and ``2*kh*kw <= 64`` is ONE unit: the reference's own
  matricization ``(O*I/2, 2*kh*kw)`` (``svd.py:12-28``), so it is coded exactly like ``--code svd``;
* any other matrix-shaped tensor (fc layers, 1x1 convolutions, ...) is put in tall orientation and cut into column
  blocks of at most 32 columns; every block is coded on its own with budget ``ceil(rank / blocks)`` (at least 1).

A block estimate is ``sum_i b_i/p_i * (A v_i) v_i^T`` with ``v_i`` the eigenvectors of ``A^T A`` and ``b_i`` ~
Bernoulli(``p_i``), ``p_i = min(1, budget * sigma_i / sum(sigma))``: unbiased for ANY complete orthonormal basis, so
the blocks are unbiased individually and the tensor estimate is too — this replaces round 1's truncated range-finder
route for square-ish layers, which was biased.  No redraw when nothing is sampled (the reference redraws,
``svd.py:57-67``, which biases small budgets: measured +15 % at budget 1 of 18 atoms).

This class shares the unit decomposition with the GPU planner (``ops/plan2.py``), which makes it the oracle of
``tests/test_gpu_v2.py`` in spirit and gives the gloo role path the same estimator (``--code bsvd``).
"""
from __future__ import annotations

from functools import lru_cache
from typing import List, Optional, Tuple

import torch

from .coding import Coding, register
from .sampling import atom_probabilities, sample_atoms


@lru_cache(maxsize=512)
def unit_table(shape: Tuple[int, ...], rank: int, block_cols: int = 32) -> Tuple[Tuple, ...]:
    """Units of one tensor as the GPU planner cuts them: tuples ``(kind, rows, cols, col0, budget)``.

    ``kind`` is ``"slab"`` (whole conv tensor, reference matricization), ``"block"`` (columns ``col0..col0+cols`` of
    the tall orientation of ``tensor.reshape(shape[0], -1)``) or ``"dense"`` (sent as is)."""
    from ..ops import plan2 as P
    if len(shape) < 2:
        return (("dense", 0, 0, 0, 0.0),)
    pl = P.build_plan2([tuple(shape)], "svd", int(rank), False, n_owners=1, n_groups=1, block_cols=block_cols)
    out = []
    for u in pl.units:
        if u.kind == P.KIND_SLAB:
            out.append(("slab", u.rows, u.cols, 0, float(u.budget)))
        elif u.kind == P.KIND_MAT:
            out.append(("block", u.rows, u.cols, u.g_off // u.cs if u.cs > 1 else u.g_off, float(u.budget)))
        else:
            out.append(("dense", 0, 0, 0, 0.0))
    return tuple(out)


def _tall(grad: torch.Tensor) -> Tuple[torch.Tensor, bool]:
    m = grad.reshape(grad.shape[0], -1)
    return (m, False) if m.shape[0] >= m.shape[1] else (m.t(), True)


@register("bsvd")
class BlockSVD(Coding):
    def __init__(self, rank: int = 3, random_sample: bool = True, prob_rule: str = "reference",
                 scheme: str = "bernoulli", block_cols: int = 32, generator: Optional[torch.Generator] = None,
                 allocation: str = "per_block", *args, **kwargs):
        """``allocation="per_block"`` is what the sm_90a engine does today (every block samples with its own budget
        ``ceil(rank / blocks)``).  ``"global"`` treats the atoms of ALL blocks of a tensor as one atom set with
        ``p_i = min(1, rank * sigma_i / sum_all sigma)`` — ATOMO's optimal allocation for this decomposition, ``rank``
        expected atoms per tensor instead of per block; still unbiased (any probabilities are).  It needs one number
        per tensor shared by its blocks, which the fused kernel could take from the previous step; evaluated here on
        CPU first (``docs/experiments/variance_*.md``)."""
        super().__init__()
        if allocation not in ("per_block", "global"):
            raise ValueError("allocation: per_block | global")
        self.allocation = allocation
        self.svd_rank = max(int(rank), 1)
        self.random_sample = random_sample
        self.prob_rule = prob_rule
        self.scheme = scheme
        self.block_cols = int(block_cols)
        self.generator = generator

    # ------------------------------------------------------------------
    def _code_unit(self, a: torch.Tensor, budget: float, total_sigma: Optional[float] = None,
                   max_atoms: Optional[int] = None):
        """One unit ``a`` (rows x cols, fp32): Gram -> eigenvectors -> sampled atoms ``(U, s/p, V^T)``.
        ``total_sigma`` (global allocation): nuclear-norm normaliser shared by all blocks of the tensor.
        ``max_atoms`` (the engine's slot capacity): a draw with more atoms is redrawn, as the kernel does.

        The rules of the kernel (``csrc/spectral_sample.cuh``):

        * ``sigma_max < 1e-6``: the top atom is sent with ``p = 1`` (the reference's rule, ``svd.py:50-51``).  This
          estimate ``A v_0 v_0^T`` is biased by at most ``||A||_F <= sqrt(cols) sigma_max < sqrt(cols) * 1e-6``.
        * An atom with ``sigma_i <= 1e-7 sigma_max`` (a null direction) is counted and sent, with a zero column of
          ``U`` instead of ``A v_i / 0``.
        """
        lam, v = torch.linalg.eigh(a.t() @ a)
        lam, v = lam.flip(0).clamp_min(0), v.flip(1)
        sigma = lam.sqrt()
        smax = float(sigma[0])
        cols = a.shape[1]
        if not smax >= 1e-6:
            idx = torch.zeros(1, dtype=torch.long)
            scale = torch.ones(1, dtype=sigma.dtype)
        elif self.random_sample:
            if total_sigma is not None:
                p = (budget * sigma / total_sigma).clamp(max=1.0)
            else:
                p = atom_probabilities(sigma, budget, self.prob_rule)
            idx = sample_atoms(p, scheme=self.scheme, generator=self.generator, allow_empty=True,
                               max_atoms=max_atoms)
            scale = 1.0 / p[idx].to(sigma.dtype)
        else:
            k = min(int(budget) if budget > 0 else cols, cols)
            idx = torch.arange(k if max_atoms is None else min(k, max_atoms))
            scale = torch.ones(len(idx), dtype=sigma.dtype)
        vs = v[:, idx]
        live = sigma[idx] > 1e-7 * smax
        u = torch.where(live, a @ vs, 0.0) / torch.where(live, sigma[idx], 1.0)
        return u.contiguous(), (sigma[idx] * scale).contiguous(), vs.t().contiguous()

    def encode(self, grad: torch.Tensor, **kwargs) -> dict:
        g = grad.detach().to(torch.float32)
        table = unit_table(tuple(g.shape), self.svd_rank, self.block_cols)
        if table[0][0] == "dense":
            return {"grad": g, "encode": False}
        units: List[dict] = []
        if table[0][0] == "slab":
            _, rows, cols, _, budget = table[0]
            u, s, vT = self._code_unit(g.reshape(rows, cols), budget)
            units.append({"u": u, "s": s, "vT": vT})
        else:
            tall, _ = _tall(g)
            total = None
            if self.allocation == "global" and self.random_sample and len(table) > 1:
                total = float(sum(torch.linalg.svdvals(tall[:, c0:c0 + cols]).sum() for _, _, cols, c0, _ in table))
            for _, rows, cols, c0, budget in table:
                if total is not None:
                    u, s, vT = self._code_unit(tall[:, c0:c0 + cols], float(self.svd_rank), max(total, 1e-30))
                else:
                    u, s, vT = self._code_unit(tall[:, c0:c0 + cols], budget)
                units.append({"u": u, "s": s, "vT": vT})
        return {"units": units, "orig_size": list(g.shape), "encode": True, "rank": self.svd_rank,
                "block_cols": self.block_cols}

    def decode(self, code, cuda: bool = False, **kwargs) -> torch.Tensor:
        if isinstance(code, tuple) and len(code) == 1:
            code = code[0]
        if not code.get("encode", False):
            return torch.as_tensor(code["grad"], dtype=torch.float32)
        shape = tuple(code["orig_size"])
        table = unit_table(shape, int(code["rank"]), int(code.get("block_cols", self.block_cols)))
        mats = [(c["u"] * c["s"].unsqueeze(0)) @ c["vT"] for c in code["units"]]
        if table[0][0] == "slab":
            return mats[0].reshape(shape)
        numel = 1
        for d in shape:
            numel *= d
        transposed = shape[0] < numel // shape[0]          # encode() coded the transpose (tall orientation)
        tall = torch.cat(mats, dim=1)
        return (tall.t() if transposed else tall).reshape(shape)

"""Spectral ATOMO: SVD atoms + unbiased atom sampling.

Behavioural parity with ``/root/reference/src/codings/svd.py``:

* matricization rules of ``_resize_to_2d`` (svd.py:12-28): 1-D ``(n,) ->
  (n/2, 2)``; trailing-ones N-D ``(a,b,1,1) -> (a,b)``; 4-D ``(a,b,h,w) ->
  (a*b/2, 2*h*w)``; 2-D untouched;
* ``encode`` (svd.py:79-118) -> ``{'u','s','vT','orig_size','reshaped',
  'encode','rank'}`` with ``s`` already divided by the sampling probability;
* ``decode`` (svd.py:160-178) -> ``(u * s) @ vT`` viewed as ``orig_size``;
* ``random_sample=False`` keeps the top-``rank`` atoms (svd.py:109-113).

Divergences (intentional, see SURVEY.md 2.9): odd-length vectors are
matricized as ``(n, 1)`` instead of crashing, tensors stay ``torch.Tensor``
(no numpy), the ``fetch_indicator`` path works, and the sampling rule/scheme
are selectable (``sampling.py``).  This per-tensor class is the oracle and the
gloo/NCCL-path coder (it runs ``torch.linalg.svd`` on whatever device the
gradient lives on); the fused engine encodes ALL layers at once with the
sm_90a kernels of ``csrc/svd_kernels.cu`` and is tested against this class.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from .coding import Coding, register
from .sampling import atom_probabilities, sample_atoms
from .utils import l1_indicator, nuclear_indicator


def matricize_shape(shape) -> Tuple[int, int]:
    """2-D shape the reference would factorize for a tensor of ``shape``."""
    shape = tuple(int(s) for s in shape)
    if len(shape) == 0:
        return (1, 1)
    if len(shape) == 1:
        n = shape[0]
        return (n // 2, 2) if n % 2 == 0 and n >= 2 else (n, 1)
    if len(shape) == 2:
        return shape
    if all(s == 1 for s in shape[2:]):
        return (shape[0], shape[1])
    rows = shape[0] * shape[1]
    cols = 1
    for s in shape[2:]:
        cols *= s
    if rows % 2 == 0:
        return (rows // 2, cols * 2)
    return (rows, cols)


def resize_to_2d(x: torch.Tensor) -> torch.Tensor:
    """Matricize ``x`` (a view when ``x`` is contiguous)."""
    m, n = matricize_shape(x.shape)
    return x.reshape(m, n)


def _gram_applicable(m: int, n: int) -> bool:
    small, big = min(m, n), max(m, n)
    return 0 < small <= 64 and big >= 4 * small


def gram_basis(mat32: torch.Tensor):
    """``(tall, V, sigma_est, transposed)``: ``tall`` is the tall orientation of the matrix, ``V`` a complete
    orthonormal basis of its row space (eigenvectors of the small Gram matrix, fp32 Gram / fp64 eigenproblem) sorted
    by ``sigma_est = sqrt(eigenvalue)`` descending."""
    m, n = mat32.shape
    tall = mat32 if m >= n else mat32.t()
    lam, v = torch.linalg.eigh((tall.t() @ tall).to(torch.float64))
    return tall, v.flip(1).to(torch.float32), lam.flip(0).clamp_min(0).sqrt().to(torch.float32), m < n


def thin_svd(mat32: torch.Tensor, gram_route: bool = True):
    """``(u, s, vT)`` of a 2-D fp32 matrix.  Tall-skinny (or short-fat) matrices — every convolution under the
    reference's matricization has 18..98 columns and 10^3..10^5 rows — go through the Gram matrix of the small side,
    exactly like the sm_90a kernels: ``V`` = eigenvectors of ``A^T A``, ``sigma_i = ||A v_i||`` measured on the
    product itself, ``u_i = A v_i / sigma_i``.  Two streaming passes over the matrix instead of LAPACK's
    bidiagonalisation (131072 x 18 on 4 CPU threads: 16 ms instead of 28 ms).  ``u_i sigma_i`` is ``A v_i`` by
    construction and ``V`` is a complete orthonormal basis, so the atoms reproduce the matrix exactly even where fp32
    cannot resolve a small singular value.  (``SVD.encode`` goes one step further and forms ``A v_i`` only for the
    atoms it sampled.)"""
    m, n = mat32.shape
    if not gram_route or not _gram_applicable(m, n):
        return torch.linalg.svd(mat32, full_matrices=False)
    tall, v, _, transposed = gram_basis(mat32)
    av = tall @ v
    s = av.norm(dim=0)
    order = torch.argsort(s, descending=True)
    s, v, av = s[order], v[:, order], av[:, order]
    u = torch.where(s > 0, av / s.clamp_min(torch.finfo(torch.float32).tiny), torch.zeros((), dtype=av.dtype))
    return (v, s, u.t()) if transposed else (u, s, v.t())


@register("svd")
class SVD(Coding):
    """Spectral-ATOMO coder.

    Parameters mirror the reference constructor (svd.py:71-77):
    ``compress``, ``rank`` (the sparsity budget ``s``; 0 -> ``p = s_i/s_0``),
    ``random_sample``, ``fetch_indicator``; plus ``prob_rule`` /
    ``scheme`` / ``max_atoms`` for the sampling variants.
    """

    def __init__(
        self,
        compress: bool = True,
        rank: int = 0,
        random_sample: bool = True,
        fetch_indicator: Optional[bool] = None,
        prob_rule: str = "reference",
        scheme: str = "bernoulli",
        max_atoms: Optional[int] = None,
        generator: Optional[torch.Generator] = None,
        gram_route: bool = True,
        *args,
        **kwargs,
    ):
        super().__init__()
        self.gram_route = bool(gram_route)      # False = always torch.linalg.svd (the NCCL baseline arm)
        self.svd_rank = int(rank)
        self.random_sample = random_sample
        self.compress = compress
        self.prob_rule = prob_rule
        self.scheme = scheme
        self.max_atoms = max_atoms
        self.generator = generator
        self._fetch_indicator = fetch_indicator

    # ------------------------------------------------------------------
    def encode(self, grad: torch.Tensor, **kwargs) -> dict:
        if not self.compress:
            return {"grad": grad, "encode": False}
        orig_size = list(grad.shape)
        reshaped = grad.dim() != 2
        mat = resize_to_2d(grad) if reshaped else grad
        mat32 = mat.detach().to(torch.float32)
        lazy = self.gram_route and _gram_applicable(*mat32.shape)
        if lazy:
            # like the kernels: basis + singular-value estimates from the small Gram matrix, sample, and only then
            # form A v_i for the atoms that were kept (ResNet-18 on 4 CPU threads: 0.15 -> 0.06 s per step)
            tall, v_all, s, transposed = gram_basis(mat32)
            u = vT = None
        else:
            u, s, vT = thin_svd(mat32, False)

        if self._fetch_indicator:
            print(
                "Step: {}, Nuclear Indicator: {}, L1 Indicator: {}".format(
                    kwargs.get("step", -1), nuclear_indicator(mat32, s), l1_indicator(mat32)
                )
            )

        if self.random_sample:
            if float(s[0]) < 1e-6:  # degenerate spectrum (svd.py:50-51)
                idx = torch.zeros(1, dtype=torch.long)
                probs = torch.ones(1, dtype=s.dtype)
            else:
                p = atom_probabilities(s, self.svd_rank, self.prob_rule)
                idx = sample_atoms(
                    p,
                    scheme=self.scheme,
                    generator=self.generator,
                    uniforms=kwargs.get("uniforms"),
                    max_atoms=self.max_atoms,
                )
                probs = p.cpu()[idx]
            idx_d = idx.to(s.device)
            scale = 1.0 / probs.to(s.device, s.dtype)
        elif self.svd_rank > 0:
            idx_d = torch.arange(min(self.svd_rank, s.numel()), device=s.device)
            scale = torch.ones(idx_d.numel(), dtype=s.dtype, device=s.device)
        else:
            idx_d = torch.arange(s.numel(), device=s.device)
            scale = torch.ones(idx_d.numel(), dtype=s.dtype, device=s.device)
        if lazy:
            v_sel = v_all[:, idx_d]
            av = tall @ v_sel                                  # the only pass over the matrix besides the Gram
            norm = av.norm(dim=0)
            u_sel = torch.where(norm > 0, av / norm.clamp_min(torch.finfo(torch.float32).tiny),
                                torch.zeros((), dtype=av.dtype))
            s = norm * scale                                   # u_i s_i = (A v_i) / p_i exactly
            u, vT = (v_sel, u_sel.t()) if transposed else (u_sel, v_sel.t())
        else:
            u, s, vT = u[:, idx_d], s[idx_d] * scale, vT[idx_d, :]

        return {
            "u": u.contiguous(),
            "s": s.contiguous(),
            "vT": vT.contiguous(),
            "orig_size": orig_size,
            "reshaped": reshaped,
            "encode": True,
            "rank": self.svd_rank,
        }

    # kept for API parity with svd.py:120-158; CUDA tensors take the same path
    def encode_cuda(self, grad: torch.Tensor, device=None, **kwargs) -> dict:
        if not grad.is_cuda:
            raise ValueError("Object passed wasn't set on CUDA, please check CUDA availability!")
        return self.encode(grad, **kwargs)

    def decode(self, encode_output, cuda: bool = False, **kwargs) -> torch.Tensor:
        if isinstance(encode_output, tuple) and len(encode_output) == 1:
            encode_output = encode_output[0]
        if not encode_output.get("encode", False):
            grad = torch.as_tensor(encode_output["grad"], dtype=torch.float32)
            return grad.cuda(non_blocking=True) if cuda else grad
        u, s, vT = (encode_output[k] for k in ("u", "s", "vT"))
        grad = (u * s.unsqueeze(0)) @ vT
        grad = grad.reshape(encode_output["orig_size"])
        return grad.cuda(non_blocking=True) if cuda else grad

"""QSGD / TernGrad stochastic quantizer with uint64-style bit packing.

Behavioural parity with ``/root/reference/src/codings/qsgd.py``:

* ``scheme in {'qsgd','terngrad'}``, ``bucket_size`` (default 512, 0 = whole
  tensor), ``quantization_level`` q -> ``s = 2**q - 1`` levels (qsgd.py:14-17,49);
* qsgd norm = L2 of the bucket; terngrad norm = L-inf after clipping to
  ``2.5*std`` (qsgd.py:42-47, 212-216), and decode can use the max norm over a
  list of codes (qsgd.py:103-104);
* packing: ``E = floor(64/(2+q))`` elements per 64-bit word, *section-major*:
  word ``j`` of a bucket holds elements ``j, j+L, j+2L, ...`` (``L`` words per
  bucket) with section 0 in the most significant bits; each element is
  ``(sign+1) << q | level`` (qsgd.py:52-78).

TernGrad differences from the reference, on purpose: the clip limit ``2.5*std`` is taken over the WHOLE tensor
(not per bucket) and the per-bucket L-inf norm is taken AFTER clipping, so a clipped element quantizes to the top
level instead of overflowing it.

Fixed defects (SURVEY.md 2.9): stochastic rounding is *unbiased* (round up with
probability ``frac``; the reference rounds up with ``1-frac``), the level never
overflows into the sign bits, and buckets need not divide the tensor (the tail
bucket is zero-padded).  The code is a flat dict of tensors
(``words`` int64 ``[B, L]``, ``norms`` fp32 ``[B]``) — the same layout the
sm_90a kernel (``csrc/qsgd_kernels.cu``) writes into PS peer memory.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from .coding import Coding, register


def words_per_bucket(bucket: int, q: int) -> int:
    e = 64 // (2 + q)
    return (bucket + e - 1) // e


def grad_clip_limit(grad: torch.Tensor, clip_factor: float = 2.5) -> float:
    """qsgd.py:212-216"""
    if clip_factor > 1.0e-5:
        return clip_factor * float(grad.reshape(-1).std(unbiased=False))
    return float(grad.abs().max())


@register("qsgd")
class QSGD(Coding):
    def __init__(self, scheme: str = "qsgd", bucket_size: int = 512, quantization_level: int = 4,
                 generator: Optional[torch.Generator] = None, *args, **kwargs):
        super().__init__()
        if scheme not in ("qsgd", "terngrad"):
            raise ValueError("scheme must be 'qsgd' or 'terngrad'")
        self.scheme = scheme
        self._quantization_level = int(quantization_level)
        self._bucket_size = int(bucket_size)
        self.generator = generator
        if not 1 <= self._quantization_level <= 30:
            raise ValueError("quantization_level must be in [1, 30]")

    # ------------------------------------------------------------------
    @property
    def levels(self) -> int:
        return (1 << self._quantization_level) - 1

    @property
    def elems_per_word(self) -> int:
        return 64 // (2 + self._quantization_level)

    def _bucketize(self, flat: torch.Tensor):
        n = flat.numel()
        bucket = self._bucket_size if self._bucket_size > 0 else max(n, 1)
        # a tensor smaller than one bucket (biases, BN vectors, a 10-way fc bias) is ONE bucket of its own length:
        # padding it to 512 elements would send 416 B for a 40 B tensor (the reference's np.split gives
        # ceil(n/512) short buckets, qsgd.py:32-40)
        bucket = max(1, min(bucket, n))
        nb = (n + bucket - 1) // bucket
        padded = torch.zeros(nb * bucket, dtype=torch.float32, device=flat.device)
        padded[:n] = flat
        return padded.view(nb, bucket), bucket, nb

    def encode(self, v: torch.Tensor, uniforms: Optional[torch.Tensor] = None, **kwargs) -> dict:
        q = self._quantization_level
        s = self.levels
        E = self.elems_per_word
        shape = list(v.shape)
        flat = v.detach().reshape(-1).to(torch.float32)
        w, bucket, nb = self._bucketize(flat)

        if self.scheme == "terngrad":
            # clip the whole tensor to 2.5 sigma, then per-bucket L-inf norm
            limit = grad_clip_limit(flat) if flat.numel() > 1 else float(flat.abs().max())
            if limit > 0:
                w = w.clamp(-limit, limit)
            norms = w.abs().amax(dim=1)
        else:
            norms = w.norm(dim=1)

        safe = torch.where(norms > 0, norms, torch.ones_like(norms)).unsqueeze(1)
        a = (w.abs() / safe * s).clamp(max=float(s))
        low = torch.floor(a)
        frac = a - low
        if uniforms is None:
            dice = torch.rand(w.shape, generator=self.generator, dtype=torch.float32).to(w.device)
        else:
            dice = uniforms.reshape(-1)[: w.numel()].view_as(w).to(w.device, torch.float32)
        xi = (low + (dice < frac).to(torch.float32)).to(torch.int64).clamp_(max=s)
        sign = (torch.sign(w) + 1).to(torch.int64)  # {0,1,2}
        elem = (sign << q) | xi

        L = words_per_bucket(bucket, q)
        pad = L * E - bucket
        if pad:
            elem = torch.cat(
                [elem, torch.full((nb, pad), 1 << q, dtype=torch.int64, device=elem.device)], dim=1
            )  # padding encodes sign=+0 (value 1<<q -> sign field 1, level 0)
        elem = elem.view(nb, E, L)
        words = torch.zeros(nb, L, dtype=torch.int64, device=elem.device)
        for i in range(E):
            words = (words << (2 + q)) | elem[:, i, :]
        return {
            "words": words,
            "norms": norms.to(torch.float32),
            "quantization_level": q,
            "bucket_size": bucket,
            "shape": shape,
            "scheme": self.scheme,
        }

    def encode_cuda(self, v: torch.Tensor, **kwargs) -> dict:
        if not v.is_cuda:
            raise ValueError("Object passed wasn't set on CUDA, please check CUDA availability!")
        return self.encode(v, **kwargs)

    def _get_max_norm(self, codes: List[dict]) -> torch.Tensor:
        out = codes[0]["norms"]
        for c in codes[1:]:
            out = torch.maximum(out, c["norms"].to(out.device))
        return out

    def decode(self, code: dict, cuda: bool = False, codes: Optional[List[dict]] = None, **kwargs) -> torch.Tensor:
        q = int(code["quantization_level"])
        s = (1 << q) - 1
        E = 64 // (2 + q)
        words = code["words"]
        norms = code["norms"]
        if code.get("scheme", self.scheme) == "terngrad" and codes:
            norms = self._get_max_norm(codes)
        nb, L = words.shape
        bucket = int(code["bucket_size"])
        mask_xi = (1 << q) - 1
        elems = torch.empty(nb, E, L, dtype=torch.int64, device=words.device)
        wcur = words.clone()
        for i in range(E - 1, -1, -1):
            elems[:, i, :] = wcur & ((1 << (2 + q)) - 1)
            wcur = wcur >> (2 + q)
        elems = elems.view(nb, E * L)[:, :bucket]
        xi = (elems & mask_xi).to(torch.float32)
        sign = ((elems >> q) & 3).to(torch.float32) - 1.0
        vals = sign * xi * (norms.to(torch.float32).unsqueeze(1) / s)
        numel = 1
        for d in code["shape"]:
            numel *= d
        out = vals.reshape(-1)[:numel].reshape(code["shape"])
        return out.cuda() if cuda else out


@register("terngrad")
class TernGrad(QSGD):
    """``--code terngrad``: QSGD machinery with the TernGrad norm/clipping."""

    def __init__(self, *args, **kwargs):
        kwargs["scheme"] = "terngrad"
        super().__init__(*args, **kwargs)

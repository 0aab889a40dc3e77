"""Scaled sign: one bit per element and one fp32 scale per bucket (EF-SignSGD).

The dense contractive code for error feedback (Karimireddy et al. 2019, "Error Feedback Fixes SignSGD"): a bucket ``b``
is sent as ``C(b) = (||b||_1 / |b|) * sign(b)``.  Its error has a closed form,
``||b - C(b)||^2 = ||b||^2 - ||b||_1^2 / |b| <= (1 - 1/|b|) ||b||^2``, so a residual fed back step after step stays
bounded.  Without error feedback the code is biased.

This coder is the oracle of the bf16 engine's sign units (``csrc/v2_sign.cu``), applied to the physical-order bf16
vector of a weight tensor:

* the input is the bf16 rounding of the tensor with bf16 subnormals (``|x| < 2^-126``) flushed to zero, so the result
  does not depend on how a compiler treats fp32 subnormals (:func:`bf16_flushed`);
* buckets of ``bucket = min(bucket_size, numel)`` elements; the last bucket has ``blen <= bucket`` real elements;
* ``scale = fp32(L1 / blen)`` with ``L1 = sum |x_i|`` over the real elements in fp64, summed in the kernel's fixed
  order (:func:`bucket_l1`), so the scale has the kernel's bits;
* ``L = ceil(bucket / 64)`` uint64 words per bucket; bit ``i`` of word ``j`` is element ``64 j + i`` and is set when
  ``x < 0`` (``+0``, ``-0`` and NaN decode to ``+scale``); padding bits are 0;
* element ``i`` decodes to ``bit ? -scale : +scale``.  A bucket holding an Inf or NaN has a non-finite scale and
  decodes to non-finite values; the other buckets are unaffected;
* no random numbers: the code depends only on the bf16 values.
"""
from __future__ import annotations

import numpy as np
import torch

from .coding import Coding, register

SIGN_MIN_BUCKET, SIGN_MAX_BUCKET = 64, 4096


def check_bucket_size(bucket_size: int, code: str = "sign") -> int:
    """The bucket rule of the sign and fp8 codes: a multiple of 64 in ``[64, 4096]``."""
    b = int(bucket_size)
    if not (SIGN_MIN_BUCKET <= b <= SIGN_MAX_BUCKET and b % 64 == 0):
        raise ValueError("%s: bucket_size must be a multiple of 64 in [%d, %d] (got %r)"
                         % (code, SIGN_MIN_BUCKET, SIGN_MAX_BUCKET, bucket_size))
    return b


def bucket_l1(a: np.ndarray) -> np.ndarray:
    """fp64 L1 norm of each row of ``a`` (``[buckets, bucket]`` magnitudes, zero past ``blen``) in the kernel's order:
    lane ``l`` of a warp adds elements ``8c .. 8c+7`` of chunks ``c = l, l + 32, ...`` one after the other, then the
    32 lane sums are combined by a butterfly (``v_l += v_{l ^ o}`` for ``o = 16, 8, 4, 2, 1``)."""
    nb, bucket = a.shape
    rounds = -(-bucket // 256)
    pad = np.zeros((nb, rounds * 256), dtype=np.float64)
    pad[:, :bucket] = a
    pad = pad.reshape(nb, rounds, 32, 8)
    acc = np.zeros((nb, 32), dtype=np.float64)
    for r in range(rounds):
        for i in range(8):
            acc = acc + pad[:, r, :, i]
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, lanes ^ o]
    return acc[:, 0]


def bf16_flushed(grad: torch.Tensor) -> np.ndarray:
    """The flat fp32 values of ``bf16(grad)`` with subnormals replaced by zero (what the kernels read)."""
    x = grad.detach().reshape(-1).to(torch.bfloat16).float().cpu().numpy().copy()
    x[np.abs(x) < np.float32(2.0 ** -126)] = 0.0
    return x


@register("sign")
class ScaledSign(Coding):
    def __init__(self, bucket_size: int = 512, *args, **kwargs):
        super().__init__()
        self.bucket_size = check_bucket_size(bucket_size)

    def bucket_for(self, numel: int) -> int:
        return min(self.bucket_size, max(int(numel), 1))

    def encode(self, grad: torch.Tensor, **kwargs) -> dict:
        shape = list(grad.shape)
        x = bf16_flushed(grad)
        n = x.size
        bucket = self.bucket_for(n)
        nb = -(-n // bucket)
        L = -(-bucket // 64)
        xb = np.zeros(nb * bucket, dtype=np.float32)
        xb[:n] = x
        xb = xb.reshape(nb, bucket)
        blen = np.minimum(bucket, n - np.arange(nb) * bucket)
        l1 = bucket_l1(np.abs(xb).astype(np.float64))
        with np.errstate(invalid="ignore"):
            scales = (l1 / blen.astype(np.float64)).astype(np.float32)
        bits = np.zeros((nb, L * 64), dtype=np.uint64)
        bits[:, :bucket] = (xb < 0).astype(np.uint64)
        weights = np.left_shift(np.uint64(1), np.arange(64, dtype=np.uint64))
        words = (bits.reshape(nb, L, 64) * weights).sum(axis=2, dtype=np.uint64)
        return {"words": torch.from_numpy(words.view(np.int64).copy()), "scales": torch.from_numpy(scales),
                "bucket_size": bucket, "numel": n, "shape": shape}

    @staticmethod
    def decode_flat(code: dict) -> torch.Tensor:
        words = code["words"].cpu().numpy().view(np.uint64)
        nb, L = words.shape
        bits = (words[:, :, None] >> np.arange(64, dtype=np.uint64)) & np.uint64(1)
        bits = bits.reshape(nb, L * 64)[:, :int(code["bucket_size"])]
        scales = code["scales"].cpu().numpy().astype(np.float32)[:, None]
        out = np.where(bits != 0, -scales, scales).astype(np.float32).reshape(-1)[:int(code["numel"])]
        return torch.from_numpy(out.copy())

    def decode(self, code: dict, cuda: bool = False, **kwargs) -> torch.Tensor:
        out = self.decode_flat(code).reshape(code["shape"])
        return out.cuda() if cuda else out

    def error_sq(self, grad: torch.Tensor) -> float:
        """Exact ``sum (x - C(x))^2`` in fp64 of one encode of ``grad`` (``x`` = :func:`bf16_flushed`)."""
        x = torch.from_numpy(bf16_flushed(grad)).double()
        return float((x - self.decode_flat(self.encode(grad)).double()).square().sum())

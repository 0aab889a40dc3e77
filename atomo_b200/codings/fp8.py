"""FP8 (e4m3) with stochastic rounding: one e4m3 byte per element and one power-of-two fp32 scale per bucket.

An unbiased dense 8-bit code.  A bucket is scaled by ``2^k`` so that its largest magnitude lands in ``(224, 448]``,
the top binade of e4m3, and each scaled magnitude ``y`` is rounded to one of its two e4m3 neighbours ``lo <= y < hi``
with ``P(hi) = (y - lo) / (hi - lo)``, so ``E[decode] = x``.  Because e4m3 spacing is relative (3 mantissa bits), the
relative variance of the code hardly depends on how the gradient is distributed.  Its expected error has the closed
form ``sum (y - lo)(hi - y) 2^-2k`` (:meth:`FP8.expected_error_sq`).

This coder is the oracle of the bf16 engine's fp8 units (``csrc/v2_fp8.cu``), applied to the physical-order bf16
vector of a weight tensor; the kernels match it bit for bit:

* the input is :func:`codings.sign.bf16_flushed` (bf16 subnormals read as zero); buckets of
  ``bucket = min(bucket_size, numel)`` elements, ``bucket_size`` a multiple of 64 in ``[64, 4096]``;
* ``amax`` is the largest magnitude of the bucket, ``k`` is taken from its exponent bits so that ``amax 2^k`` lies in
  ``(224, 448]``, clamped to ``k <= 117`` (every non-zero decoded value stays an fp32 normal); the scale stored is the
  fp32 ``2^-k``.  An all-zero bucket stores scale 0; a bucket holding an Inf or NaN, or with ``amax >= 2^126``, stores
  scale NaN and zero bytes, so it decodes to NaN and the other buckets are unaffected;
* ``y = |x| 2^k`` (exact); ``y < 2^-126`` counts as zero.  ``lo`` is ``y`` with its mantissa truncated to 3 bits when
  ``y >= 2^-6``, else ``floor(y 2^9) 2^-9``; ``ulp`` is the e4m3 spacing there and ``p = (y - lo) / ulp`` (exact);
* one 24-bit uniform per element: word ``e & 3`` of Philox4x32-10 (:func:`codings.powersgd.philox`) keyed by
  ``seed ^ FP8_KEY_XOR`` with counter ``(e >> 2, unit, step, worker)``, as ``(w >> 8) / 2^24``; the element keeps
  ``hi = lo + ulp`` when ``u < p``, else ``lo``;
* the byte is the e4m3fn encoding of the chosen value with the sign of ``x``; a zero result is ``0x00``.  Bucket ``j``
  holds ``8 ceil(bucket / 8)`` bytes (zero padded) in element order;
* decode: ``byte -> f16 -> f32`` (exact) times the scale, an exact fp32 product.
"""
from __future__ import annotations

import numpy as np
import torch

from .coding import Coding, register
from .powersgd import philox
from .sign import bf16_flushed, check_bucket_size

FP8_KEY_XOR = 0xF8E43A5C96D1B207      # the seed of the rounding draws differs from the other codes'
E4M3_MAX = 448.0
K_MAX = 117                           # 2^-9 (the least e4m3 value) * 2^-117 = 2^-126
SPECIAL_AMAX = 2.0 ** 126


def e4m3_table() -> np.ndarray:
    """fp64 value of every e4m3fn byte (``0x7f`` / ``0xff`` are NaN): sign bit 7, exponent bits 6..3 (bias 7),
    mantissa bits 2..0, subnormals at exponent 0."""
    b = np.arange(256)
    e, m = (b >> 3) & 15, (b & 7).astype(np.float64)
    mag = np.where(e == 0, m * 2.0 ** -9, (1.0 + m / 8.0) * np.exp2(e - 7.0))
    mag = np.where((e == 15) & (m == 7), np.nan, mag)
    return np.where(b >= 128, -mag, mag)


def e4m3_encode(v: np.ndarray) -> np.ndarray:
    """Byte of each non-negative e4m3 value ``v`` (exactly representable, at most 448)."""
    v = np.asarray(v, dtype=np.float64)
    mant, ex = np.frexp(np.where(v > 0, v, 1.0))          # v = mant 2^ex, mant in [0.5, 1)
    e = ex - 1
    normal = ((e + 7) << 3) + np.rint((mant * 2.0 - 1.0) * 8.0).astype(np.int64)
    sub = np.rint(v * 2.0 ** 9).astype(np.int64)
    return np.where(v >= 2.0 ** -6, normal, sub).astype(np.uint8)


def scale_exponents(amax: np.ndarray) -> np.ndarray:
    """``k`` of each finite, non-zero fp32 ``amax < 2^126``: ``amax 2^k`` in ``(224, 448]``, clamped to ``<= 117``.
    With ``amax = m 2^E`` (``m`` in ``[1, 2)``), ``k = 7 - E`` when ``m > 1.75``, else ``8 - E``."""
    bits = np.asarray(amax, dtype=np.float32).view(np.uint32).astype(np.int64)
    e = ((bits >> 23) & 0xFF) - 127
    k = np.where((bits & 0x7FFFFF) > 0x600000, 7, 8) - e
    return np.minimum(k, K_MAX)


def round_neighbours(y: np.ndarray):
    """``(lo, ulp)`` of scaled magnitudes ``y`` in ``[0, 448]`` (fp64, exact): ``lo`` is the largest e4m3 value
    ``<= y`` and ``ulp`` the e4m3 spacing above it."""
    y = np.asarray(y, dtype=np.float64)
    _, ex = np.frexp(np.where(y > 0, y, 1.0))
    ulp = np.where(y >= 2.0 ** -6, np.exp2(ex - 1.0 - 3.0), 2.0 ** -9)
    return np.floor(y / ulp) * ulp, ulp


def uniforms(seed: int, unit: int, step: int, worker: int, n: int) -> np.ndarray:
    """The kernel's ``n`` float32 uniforms of ``(seed, unit, step, worker)``: element ``e`` is word ``e & 3`` of
    Philox(seed ^ FP8_KEY_XOR, (e >> 2, unit, step, worker)) as ``(w >> 8) / 2^24``."""
    key = (int(seed) ^ FP8_KEY_XOR) & 0xFFFFFFFFFFFFFFFF
    w = philox(key, np.arange(-(-n // 4), dtype=np.uint64), unit, step, worker)
    words = np.stack(w, axis=1).reshape(-1)[:n]
    return ((words >> np.uint64(8)).astype(np.float64) / 16777216.0).astype(np.float32)


@register("fp8")
class FP8(Coding):
    def __init__(self, bucket_size: int = 512, seed: int = 1, *args, **kwargs):
        super().__init__()
        self.bucket_size = check_bucket_size(bucket_size, "fp8")
        self.seed = int(seed)

    def bucket_for(self, numel: int) -> int:
        return min(self.bucket_size, max(int(numel), 1))

    def _scaled(self, grad: torch.Tensor):
        """``(x, bucket, scales, k, y)``: the flushed input, the bucket, the fp32 scales, the exponents (0 for zero
        and special buckets) and the scaled magnitudes ``[buckets, bucket]`` (fp64, zero padded, zero in special
        buckets and below ``2^-126``)."""
        x = bf16_flushed(grad)
        n = x.size
        bucket = self.bucket_for(n)
        nb = -(-n // bucket)
        xb = np.zeros(nb * bucket, dtype=np.float32)
        xb[:n] = x
        a = np.abs(xb.reshape(nb, bucket)).astype(np.float64)
        amax = a.max(axis=1)                                   # NaN propagates
        special = ~np.isfinite(amax) | (amax >= SPECIAL_AMAX)
        zero = amax == 0
        ok = ~special & ~zero
        k = np.where(ok, scale_exponents(np.where(ok, amax, 1.0).astype(np.float32)), 0)
        scales = np.where(zero, 0.0, np.exp2(-k.astype(np.float64))).astype(np.float32)
        scales[special] = np.nan
        y = np.where(ok[:, None], a * np.exp2(k.astype(np.float64))[:, None], 0.0)
        y[y < 2.0 ** -126] = 0.0
        return x, bucket, scales, k, y

    def encode(self, grad: torch.Tensor, unit: int = 0, step: int = 1, worker: int = 0, u=None, **kwargs) -> dict:
        """One encode.  The draws are the kernel's Philox uniforms of ``(seed, unit, step, worker)``, or the explicit
        per-element uniforms ``u`` (``numel`` values in ``[0, 1)``) when given."""
        shape = list(grad.shape)
        x, bucket, scales, k, y = self._scaled(grad)
        n = x.size
        nb = y.shape[0]
        cols = -(-bucket // 8)
        if u is None:
            u = uniforms(self.seed, unit, step, worker, n)
        up = np.ones(nb * bucket, dtype=np.float64)            # padding: y = 0, never rounded up
        up[:n] = np.asarray(u, dtype=np.float32)
        lo, ulp = round_neighbours(y)
        v = np.where(up.reshape(nb, bucket) < (y - lo) / ulp, lo + ulp, lo)
        byte = e4m3_encode(v)
        neg = np.zeros(nb * bucket, dtype=bool)
        neg[:n] = x < 0
        byte = np.where(neg.reshape(nb, bucket) & (v > 0), byte | np.uint8(0x80), byte).astype(np.uint8)
        out = np.zeros((nb, 8 * cols), dtype=np.uint8)
        out[:, :bucket] = byte
        return {"bytes": torch.from_numpy(out), "scales": torch.from_numpy(scales), "bucket_size": bucket,
                "numel": n, "shape": shape}

    @staticmethod
    def decode_flat(code: dict) -> torch.Tensor:
        table = e4m3_table().astype(np.float32)
        vals = table[code["bytes"].cpu().numpy()]
        scales = code["scales"].cpu().numpy().astype(np.float32)[:, None]
        with np.errstate(invalid="ignore"):
            out = (vals * scales).astype(np.float32)
        out = out[:, :int(code["bucket_size"])].reshape(-1)[:int(code["numel"])]
        return torch.from_numpy(out.copy())

    def decode(self, code: dict, cuda: bool = False, **kwargs) -> torch.Tensor:
        out = self.decode_flat(code).reshape(code["shape"])
        return out.cuda() if cuda else out

    def expected_error_sq(self, grad: torch.Tensor) -> float:
        """``E ||decode - x||^2 = sum (y - lo)(hi - y) 2^-2k`` in fp64 over the buckets of ``grad`` (``x`` =
        :func:`bf16_flushed`); NaN when a bucket is special."""
        _, _, scales, k, y = self._scaled(grad)
        if not np.isfinite(scales).all():
            return float("nan")
        lo, ulp = round_neighbours(y)
        per = ((y - lo) * (lo + ulp - y)).sum(axis=1)
        return float((per * np.exp2(-2.0 * k.astype(np.float64))).sum())

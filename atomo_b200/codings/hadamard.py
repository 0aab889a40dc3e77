"""Randomized-Hadamard rotated quantization: each bucket is rotated by ``H D`` and quantized between its min and max.

An unbiased dense 2 / 4 / 8-bit code (Suresh et al. 2017, the rotation of DRIVE / EDEN).  A bucket ``x`` of ``d``
elements is rotated, ``y = H_d (s * x)`` with the unnormalised Sylvester Hadamard matrix ``H_d`` and random signs
``s``, which makes its coordinates close to Gaussian whatever the gradient looks like.  ``y`` is then quantized to
``L = 2^bits`` levels between ``lo = min(y)`` and ``hi = max(y)`` with stochastic rounding, which is unbiased for any
fixed rotation; since ``H_d H_d = d I`` the decode ``x_hat = s * H_d y_hat / d`` is unbiased too.  The range
``hi - lo`` is only about ``6 ||x|| / sqrt(d)``, so the variance per byte is far below QSGD's, which scales by the
bucket's norm.  The expected error given the gradient and the drawn rotation has the closed form
``sum_b (n_b / d^2) sum_i f_i (1 - f_i) step_b^2`` (:meth:`Hadamard.expected_error_sq`).

This coder is the oracle of the bf16 engine's hadamard units (``csrc/v2_hadamard.cu``), applied to the
physical-order bf16 vector of a weight tensor; the kernels match it bit for bit.  The kernels are compiled with
flush-to-zero, so every fp32 result below that would be subnormal is a (sign-preserving) zero here too:

* the input is :func:`codings.sign.bf16_flushed` with ``-0`` read as ``+0``; ``bits`` in ``{2, 4, 8}``,
  ``bucket_size`` a power of two in ``[64, 4096]``; per tensor ``d = min(bucket_size, next_pow2(max(numel, 64)))``
  and the tail bucket is zero padded to ``d``;
* signs: element ``e`` of the padded tensor is negated when bit ``e & 31`` of word ``(e >> 5) & 3`` of
  Philox4x32-10 (:func:`codings.powersgd.philox`) keyed by ``seed ^ HADAMARD_ROT_KEY`` with counter
  ``(e >> 7, unit, step, 0)`` is set.  The counter holds no worker index: every worker rotates a bucket the same way
  in a step, so the owners apply one inverse rotation to the sum of the workers' decodes;
* rotation: butterfly stages ``h = 1, 2, 4, ..., d / 2``, each mapping the pair ``(a, b)`` at positions
  ``(i, i + h)`` (``i & h == 0``) to ``(a + b, a - b)`` in fp32; a zero result is read as ``+0``;
* a bucket whose rotated values are not all finite (an Inf or NaN input, an fp32 overflow of the sums) or whose
  ``hi - lo`` overflows stores ``lo = step = NaN`` and zero codes: it decodes to NaN and the other buckets are
  unaffected;
* ``step = (hi - lo) / (L - 1)`` in fp32.  Underflow rule: a ``step`` below ``2^-126`` (an fp32 subnormal, or
  ``hi == lo``) is stored as 0 with zero codes, and the bucket decodes to ``lo`` everywhere.  That is exact when
  ``hi == lo``; otherwise every rotated value is off by less than ``(L - 1) 2^-126``;
* ``t = (y - lo) / step`` in fp32 (both steps flushed), ``c = floor(t) + [u < t - floor(t)]`` clamped to
  ``[0, L - 1]``, with one 24-bit uniform per element: word ``e & 3`` of Philox keyed by ``seed ^ HADAMARD_Q_KEY``
  with counter ``(e >> 2, unit, step, worker)``, as ``(w >> 8) / 2^24``;
* codes are packed little-endian in uint64 words in element order, ``64 / bits`` per word, ``d bits / 64`` words per
  bucket; ``lo`` and ``step`` travel as fp32 (8 bytes per bucket);
* decode: ``y_hat = fma(c, step, lo)`` (one rounding); an owner sums the counted workers' ``y_hat`` in worker order
  starting from ``+0``, runs the same butterflies, multiplies by ``2^-log2(d)`` and by ``s``, then by the fp32
  ``1 / #counted``; positions past ``numel`` are dropped.
"""
from __future__ import annotations

import numpy as np
import torch

from .coding import Coding, register
from .powersgd import philox
from .sign import bf16_flushed

HADAMARD_ROT_KEY = 0x48D2A7E13B5C9F61   # the rotation signs: no worker in the counter
HADAMARD_Q_KEY = 0x7C1E94B2D58A3F0D     # the rounding draws: keyed per worker, as fp8's
HADAMARD_BITS = (2, 4, 8)
HADAMARD_MIN_BUCKET, HADAMARD_MAX_BUCKET = 64, 4096
FLT_MIN = np.float32(2.0 ** -126)


def check_settings(bits: int, bucket_size: int):
    """``(bits, bucket_size)`` as ints, or ``ValueError``: bits in {2, 4, 8}, a power-of-two bucket in [64, 4096]."""
    b, B = int(bits), int(bucket_size)
    if b not in HADAMARD_BITS:
        raise ValueError("hadamard: quantization_level (bits) must be 2, 4 or 8 (got %r)" % (bits,))
    if not (HADAMARD_MIN_BUCKET <= B <= HADAMARD_MAX_BUCKET and B & (B - 1) == 0):
        raise ValueError("hadamard: bucket_size must be a power of two in [%d, %d] (got %r)"
                         % (HADAMARD_MIN_BUCKET, HADAMARD_MAX_BUCKET, bucket_size))
    return b, B


def bucket_for(numel: int, bucket_size: int) -> int:
    """``d = min(bucket_size, next_pow2(max(numel, 64)))``."""
    n = max(int(numel), HADAMARD_MIN_BUCKET)
    return min(int(bucket_size), 1 << (n - 1).bit_length())


def ftz(a) -> np.ndarray:
    """fp32 with subnormals replaced by a zero of the same sign (the kernels' flush-to-zero)."""
    a = np.asarray(a, dtype=np.float32)
    with np.errstate(invalid="ignore"):
        return np.where(np.abs(a) < FLT_MIN, np.copysign(np.float32(0), a), a).astype(np.float32)


def butterflies(y: np.ndarray) -> np.ndarray:
    """``H_d`` applied to every row of ``y`` ``[buckets, d]`` (fp32): stages ``h = 1, 2, ..., d / 2`` of
    ``(a, b) -> (a + b, a - b)``, each result rounded to fp32 and flushed.  Its own inverse up to the factor ``d``."""
    y = np.asarray(y, dtype=np.float32)
    nb, d = y.shape
    h = 1
    with np.errstate(over="ignore", invalid="ignore"):
        while h < d:
            v = y.reshape(nb, d // (2 * h), 2, h)
            a, b = v[:, :, 0, :], v[:, :, 1, :]
            y = np.stack([ftz(a + b), ftz(a - b)], axis=2).reshape(nb, d)
            h *= 2
    return y


def fma32(a, b, c) -> np.ndarray:
    """fp32 ``fma(a, b, c)`` with one rounding, for ``a`` an integer below ``2^24`` (so ``a b`` is exact in fp64):
    the fp64 sum and its TwoSum error decide the one case where rounding fp64 to fp32 would round twice."""
    a, b, c = (np.asarray(v, dtype=np.float64) for v in np.broadcast_arrays(a, b, c))
    p = a * b
    with np.errstate(over="ignore", invalid="ignore"):
        s = p + c
        bb = s - p
        err = (p - (s - bb)) + (c - bb)
        r = s.astype(np.float32)
        lo32 = np.where(r.astype(np.float64) > s, np.nextafter(r, np.float32(-np.inf)), r)
        hi32 = np.nextafter(lo32, np.float32(np.inf))
        mid = (lo32.astype(np.float64) + hi32.astype(np.float64)) / 2
        tie = np.isfinite(s) & (s == mid) & (err != 0)
        r = np.where(tie, np.where(err > 0, hi32, lo32), r)
    return ftz(r)


def signs(seed: int, unit: int, step: int, n: int) -> np.ndarray:
    """``True`` where element ``e < n`` of a unit is negated by the rotation of ``(seed, unit, step)``: bit
    ``e & 31`` of word ``e >> 5`` of the Philox stream (word ``(e >> 5) & 3`` of counter ``(e >> 7, unit, step, 0)``)."""
    key = (int(seed) ^ HADAMARD_ROT_KEY) & 0xFFFFFFFFFFFFFFFF
    w = philox(key, np.arange(-(-n // 128), dtype=np.uint64), unit, step, 0)
    words = np.stack(w, axis=1).reshape(-1)
    e = np.arange(n, dtype=np.uint64)
    return ((words[e >> np.uint64(5)] >> (e & np.uint64(31))) & np.uint64(1)).astype(bool)


def uniforms(seed: int, unit: int, step: int, worker: int, n: int) -> np.ndarray:
    """The kernel's ``n`` float32 rounding uniforms of ``(seed, unit, step, worker)``: element ``e`` is word ``e & 3``
    of Philox(seed ^ HADAMARD_Q_KEY, (e >> 2, unit, step, worker)) as ``(w >> 8) / 2^24``."""
    key = (int(seed) ^ HADAMARD_Q_KEY) & 0xFFFFFFFFFFFFFFFF
    w = philox(key, np.arange(-(-n // 4), dtype=np.uint64), unit, step, worker)
    words = np.stack(w, axis=1).reshape(-1)[:n]
    return ((words >> np.uint64(8)).astype(np.float64) / 16777216.0).astype(np.float32)


@register("hadamard")
class Hadamard(Coding):
    def __init__(self, quantization_level: int = 4, bucket_size: int = 512, seed: int = 1, *args, **kwargs):
        super().__init__()
        self.bits, self.bucket_size = check_settings(quantization_level, bucket_size)
        self.seed = int(seed)

    @property
    def levels(self) -> int:
        return 1 << self.bits

    def bucket_for(self, numel: int) -> int:
        return bucket_for(numel, self.bucket_size)

    def rotate(self, grad: torch.Tensor, unit: int = 0, step: int = 1):
        """``(x, d, neg, y)``: the flushed input, the bucket, the sign flips of the padded tensor and the rotated
        buckets ``[buckets, d]`` (fp32, zeros read as ``+0``)."""
        x = bf16_flushed(grad)
        x[x == 0] = 0.0
        n = x.size
        d = self.bucket_for(n)
        nb = -(-n // d)
        xp = np.zeros(nb * d, dtype=np.float32)
        xp[:n] = x
        neg = signs(self.seed, unit, step, nb * d)
        y = butterflies(np.where(neg, -xp, xp).reshape(nb, d))
        y[y == 0] = 0.0
        return x, d, neg, y

    def _range(self, y: np.ndarray):
        """``(lo, step, bad)`` per bucket: fp32, with the NaN buckets and the underflow rule applied."""
        L = self.levels
        with np.errstate(invalid="ignore", over="ignore"):
            bad = ~np.isfinite(y).all(axis=1)
            yf = np.where(bad[:, None], 0, y).astype(np.float32)
            lo, hi = yf.min(axis=1), yf.max(axis=1)
            rng = ftz(hi - lo)
            bad |= ~np.isfinite(rng)
            st = ftz(np.where(bad, 0, rng).astype(np.float32) / np.float32(L - 1))
        st = np.where(st < FLT_MIN, np.float32(0), st).astype(np.float32)
        lo = np.where(bad, np.float32(np.nan), lo).astype(np.float32)
        st = np.where(bad, np.float32(np.nan), st).astype(np.float32)
        return lo, st, bad

    def _t(self, y, lo, st):
        """``(t, ok)``: fp32 ``(y - lo) / step`` of the buckets with a positive step (0 elsewhere)."""
        ok = (st > 0)[:, None] & np.ones_like(y, dtype=bool)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            diff = ftz(np.where(ok, y - lo[:, None], 0))
            t = ftz(np.where(ok, diff / np.where(st > 0, st, 1)[:, None], 0))
        return t, ok

    def encode(self, grad: torch.Tensor, unit: int = 0, step: int = 1, worker: int = 0, u=None, **kwargs) -> dict:
        """One encode.  The rounding draws are the kernel's Philox uniforms of ``(seed, unit, step, worker)``, or the
        explicit uniforms ``u`` (one per element of the padded tensor, ``buckets * d`` values in ``[0, 1)``)."""
        shape = list(grad.shape)
        x, d, _, y = self.rotate(grad, unit, step)
        n, nb, L = x.size, y.shape[0], self.levels
        lo, st, _ = self._range(y)
        if u is None:
            u = uniforms(self.seed, unit, step, worker, nb * d)
        u = np.asarray(u, dtype=np.float32).reshape(nb, d)
        t, ok = self._t(y, lo, st)
        fl = np.floor(t)
        c = fl + (u < (t - fl))
        c = np.where(ok, np.clip(c, 0, L - 1), 0).astype(np.uint64)
        per = 64 // self.bits
        cw = c.reshape(nb, d // per, per)
        words = np.zeros((nb, d // per), dtype=np.uint64)
        for k in range(per):
            words |= cw[:, :, k] << np.uint64(k * self.bits)
        return {"codes": torch.from_numpy(c.astype(np.uint8)), "words": torch.from_numpy(words.view(np.int64)),
                "lo": torch.from_numpy(lo), "step": torch.from_numpy(st), "bucket_size": d, "bits": self.bits,
                "numel": n, "shape": shape, "unit": unit, "step_index": step}

    @staticmethod
    def unpack(code: dict) -> np.ndarray:
        """The codes ``[buckets, d]`` unpacked from the words."""
        bits = int(code["bits"])
        w = code["words"].cpu().numpy().view(np.uint64)
        per = 64 // bits
        mask = np.uint64((1 << bits) - 1)
        c = np.stack([(w >> np.uint64(k * bits)) & mask for k in range(per)], axis=2)
        return c.reshape(w.shape[0], -1)

    @staticmethod
    def rotated_decode(code: dict) -> np.ndarray:
        """``y_hat = fma(c, step, lo)`` ``[buckets, d]`` (fp32) of one worker's code."""
        c = Hadamard.unpack(code).astype(np.float64)
        return fma32(c, code["step"].numpy()[:, None], code["lo"].numpy()[:, None])

    def unrotate(self, ysum: np.ndarray, unit: int, step: int, numel: int, inv_w: float = 1.0) -> np.ndarray:
        """The owner's inverse: butterflies, ``* 2^-log2(d)``, ``* s``, ``* fp32(inv_w)``, the first ``numel``."""
        nb, d = ysum.shape
        with np.errstate(invalid="ignore", over="ignore"):
            v = ftz(butterflies(ysum) * np.float32(1.0 / d)).reshape(-1)
            v = np.where(signs(self.seed, unit, step, nb * d), -v, v)
            if inv_w != 1.0:
                v = ftz(v * np.float32(inv_w))
        return v[:numel].astype(np.float32)

    def decode_sum(self, codes, inv_w: float = 1.0) -> torch.Tensor:
        """The owner's mean of several workers' codes of one tensor and step (the same rotation): ``y_hat`` summed
        in list order from ``+0``, then :meth:`unrotate`."""
        acc = np.zeros_like(self.rotated_decode(codes[0]))
        with np.errstate(invalid="ignore", over="ignore"):
            for c in codes:
                acc = ftz(acc + self.rotated_decode(c))
        c0 = codes[0]
        return torch.from_numpy(self.unrotate(acc, c0["unit"], c0["step_index"], c0["numel"], inv_w))

    def decode(self, code: dict, cuda: bool = False, **kwargs) -> torch.Tensor:
        out = self.decode_sum([code]).reshape(code["shape"])
        return out.cuda() if cuda else out

    def decode_flat(self, code: dict) -> torch.Tensor:
        return self.decode_sum([code])

    def expected_error_sq(self, grad: torch.Tensor, unit: int = 0, step: int = 1) -> float:
        """``E ||decode - x||^2`` given ``grad`` and the rotation of ``(unit, step)``, in fp64:
        ``sum_b (n_b / d^2) sum_i f_i (1 - f_i) step_b^2`` with ``f_i = t_i - floor(t_i)`` (0 where the code is
        clamped to ``L - 1``) and ``n_b`` the bucket's real elements; NaN when a bucket is special."""
        x, d, _, y = self.rotate(grad, unit, step)
        lo, st, bad = self._range(y)
        if bad.any():
            return float("nan")
        t, ok = self._t(y, lo, st)
        fl = np.floor(t)
        f = np.where(ok & (fl < self.levels - 1), (t - fl).astype(np.float64), 0.0)
        nb = y.shape[0]
        n_b = np.minimum(d, x.size - np.arange(nb) * d).astype(np.float64)
        per = (f * (1.0 - f)).sum(axis=1) * st.astype(np.float64) ** 2
        return float((per * n_b / float(d) ** 2).sum())

"""Momentum correction with momentum-factor masking (Lin et al. 2018, Deep Gradient Compression) for top-k with error
feedback: the fp32 oracle of the bf16 engine's worker-side passes (``csrc/v2_momentum.cu`` and the masking epilogue
of ``v2_topk_encode_mc_kernel``).

Every value is float32 and every sum and product is one correctly rounded numpy operation, in the kernels' order, so
the engine matches this replay bit for bit.  Per weight tensor of one worker, in physical order:

    d = wd > 0 ? g + wd * w : g          g: the bf16 gradient, w: the worker's bf16 weight
    u = m * u + d
    s = nesterov ? d + m * u : u
    A = s + e;  b = bf16(A);  e = A - b  the coded input b, and the rounding remainder
    kept = TopK.select(b)                 the top-k encode on b, unchanged
    e = e + (b where not kept, else 0)    the error-feedback epilogue: kept entries are sent exactly
    u[kept] = 0                           momentum-factor masking

and per vector (sent exactly, not masked): ``d = wd > 0 ? v + wd * p : v``, ``u = m * u + d``, ``v = nesterov ?
d + m * u : u``.  The parameter server then runs plain SGD on the mean of what the workers sent.  With ``m = 0`` and
``wd = 0`` the weight pass is the error-feedback apply ``A = g + e`` exactly.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np
import torch

from ..codings.topk import TopK

f32 = np.float32


def _bf16(x: np.ndarray) -> np.ndarray:
    """Round-to-nearest-even bf16 of an fp32 array, as fp32."""
    return torch.from_numpy(np.ascontiguousarray(x, dtype=f32)).to(torch.bfloat16).float().numpy()


def _direction(d: np.ndarray, u: np.ndarray, m: float, nesterov: bool) -> Tuple[np.ndarray, np.ndarray]:
    u = f32(m) * u + d
    return (d + f32(m) * u if nesterov else u), u


def mc_apply(g: np.ndarray, w: np.ndarray, u: np.ndarray, e: np.ndarray, m: float, wd: float = 0.0,
             nesterov: bool = False) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The apply pass of one weight tensor: ``(b, u, e)`` after it, with ``b = bf16(A)`` the coded input (fp32
    values) and ``e = A - b``.  ``w`` is read only when ``wd > 0``."""
    g, u, e = (np.asarray(x, dtype=f32) for x in (g, u, e))
    d = g + f32(wd) * np.asarray(w, dtype=f32) if wd > 0 else g
    s, u = _direction(d, u, m, nesterov)
    a = s + e
    b = _bf16(a)
    return b, u, a - b


def mc_apply_vector(v: np.ndarray, p: np.ndarray, u: np.ndarray, m: float, wd: float = 0.0,
                    nesterov: bool = False) -> Tuple[np.ndarray, np.ndarray]:
    """The apply pass of one vector: ``(v, u)`` after it, ``v`` the direction pushed in place of the gradient."""
    v, u = np.asarray(v, dtype=f32), np.asarray(u, dtype=f32)
    d = v + f32(wd) * np.asarray(p, dtype=f32) if wd > 0 else v
    return _direction(d, u, m, nesterov)


def mc_encode(b: np.ndarray, u: np.ndarray, e: np.ndarray, coder: TopK) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The top-k encode of ``b`` with its error-feedback epilogue and momentum-factor masking: ``(kept indices,
    u, e)``."""
    kept = coder.select(torch.from_numpy(np.asarray(b, dtype=f32))).numpy()
    owed = np.asarray(b, dtype=f32).copy()
    owed[kept] = 0
    u = np.asarray(u, dtype=f32).copy()
    u[kept] = 0
    return kept, u, np.asarray(e, dtype=f32) + owed


def mc_step(g: np.ndarray, w: np.ndarray, u: np.ndarray, e: np.ndarray, coder: TopK, m: float, wd: float = 0.0,
            nesterov: bool = False) -> dict:
    """One worker step of one weight tensor: the apply pass, then the encode.  Returns the coded input ``b``, the
    kept indices and the sent values ``b[kept]``, and the state ``u`` / ``e`` after the step."""
    b, u, e = mc_apply(g, w, u, e, m, wd, nesterov)
    kept, u, e = mc_encode(b, u, e, coder)
    return {"b": b, "kept": kept, "sent": b[kept], "u": u, "e": e}

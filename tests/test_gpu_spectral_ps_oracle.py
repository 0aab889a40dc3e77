"""The bf16 engine's spectral parameter server (``ps_spectral`` in ``csrc/v2_ps.cu``) against an fp64 oracle, on worker
slots written straight into the arena.

No encode runs.  Every (unit, worker) slot gets a designed atom count and designed factors, so the test chooses what
the kernel must handle: empty tiles, ragged groups of 4 atoms, full slots, per-worker offsets that straddle the 32-atom
chunks, and totals of 31, 32, 33, 64, 65 and ``W * rcap`` atoms per unit.  The oracle is plain PyTorch in float64:

* ``oracle_decode``: the mean ``sum_w U_w[:, :c_w] diag(s_w) V_w[:c_w] / |mask|`` of a coded unit;
* ``oracle_scatter``: those means placed in the physical weight order through the reference's matricization (the
  reshape ``H2.unit_matrix`` reads with), plus the means of the dense bf16 weights and of the fp32 vectors;
* ``oracle_step``: the rule of ``opt_update`` (``csrc/v2_ps_common.cuh``).

Exact mode uses dyadic inputs whose every product and partial sum is exact in fp32, in any order, so the kernel must
equal the oracle bit for bit.  Bounded mode uses random fp32 factors and compares each step with an error bound carried
through the fp32 operations the kernel performs (``Val``).
"""
import math

import numpy as np
import pytest
import torch

from atomo_b200.ops import plan2 as P

from shadow_harness import H2, MODELS, model_shapes

gpu = pytest.mark.gpu
SIG_PUSH, SIG_PARAM, SIG_MASK = 0, 256, 320
MAX_WORKERS = 16
ERR2_SLOT_STEP = 4
KC = 32                              # atoms per chunk of the PS (PS2_KC)
U32 = 2.0 ** -24                     # unit roundoff of fp32
ETA = 2.0 ** -126                    # the kernels flush results below the smallest normal to zero
LR_EXACT = 2.0 ** -6

# the odd paths: a 5x5 slab (50 columns); 301 rows (PS tiles of 144, 144 and 13 rows) cut into blocks of 32 and 8
# columns; a wide fc (transposed, cs = 512); transposed with cs = 300 and a 7-column matrix (scalar epilogue); the
# 3-channel stem and 15- and 81-element tensors (DENSE16, tail loop); vectors of 64, 7 and 10 elements
ODD_SHAPES = [(32, 16, 5, 5), (301, 40), (10, 512), (20, 300), (300, 7), (64, 3, 3, 3), (3, 5), (9, 9),
              (64, 32, 3, 3), (64,), (7,), (10,)]

# atom-count patterns of a unit: all empty, all full, ragged per-worker counts, random, and fixed totals
PATTERNS = ("zero", "full", "ragged", "random", 31, 32, 33, 64, 65)


def f32(x):
    return float(np.float32(x))


def _coded(plan):
    return [u for u in plan.units if u.coded]


# ------------------------------------------------------------------------------------------------------- the oracle
def oracle_decode(U, S, V, counts, workers, divisor):
    """Mean of the decoded atoms of one coded unit: sum over `workers` of U[w][:, :c] diag(S[w][:c]) V[w][:c], over
    `divisor`.  U: [W][rows][rcap], S: [W][rcap], V: [W][rcap][cols], float64; counts: atoms used per worker."""
    G = torch.zeros(U.shape[1], V.shape[2], dtype=torch.float64)
    for w in workers:
        c = counts[w]
        if c > 0:
            G += U[w, :, :c] @ (S[w, :c, None] * V[w, :c])
    return G / divisor


def oracle_scatter(plan, unit_mats, dense, vec):
    """Flat fp64 arrays indexed like master / vparams: coded unit matrices (tall, the reference's matricization: a slab
    is the (o*i/2, 2*kh*kw) reshape of the logical OIHW tensor, stored channels-last; a column block sits at (rs, cs)
    strides from its w_off), dense weights (physical order) and vectors."""
    flat = torch.zeros(plan.w_total, dtype=torch.float64)
    vflat = torch.zeros(plan.v_total, dtype=torch.float64)
    for u in plan.units:
        q = plan.params[u.param]
        if u.coded:
            mat = unit_mats[u.index]
            if u.kind == P.KIND_SLAB:
                o, i, kh, kw = q.shape
                flat[q.off:q.off + q.numel] = mat.reshape(o, i, kh, kw).permute(0, 2, 3, 1).reshape(-1)
            else:
                torch.as_strided(flat, (u.rows, u.cols), (u.rs, u.cs), u.w_off).copy_(mat)
        elif u.kind == P.KIND_DENSE16:
            flat[u.w_off:u.w_off + u.numel] = dense[u.index]
        elif u.kind == P.KIND_VEC:
            vflat[u.w_off:u.w_off + u.numel] = vec[u.index]
    return flat, vflat


class Opt:
    """Optimizer settings as the kernel holds them (fp32)."""

    def __init__(self, opt=P.OPT_SGD, lr=0.05, momentum=0.0, dampening=0.0, nesterov=False, wd=0.0, first_step=1):
        self.opt, self.nesterov, self.first_step = opt, nesterov, first_step
        self.lr, self.mu, self.damp, self.wd = f32(lr), f32(momentum), f32(dampening), f32(wd)
        self.b1, self.b2, self.eps = f32(0.9), f32(0.999), f32(1e-8)

    def ctrl(self, step, **kw):
        return P.pack_ctrl2(step=step, lr=self.lr, momentum=self.mu, dampening=self.damp, weight_decay=self.wd,
                            nesterov=self.nesterov, first_step=self.first_step, opt=self.opt, beta1=self.b1,
                            beta2=self.b2, eps=self.eps, **kw)


def oracle_step(o, step, p, g, m, v, vmax):
    """One step of opt_update on fp64 tensors; returns (p, m, v, vmax)."""
    g = g + o.wd * p
    if o.opt == P.OPT_SGD:
        d = g
        if o.mu != 0:
            m = g.clone() if step == o.first_step else o.mu * m + (1 - o.damp) * g
            d = g + o.mu * m if o.nesterov else m
        return p - o.lr * d, m, v, vmax
    t = step - o.first_step + 1
    m = o.b1 * m + (1 - o.b1) * g
    v = o.b2 * v + (1 - o.b2) * g * g
    vv = v
    if o.opt == P.OPT_AMSGRAD:
        vmax = torch.maximum(vmax, v)
        vv = vmax
    denom = vv.sqrt() / math.sqrt(1 - o.b2 ** t) + o.eps
    return p - o.lr / (1 - o.b1 ** t) * (m / denom), m, v, vmax


# ---------------------------------------------------------------------------------------- error bound of the step
def gamma(n):
    return n * U32 / (1 - n * U32)


class Val:
    """An fp64 value of the exact rule and a bound on |fp32 result - value|, carried through each fp32 operation of
    opt_update.  A correctly rounded operation adds u |result|; results below 2^-126 are flushed (ETA).  The
    approximate operations of the --use_fast_math build add their documented maximum error (CUDA C++ Programming Guide,
    mathematical functions): division 2 ulp, square root 3 ulp (the larger of the two figures given).  One ulp of y is at
    most 2u |y|."""

    def __init__(self, x, e=0.0):
        self.x = x
        self.e = e if torch.is_tensor(e) else torch.full_like(x, e) if torch.is_tensor(x) else e

    def _round(self, x, e, ulps=0.5):
        return Val(x, e + ulps * 2 * U32 * (abs(x) + e) + ETA)

    def __mul__(self, b):
        b = b if isinstance(b, Val) else Val(b)
        return self._round(self.x * b.x, abs(self.x) * b.e + abs(b.x) * self.e + self.e * b.e)

    def __add__(self, b):
        b = b if isinstance(b, Val) else Val(b)
        return self._round(self.x + b.x, self.e + b.e)

    def __neg__(self):
        return Val(-self.x, self.e)

    def fma(self, b, c):
        """fl(self * b + c): one rounding (a fused multiply-add, or a contraction the compiler chose)."""
        b = b if isinstance(b, Val) else Val(b)
        return self._round(self.x * b.x + c.x, abs(self.x) * b.e + abs(b.x) * self.e + self.e * b.e + c.e)

    def __truediv__(self, b):
        b = b if isinstance(b, Val) else Val(b)
        x = self.x / b.x
        den = abs(b.x) - b.e
        e = (self.e + abs(x) * b.e) / den if not torch.is_tensor(den) else \
            torch.where(den > 0, (self.e + abs(x) * b.e) / den.clamp_min(1e-300), torch.full_like(den, math.inf))
        return self._round(x, e, ulps=2)

    def sqrt(self):
        x = self.x.sqrt()
        # |sqrt(y) - sqrt(x)| = |y - x| / (sqrt(y) + sqrt(x)) <= min(sqrt(e), e / sqrt(x))
        e = torch.minimum(self.e.sqrt(), self.e / x.clamp_min(1e-300))
        return self._round(x, e, ulps=3)

    def maximum(self, b):
        return Val(torch.maximum(self.x, b.x), torch.maximum(self.e, b.e))


def _pow_bound(b, t):
    """powf(b, t) of the fast-math build is exp2(t * log2(b)) on the hardware approximations: log2 within 2^-22 absolute
    for b in [0.5, 2], one rounding of the product, exp2 within 2 ulp.  An argument error d scales the result by 2^d."""
    assert 0.5 <= b <= 2
    d = t * 2.0 ** -22 + U32 * abs(t * math.log2(b))
    x = b ** t
    return Val(torch.tensor(x, dtype=torch.float64), torch.tensor(x * ((2.0 ** d - 1) + 4 * U32 * 2.0 ** d)))


def bound_step(o, step, p, g, m, v, vmax):
    """The fp32 operations of opt_update on Val inputs (p, m, v, vmax exact: the kernel's own pre-step state).  Returns
    Vals of (p, m, v, vmax); their .x equal oracle_step's."""
    p = Val(p)
    g1 = Val(o.wd).fma(p, g)
    if o.opt == P.OPT_SGD:
        d = g1
        if o.mu != 0:
            if step == o.first_step:
                m = g1
            else:
                t = (Val(1.0) + Val(-o.damp)) * g1
                m = Val(o.mu).fma(Val(m), t)
            d = Val(o.mu).fma(m, g1) if o.nesterov else m
        pn = Val(-o.lr).fma(d, p)
        return pn, m if isinstance(m, Val) else Val(m), Val(v), Val(vmax)
    t = step - o.first_step + 1
    m = Val(o.b1).fma(Val(m), Val(1 - o.b1) * g1)            # 1 - b1 is exact in fp32 (Sterbenz)
    v = Val(o.b2).fma(Val(v), (Val(1 - o.b2) * g1) * g1)
    vv = v
    if o.opt == P.OPT_AMSGRAD:
        vmax = Val(vmax).maximum(v)
        vv = vmax
    else:
        vmax = Val(vmax)
    bc1 = Val(1.0) + (-_pow_bound(o.b1, t))
    sbc2 = (Val(1.0) + (-_pow_bound(o.b2, t))).sqrt()
    den = vv.sqrt() / sbc2 + Val(o.eps)
    upd = (Val(torch.tensor(o.lr)) / bc1) * (m / den)
    return p + (-upd), m, v, vmax


def decode_bound(abs_sum, K, divisor_exact=True):
    """|g - g*| for a decoded element whose exact terms |u s v| / |mask| sum to abs_sum, K atoms in all.  Each term
    takes at most: one rounding of s v, one per fma of its chunk (<= min(K, 32)), one of acc * inv_w, one for inv_w
    itself when 1 / |mask| is not exact, and one per later chunk added into the tile (ceil(K / 32) - 1)."""
    if K == 0:
        return abs_sum * 0
    n = min(K, KC) + 2 + (0 if divisor_exact else 1) + (-(-K // KC) - 1)
    return gamma(n) * abs_sum + ETA


def sum_bound(abs_sum, W, divisor_exact=True):
    """The same for a dense element summed over W workers in fp32: W - 1 additions, the scaling and inv_w."""
    return gamma(W - 1 + 1 + (0 if divisor_exact else 1)) * abs_sum + ETA


# --------------------------------------------------------------------------------------------------- designed slots
def _pow2(x):
    return x > 0 and x & (x - 1) == 0


def qsvd_scale(k):
    """A row scale whose fp32(scale * fp32(1/127)) is exactly 2^k (the kernel's de-quantization factor)."""
    inv = np.float32(1.0) / np.float32(127.0)
    target = np.float32(2.0 ** k)
    x = np.float32(127.0 * 2.0 ** k)
    for _ in range(64):
        for c in (x, np.nextafter(x, np.float32(np.inf))):
            if np.float32(c * inv) == target:
                return c
        x = np.nextafter(x, np.float32(0))
    raise AssertionError("no scale for 2^%d" % k)


def _counts(u, W, pattern, rng):
    rc = u.rcap
    if pattern == "zero":
        return [0] * W
    if pattern == "full":
        return [rc] * W
    base = [1, 3, 5, rc, 0, 2, 7, 6]
    if pattern == "ragged":
        return [min(base[(w + u.index) % len(base)], rc) for w in range(W)]
    if pattern == "random":
        return rng.integers(0, rc + 1, W).tolist()
    T = min(pattern, W * rc)          # a total: start ragged, then move atoms until the sum is T
    c = [min(base[w % len(base)], rc) for w in range(W)]
    while sum(c) > T:
        c[int(np.argmax(c))] -= 1
    w = 0
    while sum(c) < T:
        if c[w % W] < rc:
            c[w % W] += 1
        w += 1
    return c


class Design:
    """Worker slots, staged dense weights and vector gradients of one step, and the oracle's view of them.

    exact: U and V are multiples of 1/4 in [-3/4, 3/4], s a power of two in [1/4, 2] (QSVD: int8 codes in [-15, 15]
    and row scales de-quantizing to 2^-4 or 2^-3), staged weights multiples of 1/16 and vector gradients multiples of
    1/64.  Every product is then a multiple of 2^-8 and every partial sum stays below 2^16 (|u s v| <= 2.25 and
    K <= 320), far inside the 2^24 ulps fp32 holds exactly; so does the step p - 2^-6 g (p a multiple of 2^-8 in
    [-1, 1]).  Otherwise random fp32 factors."""

    def __init__(self, plan, W, step, exact, seed, shift=0, counts=None):
        self.plan, self.W, self.step, self.exact = plan, W, step, exact
        g = torch.Generator().manual_seed(seed)
        rng = np.random.default_rng(seed)
        self.units = {}
        for u in _coded(plan):
            rc, n, rows = u.rcap, u.cols, u.rows
            c = counts(u) if counts is not None else _counts(u, W, PATTERNS[(u.index + shift) % len(PATTERNS)], rng)
            if exact:
                S = 2.0 ** torch.randint(-2, 2, (W, rc), generator=g).double()
                V = torch.randint(-3, 4, (W, rc, n), generator=g).double() / 4
                if u.ubits == 8:
                    codes = torch.randint(-15, 16, (W, rows, rc), generator=g, dtype=torch.int8)
                    scales = torch.where(torch.rand(W, rows, generator=g) < 0.5, float(qsvd_scale(-4)),
                                         float(qsvd_scale(-3)))
                    deq = torch.tensor((scales.numpy() * (np.float32(1.0) / np.float32(127.0))).astype(np.float32))
                    U = codes.double() * deq.double()[:, :, None]
                else:
                    U = torch.randint(-3, 4, (W, rows, rc), generator=g).double() / 4
            else:
                assert u.ubits == 0
                S = (torch.rand(W, rc, generator=g) * 1.5 + 0.5).double()
                V = torch.randn(W, rc, n, generator=g).float().double()
                U = torch.randn(W, rows, rc, generator=g).float().double()
            d = dict(counts=list(c), hdr_count=list(c), hdr_step=[step] * W, S=S, V=V, U=U.float())
            if u.ubits == 8:
                d.update(codes=codes, scales=scales)
            self.units[u.index] = d
        self.stage = torch.zeros(W, plan.stage_total, dtype=torch.bfloat16)
        self.vgrads = torch.zeros(W, plan.v_total)
        for u in plan.units:
            if u.kind == P.KIND_DENSE16:
                x = torch.randint(-16, 17, (W, u.numel), generator=g).float() / 16 if exact else \
                    torch.randn(W, u.numel, generator=g)
                self.stage[:, u.rs:u.rs + u.numel] = x.to(torch.bfloat16)
            elif u.kind == P.KIND_VEC:
                self.vgrads[:, u.w_off:u.w_off + u.numel] = \
                    torch.randint(-64, 65, (W, u.numel), generator=g).float() / 64 if exact else \
                    torch.randn(W, u.numel, generator=g)

    def arena(self, garbage=()):
        """[W][arena_floats] fp32: the designed slots; atoms past a slot's count hold NaN (they must never be read into
        the sum), and workers in `garbage` hold NaN everywhere."""
        plan, W = self.plan, self.W
        A = torch.full((W, plan.arena_floats), float("nan"))
        for u in _coded(plan):
            d = self.units[u.index]
            rc, n, rows, b = u.rcap, u.cols, u.rows, u.slot_off
            live = torch.arange(rc)[None, :] < torch.tensor(d["counts"])[:, None].clamp(0, rc)     # [W][rcap]
            nan = torch.tensor(float("nan"), dtype=torch.float64)
            hdr = A[:, b:b + 4].view(torch.int32)
            hdr[:, 0] = torch.tensor(d["hdr_count"], dtype=torch.int32)
            hdr[:, 1] = torch.tensor(d["hdr_step"], dtype=torch.int32)
            A[:, b + 4:b + 4 + rc] = torch.where(live, d["S"], nan).float()
            A[:, b + 4 + rc:b + 4 + rc + rc * n] = torch.where(live[:, :, None], d["V"], nan).float().reshape(W, -1)
            uo = b + P.slot_u_off(rc, n)
            if u.ubits == 8:
                A[:, uo:uo + rows * rc // 4].view(torch.int8)[:] = d["codes"].reshape(W, -1)
                so = b + P.slot_scale_off(rows, n, rc)
                A[:, so:so + rows] = d["scales"]
            else:
                A[:, uo:uo + rows * rc] = torch.where(live[:, None, :], d["U"], nan.float()).reshape(W, -1)
        for w in garbage:
            A[w] = float("nan")
        return A

    def oracle(self, workers=None):
        """(g, gv, e, ev): the mean gradient (flat, fp64) and the bound on its fp32 decode error."""
        plan, W = self.plan, self.W
        workers = list(range(W)) if workers is None else list(workers)
        div = len(workers)
        exact_div = _pow2(div)
        mats, emats, dense, edense, vec, evec = {}, {}, {}, {}, {}, {}
        for u in _coded(plan):
            d = self.units[u.index]
            U = d["U"].double()
            mats[u.index] = oracle_decode(U, d["S"], d["V"], d["counts"], workers, div)
            absm = oracle_decode(U.abs(), d["S"].abs(), d["V"].abs(), d["counts"], workers, div)
            emats[u.index] = decode_bound(absm, sum(max(d["counts"][w], 0) for w in workers), exact_div)
        st = self.stage.double()
        for u in plan.units:
            if u.kind == P.KIND_DENSE16:
                x = st[workers, u.rs:u.rs + u.numel]
                dense[u.index] = x.sum(0) / div
                edense[u.index] = sum_bound(x.abs().sum(0) / div, div, exact_div)
            elif u.kind == P.KIND_VEC:
                x = self.vgrads.double()[workers, u.w_off:u.w_off + u.numel]
                vec[u.index] = x.sum(0) / div
                evec[u.index] = sum_bound(x.abs().sum(0) / div, div, exact_div)
        g, gv = oracle_scatter(plan, mats, dense, vec)
        e, ev = oracle_scatter(plan, emats, edense, evec)
        self.mats = mats
        return g, gv, e, ev

    def load(self, h, garbage=(), pushed=None):
        """Write the design into harness h and raise the push flags of every group (workers not in `pushed` keep the
        previous step's flag)."""
        h.arena.copy_(self.arena(garbage).reshape(-1))
        for w in range(self.W):
            bad = w in garbage
            h.stage[w].copy_(self.stage[w] if not bad else torch.full_like(self.stage[w], float("nan")))
            h.vgrads[w].copy_(self.vgrads[w] if not bad else torch.full_like(self.vgrads[w], float("nan")))
        pushed = range(self.W) if pushed is None else pushed
        for g in range(self.plan.n_groups):
            for w in range(self.W):
                h.signals[SIG_PUSH + g * MAX_WORKERS + w] = self.step if w in pushed else self.step - 1
        h.ctrl.view(torch.int32)[0] = self.step


def _harness(shapes, rank, W, code="svd", opt=None, step=1, **kw):
    h = H2(shapes, code=code, rank=rank, W=W, groups=5)
    o = opt or Opt(lr=LR_EXACT)
    h.ctrl.copy_(torch.frombuffer(bytearray(o.ctrl(step, **kw)), dtype=torch.uint8).to(h.dev))
    return h, o


def _grids(h):
    return (3 * torch.cuda.get_device_properties(h.dev).multi_processor_count, 7, 1)


def _exact_state(h, seed):
    """Dyadic master (multiples of 2^-8 in [-1, 1]) and momentum buffers that momentum 0 must leave alone."""
    g = torch.Generator().manual_seed(seed)
    pl = h.plan
    st = {"master": torch.randint(-256, 257, (pl.w_total,), generator=g).float() / 256,
          "mom": torch.randint(-256, 257, (pl.w_total,), generator=g).float() / 256,
          "vparams": torch.randint(-256, 257, (pl.v_total,), generator=g).float() / 256,
          "vmom": torch.randint(-256, 257, (pl.v_total,), generator=g).float() / 256}
    return {k: v.to(h.dev) for k, v in st.items()}


def _put(h, st):
    for k, v in st.items():
        getattr(h, k).copy_(v)
    h.wshadow.copy_(h.master.to(torch.bfloat16))


def _check_exact(h, st, g, gv, step, error=0):
    """The kernel's state after a momentum-0 SGD step of lr 2^-6 equals the oracle bit for bit."""
    want = (st["master"].double().cpu() - LR_EXACT * g).float().to(h.dev)
    vwant = (st["vparams"].double().cpu() - LR_EXACT * gv).float().to(h.dev)
    assert torch.equal(want.double().cpu(), st["master"].double().cpu() - LR_EXACT * g), "oracle step not exact"
    bad = (h.master != want).nonzero().flatten()
    assert bad.numel() == 0, ("master differs", bad[:8].tolist(), h.master[bad[:8]].tolist(), want[bad[:8]].tolist())
    assert torch.equal(h.wshadow, h.master.to(torch.bfloat16))
    assert torch.equal(h.mom, st["mom"]) and torch.equal(h.vmom, st["vmom"])
    assert torch.equal(h.vparams, vwant)
    assert int(h.ctrl.view(torch.int32)[1]) == error
    assert int(h.signals[SIG_PARAM]) == step + 1


def _run_exact(h, design, seed, grids=None, garbage=(), pushed=None, workers=None, error=0):
    g, gv, _, _ = design.oracle(workers)
    design.load(h, garbage, pushed)
    st = _exact_state(h, seed)
    for grid in grids or _grids(h):
        _put(h, st)
        h.ctrl.view(torch.int32)[1] = 0
        h.signals[SIG_PARAM] = 0
        h.ps(grid)
        _check_exact(h, st, g, gv, design.step, error)


# ------------------------------------------------------------------------------------------- CPU: oracle self-checks
class _PlanOnly:
    """What H2.unit_matrix needs, without a device."""

    def __init__(self, plan):
        self.plan, self.P = plan, P


@pytest.mark.parametrize("model", list(MODELS))
def test_scatter_inverts_unit_matrix(model):
    """oracle_scatter puts every coded unit's matrix (H2.unit_matrix of a logical gradient) back where the physical
    channels-last weight holds it; with the DENSE16 units this covers every weight element exactly once."""
    net, ds = MODELS[model]
    shapes = model_shapes(net, ds)
    pl = P.build_plan2(shapes, "svd", 3, n_groups=5)
    g = torch.Generator().manual_seed(3)
    logical, phys = {}, torch.zeros(pl.w_total, dtype=torch.float64)
    for q in pl.params:
        if q.is_w:
            t = torch.randn(q.shape, generator=g, dtype=torch.float64)
            logical[q.index] = t
            phys[q.off:q.off + q.numel] = t.permute(0, 2, 3, 1).reshape(-1) if t.dim() == 4 else t.reshape(-1)
    stub = _PlanOnly(pl)
    mats = {u.index: H2.unit_matrix(stub, u, logical).double() for u in _coded(pl)}
    dense = {u.index: phys[u.w_off:u.w_off + u.numel] for u in pl.units if u.kind == P.KIND_DENSE16}
    vec = {u.index: torch.zeros(u.numel, dtype=torch.float64) for u in pl.units if u.kind == P.KIND_VEC}
    flat, _ = oracle_scatter(pl, mats, dense, vec)
    assert torch.equal(flat, phys)
    # coverage: ones scattered from every unit reach every weight element and no padding, and the units hold as many
    # elements as the weights, so none is reached twice
    ones = {u.index: torch.ones(u.rows, u.cols, dtype=torch.float64) for u in _coded(pl)}
    dn = {u.index: torch.ones(u.numel, dtype=torch.float64) for u in pl.units if u.kind == P.KIND_DENSE16}
    count, _ = oracle_scatter(pl, ones, dn, vec)
    want = torch.zeros(pl.w_total, dtype=torch.float64)
    for q in pl.params:
        if q.is_w:
            want[q.off:q.off + q.numel] = 1
    assert torch.equal(count, want)
    assert sum(u.rows * u.cols for u in _coded(pl)) + sum(x.numel() for x in dn.values()) == int(want.sum())


OPTS = {"sgd": dict(), "momentum": dict(momentum=0.9, wd=1e-3), "dampening": dict(momentum=0.9, dampening=0.1, wd=1e-3),
        "nesterov": dict(momentum=0.9, nesterov=True, wd=1e-3), "adam": dict(opt=P.OPT_ADAM, lr=1e-2, wd=1e-3),
        "amsgrad": dict(opt=P.OPT_AMSGRAD, lr=1e-2, wd=1e-3)}


def _torch_opt(name, o, p):
    if o.opt == P.OPT_SGD:
        return torch.optim.SGD([p], lr=o.lr, momentum=o.mu, dampening=o.damp, nesterov=o.nesterov, weight_decay=o.wd)
    return torch.optim.Adam([p], lr=o.lr, betas=(o.b1, o.b2), eps=o.eps, weight_decay=o.wd,
                            amsgrad=o.opt == P.OPT_AMSGRAD)


@pytest.mark.parametrize("name", list(OPTS))
def test_step_oracle_matches_torch_optim(name):
    """oracle_step over 4 steps (first_step 3, so t = step - first_step + 1 is what matters) equals torch.optim in
    float64, and bound_step carries the same values."""
    o = Opt(first_step=3, **OPTS[name])
    g = torch.Generator().manual_seed(1)
    p0 = torch.randn(257, generator=g, dtype=torch.float64)
    p = p0.clone().requires_grad_(True)
    ref = _torch_opt(name, o, p)
    q, m, v, vmax = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0), torch.zeros_like(p0)
    for step in range(3, 7):
        grad = torch.randn(257, generator=g, dtype=torch.float64)
        p.grad = grad.clone()
        ref.step()
        bp, bm, bv, bvm = bound_step(o, step, q, Val(grad), m, v, vmax)
        q, m, v, vmax = oracle_step(o, step, q, grad, m, v, vmax)
        assert torch.allclose(q, p.detach(), rtol=1e-13, atol=1e-15), (step, float((q - p.detach()).abs().max()))
        for a, b in ((bp, q), (bm, m), (bv, v), (bvm, vmax)):
            assert torch.allclose(a.x, b, rtol=1e-13, atol=1e-15)
        if o.opt == P.OPT_SGD and o.mu:
            assert torch.allclose(m, ref.state[p]["momentum_buffer"], rtol=1e-13, atol=1e-15)
        elif o.opt != P.OPT_SGD:
            assert torch.allclose(v, ref.state[p]["exp_avg_sq"], rtol=1e-13, atol=1e-15)


def _f32_update(o, step, p, g, m, v, vmax):
    """opt_update in numpy float32 (correctly rounded operations; fmaf as one rounding of the fp64 value, which holds
    every product of two floats exactly; powf in fp64, then rounded): a stand-in for the kernel that bound_step must
    cover."""
    F = np.float32
    p, g, m, v, vmax = (np.asarray(x, dtype=F) for x in (p, g, m, v, vmax))

    def fma(a, b, c):
        return (np.float64(a) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F)
    g = fma(o.wd, p, g)
    if o.opt == P.OPT_SGD:
        d = g
        if o.mu:
            m = g if step == o.first_step else fma(o.mu, m, (F(1) - F(o.damp)) * g)
            d = fma(o.mu, m, g) if o.nesterov else m
        return fma(-o.lr, d, p), m, v, vmax
    t = step - o.first_step + 1
    m = fma(o.b1, m, (F(1) - F(o.b1)) * g)
    v = fma(o.b2, v, (F(1) - F(o.b2)) * g * g)
    vv = v
    if o.opt == P.OPT_AMSGRAD:
        vmax = np.maximum(vmax, v)
        vv = vmax
    bc1 = F(1) - F(o.b1 ** t)
    sbc2 = np.sqrt(F(1) - F(o.b2 ** t))
    return p - (F(o.lr) / bc1) * (m / (np.sqrt(vv) / sbc2 + F(o.eps))), m, v, vmax


@pytest.mark.parametrize("name", list(OPTS))
def test_step_bound_covers_an_fp32_evaluation(name):
    """A float32 evaluation of the rule, fed a gradient off by up to its decode bound, stays within bound_step of the
    fp64 oracle at every step, and the bound is small against the step (the check has teeth)."""
    o = Opt(**OPTS[name])
    g = torch.Generator().manual_seed(2)
    n = 4096
    p = torch.randn(n, generator=g).double()
    m, v, vmax = torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    for step in range(1, 5):
        gs = torch.randn(n, generator=g).double()
        eg = decode_bound(gs.abs() * 3, 100, False)
        gk = (gs + eg * (2 * torch.rand(n, generator=g).double() - 1)).float().double()
        bp, bm, bv, bvm = bound_step(o, step, p, Val(gs, eg + (gk - gs).abs()), m, v, vmax)
        kp, km, kv, kvm = (torch.from_numpy(np.asarray(x)).double() for x in _f32_update(o, step, p, gk, m, v, vmax))
        for got, b in ((kp, bp), (km, bm), (kv, bv), (kvm, bvm)):
            assert bool(((got - b.x).abs() <= b.e).all()), (step, float(((got - b.x).abs() - b.e).max()))
        assert float(bp.e.sum()) <= 1e-3 * float((bp.x - p).abs().sum())
        p, m, v, vmax = kp, km, kv, kvm


# --------------------------------------------------------------------------------------------- GPU: exact, bitwise
@gpu
@pytest.mark.parametrize("model", list(MODELS))
@pytest.mark.parametrize("rank", [1, 3, 8])
def test_ps_equals_oracle_bitwise_on_models(model, rank):
    """Every unit of the model plan at 5 groups, 16 workers (8 at rank 8: up to 160 atoms, 5 chunks): designed counts
    cover empty, ragged, full and 31 / 32 / 33 / 64 / 65 / W * rcap atoms (those rcap allows); the production grid, 7
    CTAs and one CTA give the same bits."""
    net, ds = MODELS[model]
    W = 16 if rank < 8 else 8
    h, _ = _harness(model_shapes(net, ds), rank, W)
    d = Design(h.plan, W, 1, True, seed=rank, shift=rank)
    _run_exact(h, d, seed=rank)


@gpu
@pytest.mark.parametrize("W", [1, 2, 8, 16])
@pytest.mark.parametrize("rank", [3, 8])
def test_ps_equals_oracle_bitwise_on_odd_shapes(W, rank):
    h, _ = _harness(ODD_SHAPES, rank, W)
    for shift in range(0, len(PATTERNS), 3):
        _run_exact(h, Design(h.plan, W, 1, True, seed=10 * W + shift, shift=shift + W), seed=shift)


@gpu
@pytest.mark.parametrize("shapes", ["ResNet18", "odd"])
def test_qsvd_ps_equals_oracle_bitwise(shapes):
    """int8 U with row scales whose de-quantization factor fp32(scale * fp32(1/127)) is a power of two."""
    sh = model_shapes("ResNet18") if shapes == "ResNet18" else ODD_SHAPES
    h, _ = _harness(sh, 3, 8, code="qsvd")
    assert all(u.ubits == 8 for u in _coded(h.plan))
    _run_exact(h, Design(h.plan, 8, 1, True, seed=5, shift=2), seed=5)


@gpu
@pytest.mark.parametrize("shapes", ["ResNet18", "odd"])
def test_gather_stores_the_oracle_mean_and_tile_sums(shapes):
    """The gather instantiation (clipping phase 1, as ShadowEngine._launch_ps_clip launches it): the stored mean
    gradient is the oracle's bit for bit; part[tile].x is sum g^2 of the tile within gamma_{N + 12} sum g^2 (N
    products of one thread's chain at most, then 5 shuffle and 7 warp additions)."""
    sh = model_shapes("ResNet18") if shapes == "ResNet18" else ODD_SHAPES
    W = 16
    h, _ = _harness(sh, 3, W)
    pl, C = h.plan, h.C
    d = Design(pl, W, 1, True, seed=21, shift=4)
    g, gv, _, _ = d.oracle()
    d.load(h)
    z = lambda n: torch.zeros(n, device=h.dev)
    for grid in _grids(h):
        grad, vgrad, part = z(pl.w_total), z(pl.v_total), z(2 * len(pl.ps_tiles))
        for grp in range(pl.n_groups):
            t0, nt = pl.ps_range[grp][0]
            C.v2_ps_gather(0, h.t_units.data_ptr(), h.t_ps.data_ptr(), t0, nt, W, 1, grp, 0, 0,
                           h.t_vgrads_peer.data_ptr(), h.t_stage_peer.data_ptr(), h.arena.data_ptr(), pl.arena_floats,
                           h.signals.data_ptr(), h.t_sig_peer.data_ptr(), h.ctrl.data_ptr(),
                           h.counters.data_ptr() + 4 * (pl.n_coded + 8 + grp), int(5e9), h.tstats.data_ptr(), 1.0 / W,
                           grad.data_ptr(), vgrad.data_ptr(), part.data_ptr() + 8 * t0, max(1, min(grid, nt)), 0, 0)
        torch.cuda.synchronize()
        assert int(h.ctrl.view(torch.int32)[1]) == 0
        assert torch.equal(grad.double().cpu(), g) and torch.equal(vgrad.double().cpu(), gv)
        got = part.view(-1, 2)[:, 0].double().cpu()
        for ti, (ui, a, b, _o) in enumerate(pl.ps_tiles):
            u = pl.units[ui]
            x = d.mats[ui][a:a + b] if u.coded else (g if u.kind == P.KIND_DENSE16 else gv)[u.w_off + a:u.w_off + a + b]
            want = float((x * x).sum())
            assert abs(float(got[ti]) - want) <= gamma(x.numel() + 12) * want, (ti, u.kind, float(got[ti]), want)


# ----------------------------------------------------------------------------------------------- GPU: the guards
@gpu
def test_stale_slot_adds_nothing_and_raises_the_error():
    """Worker 5's slots carry the previous step: its atoms are left out, the mean still divides by W = 8 (its dense and
    vector gradients count), and ERR2_SLOT_STEP is set."""
    W, step = 8, 3
    h, _ = _harness(ODD_SHAPES, 3, W, step=step)
    d = Design(h.plan, W, step, True, seed=31, shift=1)
    for u in _coded(h.plan):
        d.units[u.index]["hdr_step"][5] = step - 1
    g_all, _, _, _ = d.oracle()
    for u in _coded(h.plan):
        d.units[u.index]["counts"][5] = 0
    assert any(d.units[u.index]["hdr_count"][5] > 0 for u in _coded(h.plan))
    g, _, _, _ = d.oracle()
    assert not torch.equal(g, g_all)
    _run_exact(h, d, seed=31, error=ERR2_SLOT_STEP)


@gpu
def test_header_count_is_clamped_to_the_slot():
    """A header count above rcap reads rcap atoms; a negative one reads none."""
    W = 2
    h, _ = _harness(ODD_SHAPES, 3, W)
    d = Design(h.plan, W, 1, True, seed=41, counts=lambda u: [u.rcap, 0])
    for u in _coded(h.plan):
        d.units[u.index]["hdr_count"] = [u.rcap + 5, -3]
    _run_exact(h, d, seed=41)


@gpu
def test_num_aggregate_averages_exactly_the_workers_that_pushed():
    """--num-aggregate 2 of W = 3: worker 1 has not pushed this step and its slots, staging and vector gradients hold
    NaN; the mean is over workers 0 and 2 (inv_w = 1/2) and the published mask is 0b101."""
    W, step = 3, 2
    h, _ = _harness(ODD_SHAPES, 3, W, step=step, num_aggregate=2)
    d = Design(h.plan, W, step, True, seed=51, shift=5)
    _run_exact(h, d, seed=51, garbage=(1,), pushed=(0, 2), workers=(0, 2))
    for grp in range(h.plan.n_groups):
        assert int(h.signals[SIG_MASK + 2 * grp]) == 0b101 and int(h.signals[SIG_MASK + 2 * grp + 1]) == step


# ----------------------------------------------------------------------------------------- GPU: bounded, optimizers
@gpu
@pytest.mark.parametrize("W", [3, 5, 12])
@pytest.mark.parametrize("name", ["momentum", "dampening", "nesterov", "adam", "amsgrad"])
def test_ps_step_within_the_fp32_bound(name, W):
    """Random fp32 factors, 4 steps.  At each step the oracle starts from the kernel's own pre-step state, so errors
    do not compound; the step p_new - p_old, the momentum and the second moments must lie within bound_step of it,
    with the decode error of decode_bound / sum_bound.  The first step checks m = g (SGD) and t = 1 (Adam)."""
    o = Opt(**OPTS[name])
    h, _ = _harness(ODD_SHAPES, 8, W, opt=o)
    grid = _grids(h)[[3, 5, 12].index(W)]
    g0 = torch.Generator(device="cuda").manual_seed(W)
    h.master.copy_(torch.randn(h.plan.w_total, device=h.dev, generator=g0))
    h.vparams.copy_(torch.randn(h.plan.v_total, device=h.dev, generator=g0))
    h.wshadow.copy_(h.master.to(torch.bfloat16))
    used = torch.zeros(h.plan.w_total, dtype=torch.bool)
    vused = torch.zeros(h.plan.v_total, dtype=torch.bool)
    for q in h.plan.params:
        (used if q.is_w else vused)[q.off:q.off + q.numel] = True
    for step in range(1, 5):
        d = Design(h.plan, W, step, False, seed=100 * W + step, shift=step)
        g, gv, e, ev = d.oracle()
        d.load(h)
        pre = {k: getattr(h, k).double().cpu() for k in ("master", "mom", "sq", "sqmax", "vparams", "vmom", "vsq",
                                                         "vsqmax")}
        h.ps(grid)
        assert int(h.ctrl.view(torch.int32)[1]) == 0 and int(h.signals[SIG_PARAM]) == step + 1
        for names, gg, ee, mask in ((("master", "mom", "sq", "sqmax"), g, e, used),
                                    (("vparams", "vmom", "vsq", "vsqmax"), gv, ev, vused)):
            st = [pre[k] for k in names]
            bp, bm, bv, bvm = bound_step(o, step, st[0], Val(gg, ee), st[1], st[2], st[3])
            rp = oracle_step(o, step, st[0], gg, st[1], st[2], st[3])[0]
            assert torch.allclose(bp.x, rp, rtol=1e-12, atol=1e-15)
            step_k = getattr(h, names[0]).double().cpu() - st[0]
            step_o = bp.x - st[0]
            err = (step_k - step_o).abs()
            assert bool((err[mask] <= bp.e[mask]).all()), (names[0], step, float((err - bp.e)[mask].max()))
            # an element whose gradient lies within its decode error of zero has no finite Adam bound (m / sqrt(v) is
            # then ill-conditioned); such elements are rare, and elsewhere the bound is far below the step
            fin = mask & torch.isfinite(bp.e)
            assert int(fin.sum()) >= 0.999 * int(mask.sum())
            assert float(bp.e[fin].sum()) <= 1e-3 * float(step_o[fin].abs().sum())
            checks = [(names[1], bm)] + ([(names[2], bv)] if o.opt != P.OPT_SGD else []) + \
                ([(names[3], bvm)] if o.opt == P.OPT_AMSGRAD else [])
            for k, b in checks:
                got = getattr(h, k).double().cpu()
                assert bool(((got - b.x).abs()[mask] <= b.e[mask]).all()), (k, step, float(((got - b.x).abs() - b.e)[mask].max()))
        assert torch.equal(h.wshadow[used.to(h.dev)], h.master.to(torch.bfloat16)[used.to(h.dev)])

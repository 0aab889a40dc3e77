"""The bf16 engine's spectral ATOMO encode (``csrc/v2_encode.cu`` with ``csrc/spectral_sample.cuh``), atom by atom,
against an fp64 oracle built on the kernel's own eigenbasis.

Eigenvectors inside a cluster of equal singular values are not unique, so the oracle never re-derives them: it reads
the basis ``V`` that the Jacobi solver wrote to the warm-start buffer (solver column order, the order in which the
uniforms are indexed) and computes everything else in fp64 on the bf16-rounded unit matrix ``A``:
``sigma_j = ||A v_j||``, ``p_j`` (``codings/sampling.atom_probabilities``) and the decoded atoms ``A v_j v_j^T / p_j``.
The Gram matrix is deterministic, so a second encode of the same gradient gives the same ``V`` bit for bit; that
encode is fed *designed* uniforms: ``p_j / 2`` for the atoms of a chosen set ``S`` and ``p_j + (1 - p_j) / 2`` for
the others, half a probability away from every threshold.  Redraws (a draw over the slot capacity, or an empty one
with ``resample_empty``) use Philox, reproduced with ``codings/powersgd.philox`` at seeds whose uniforms all stay
``1e-4`` away from their thresholds.
"""
import math

import numpy as np
import pytest
import torch

from atomo_b200.codings.sampling import atom_probabilities

from test_gpu_kernels import Harness
from test_gpu_v2 import H2

gpu = pytest.mark.gpu
ERR2_NONFINITE = 8
EPS32 = 2.0 ** -24
MARGIN = 1e-4            # closest a reproduced Philox uniform may come to its threshold


def _coded(h):
    return [u for u in h.plan.units if u.coded]


def _basis(h, u):
    """The unit's Jacobi basis (columns = eigenvectors, solver order), fp32 as the kernel stored it."""
    o = u.ts_index * 4096
    return h.vprev[o:o + u.cols * u.cols].view(u.cols, u.cols).clone()


def _set_basis(h, bases=None):
    """Identity (a cold start from the warm-start path), or the saved bases."""
    for u in _coded(h):
        o = u.ts_index * 4096
        v = torch.eye(u.cols, device=h.dev) if bases is None else bases[u.index]
        h.vprev[o:o + u.cols * u.cols] = v.reshape(-1)


def _set_seed(h, seed):
    h.ctrl.view(torch.int64)[4] = seed


def _set_step(h, step):
    h.ctrl.view(torch.int32)[0] = step


class Oracle:
    def __init__(self, A, V, rule, budget):
        self.A, self.V = A, V                                    # fp64 unit matrix, fp32 kernel basis
        self.AV = A @ V.double()
        self.sig = self.AV.norm(dim=0)
        b = 0.0 if budget <= 0 else budget
        self.p = atom_probabilities(self.sig, b, "waterfill" if rule == "waterfill" else "reference")

    def order(self, idx):
        """Descending sigma, ties by index (the kernel's order)."""
        return sorted(idx, key=lambda j: (-float(self.sig[j]), j))


def _oracles(h, logical, rule):
    return {u.index: Oracle(h.unit_matrix(u, logical).double(), _basis(h, u), rule, u.budget) for u in _coded(h)}


def _encode(h, rule, **kw):
    h.encode(0, waterfill=rule == "waterfill", **kw)


def _designed(h, orc, picks):
    """ext_uniforms selecting exactly picks[unit] on the first draw."""
    uni = torch.ones(max(h.plan.n_coded, 1) * 64, dtype=torch.float64, device=h.dev)
    for u in _coded(h):
        p = orc[u.index].p
        x = torch.where(1 - p > 2e-3, p + (1 - p) / 2, torch.ones_like(p))
        S = list(picks[u.index])
        if S:
            x[S] = p[S] / 2
        uni[u.ts_index * 64:u.ts_index * 64 + u.cols] = x
    return uni.float()


def _slot_atoms(h, u, o):
    """Slot rows identified bit for bit with solver columns of V."""
    count, s, Vs, U, step = h.slot(u, 0)
    eq = (Vs[:, None, :] == o.V.t()[None, :, :]).all(-1)
    assert bool((eq.sum(1) == 1).all()), ("slot V rows are not columns of the solver basis", u.index)
    return count, s, Vs, U, eq.float().argmax(1).tolist()


def _check_slot(h, u, o, S, rtol=2e-3, scale=None):
    """count, atom choice and order, s = sigma / p (scale: 1 / p override), decoded atoms A v v^T / p."""
    count, s, Vs, U, got = _slot_atoms(h, u, o)
    assert count == len(S), (u.index, u.rows, u.cols, count, sorted(S))
    want = o.order(S)
    assert sorted(got) == sorted(want), (u.index, got, want)
    for a, b in zip(got, got[1:]):            # descending sigma; near-ties (fp32 vs fp64) may swap, exact ties may not
        sa, sb = float(o.sig[a]), float(o.sig[b])
        assert sa >= sb * (1 - 1e-4) and (sa != sb or a < b), (u.index, got, want)
    if not count:
        return
    inv_p = (1.0 / o.p[got]) if scale is None else scale[got]
    ref_s = o.sig[got] * inv_p
    assert torch.allclose(s.double(), ref_s, rtol=rtol, atol=0), (u.index, s, ref_s)
    ref_u = o.AV[:, got] * inv_p                                # A v_j / p_j: column k of U diag(s)
    err = ((U.double() * s.double()) - ref_u).norm(dim=0)
    assert bool((err <= rtol * ref_u.norm(dim=0) + 1e-30).all()), (u.index, err / ref_u.norm(dim=0))
    dec = (U.double() * s.double()) @ Vs.double()
    ref = ref_u @ o.V.double()[:, got].t()
    assert float((dec - ref).norm()) <= rtol * float(ref.norm()), u.index


def _picks(h, orc, kind, rng):
    out = {}
    for u in _coded(h):
        o = orc[u.index]
        ok = [j for j in range(u.cols) if float(o.p[j]) >= 0.02]        # selectable with a wide margin
        ones = [j for j in range(u.cols) if float(o.p[j]) >= 1 - 2e-3]  # excluded only through u = 1
        if kind == "empty":
            S = []
        elif kind == "one":
            S = [ok[int(rng.integers(len(ok)))]]
        elif kind == "ones":
            S = ones[:u.rcap]
        else:
            k = int(rng.integers(1, min(len(ok), u.rcap) + 1))
            S = sorted(rng.choice(ok, size=k, replace=False).tolist())
        out[u.index] = S
    return out


def _philox_uniforms(seed, n, attempt, unit, tag):
    from atomo_b200.codings.powersgd import philox
    w0 = philox(seed, np.arange(n), attempt, unit, tag)[0]
    return torch.from_numpy((w0 >> np.uint64(8)).astype(np.float64) / 16777216.0)


def _redraw(o, u, seed, tag, resample_empty):
    """The kernel's redraws after a rejected first draw: (attempt, selected indices, closest |uniform - p|)."""
    p = o.p.cpu()
    margin = 1.0
    for attempt in range(1, 16):
        x = _philox_uniforms(seed, u.cols, attempt, u.index, tag)
        margin = min(margin, float((x - p).abs().min()))
        keep = (x < p).nonzero().flatten().tolist()
        if len(keep) <= u.rcap and (keep or not resample_empty):
            return attempt, keep, margin
    raise AssertionError("no accepted draw in 15 redraws")


def _fill_mats(h, mats, seed=0):
    """Gradients whose unit matrices are mats[unit index] (fp32 tall, bf16-representable or rounded here); every
    other weight gets random values.  Returns {param index: fp32 logical tensor}."""
    P = h.P
    g = torch.Generator(device="cuda").manual_seed(seed)
    by_param = {}
    for u in _coded(h):
        by_param.setdefault(u.param, []).append(u)
    grads, logical = [], {}
    for q in h.plan.params:
        if q.is_w:
            x = torch.randn(q.shape, device=h.dev, generator=g)
            for u in by_param.get(q.index, []):
                if u.index not in mats:
                    continue
                m = mats[u.index].to(h.dev, torch.float32)
                if u.kind == P.KIND_SLAB:
                    x = m.reshape(q.shape)
                else:
                    tall = x.reshape(q.shape[0], -1)
                    tall = tall if tall.shape[0] >= tall.shape[1] else tall.t()
                    c0 = u.g_off // u.cs if u.cs > 1 else u.g_off
                    tall[:, c0:c0 + u.cols] = m
            xb = x.to(torch.bfloat16)
            grads.append(xb.contiguous(memory_format=torch.channels_last) if xb.dim() == 4 else xb.contiguous())
            logical[q.index] = grads[-1].float()
        else:
            v = torch.randn(q.numel, device=h.dev, generator=g)
            h.vgrads[0][q.off:q.off + q.numel] = v
            logical[q.index] = v
    h.wgrads = [grads]
    return logical


def _read_basis(h, rule, uniforms=None):
    """Encode twice from the identity; the basis must repeat bit for bit."""
    _set_basis(h)
    _encode(h, rule)
    first = h.vprev.clone()
    _set_basis(h)
    _encode(h, rule)
    assert torch.equal(h.vprev, first), "the Jacobi basis of a fixed gradient must be deterministic"


def _model_shapes(net, dataset=""):
    from atomo_b200.models import build_model
    return [tuple(p.shape) for p in build_model(net, 10, dataset).parameters()]


MODELS = {"ResNet18": ("ResNet18", ""), "VGG11": ("VGG11", ""), "ResNet50-ImageNet": ("ResNet50", "ImageNet")}


# ------------------------------------------------------------------------------------------------- items 1, 2, 5
def _spectrum_bound(h, u, A):
    """Bound on |sigma_out_k^2 - sigma_k^2| (sigma_k: fp64 singular values of the bf16 unit matrix).

    sigma_out^2 are the eigenvalues Jacobi leaves on the diagonal of the fp32 Gram matrix G^ that the encode summed.
    By Weyl's inequality they differ from those of A^T A by at most ||G^ - A^T A||_2 (the Gram's fp32 accumulation
    error, measured here from the kernel's own Gram partials) plus the eigensolver's own error relative to G^, which
    has two parts: (a) the sweep loop stops after a sweep that started with every coupling below 1e-3 gmax, and
    Jacobi converges quadratically, so the couplings left are below 1e-6 gmax and move the diagonal by at most
    n * 1e-6 gmax (Gershgorin); (b) each of at most 12 sweeps applies one plane rotation to every entry per round,
    n - 1 rounds, each with a relative rounding error of a few u = 2^-24, so at most 12 * 2 * n * u * gmax in all.
    gmax <= sigma_max^2.  An fp32 Gram matrix therefore cannot resolve sigma_k far below sqrt(u) sigma_max, which
    is why the error is bounded relative to sigma_max^2 and not to sigma_k^2."""
    n = u.cols
    G = h.gpart[u.gpart_off:u.gpart_off + u.n_enc * n * n].view(u.n_enc, n, n).double().sum(0)
    eg = float(torch.linalg.matrix_norm(G - A.t() @ A, ord=2))
    gmax = float(torch.diagonal(G).abs().max())
    return eg + (n * 1e-6 + 24 * n * EPS32) * gmax


def _check_spectrum(h, logical, cold=True):
    worst = 0.0
    for u in _coded(h):
        A = h.unit_matrix(u, logical).double()
        V = _basis(h, u).double()
        eye = torch.eye(u.cols, device=h.dev, dtype=torch.float64)
        # each rotation is orthogonal to a few u; 12 sweeps of n - 1 rounds
        assert float((V.t() @ V - eye).abs().max()) <= 24 * u.cols * EPS32 * 4, u.index
        if not cold:
            continue
        sv = torch.linalg.svdvals(A)
        got = h.sigma[u.ts_index * 64:u.ts_index * 64 + u.cols].double()
        assert bool((got[:-1] >= got[1:]).all()), "sigma_out must be sorted"
        bound = _spectrum_bound(h, u, A)
        err = float((got ** 2 - sv ** 2).abs().max())
        assert err <= bound, (u.index, u.rows, u.cols, err, bound)
        worst = max(worst, err / bound) if bound > 0 else worst
    return worst


@gpu
@pytest.mark.parametrize("model", list(MODELS))
@pytest.mark.parametrize("rank", [3, 1])
def test_encode_selects_orders_and_scales_like_the_oracle(model, rank):
    """Every coded unit of the model, batched: for S = {}, one atom, every atom with p = 1 and a random subset, under
    the reference rule and water-filling, the slot holds exactly S in the kernel's order with s = sigma / p, and the
    decoded atoms are A v v^T / p; the sorted spectrum is within the fp32 Gram bound (_spectrum_bound)."""
    net, ds = MODELS[model]
    shapes = _model_shapes(net, ds)
    rng = np.random.default_rng(rank)
    h = H2(shapes, rank=rank, warm=True, max_sweeps=0)
    logical = h.fill(0, 11 + rank)
    for rule in ("reference", "waterfill"):
        _read_basis(h, rule)
        if rule == "reference":
            _check_spectrum(h, logical)
        orc = _oracles(h, logical, rule)
        for kind in ("empty", "one", "ones", "random"):
            picks = _picks(h, orc, kind, rng)
            _set_basis(h)
            _encode(h, rule, uniforms=_designed(h, orc, picks))
            assert int(h.ctrl.view(torch.int32)[1]) == 0
            for u in _coded(h):
                _check_slot(h, u, orc[u.index], picks[u.index])


@gpu
@pytest.mark.parametrize("model", list(MODELS))
def test_encode_budget_zero_rule(model):
    """budget <= 0 (rank 0): p = sigma / sigma_max, the top atom always sent."""
    net, ds = MODELS[model]
    h = H2(_model_shapes(net, ds), rank=0, warm=True, max_sweeps=0)
    logical = h.fill(0, 5)
    _read_basis(h, "reference")
    orc = _oracles(h, logical, "reference")
    rng = np.random.default_rng(0)
    for u in _coded(h):
        if u.budget <= 0:
            o = orc[u.index]
            assert float(o.p.max()) == 1.0 and torch.allclose(o.p, o.sig / o.sig.max())
    for kind in ("ones", "random"):
        picks = _picks(h, orc, kind, rng)
        _set_basis(h)
        _encode(h, "reference", uniforms=_designed(h, orc, picks))
        for u in _coded(h):
            _check_slot(h, u, orc[u.index], picks[u.index])


# ----------------------------------------------------------------------------------------------------- item 3
@gpu
@pytest.mark.parametrize("warm", [False, True])
def test_redraws_follow_philox(warm):
    """A first draw over the slot capacity, or an empty one with resample_empty, is redrawn from Philox(seed;
    atom, attempt, unit, (worker << 24) ^ step).  warm=True is the production setting (warm start, one sweep): the
    basis is then approximate but orthonormal, and the same checks hold on it."""
    shapes = _model_shapes("ResNet18")
    h = H2(shapes, rank=3, warm=True, max_sweeps=1 if warm else 0)
    logical = h.fill(0, 21)
    step = 2
    if warm:
        _set_basis(h)
        _encode(h, "reference")                       # step 1: one sweep from the identity
        start = {u.index: _basis(h, u) for u in _coded(h)}
        _set_step(h, step)
        _encode(h, "reference")
        bases = {u.index: _basis(h, u) for u in _coded(h)}
        _set_basis(h, start)
        _encode(h, "reference")
        for u in _coded(h):
            assert torch.equal(_basis(h, u), bases[u.index])
        _check_spectrum(h, logical, cold=False)
    else:
        _set_step(h, step)
        _read_basis(h, "reference")
    orc = _oracles(h, logical, "reference")
    reset = start if warm else None
    tag = (0 << 24) ^ step
    assert all(u.cols > u.rcap for u in _coded(h))
    for resample_empty, kind in ((False, "over"), (True, "over"), (True, "empty")):
        # a seed whose redraws all stay MARGIN away from their thresholds
        for seed in range(100, 400):
            res = {u.index: _redraw(orc[u.index], u, seed, tag, resample_empty) for u in _coded(h)}
            if min(m for _, _, m in res.values()) > MARGIN:
                break
        else:
            raise AssertionError("no seed with every redraw uniform %g away from its threshold" % MARGIN)
        assert all(m > MARGIN for _, _, m in res.values())
        _set_seed(h, seed)
        _set_basis(h, reset)
        if kind == "over":      # u = 0 < p_j selects every atom: cols > rcap atoms overflow the slot
            uni = torch.zeros(max(h.plan.n_coded, 1) * 64, device=h.dev)
        else:
            uni = _designed(h, orc, {u.index: [] for u in _coded(h)})
        _encode(h, "reference", uniforms=uni, resample_empty=resample_empty)
        for u in _coded(h):
            _check_slot(h, u, orc[u.index], res[u.index][1])


@gpu
def test_empty_draw_is_kept_without_resample_empty():
    h = H2([(64, 32, 3, 3), (100, 34)], rank=3, warm=True, max_sweeps=0)
    logical = h.fill(0, 3)
    _read_basis(h, "reference")
    orc = _oracles(h, logical, "reference")
    picks = {u.index: [] for u in _coded(h)}
    _set_basis(h)
    _encode(h, "reference", uniforms=_designed(h, orc, picks), resample_empty=False)
    for u in _coded(h):
        _check_slot(h, u, orc[u.index], [])
        assert int(h.selcount[u.ts_index]) == 0


# ----------------------------------------------------------------------------------------------------- item 4
def _systematic_x(p_sorted):
    """A uniform x that keeps every frac(c_k + x) at least 1 / (2 (n + 1)) from 0 and 1 (c: cumulative sums)."""
    c = torch.cat([torch.zeros(1, dtype=torch.float64), torch.cumsum(p_sorted.cpu(), 0)])
    f = torch.sort(torch.frac(c)).values
    gaps = torch.cat([f[1:] - f[:-1], (f[:1] + 1 - f[-1:])])
    k = int(torch.argmax(gaps))
    mid = float(f[k] + gaps[k] / 2) % 1.0
    x = (1.0 - mid) % 1.0
    d = torch.frac(c + x)
    assert float(torch.minimum(d, 1 - d).min()) >= 1.0 / (2 * (len(c))) - 1e-12
    return x


@gpu
@pytest.mark.parametrize("rule", ["reference", "waterfill"])
def test_systematic_and_topk_selection(rule):
    from atomo_b200.codings.sampling import sample_atoms
    shapes = _model_shapes("ResNet18")
    h = H2(shapes, rank=3, warm=True, max_sweeps=0, systematic=True)
    logical = h.fill(0, 31)
    _read_basis(h, rule)
    orc = _oracles(h, logical, rule)
    uni = torch.zeros(max(h.plan.n_coded, 1) * 64, device=h.dev)
    want = {}
    for u in _coded(h):
        o = orc[u.index]
        order = o.order(range(u.cols))
        ps = o.p[order]
        x = _systematic_x(ps)
        uni[u.ts_index * 64] = x
        keep = sample_atoms(ps, "systematic", uniforms=torch.tensor([x])).tolist()
        total = float(ps.sum())
        assert math.floor(total) <= len(keep) <= math.ceil(total)
        want[u.index] = [order[k] for k in keep]
    _set_basis(h)
    h.encode(0, waterfill=rule == "waterfill", systematic=True, uniforms=uni)
    for u in _coded(h):
        _check_slot(h, u, orc[u.index], want[u.index])
    # random_sample=False: exactly the top min(budget, n, rcap) atoms, s = sigma
    _set_basis(h)
    h.encode(0, random_sample=False)
    for u in _coded(h):
        o = orc[u.index]
        k = min(int(u.budget) if u.budget > 0 else u.cols, u.cols, u.rcap)
        _check_slot(h, u, o, o.order(range(u.cols))[:k], scale=torch.ones_like(o.p))


# ----------------------------------------------------------------------------------------------------- item 6
def _hadamard(n):
    H = torch.ones(1, 1)
    while H.shape[0] < n:
        H = torch.cat([torch.cat([H, H], 1), torch.cat([H, -H], 1)], 0)
    return H


# odd cols (7, 35 -> 32 + 3), the narrowest block the planner cuts (34 -> 32 + 2), slabs of 18 and 50 columns
EDGE_SHAPES = [(64, 32, 3, 3), (16, 16, 5, 5), (7, 300), (300, 34), (300, 35)]


def _edge_mats(h, kind):
    gen = torch.Generator().manual_seed(5)
    mats = {}
    for u in _coded(h):
        r, n = u.rows, u.cols
        if kind == "zero":
            m = torch.zeros(r, n)
        elif kind == "rank1":      # small-mantissa factors: the product is exact in bf16, so A is exactly rank 1
            x = torch.randint(-3, 4, (r, 1), generator=gen).float() * 0.5
            x[0] = 1.0
            y = torch.randint(1, 4, (1, n), generator=gen).float() * torch.where(torch.rand(1, n, generator=gen) < .5, -1., 1.)
            m = x @ y
        elif kind == "equal":      # Hadamard columns: A^T A = r I exactly, every sigma equal
            m = _hadamard(max(r, n))[:r, :n] if r & (r - 1) == 0 else None
            if m is None:
                continue
        else:                      # tiny: sigma_max near 1e-8 or 1e-5
            target = {"tiny8": 1e-8, "tiny5": 1e-5}[kind]
            m = torch.randn(r, n, generator=gen) * torch.logspace(0, -1, n)
            m = m / torch.linalg.matrix_norm(m, ord=2) * target
        mats[u.index] = m
    return mats


@gpu
@pytest.mark.parametrize("kind", ["zero", "tiny8", "tiny5", "rank1", "equal"])
def test_edge_spectra(kind):
    shapes = EDGE_SHAPES + ([(64, 8)] if kind == "equal" else [])   # 64 x 8: Hadamard-able MAT unit
    h = H2(shapes, rank=3, warm=True, max_sweeps=0)
    mats = _edge_mats(h, kind)
    logical = _fill_mats(h, mats)
    _read_basis(h, "reference")
    orc = _oracles(h, logical, "reference")
    for u in _coded(h):
        if u.index not in mats:
            continue
        o = orc[u.index]
        A = o.A
        smax = float(torch.linalg.svdvals(A)[0])
        if kind in ("zero", "tiny8"):
            # sigma_max < 1e-6: the top atom with p = 1, whatever the draw
            assert smax < 1e-6
            for uni in (None, torch.ones(max(h.plan.n_coded, 1) * 64, device=h.dev)):
                _set_basis(h)
                _encode(h, "reference", uniforms=uni)
                count, s, Vs, U, got = _slot_atoms(h, u, o)
                top = o.order(range(u.cols))[0] if kind == "tiny8" else 0
                assert count == 1 and got == [top], (u.index, count, got)
                if kind == "zero":
                    assert float(s[0]) == 0.0 and float(U.abs().max()) == 0.0
                else:
                    _check_slot(h, u, o, [top], scale=torch.ones_like(o.p), rtol=5e-3)
        elif kind == "tiny5":
            assert 1e-6 < smax < 1e-4
            rng = np.random.default_rng(u.index)
            for k in ("empty", "one", "random"):
                picks = _picks(h, orc, k, rng)
                _set_basis(h)
                _encode(h, "reference", uniforms=_designed(h, orc, picks))
                _check_slot(h, u, o, picks[u.index])
        elif kind == "rank1":
            assert int(torch.linalg.matrix_rank(A)) == 1
            # p_0 = 1; the null directions have p ~ sqrt(u) at most in fp32 and are not drawn
            top = o.order(range(u.cols))[0]
            picks = {k: [] for k in orc}
            picks[u.index] = [top]
            _set_basis(h)
            _encode(h, "reference", uniforms=_designed(h, orc, picks))
            count, s, Vs, U, got = _slot_atoms(h, u, o)
            assert count == 1 and got == [top]
            dec = (U.double() * s.double()) @ Vs.double()
            assert float((dec - A).norm()) <= 1e-3 * float(A.norm()), u.index
        elif kind == "equal":
            # exact ties: Jacobi has nothing to rotate, sigma_j all equal, order = index order
            assert torch.equal(o.V, torch.eye(u.cols, device=h.dev))
            S = [1, u.cols - 1, 2]
            picks = {k: [] for k in orc}
            picks[u.index] = S
            _set_basis(h)
            _encode(h, "reference", uniforms=_designed(h, orc, picks))
            count, s, Vs, U, got = _slot_atoms(h, u, o)
            assert got == sorted(S), got
            _check_slot(h, u, o, S)
    if kind in ("zero", "rank1", "equal", "tiny5"):
        _check_spectrum(h, logical)


@gpu
@pytest.mark.parametrize("bad", [float("inf"), float("nan")])
def test_nonfinite_unit_raises_the_error_and_leaves_the_others_alone(bad):
    """One unit holding an Inf or a NaN: ERR2_NONFINITE is raised in ctrl.error, every other unit's slot is bitwise
    what a clean run writes, and the bad unit's slot holds what DESIGN.md documents."""
    h = H2(EDGE_SHAPES, rank=3, warm=True, max_sweeps=0)
    logical = h.fill(0, 41)
    _set_basis(h)
    _encode(h, "reference")
    assert int(h.ctrl.view(torch.int32)[1]) == 0
    clean = h.arena.clone()
    victim = _coded(h)[0]
    q = h.plan.params[victim.param]
    g = h.wgrads[0][q.widx]
    g[1, 5, 1, 2] = bad
    _set_basis(h)
    _encode(h, "reference")
    assert int(h.ctrl.view(torch.int32)[1]) & ERR2_NONFINITE
    for u in _coded(h):
        sl = slice(u.slot_off, u.slot_off + h.P.slot_floats(u.rows, u.cols, u.rcap))
        if u.index != victim.index:
            assert torch.equal(h.arena[sl], clean[sl]), u.index
    # every eigenvalue of the poisoned Gram is non-finite and zeroed: the degenerate rule sends one atom with s = 0,
    # a finite unit V row, and U is non-finite exactly in the row that holds the bad entry (row (o, i // 2) of the
    # (O*I/2, 2*kh*kw) matricization)
    count, s, V, U, step = h.slot(victim, 0)
    assert count == 1 and step == 1 and float(s[0]) == 0.0
    assert bool(torch.isfinite(V).all()) and abs(float(V.norm()) - 1.0) < 1e-5
    bad_rows = (~torch.isfinite(U)).any(1).nonzero().flatten().tolist()
    assert bad_rows == [1 * q.shape[1] // 2 + 5 // 2], bad_rows


# ----------------------------------------------------------------------------------------------------- item 8
FP32_SHAPES = [(64, 32, 3, 3), (10, 128), (300, 25)]       # cols 18, 10, 25 (odd); rcap >= cols at rank 0


@gpu
def test_fp32_engine_eig_sample_matches_the_oracle():
    """The round-1 engine's eig_sample_kernel shares spectral_sample.cuh.  It has no warm-start buffer, so its solver
    order is read with probes: with budget 0 every atom has p > 0, u = 0 selects it and u = 1 never does, so
    ceil(log2 n) encodes with u_i = 0 iff bit b of i is set name the solver index of every slot row."""
    h = Harness(FP32_SHAPES, rank=0)
    g = torch.Generator(device="cuda").manual_seed(9)
    for l, v in zip(h.plan.layers, h.grad_views()):
        k = l.cols
        tall = torch.randn(l.rows, k, device=h.dev, generator=g) * torch.logspace(0, -1.5, k, device=h.dev)
        mix = torch.linalg.qr(torch.randn(k, k, device=h.dev, generator=g)).Q
        h.tall(l, h.grads).copy_(tall @ mix)
    layers = [l for l in h.plan.layers if l.route == 1]
    row = {l.index: l.ts_index for l in layers}
    n_ts = max(len(layers), 1)

    # the fp32 Gram kernel sums in shared-memory atomics (not bitwise reproducible): one Gram, several eig_samples
    pl = h.plan
    h.C.gram(h.grads, h.t_layers, h.t_enc, len(pl.enc_tiles), h.gpart)

    def run(uni, rank=0, waterfill=False):
        h.C.eig_sample(h.t_layers, h.t_ts, h.gpart, h.vsel, h.selcount, h.sigma, h.arena.data_ptr(), pl.arena_floats,
                       h.ctrl, uni, rank, True, waterfill, False, 0, 1024)
        h.C.project_push(h.grads, h.t_layers, h.t_enc, len(pl.enc_tiles), h.vsel, h.selcount, h.arena.data_ptr(),
                         pl.arena_floats, h.flags.data_ptr(), h.ctrl, 0, True)
        torch.cuda.synchronize()

    run(torch.zeros(n_ts * 64, device=h.dev))
    V = {}
    for l in layers:
        c, s, Vs, U = h.slot(l)
        assert c == l.cols <= l.rcap
        V[l.index] = Vs.clone()                  # all atoms, descending sigma
    idx = {l.index: [0] * l.cols for l in layers}
    for b in range(5):
        uni = torch.ones(n_ts * 64, device=h.dev)
        for l in layers:
            for i in range(l.cols):
                if (i >> b) & 1:
                    uni[row[l.index] * 64 + i] = 0.0
        run(uni)
        for l in layers:
            if l.cols <= 1 << b:          # no index has bit b: the empty draw was redrawn
                continue
            c, s, Vs, U = h.slot(l)
            for k in range(l.cols):
                hit = (Vs == V[l.index][k]).all(1).any()
                idx[l.index][k] |= int(bool(hit)) << b
    rng = np.random.default_rng(1)
    for rank, rule in ((0, "reference"), (3, "reference"), (3, "waterfill")):
        orc, picks = {}, {}
        uni = torch.ones(n_ts * 64, dtype=torch.float64, device=h.dev)
        for l in layers:
            assert sorted(idx[l.index]) == list(range(l.cols))
            Vb = torch.zeros(l.cols, l.cols, device=h.dev)
            for k, i in enumerate(idx[l.index]):
                Vb[:, i] = V[l.index][k]
            A = h.tall(l, h.grads).double()
            o = orc[l.index] = Oracle(A, Vb, rule, rank)
            ok = [j for j in range(l.cols) if float(o.p[j]) >= 0.02]
            S = sorted(rng.choice(ok, size=min(len(ok), 3), replace=False).tolist())
            picks[l.index] = S
            x = torch.where(1 - o.p > 2e-3, o.p + (1 - o.p) / 2, torch.ones_like(o.p))
            x[S] = o.p[S] / 2
            uni[row[l.index] * 64:row[l.index] * 64 + l.cols] = x
        run(uni.float(), rank, rule == "waterfill")
        for l in layers:
            o = orc[l.index]
            c, s, Vs, U = h.slot(l)
            eq = (Vs[:, None, :] == o.V.t()[None, :, :]).all(-1)
            got = eq.float().argmax(1).tolist()
            assert c == len(picks[l.index]) and got == o.order(picks[l.index]), (l.index, got)
            ref_s = o.sig[got] / o.p[got]
            assert torch.allclose(s.double(), ref_s, rtol=2e-3)
            ref_u = o.AV[:, got] / o.p[got]
            assert float(((U.double() * s.double()) - ref_u).norm()) <= 2e-3 * float(ref_u.norm())


# ----------------------------------------------------------------------------------------------------- item 9
def _poisson_binomial_tail(p, k):
    """P(sum of independent Bernoulli(p_i) > k), exactly, in fp64."""
    dist = np.zeros(len(p) + 1)
    dist[0] = 1.0
    for x in np.asarray(p, dtype=np.float64):
        dist[1:] = dist[1:] * (1 - x) + dist[:-1] * x
        dist[0] *= 1 - x
    return float(dist[k + 1:].sum())


OVERFLOW_BOUND = 3e-3        # per unit and step


@pytest.mark.parametrize("rank", [3, 1])
def test_slot_overflow_probability_is_small(rank):
    """The encode redraws a draw with more atoms than the slot holds (rcap = round4(min(cols, 2 rank + 2))), which
    biases the estimate by up to P(count > rcap).  Exactly, for the ResNet-18 units: on the spectra of a real gradient
    (one CPU backward of ResNet-18 on a synthetic batch), and on the worst case for the reference rule, equal p_i =
    budget / cols (Hoeffding 1956, Thm. 4: for a fixed mean, a Poisson-binomial tail at least one above the mean is
    largest when all p_i are equal; sum p_i <= budget, and the tail grows with the mean).  Numbers in DESIGN.md."""
    from atomo_b200.codings.block_svd import unit_table
    from atomo_b200.models import build_model
    from atomo_b200.ops import plan2 as P
    torch.manual_seed(0)
    net = build_model("ResNet18", 10)
    x = torch.randn(8, 3, 32, 32)
    torch.nn.functional.cross_entropy(net(x), torch.arange(8) % 10).backward()
    worst_real = worst_flat = 0.0
    for prm in net.parameters():
        shape = tuple(prm.shape)
        g = prm.grad.detach().double()
        for kind, rows, cols, c0, budget in unit_table(shape, rank):
            if kind == "dense":
                continue
            rcap = P.slot_capacity(cols, max(1, int(budget)), False)
            if kind == "slab":
                a = g.reshape(rows, cols)
            else:
                m = g.reshape(shape[0], -1)
                a = (m if m.shape[0] >= m.shape[1] else m.t())[:, c0:c0 + cols]
            sig = torch.linalg.svdvals(a)
            real = _poisson_binomial_tail(atom_probabilities(sig, budget).numpy(), rcap)
            flat = _poisson_binomial_tail(np.full(cols, min(1.0, budget / cols)), rcap)
            assert real <= flat + 1e-15, (shape, real, flat)
            worst_real, worst_flat = max(worst_real, real), max(worst_flat, flat)
    print("rank", rank, "P(count > rcap): real gradient max %.3e, equal-p worst case max %.3e" % (worst_real, worst_flat))
    assert worst_real <= worst_flat < OVERFLOW_BOUND

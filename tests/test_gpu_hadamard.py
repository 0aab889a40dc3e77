"""Randomized-Hadamard rotated quantization on the bf16 engine (``code="hadamard"``, csrc/v2_hadamard.cu): the
``codings.hadamard`` oracle, the planner, the refusals and the launcher routing (CPU); the encode against the oracle
bit for bit with the in-graph Philox draws, the PS, error feedback and ``--code-stats`` (GPU loopback harness); and the
engine end to end (GPU)."""
import argparse
import functools
import hashlib
import json
import math
import os

import numpy as np
import pytest
import torch

from atomo_b200.ops import plan2 as P
from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils.flags import add_fit_args

from shadow_harness import (LoopbackPS, Loopback, ef_grads, fit_args, flat, forbid_cuda, opt_ref, physical, run_mp,
                            train)

NET_SHAPES = [(64, 3, 3, 3), (64,), (64,), (128, 64, 3, 3), (128,), (256, 128, 3, 3), (512, 256, 1, 1), (300, 200),
              (10, 512), (7, 20), (10,)]
# the 1728-element stem, 3x3 convs (one a multiple of the 4096-element tile, one not), fc layers, tensors smaller than
# a bucket, a vector, then an all-zero tensor (ZERO), one spike (SPIKE), one with an Inf (INF), 1e-20 magnitudes (TINY)
ORACLE_SHAPES = [(64, 3, 3, 3), (64, 32, 3, 3), (128, 64, 3, 3), (96, 64, 3, 3), (10, 512), (300, 200), (7, 20), (5, 3),
                 (64,), (32, 16, 3, 3), (40, 30), (48, 16, 3, 3), (24, 16, 3, 3)]
ZERO, SPIKE, INF, TINY = 9, 10, 11, 12
BUCKETS = [64, 512, 4096]
BITS = [2, 4, 8]


def _coder(bits=4, bucket=512, seed=7):
    from atomo_b200.codings.hadamard import Hadamard
    return Hadamard(bits, bucket, seed=seed)


# ---------------------------------------------------------------------------------------------------- CPU: coder
def test_transform_is_its_own_inverse():
    from atomo_b200.codings.hadamard import butterflies
    rng = np.random.default_rng(0)
    for d in (64, 512, 4096):
        y = rng.standard_normal((3, d)).astype(np.float32)
        back = butterflies(butterflies(y)) / np.float32(d)
        assert np.abs(back - y).max() <= 2e-6 * np.log2(d) * np.abs(y).max()
        # power-of-two values of one binade range: every butterfly sum is exact
        p = (rng.choice([-1.0, 1.0], (3, d)) * 2.0 ** rng.integers(-3, 4, (3, d))).astype(np.float32)
        assert np.array_equal(butterflies(butterflies(p)) / np.float32(d), p)
        # against the dense Sylvester matrix in fp64
        h = np.array([[1.0]])
        while h.shape[0] < d:
            h = np.block([[h, h], [h, -h]])
        assert np.allclose(butterflies(y), y.astype(np.float64) @ h.T, rtol=0, atol=1e-4 * np.abs(y).sum(axis=1).max())


@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("bucket", BUCKETS)
def test_coder_codes_are_floor_or_ceil(bits, bucket):
    rng = np.random.default_rng(bits * bucket)
    x = torch.from_numpy(np.concatenate([rng.standard_normal(3 * bucket + 70) * 10.0 ** rng.integers(-6, 4),
                                         rng.standard_t(1.5, 2 * bucket)])).float()
    c = _coder(bits, bucket)
    code = c.encode(x, unit=5, step=3, worker=1)
    codes = code["codes"].numpy().astype(np.int64)
    assert codes.min() >= 0 and codes.max() <= (1 << bits) - 1
    assert np.array_equal(c.unpack(code), codes)
    _, d, _, y = c.rotate(x, 5, 3)
    lo, st, bad = c._range(y)
    assert not bad.any() and np.array_equal(code["lo"].numpy(), lo) and np.array_equal(code["step"].numpy(), st)
    assert np.array_equal(lo, y.min(axis=1)) and bool((st > 0).all())
    t, _ = c._t(y, lo, st)
    fl = np.floor(t)
    assert np.all((codes == fl) | (codes == np.minimum(fl + 1, (1 << bits) - 1)))
    assert code["words"].shape == (y.shape[0], d * bits // 64)


@pytest.mark.parametrize("bucket", BUCKETS)
def test_coder_tail_bucket_and_small_tensor(bucket):
    from atomo_b200.codings.hadamard import bucket_for
    g = torch.Generator().manual_seed(bucket + 1)
    for n in (1, 40, 63, 64, 65, 140, bucket - 1, bucket, bucket + 3, 3 * bucket + 70):
        x = torch.randn(n, generator=g).bfloat16().float()
        c = _coder(8, bucket)
        code = c.encode(x)
        d = code["bucket_size"]
        assert d == bucket_for(n, bucket) == min(bucket, 1 << max(n - 1, 63).bit_length())
        nb = -(-n // d)
        assert code["words"].shape == (nb, d // 8) and code["lo"].shape == (nb,)
        dec = c.decode(code)
        assert dec.shape == x.shape and bool(torch.isfinite(dec).all())
        assert float((dec - x).norm()) <= 0.05 * float(x.norm()) + 1e-6


def test_coder_special_buckets():
    c = _coder(4, 64)
    # all zero: step 0, zero codes, decoded exactly
    z = c.encode(torch.zeros(100))
    assert bool((z["step"] == 0).all()) and bool((z["lo"] == 0).all()) and bool((z["words"] == 0).all())
    assert bool((c.decode(z) == 0).all())
    # one non-zero at the start of a bucket: every rotated value is equal (hi == lo), so it decodes exactly
    x = torch.zeros(128)
    x[64] = 3.25
    code = c.encode(x)
    assert float(code["step"][1]) == 0 and torch.equal(c.decode(code), x)
    # a spike: finite, and the bucket's error stays a fraction of the spike
    x = torch.randn(256) * 1e-3
    x[70] = 1e4
    code = c.encode(x)
    dec = c.decode(code)
    assert bool(torch.isfinite(dec).all()) and abs(float(dec[70]) - 1e4) < 1e3
    # tiny magnitudes: no Inf / NaN, positive normal steps
    x = torch.randn(512) * 1e-20
    code = c.encode(x)
    assert bool(torch.isfinite(code["lo"]).all()) and bool((code["step"] >= 2.0 ** -126).all())
    dec = c.decode(code)
    assert bool(torch.isfinite(dec).all()) and float((dec - x.bfloat16().float()).norm()) < 0.3 * float(x.norm())
    ex = c.expected_error_sq(x)
    assert math.isfinite(ex) and 0 < ex < 0.1 * float(x.bfloat16().double().square().sum())
    # underflow rule: a step below 2^-126 is stored as 0 and the bucket decodes to lo, off by < (L - 1) 2^-126
    x = torch.zeros(64)
    x[5] = 2.0 ** -126
    c2 = _coder(2, 64)
    code = c2.encode(x)
    assert float(code["step"][0]) == 0 and bool((code["words"] == 0).all())
    assert abs(float(code["lo"][0])) == 2.0 ** -126
    dec = c2.decode(code)
    assert bool(torch.isfinite(dec).all()) and float((dec - x).abs().max()) <= 3 * 2.0 ** -126
    assert c2.expected_error_sq(x) == 0.0
    # an Inf, a NaN or an fp32 overflow of the sums poisons its bucket only
    for bad in (float("inf"), float("nan"), None):
        x = torch.randn(256)
        if bad is None:
            x[64:128] = 3.0e38                         # finite in bf16, the butterflies overflow
        else:
            x[70] = bad
        code = c.encode(x)
        assert bool(torch.isnan(code["lo"][1])) and bool(torch.isnan(code["step"][1]))
        assert bool(torch.isfinite(code["lo"][[0, 2, 3]]).all()) and bool((code["words"][1] == 0).all())
        dec = c.decode(code)
        assert bool(torch.isnan(dec[64:128]).all()) and bool(torch.isfinite(dec[:64]).all())
        assert bool(torch.isfinite(dec[128:]).all())
        assert math.isnan(c.expected_error_sq(x))


def test_coder_explicit_uniforms():
    from atomo_b200.codings.hadamard import uniforms
    c = _coder(4, 64)
    x = torch.randn(200).bfloat16().float()
    n = 4 * 64
    down = c.encode(x, u=np.full(n, 1.0 - 2.0 ** -24, dtype=np.float32))
    up = c.encode(x, u=np.zeros(n, dtype=np.float32))
    _, _, _, y = c.rotate(x)
    lo, st, _ = c._range(y)
    t, _ = c._t(y, lo, st)
    fl = np.floor(t)
    assert np.array_equal(down["codes"].numpy(), fl)
    assert np.array_equal(up["codes"].numpy(), np.where(t > fl, np.minimum(fl + 1, 15), fl))
    # the keyed draws are the default uniforms
    u = uniforms(7, 4, 9, 2, n)
    assert torch.equal(c.encode(x, unit=4, step=9, worker=2)["words"], c.encode(x, unit=4, step=9, worker=2, u=u)["words"])
    assert not torch.equal(c.encode(x, unit=4, step=9, worker=2)["words"], c.encode(x, unit=4, step=10, worker=2)["words"])


def test_shared_rotation_and_per_worker_draws():
    """Two workers of one (seed, unit, step) rotate identically and draw different roundings; the owner's decode of
    their sum is the mean of their decodes (the rotation is linear)."""
    from atomo_b200.codings.hadamard import signs
    c = _coder(4, 512)
    assert np.array_equal(signs(7, 3, 5, 4096), signs(7, 3, 5, 4096))
    assert not np.array_equal(signs(7, 3, 5, 4096), signs(7, 3, 6, 4096))
    assert 0.45 < signs(7, 3, 5, 4096).mean() < 0.55
    x = torch.randn(1500)
    a, b = c.encode(x, unit=3, step=5, worker=0), c.encode(x, unit=3, step=5, worker=1)
    assert np.array_equal(c.rotate(x, 3, 5)[3], c.rotate(x, 3, 5)[3])
    assert torch.equal(a["lo"], b["lo"]) and torch.equal(a["step"], b["step"])
    assert not torch.equal(a["words"], b["words"])
    mean = c.decode_sum([a, b], inv_w=0.5)
    assert torch.allclose(mean, (c.decode(a) + c.decode(b)) / 2, rtol=0, atol=1e-5 * float(x.abs().max()))


@pytest.mark.parametrize("dist", ["normal", "laplace", "student1.5"])
def test_coder_unbiased_and_variance_matches_closed_form(dist):
    """Over T keyed draws (steps 1..T: fresh signs and roundings) the mean converges to x and the squared error to the
    mean of expected_error_sq() over the drawn rotations, within CLT bounds."""
    rng = np.random.default_rng(3)
    n = 512
    x = {"normal": lambda k: rng.standard_normal(k), "laplace": lambda k: rng.laplace(size=k),
         "student1.5": lambda k: rng.standard_t(1.5, k)}[dist](n)
    x = torch.from_numpy(x).float().bfloat16().float()
    c = _coder(4, 64)
    T = 800
    dec = torch.stack([c.decode(c.encode(x, unit=2, step=t)) for t in range(1, T + 1)]).double()
    want = np.array([c.expected_error_sq(x, unit=2, step=t) for t in range(1, T + 1)])
    err = dec - x.double()
    per = err.square().sum(dim=1).numpy()
    assert abs(per.mean() - want.mean()) <= 5 * per.std() / math.sqrt(T), (per.mean(), want.mean())
    assert float(err.mean(dim=0).square().sum()) <= 3.0 * want.mean() / T
    assert 0.01 < want.mean() / float(x.double().square().sum()) < 0.05      # ~0.026 whatever the distribution


def test_coder_refuses_settings():
    for bits in (0, 1, 3, 5, 16):
        with pytest.raises(ValueError, match="hadamard: quantization_level"):
            _coder(bits, 512)
    for b in (0, 32, 96, 100, 8192):
        with pytest.raises(ValueError, match="hadamard: bucket_size must be a power of two"):
            _coder(4, b)


# ---------------------------------------------------------------------------------------------------- CPU: planner
def _check_hadamard_plan(pl, owners, bits, bucket):
    for p in pl.params:
        units = [u for u in pl.units if u.param == p.index]
        assert len(units) == 1
        u = units[0]
        if not p.is_w:
            assert u.kind == P.KIND_VEC
            continue
        d = P.hadamard_bucket(p.numel, bucket)
        assert d & (d - 1) == 0 and 64 <= d <= bucket and (d >= p.numel or d == bucket)
        bpt = max(1, 4096 // d)
        assert u.kind == P.KIND_HADAMARD and (u.K, u.I, u.numel, u.w_off, u.rs) == (d, bits, p.numel, p.off, 0)
        assert u.rows == -(-p.numel // d) and u.cols == d * bits // 64 and u.cs == bpt and u.ps_rows == bpt * d
        tiles = sorted((a, n, o) for (ui, a, n, o) in pl.ps_tiles if ui == u.index)
        assert len(tiles) == u.n_ps
        assert [a for a, _, _ in tiles] == list(range(0, p.numel, u.ps_rows))
        assert all(n == min(u.ps_rows, p.numel - a) for a, n, _ in tiles)
        assert [o for _, _, o in tiles] == [(u.own0 + j) % owners for j in range(u.n_ps)]
        enc = [(a, n, j) for (ui, a, n, j) in pl.enc_tiles if ui == u.index]
        assert enc == [(a, n, j) for j, (a, n, _) in enumerate(tiles)]
    assert pl.n_coded == sum(1 for p in pl.params if p.is_w)
    spans = []
    for u in pl.units:
        if u.kind == P.KIND_HADAMARD:
            po, wo = u.slot_off + P.hadamard_params_off(u.n_ps), u.slot_off + P.hadamard_words_off(u.n_ps, u.rows)
            assert u.slot_off % 4 == 0 and po % 2 == 0 and wo % 4 == 0 and po + 2 * u.rows <= wo
            spans.append((u.slot_off, u.slot_off + P.hadamard_slot_floats(u.n_ps, u.rows, u.cols)))
            assert wo + 2 * u.rows * u.cols <= spans[-1][1]
    spans.sort()
    assert all(a1 >= b0 for (a0, b0), (a1, b1) in zip(spans, spans[1:]))
    assert not spans or spans[-1][1] <= pl.arena_floats


@pytest.mark.parametrize("owners", [1, 2, 8])
@pytest.mark.parametrize("bucket", BUCKETS)
@pytest.mark.parametrize("bits", BITS)
def test_plan2_hadamard_units_tiles_and_slots(bits, bucket, owners):
    pl = P.build_plan2(NET_SHAPES, "hadamard", n_owners=owners, n_groups=3, quantization_level=bits,
                       bucket_size=bucket)
    _check_hadamard_plan(pl, owners, bits, bucket)
    c = _coder(bits, bucket)
    want = 0
    for s in NET_SHAPES:
        if len(s) >= 2:
            code = c.encode(torch.zeros(s))
            want += 8 * code["words"].numel() + 4 * (code["lo"].numel() + code["step"].numel())
    assert pl.hadamard_bytes() == want and pl.expected_factor_bytes() == want and pl.qsgd_bytes() == 0
    assert pl.dense_bytes() == 4 * sum(p.numel for p in pl.params if not p.is_w)


@pytest.mark.parametrize("net,want", [("ResNet18", (2.83, 5.49, 10.81)), ("VGG11", (2.47, 4.79, 9.44))])
def test_plan2_hadamard_push_bytes_from_shapes(net, want):
    from atomo_b200.models import build_model
    shapes = [tuple(p.shape) for p in build_model(net, 10).parameters()]
    for bits, mib in zip(BITS, want):
        pl = P.build_plan2(shapes, "hadamard", quantization_level=bits, bucket_size=512)
        assert round(pl.hadamard_bytes() / 2 ** 20, 2) == mib
        n = sum(math.prod(s) for s in shapes if len(s) >= 2)
        assert n * bits / 8 < pl.hadamard_bytes() < n * (bits / 8 + 8 / 512) + 512 * len(shapes)


def test_plan2_hadamard_refuses_settings():
    for bits in (0, 1, 3, 16):
        with pytest.raises(ValueError, match="hadamard: quantization_level"):
            P.build_plan2(NET_SHAPES, "hadamard", quantization_level=bits)
    for b in (0, 32, 96, 100, 8192):
        with pytest.raises(ValueError, match="hadamard: bucket_size must be a power of two"):
            P.build_plan2(NET_SHAPES, "hadamard", bucket_size=b)


def test_plan2_other_codes_unchanged_by_the_new_code():
    """Digests of the plans of the existing codes, taken from the planner before the hadamard code was added."""
    want = {"svd": "917543867e0167683f770150a43eaf4c129e4d461aa989111b2a491e5eeca388",
            "qsvd": "6ea73c4cd4a95d51288ea6c2a2053f66ff7800fc277120bdccfda766e92e3cf9",
            "sgd": "6d3fd294b9211300d2945b4d3f20d6bf9615e56c5dfa3bab6b294fa9370a37d8",
            "qsgd": "1f34b0853ed1349c3ede1baad5eecd6d7a8e9d4bd571740ec8e531cedbfe275c",
            "terngrad": "5ab388e54d2c51d29226927eaa996c37b3173a968114dce188b5cb8121895e57",
            "entrywise": "5ec97d1b33d12cee3ed4b7b6466f49526420e0442c54d8d8aa9634e1cfe73dcf",
            "topk": "0fed82b9ada85f2510d5f1e0b047978d4124c2a1bd1557bba9353e0d7fae72f0",
            "sign": "81b324f24294287fe7a390c33fc80496d4e05e4f6e2236d722a14a87cc73cb97",
            "powersgd": "dd44d14dac1cdad253f1ff4a89cb2423202cac1056532f643b917a03966a9ffc",
            "fp8": "f7e2ad88e0d238d07dd65acc802e9c64f6375d2bfc56ff7813b3367aa177dffb"}
    for code, digest in want.items():
        pl = P.build_plan2(NET_SHAPES, code, 3, n_owners=2, n_groups=3, entry_budget=0.05)
        b = pl.units_bytes() + P.Plan2.tiles_bytes(pl.enc_tiles) + P.Plan2.tiles_bytes(pl.ps_tiles) + \
            repr((pl.enc_range, pl.ps_range, pl.arena_floats, pl.n_coded)).encode()
        assert hashlib.sha256(b).hexdigest() == digest, code


def test_plan2_hadamard_fuzz():
    """Random architectures, owners, groups, bits and buckets: every weight element is owned by exactly one PS tile
    of its unit, and the slots are disjoint and inside the arena."""
    rng = np.random.default_rng(11)
    for _ in range(60):
        shapes = []
        for _ in range(int(rng.integers(1, 9))):
            kind = int(rng.integers(0, 4))
            if kind == 0:
                shapes.append((int(rng.integers(1, 300)),))
            elif kind == 1:
                shapes.append((int(rng.integers(1, 600)), int(rng.integers(1, 600))))
            else:
                k = int(rng.choice([1, 3, 5]))
                shapes.append((int(rng.integers(1, 160)), int(rng.integers(1, 160)), k, k))
        owners, groups = int(rng.choice([1, 2, 3, 8])), int(rng.integers(1, 6))
        bits, bucket = int(rng.choice(BITS)), int(rng.choice([64, 128, 256, 512, 1024, 2048, 4096]))
        pl = P.build_plan2(shapes, "hadamard", n_owners=owners, n_groups=groups, quantization_level=bits,
                           bucket_size=bucket)
        _check_hadamard_plan(pl, owners, bits, bucket)
        cover = np.zeros(pl.w_total, dtype=np.int32)
        for (ui, a, b, o) in pl.ps_tiles:
            u = pl.units[ui]
            if u.kind == P.KIND_HADAMARD:
                assert a % u.K == 0 and b <= 4096 and a + b <= u.numel
                cover[u.w_off + a:u.w_off + a + b] += 1
        for q in pl.params:
            if q.is_w:
                assert (cover[q.off:q.off + q.numel] == 1).all()
        assert cover.sum() == sum(q.numel for q in pl.params if q.is_w)


@pytest.mark.parametrize("kw,msg", [(dict(quantization_level=3), "hadamard: quantization_level"),
                                    (dict(quantization_level=1), "hadamard: quantization_level"),
                                    (dict(bucket_size=96), "hadamard: bucket_size"),
                                    (dict(bucket_size=8192), "hadamard: bucket_size")])
def test_shadow_engine_hadamard_refuses_before_cuda(kw, msg, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    forbid_cuda(monkeypatch)
    with pytest.raises(ValueError, match=msg):
        S.ShadowEngine(None, 0, 1, code="hadamard", **kw)
    with pytest.raises(ValueError, match="num_aggregate"):     # the error-feedback rule applies unchanged
        S.ShadowEngine(None, 0, 4, code="hadamard", error_feedback=True, num_aggregate=2)


# ---------------------------------------------------------------------------------------------------- CPU: launcher
def test_launcher_routes_hadamard(tmp_path, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    seen = []

    class Fake:
        def __init__(self, model, rank, world, **kw):
            seen.append(kw)
    monkeypatch.setattr(S, "ShadowEngine", Fake)
    model = torch.nn.Linear(4, 4)
    for engine in ("auto", "shadow"):
        _, kind = L._build_engine(fit_args(tmp_path, "--code", "hadamard", "--dtype", "bf16", "--engine", engine,
                                        "--quantization-level", "2", "--bucket-size", "256", "--error-feedback", "1",
                                        "--code-stats", "1"), model, 0, 1)
        assert kind == "shadow" and seen[-1]["code"] == "hadamard" and seen[-1]["bucket_size"] == 256
        assert seen[-1]["quantization_level"] == 2
        assert seen[-1]["error_feedback"] is True and seen[-1]["code_stats"] is True
    n = len(seen)
    for extra in (("--dtype", "fp32"), ("--dtype", "bf16", "--engine", "fused")):
        with pytest.raises(SystemExit, match="hadamard"):
            L._build_engine(fit_args(tmp_path, "--code", "hadamard", *extra), model, 0, 1)
    assert len(seen) == n


def test_role_paths_refuse_hadamard(monkeypatch, tmp_path):
    from atomo_b200 import distributed_nn
    from atomo_b200.runtime.master import build_coder
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    with pytest.raises(SystemExit, match="p2p bf16 engine"):
        distributed_nn.run_rank(fit_args(tmp_path, "--code", "hadamard", "--backend", "gloo"))
    with pytest.raises(ValueError, match="p2p bf16 engine"):
        build_coder({"code": "hadamard", "bucket_size": 512}, worker_side=True)


# ---------------------------------------------------------------------------------------------------- GPU harness
class HH(LoopbackPS):
    """Randomized-Hadamard quantization; with ``special``, ``fill`` gives the ZERO / SPIKE / INF / TINY tensors of
    ORACLE_SHAPES their content."""

    PS = "v2_ps_hadamard"

    def __init__(self, shapes, bits=4, bucket=512, W=1, lr=0.1, momentum=0.0, wd=0.0, nesterov=False, opt=0, seed=7,
                 num_aggregate=0):
        super().__init__(shapes, "hadamard", W, lr, momentum, wd, nesterov, opt, seed, num_aggregate,
                         quantization_level=bits, bucket_size=bucket)
        self.bits, self.bucket = bits, bucket
        self.spart = self.zeros(5 * max(len(self.plan.enc_tiles), 1), torch.float64)
        self.acc = self.zeros(7 * self.nc, torch.float64)

    def coder(self):
        return _coder(self.bits, self.bucket, self.seed)

    def tensor(self, q, x, g, special=False):
        if special and q.index == ZERO:
            x.zero_()
        elif special and q.index == TINY:
            x = x * 1e-20
        elif special and q.index == INF:
            x = physical(x)
            flat(x)[1234] = float("inf")
        elif special and q.index == SPIKE:
            x = physical(x)
            flat(x)[700] = 5e3
        return x

    def encode(self, w, residual=0, stats=False):
        C, pl = self.C, self.plan
        gptr = self.gptr(w)
        t0, nt = pl.enc_range[0]
        C.v2_hadamard_encode(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr,
                             self.t_arena_peer.data_ptr(), self.t_sig_peer.data_ptr(), 1, pl.arena_floats, w, 0,
                             self.ctrl.data_ptr(), self.counter(), 0, False, residual)
        if stats:
            C.v2_hadamard_code_stats(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr,
                                     self.t_arena_peer.data_ptr(), 1, pl.arena_floats, w, self.ctrl.data_ptr(),
                                     self.spart.data_ptr(), self.counters.data_ptr(), self.acc.data_ptr())
        torch.cuda.synchronize()

    def slot(self, u, w):
        """(stamps, lo, step, words [buckets, cols] int64) of unit u in worker w's slot."""
        base = self.arena[w * self.plan.arena_floats + u.slot_off:]
        stamps = base[:u.n_ps].view(torch.int32).clone()
        po, wo = P.hadamard_params_off(u.n_ps), P.hadamard_words_off(u.n_ps, u.rows)
        par = base[po:po + 2 * u.rows].view(u.rows, 2).clone()
        words = base[wo:wo + 2 * u.rows * u.cols].view(torch.int64).view(u.rows, u.cols).clone()
        return stamps, par[:, 0].contiguous(), par[:, 1].contiguous(), words

    def slot_code(self, u, w):
        """The slot of unit u / worker w as an oracle code dict (for the oracle's decode)."""
        _, lo, st, words = self.slot(u, w)
        return {"words": words.cpu(), "lo": lo.cpu(), "step": st.cpu(), "bucket_size": u.K, "bits": self.bits,
                "numel": u.numel, "shape": [u.numel], "unit": u.index, "step_index": self.step}

    def oracle(self, u, x, w):
        """The oracle's encode of unit u's physical-order gradient x by worker w at the current step."""
        return self.coder().encode(x.cpu(), unit=u.index, step=self.step, worker=w)


def _decoded_mean(h, phys_by_worker, workers=None, inv_w=None):
    """The oracle owner's mean over the counted workers (sum of y_hat in worker order, one inverse transform, times
    fp32(inv_w)), physical order."""
    workers = list(range(len(phys_by_worker))) if workers is None else workers
    inv_w = float(np.float32(1.0 / len(workers))) if inv_w is None else inv_w
    est = torch.zeros(h.plan.w_total)
    c = h.coder()
    for u in h.plan.units:
        if u.kind == P.KIND_HADAMARD:
            codes = [h.oracle(u, phys_by_worker[w][u.param], w) for w in workers]
            est[u.w_off:u.w_off + u.numel] = c.decode_sum(codes, inv_w=inv_w)
    return est


# ---------------------------------------------------------------------------------------------------- GPU: encode
@pytest.mark.gpu
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("bucket", BUCKETS)
def test_v2_hadamard_encode_matches_oracle_bitwise(bits, bucket):
    h = HH(ORACLE_SHAPES, bits, bucket)
    h.set_step(3)
    phys = h.fill(0, 11, special=True)
    h.encode(0)
    first = h.arena.clone()
    for u in h.plan.units:
        if u.kind != P.KIND_HADAMARD:
            continue
        ref = h.oracle(u, phys[u.param], 0)
        stamps, lo, st, words = h.slot(u, 0)
        assert bool((stamps == 3).all()), u.param
        assert torch.equal(lo.cpu().view(torch.int32), ref["lo"].view(torch.int32)), u.param
        assert torch.equal(st.cpu().view(torch.int32), ref["step"].view(torch.int32)), u.param
        assert torch.equal(words.cpu(), ref["words"]), u.param
        if u.param == ZERO:
            assert bool((st == 0).all()) and bool((words == 0).all())
        if u.param == INF:          # only the bucket holding the Inf is non-finite
            bad = (~torch.isfinite(st)).nonzero().flatten().tolist()
            assert bad == [1234 // u.K]
        if u.param == TINY:
            assert bool(torch.isfinite(lo).all()) and bool((st > 0).all())
    assert int(h.signals[0]) == 3
    h.arena.zero_()                  # a second encode of the same gradient and step: the same bits
    h.encode(0)
    assert torch.equal(h.arena.view(torch.int32), first.view(torch.int32))
    u = next(u for u in h.plan.units if u.kind == P.KIND_HADAMARD and u.param == 2)
    ref3 = h.oracle(u, phys[u.param], 0)["words"]
    h.set_step(4)                    # the next step draws afresh, still the oracle's draws
    h.encode(0)
    assert torch.equal(h.slot(u, 0)[3].cpu(), h.oracle(u, phys[u.param], 0)["words"])
    assert not torch.equal(h.slot(u, 0)[3].cpu(), ref3)


# ---------------------------------------------------------------------------------------------------- GPU: PS
@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 2])
@pytest.mark.parametrize("bucket", [64, 4096])
@pytest.mark.parametrize("bits", [2, 8])
def test_v2_ps_hadamard_decoded_mean_is_bitwise_the_oracles(W, bucket, bits):
    """lr = 1, no momentum, a zero master: the PS writes minus the oracle owner's mean."""
    h = HH(NET_SHAPES, bits, bucket, W=W, lr=1.0)
    h.set_step(2)
    phys = []
    for w in range(W):
        phys.append(h.fill(w, 70 + w))
        h.encode(w)
    want = _decoded_mean(h, phys).to(h.dev)
    h.master.zero_()
    h.ps()
    assert int(h.ctrl.view(torch.int32)[1]) == 0
    used, _ = h.used()
    assert torch.equal(-h.master[used], want[used])


@pytest.mark.gpu
@pytest.mark.parametrize("momentum,nesterov,wd,opt", [(0.0, False, 0.0, 0), (0.9, True, 1e-3, 0), (0.9, False, 0.0, 0),
                                                      (0.0, False, 0.0, 1), (0.0, False, 1e-3, 2)])
def test_v2_ps_hadamard_matches_reference(momentum, nesterov, wd, opt):
    W, lr = 3, 0.05
    h = HH(NET_SHAPES, 4, 512, W=W, lr=lr, momentum=momentum, wd=wd, nesterov=nesterov, opt=opt)
    used, vused = h.used()
    for step in (1, 2):
        h.set_step(step)
        phys = []
        for w in range(W):
            phys.append(h.fill(w, 10 * step + w))
            h.encode(w)
        gw = _decoded_mean(h, phys).to(h.dev)
        gv = sum(h.vgrads) / W
        rp, _ = opt_ref(h.master.clone(), gw, h.mom.clone(), h.sq.clone(), h.sqmax.clone(), step, lr, momentum,
                         nesterov, wd, opt)
        rv, _ = opt_ref(h.vparams.clone(), gv, h.vmom.clone(), h.vsq.clone(), h.vsqmax.clone(), step, lr, momentum,
                         nesterov, wd, opt)
        h.ps()
        assert int(h.ctrl.view(torch.int32)[1]) == 0
        assert int(h.signals[256]) == step + 1
        tol = dict(rtol=3e-4, atol=3e-5) if opt == 0 else dict(rtol=2e-3, atol=2e-4)
        assert torch.allclose(h.master[used], rp[used], **tol), float((h.master - rp)[used].abs().max())
        assert torch.allclose(h.vparams[vused], rv[vused], **tol)
        assert torch.equal(h.wshadow[used], h.master.to(torch.bfloat16)[used])


@pytest.mark.gpu
def test_v2_ps_hadamard_num_aggregate_and_stale_slots():
    """num_aggregate = 2 of 3 workers, worker 1 never pushes: only {0, 2} are averaged.  Then a slot whose stamp is of
    another step is skipped and flagged with ERR2_SLOT_STEP."""
    lr = 0.1
    h = HH(NET_SHAPES, 4, 512, W=3, lr=lr, num_aggregate=2)
    phys = [None, None, None]
    for w in (0, 2):
        phys[w] = h.fill(w, 40 + w)
        h.encode(w)
    h.vgrads[1].fill_(1e6)                         # garbage a skipped worker may hold
    assert int(h.signals[0]) == 1 and int(h.signals[1]) == 0 and int(h.signals[2]) == 1
    est = _decoded_mean(h, phys, workers=[0, 2], inv_w=1.0).to(h.dev)
    p0, v0 = h.master.clone(), h.vparams.clone()
    h.ps()
    assert int(h.ctrl.view(torch.int32)[1]) == 0 and int(h.signals[256]) == 2
    assert int(h.signals[320]) == 0b101 and int(h.signals[321]) == 1
    used, vused = h.used()
    assert torch.allclose(h.master[used], (p0 - lr * est / 2)[used], rtol=3e-4, atol=3e-5)
    assert torch.allclose(h.vparams[vused], (v0 - lr * (h.vgrads[0] + h.vgrads[2]) / 2)[vused], rtol=3e-4, atol=3e-5)

    hs = HH(NET_SHAPES, 4, 512, W=2, lr=lr)        # worker 1's slot holds step 0 while its flag claims step 1
    hs.fill(0, 1)
    hs.encode(0)
    hs.signals[1] = 1
    hs.ps()
    assert int(hs.ctrl.view(torch.int32)[1]) & 4          # ERR2_SLOT_STEP


# ---------------------------------------------------------------------------------------------------- GPU: stats
@pytest.mark.gpu
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("bucket", BUCKETS)
def test_v2_hadamard_code_stats_match_fp64(bits, bucket):
    h = HH(ORACLE_SHAPES, bits, bucket)
    h.set_step(2)
    phys = h.fill(0, 21, special=True)
    h.encode(0, stats=True)
    acc = h.acc.view(-1, 7).tolist()
    from atomo_b200.codings.sign import bf16_flushed
    c = h.coder()
    for u in h.plan.units:
        if u.kind != P.KIND_HADAMARD:
            continue
        gsq, mse, ex, bias, real, real4, n = acc[u.ts_index]
        if u.param == INF:
            assert math.isnan(mse)
            continue
        x = torch.from_numpy(bf16_flushed(phys[u.param].cpu())).double()
        assert n == 1 and bias == 0 and ex == real == real4 == u.numel
        assert gsq == pytest.approx(float(x.square().sum()), rel=1e-12, abs=0)
        want = c.expected_error_sq(phys[u.param].cpu(), unit=u.index, step=2)
        assert mse == pytest.approx(want, rel=1e-10, abs=1e-300)
        if u.param != ZERO:
            assert 0 < mse < 1.5 * gsq


@pytest.mark.gpu
def test_v2_hadamard_code_stats_agree_with_sampled_error():
    """The closed-form expected error against the error of 400 encodes (steps 1..400) decoded from the GPU's slots."""
    h = HH([(64, 32, 3, 3), (300, 200), (7, 20)], 4, 512)
    phys = h.fill(0, 5)
    c = h.coder()
    T = 400
    per_step = []
    for step in range(1, T + 1):
        h.set_step(step)
        h.encode(0, stats=True)
        tot = 0.0
        for u in h.plan.units:
            if u.kind != P.KIND_HADAMARD:
                continue
            dec = c.decode_flat(h.slot_code(u, 0)).double()
            tot += float((dec - phys[u.param].cpu().double()).square().sum())
        per_step.append(tot)
    acc = h.acc.view(-1, 7)
    assert float(acc[0, 6]) == T
    want = float(acc[:, 1].sum()) / T
    per = torch.tensor(per_step, dtype=torch.float64)
    assert abs(float(per.mean()) - want) <= 5 * float(per.std()) / math.sqrt(T), (float(per.mean()), want)


# ---------------------------------------------------------------------------------------------------- GPU: feedback
@pytest.mark.gpu
@pytest.mark.parametrize("bits,bucket", [(2, 512), (4, 64), (4, 4096), (8, 512)])
def test_error_feedback_identity(bits, bucket):
    h = Loopback("hadamard", ef_grads(1), quantization_level=bits, bucket_size=bucket)
    try:
        g, e_old = h.g, h.residual()
        for _ in range(4):
            A = g + e_old
            ghat, e_new = h.step()
            scale = g.abs() + e_old.abs() + ghat.abs() + e_new.abs()
            assert bool(((A - (ghat + e_new)).abs() <= 1e-6 * scale + 1e-7 * float(scale.max())).all())
            assert 0 < float(e_new.norm()) <= {2: 1.0, 4: 0.3, 8: 0.03}[bits] * float(A.norm())
            e_old = e_new
    finally:
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [2, 4])
def test_error_feedback_residual_stays_bounded(bits):
    """A fixed gradient for 200 steps: every step leaves ||e_{t+1}|| <= rho ||g + e_t|| with rho < 1 (the code's
    relative error), so ||e|| stays below rho / (1 - rho) ||g||; the pushed sum misses 200 g by exactly the final
    residual."""
    h = Loopback("hadamard", ef_grads(2), quantization_level=bits, bucket_size=512)
    try:
        s = torch.zeros_like(h.g)
        e = h.residual()
        rho, norms = 0.0, []
        for _ in range(200):
            A = h.g + e
            ghat, e = h.step()
            s += ghat
            rho = max(rho, float(e.norm()) / float(A.norm()))
            norms.append(float(e.norm()))
        assert rho < {2: 0.95, 4: 0.3}[bits]
        assert max(norms) <= rho / (1 - rho) * float(h.g.norm()) * (1 + 1e-4)
        tol = 200 * 1e-6 * (float(h.g.abs().max()) + float(e.abs().max()) + float(s.abs().max()) / 200)
        assert torch.allclose(s - 200 * h.g, -e, rtol=0, atol=tol)
    finally:
        h.close()


@pytest.mark.gpu
def test_code_stats_bytes_follow_the_plan():
    h = Loopback("hadamard", ef_grads(4), quantization_level=4, bucket_size=256, code_stats=True)
    try:
        h.step()
        st = h.eng.code_stats()
        pl = h.eng.plan
        assert st["code"] == "hadamard" and st["steps"] == 1
        names = {id(p): n for n, p in h.eng.model.named_parameters()}
        for u in pl.units:
            t = st["tensors"][names[id(h.eng.params[u.param])]]
            if u.kind == P.KIND_HADAMARD:
                assert t["bytes"] == 8 * u.rows * u.cols + 8 * u.rows
                assert t["atoms"] == t["exp_atoms"] == u.numel and 0 < t["rel_var"] < 0.1
        assert st["model"]["bytes"] == pl.hadamard_bytes() + pl.dense_bytes()
    finally:
        h.close()


# ---------------------------------------------------------------------------------------------------- GPU: engine
_train = functools.partial(train, code="hadamard", quantization_level=4, bucket_size=512)


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["ResNet18", "VGG11"])
@pytest.mark.parametrize("ef", [False, True])
def test_graph_replay_equals_eager(net, ef, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    mg, _, _ = _train(net, True, ef)
    me, _, _ = _train(net, False, ef)
    assert torch.equal(mg, me)


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["ResNet18", "VGG11"])
@pytest.mark.parametrize("ef", [False, True])
def test_training_stays_finite(net, ef):
    _, losses, norms = _train(net, True, ef, steps=30)
    assert all(math.isfinite(v) for v in losses + norms)
    if ef:
        assert max(norms[10:]) < 20 * max(norms[:10]), norms
    assert losses[-1] < losses[0], losses


@pytest.mark.gpu
def test_checkpoint_round_trip(tmp_path):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.cuda.set_device(0)
    x, y = SyntheticImageDataset((3, 32, 32), 10, 256).materialize(32)

    def mk():
        torch.manual_seed(0)
        return ShadowEngine(build_model("VGG11", 10), 0, 1, code="hadamard", quantization_level=8, bucket_size=256,
                            lr=0.05, momentum=0.9, use_graph=False)
    a = mk()
    a.prepare(x.pin_memory(), y.pin_memory(), warmup=0)
    for _ in range(3):
        a.train_step(x, y)
    path = a.save_checkpoint(str(tmp_path) + "/")
    side = torch.load(path + "_optim", weights_only=False)
    assert side["code"] == "hadamard" and side["bucket_size"] == 256 and side["quantization_level"] == 8
    want = a.gather_fp32("master").clone()
    a.close()
    b = mk()
    b.prepare(x.pin_memory(), y.pin_memory(), warmup=0)
    b.load_checkpoint(str(tmp_path) + "/", 3)
    assert b.device_step() == 4 and torch.equal(b.gather_fp32("master"), want)
    b.train_step(x, y)
    torch.cuda.synchronize()
    assert b.error_code() == 0
    b.close()


@pytest.mark.gpu
def test_launcher_hadamard_writes_ef_norm_and_code_stats(tmp_path, monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    args = add_fit_args(argparse.ArgumentParser(), [
        "--network", "ResNet18", "--dataset", "Cifar10", "--synthetic", "1", "--train-len", "512", "--test-len", "64",
        "--batch-size", "32", "--test-batch-size", "64", "--backend", "p2p", "--dtype", "bf16", "--max-steps", "6",
        "--log-interval", "2", "--eval-freq", "100", "--train-dir", str(tmp_path) + "/",
        "--metrics-file", str(tmp_path / "m"), "--code", "hadamard", "--quantization-level", "4", "--bucket-size",
        "512", "--error-feedback", "1", "--code-stats", "1"])
    L.run_p2p_training(args)
    recs = [json.loads(l) for l in open(str(tmp_path / "m") + ".rank0.jsonl")]
    assert recs and all(r["ef_norm"] > 0 and math.isfinite(r["ef_norm"]) for r in recs)
    m = recs[-1]["code_stats"]["model"]
    assert m["atoms"] > 0 and 0 < m["rel_var"] < 0.1


@pytest.mark.gpu
@pytest.mark.multigpu
def test_shadow_engine_hadamard_multi_gpu_replicas_identical():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 8 else (8 if os.environ.get("ATOMO_TEST_WORLD8") else 2)
    res = run_mp(world, {"code": "hadamard", "ps_mode": "sharded", "net": "VGG11"}, 29813)
    for rank, err, same, l0, l1, mode, mc, _ in res:
        assert err == 0 and same, res

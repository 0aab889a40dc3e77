"""FP8 (e4m3, stochastic rounding) on the bf16 engine (``code="fp8"``, csrc/v2_fp8.cu): the ``codings.fp8`` oracle,
the planner, the refusals and the launcher routing (CPU); the encode against the oracle bit for bit with the in-graph
Philox draws, the PS, error feedback and ``--code-stats`` (GPU loopback harness); and the engine end to end (GPU)."""
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
# the 1728-element stem, 3x3 convs (one a multiple of the 4096-element tile, one not), fc layers, a tensor smaller than
# a bucket, a vector, an all-zero tensor (ZERO), one with zeros and -0 (SIGNED_ZERO), one with an Inf (INF)
ORACLE_SHAPES = [(64, 3, 3, 3), (64, 32, 3, 3), (128, 64, 3, 3), (96, 64, 3, 3), (10, 512), (300, 200), (7, 20), (5, 3),
                 (64,), (32, 16, 3, 3), (40, 30), (48, 16, 3, 3)]
ZERO, SIGNED_ZERO, INF = 9, 10, 11
BUCKETS = [64, 512, 4096]


def _coder(bucket, seed=7):
    from atomo_b200.codings.fp8 import FP8
    return FP8(bucket, seed=seed)


# ---------------------------------------------------------------------------------------------------- CPU: coder
def test_e4m3_table_matches_torch():
    from atomo_b200.codings.fp8 import e4m3_encode, e4m3_table
    t = e4m3_table()
    ref = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).double().numpy()
    fin = np.isfinite(ref)
    assert fin.sum() == 254 and np.array_equal(np.isnan(t), ~fin)
    assert np.array_equal(t[fin], ref[fin])
    pos = fin & (np.arange(256) < 128)
    assert np.array_equal(e4m3_encode(t[pos]), np.arange(256)[pos])


@pytest.mark.parametrize("bucket", BUCKETS)
def test_coder_bytes_scales_and_neighbours(bucket):
    """Every byte is a finite e4m3 value, every scale a power of two with amax 2^k in (224, 448], and every decoded
    element is lo or hi of its scaled magnitude."""
    from atomo_b200.codings.fp8 import e4m3_table, round_neighbours
    rng = np.random.default_rng(bucket)
    x = torch.from_numpy(np.concatenate([rng.standard_normal(3 * bucket + 70) * 10.0 ** rng.integers(-6, 4),
                                         rng.standard_t(1.5, 2 * bucket)])).float().bfloat16().float()
    c = _coder(bucket)
    code = c.encode(x, unit=5, step=3, worker=1)
    b = code["bytes"].numpy()
    assert not np.isin(b, [0x7F, 0xFF]).any()
    s = code["scales"].numpy().astype(np.float64)
    m, _ = np.frexp(s)
    assert np.all(m == 0.5)                                # powers of two
    xs = np.zeros(len(s) * bucket)
    xs[:x.numel()] = x.numpy()
    xs = xs.reshape(len(s), bucket)
    xb = np.abs(xs)
    amax = xb.max(axis=1)
    assert np.all((amax / s > 224) & (amax / s <= 448))
    y = xb / s[:, None]
    lo, ulp = round_neighbours(y)
    v = np.abs(e4m3_table()[b[:, :bucket]])
    assert np.all((v == lo) | (v == lo + ulp))
    assert np.array_equal(b[:, :bucket] >= 128, (xs < 0) & (v > 0))    # the sign of x, never -0
    dec = c.decode(code)
    assert torch.equal(dec.view(-1).abs().double(), torch.from_numpy((v * s[:, None]).reshape(-1)[:x.numel()]))


def test_coder_zeros_signed_zero_and_padding():
    c = _coder(64)
    x = torch.tensor([1.0, -2.0, 0.0, -0.0, 3.0] + [-1.0] * 59 + [0.5, -0.5, -0.0])
    code = c.encode(x)
    b = code["bytes"]
    assert b.shape == (2, 64) and code["scales"].shape == (2,)
    assert int(b[0, 2]) == 0 and int(b[0, 3]) == 0 and int(b[1, 2]) == 0        # +0 and -0 are 0x00
    assert bool((b[1, 3:] == 0).all())                                           # padding of the tail bucket
    assert float(code["scales"][0]) == 2.0 ** -7 and float(code["scales"][1]) == 2.0 ** -9   # 3 * 2^7, 0.5 * 2^9
    z = c.encode(torch.zeros(100))
    assert bool((z["scales"] == 0).all()) and bool((z["bytes"] == 0).all())
    assert bool((c.decode(z) == 0).all())


@pytest.mark.parametrize("bucket", BUCKETS)
def test_coder_tail_bucket_and_small_tensor(bucket):
    g = torch.Generator().manual_seed(bucket + 1)
    for n in (1, 40, bucket - 1, bucket, bucket + 3, 3 * bucket + 70):
        x = torch.randn(n, generator=g).bfloat16().float()
        c = _coder(bucket)
        code = c.encode(x)
        b = min(bucket, n)
        nb = -(-n // b)
        assert code["bucket_size"] == b and code["bytes"].shape == (nb, 8 * -(-b // 8))
        dec = c.decode(code)
        assert dec.shape == x.shape and bool(torch.isfinite(dec).all())
        s = code["scales"].repeat_interleave(b)[:n]
        assert bool(((dec - x).abs() <= torch.maximum(x.abs() / 8, s * 2.0 ** -9)).all())   # one e4m3 step at most


def test_coder_special_buckets_clamp_and_flush():
    c = _coder(64)
    # k clamp: amax = 2^-120 wants k = 128; clamped to 117 so the least decoded value 2^-126 stays normal
    x = torch.full((64,), 2.0 ** -125)
    x[1] = 2.0 ** -120
    x[2:10] = 1.5 * 2.0 ** -126                           # between the two least e4m3 steps after scaling
    code = c.encode(x)
    assert float(code["scales"][0]) == 2.0 ** -117
    dec = c.decode(code)
    assert bool(torch.isfinite(dec).all()) and float(dec[1]) == 2.0 ** -120
    assert bool(((dec == 0) | (dec.abs() >= 2.0 ** -126)).all())
    # bf16 subnormals read as zero
    sub = torch.zeros(64)
    sub[:8] = 2.0 ** -130
    code = c.encode(sub)
    assert float(code["scales"][0]) == 0 and bool((code["bytes"] == 0).all())
    # an Inf, a NaN or amax >= 2^126 poisons its bucket only
    for bad in (float("inf"), float("nan"), 2.0 ** 126):
        x = torch.randn(256)
        x[70] = bad
        code = c.encode(x)
        s = code["scales"]
        assert torch.isnan(s[1]) and bool(torch.isfinite(s[[0, 2, 3]]).all())
        assert bool((code["bytes"][1] == 0).all())
        dec = c.decode(code)
        assert bool(torch.isnan(dec[64:128]).all()) and bool(torch.isfinite(dec[:64]).all())
        assert math.isnan(c.expected_error_sq(x))
    x = torch.randn(256)
    x[70] = 2.0 ** 125                                     # below 2^126: a normal bucket
    assert bool(torch.isfinite(c.encode(x)["scales"]).all())


def test_coder_explicit_uniforms():
    from atomo_b200.codings.fp8 import round_neighbours
    c = _coder(64)
    x = torch.randn(200).bfloat16().float()
    lo_code = c.encode(x, u=np.full(200, 1.0 - 2.0 ** -24, dtype=np.float32))
    hi_code = c.encode(x, u=np.zeros(200, dtype=np.float32))
    s = np.repeat(lo_code["scales"].numpy().astype(np.float64), 64)[:200]
    lo, ulp = round_neighbours(np.abs(x.numpy()) / s)
    exact = lo == np.abs(x.numpy()) / s
    assert np.array_equal(c.decode(lo_code).abs().numpy() / s, lo)
    assert np.array_equal(c.decode(hi_code).abs().numpy() / s, np.where(exact, lo, lo + ulp))
    # the keyed draws are the default uniforms
    from atomo_b200.codings.fp8 import uniforms
    u = uniforms(7, 4, 9, 2, 200)
    assert torch.equal(c.encode(x, unit=4, step=9, worker=2)["bytes"], c.encode(x, u=u)["bytes"])
    assert not torch.equal(c.encode(x, unit=4, step=9, worker=2)["bytes"], c.encode(x, unit=4, step=10, worker=2)["bytes"])


@pytest.mark.parametrize("dist", ["normal", "laplace", "student1.5"])
def test_coder_unbiased_and_variance_matches_closed_form(dist):
    """Over T keyed draws (steps 1..T) the mean converges to x and the summed squared error to expected_error_sq(),
    within CLT bounds."""
    from atomo_b200.codings.fp8 import round_neighbours
    rng = np.random.default_rng(3)
    n = 512
    x = {"normal": lambda k: rng.standard_normal(k), "laplace": lambda k: rng.laplace(size=k),
         "student1.5": lambda k: rng.standard_t(1.5, k)}[dist](n)
    x = torch.from_numpy(x).float().bfloat16().float()
    c = _coder(64)
    T = 1500
    dec = torch.stack([c.decode(c.encode(x, unit=2, step=t)) for t in range(1, T + 1)]).double()
    xd = x.double()
    err = dec - xd
    # per element: the mean error has sd sqrt(var_i / T) with var_i = (y - lo)(hi - y) 2^-2k; one draw's ulp of
    # slack for the binomial's discreteness when p is near 0 or 1
    s = np.repeat(c.encode(x)["scales"].numpy().astype(np.float64), 64)[:n]
    y = np.abs(x.numpy()) / s
    lo, ulp = round_neighbours(y)
    var_i = torch.from_numpy((y - lo) * (lo + ulp - y) * s * s)
    assert bool((err.mean(dim=0).abs() <= 6 * torch.sqrt(var_i / T) + torch.from_numpy(ulp * s) / T).all())
    want = c.expected_error_sq(x)
    got = float(err.square().sum(dim=1).mean())
    sd = float(err.square().sum(dim=1).std()) / math.sqrt(T)
    assert abs(got - want) <= 5 * sd, (got, want, sd)
    assert 5e-4 < want / float(xd.square().sum()) < 3e-3          # ~0.0014 whatever the distribution


def test_coder_refuses_bucket_sizes():
    for b in (0, 32, 100, 4160, 8192):
        with pytest.raises(ValueError, match="fp8: bucket_size must be a multiple of 64"):
            _coder(b)


# ---------------------------------------------------------------------------------------------------- CPU: planner
@pytest.mark.parametrize("owners", [1, 2, 8])
@pytest.mark.parametrize("bucket", BUCKETS)
def test_plan2_fp8_units_tiles_and_slots(bucket, owners):
    pl = P.build_plan2(NET_SHAPES, "fp8", n_owners=owners, n_groups=3, bucket_size=bucket)
    for p in pl.params:
        units = [u for u in pl.units if u.param == p.index]
        assert len(units) == 1
        u = units[0]
        if not p.is_w:
            assert u.kind == P.KIND_VEC
            continue
        b = min(bucket, p.numel)
        bpt = max(1, 4096 // b)
        assert u.kind == P.KIND_FP8 and (u.K, u.numel, u.w_off, u.I, u.rs) == (b, p.numel, p.off, 0, 0)
        assert u.rows == -(-p.numel // b) and u.cols == -(-b // 8) and u.cs == bpt and u.ps_rows == bpt * b
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
        if u.kind == P.KIND_FP8:
            wo = u.slot_off + P.qsgd_words_off(u.n_ps, u.rows)
            assert u.slot_off % 4 == 0 and wo % 4 == 0
            spans.append((u.slot_off, u.slot_off + P.qsgd_slot_floats(u.n_ps, u.rows, u.cols)))
            assert wo + 2 * u.rows * u.cols <= spans[-1][1]
            # the encode's last 16-byte store of a one-bucket tensor stays inside the slot
            assert wo + (2 * u.rows * u.cols + 3) // 4 * 4 <= spans[-1][1]
    spans.sort()
    assert all(a1 >= b0 for (a0, b0), (a1, b1) in zip(spans, spans[1:])) and spans[-1][1] <= pl.arena_floats
    c = _coder(bucket)
    want = 0
    for s in NET_SHAPES:
        if len(s) >= 2:
            code = c.encode(torch.zeros(s))
            want += code["bytes"].numel() + 4 * code["scales"].numel()
    assert pl.qsgd_bytes() == want and pl.expected_factor_bytes() == want
    assert pl.dense_bytes() == 4 * sum(p.numel for p in pl.params if not p.is_w)


def test_plan2_fp8_push_bytes_from_shapes():
    """One byte per weight element (tail buckets padded) plus 4 per bucket: ResNet-18 at bucket 512 pushes ~10.7 MiB per step."""
    from atomo_b200.models import build_model
    shapes = [tuple(p.shape) for p in build_model("ResNet18", 10).parameters()]
    pl = P.build_plan2(shapes, "fp8", bucket_size=512)
    n = sum(math.prod(s) for s in shapes if len(s) >= 2)
    assert pl.qsgd_bytes() == sum(u.rows * 8 * u.cols + 4 * u.rows for u in pl.units if u.kind == P.KIND_FP8)
    n_units = sum(1 for u in pl.units if u.kind == P.KIND_FP8)
    assert n <= pl.qsgd_bytes() <= n * (1 + 4 / 512) + n_units * (512 + 4)     # padded tail buckets
    assert 10.6 < pl.qsgd_bytes() / 2 ** 20 < 10.8


def test_plan2_fp8_refuses_bucket_sizes():
    for b in (0, 32, 100, 4160, 8192):
        with pytest.raises(ValueError, match="fp8: bucket_size must be a multiple of 64"):
            P.build_plan2(NET_SHAPES, "fp8", bucket_size=b)


def test_plan2_other_codes_unchanged_by_the_new_code():
    """Digests of the plans of the existing codes, taken from the planner before the fp8 code was added."""
    want = {"svd": "917543867e0167683f770150a43eaf4c129e4d461aa989111b2a491e5eeca388",
            "qsvd": "6ea73c4cd4a95d51288ea6c2a2053f66ff7800fc277120bdccfda766e92e3cf9",
            "sgd": "6d3fd294b9211300d2945b4d3f20d6bf9615e56c5dfa3bab6b294fa9370a37d8",
            "qsgd": "1f34b0853ed1349c3ede1baad5eecd6d7a8e9d4bd571740ec8e531cedbfe275c",
            "terngrad": "5ab388e54d2c51d29226927eaa996c37b3173a968114dce188b5cb8121895e57",
            "entrywise": "5ec97d1b33d12cee3ed4b7b6466f49526420e0442c54d8d8aa9634e1cfe73dcf",
            "topk": "0fed82b9ada85f2510d5f1e0b047978d4124c2a1bd1557bba9353e0d7fae72f0",
            "sign": "81b324f24294287fe7a390c33fc80496d4e05e4f6e2236d722a14a87cc73cb97",
            "powersgd": "dd44d14dac1cdad253f1ff4a89cb2423202cac1056532f643b917a03966a9ffc"}
    for code, digest in want.items():
        pl = P.build_plan2(NET_SHAPES, code, 3, n_owners=2, n_groups=3, entry_budget=0.05)
        b = pl.units_bytes() + P.Plan2.tiles_bytes(pl.enc_tiles) + P.Plan2.tiles_bytes(pl.ps_tiles) + \
            repr((pl.enc_range, pl.ps_range, pl.arena_floats, pl.n_coded)).encode()
        assert hashlib.sha256(b).hexdigest() == digest, code


@pytest.mark.parametrize("bucket", [0, 32, 100, 4160])
def test_shadow_engine_fp8_refuses_before_cuda(bucket, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    forbid_cuda(monkeypatch)
    with pytest.raises(ValueError, match="fp8: bucket_size must be a multiple of 64"):
        S.ShadowEngine(None, 0, 1, code="fp8", bucket_size=bucket)
    with pytest.raises(ValueError, match="num_aggregate"):     # the error-feedback rule applies unchanged
        S.ShadowEngine(None, 0, 4, code="fp8", error_feedback=True, num_aggregate=2)


# ---------------------------------------------------------------------------------------------------- CPU: launcher
def test_launcher_routes_fp8(tmp_path, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    seen = []

    class Fake:
        def __init__(self, model, rank, world, **kw):
            seen.append(kw)
    monkeypatch.setattr(S, "ShadowEngine", Fake)
    model = torch.nn.Linear(4, 4)
    for engine in ("auto", "shadow"):
        _, kind = L._build_engine(fit_args(tmp_path, "--code", "fp8", "--dtype", "bf16", "--engine", engine,
                                        "--bucket-size", "256", "--error-feedback", "1", "--code-stats", "1"),
                                  model, 0, 1)
        assert kind == "shadow" and seen[-1]["code"] == "fp8" and seen[-1]["bucket_size"] == 256
        assert seen[-1]["error_feedback"] is True and seen[-1]["code_stats"] is True
    n = len(seen)
    for extra in (("--dtype", "fp32"), ("--dtype", "bf16", "--engine", "fused")):
        with pytest.raises(SystemExit, match="fp8"):
            L._build_engine(fit_args(tmp_path, "--code", "fp8", *extra), model, 0, 1)
    assert len(seen) == n


def test_role_paths_refuse_fp8(monkeypatch, tmp_path):
    from atomo_b200 import distributed_nn
    from atomo_b200.runtime.master import build_coder
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    with pytest.raises(SystemExit, match="p2p bf16 engine"):
        distributed_nn.run_rank(fit_args(tmp_path, "--code", "fp8", "--backend", "gloo"))
    with pytest.raises(ValueError, match="p2p bf16 engine"):
        build_coder({"code": "fp8", "bucket_size": 512}, worker_side=True)


# ---------------------------------------------------------------------------------------------------- GPU harness
class HF(LoopbackPS):
    """FP8 e4m3; with ``special``, ``fill`` gives the ZERO / SIGNED_ZERO / INF tensors of ORACLE_SHAPES their
    content."""

    PS = "v2_ps_fp8"

    def __init__(self, shapes, bucket=512, W=1, lr=0.1, momentum=0.0, wd=0.0, nesterov=False, opt=0, seed=7,
                 num_aggregate=0):
        super().__init__(shapes, "fp8", W, lr, momentum, wd, nesterov, opt, seed, num_aggregate, bucket_size=bucket)
        self.bucket = bucket
        self.spart = self.zeros(5 * max(len(self.plan.enc_tiles), 1), torch.float64)
        self.acc = self.zeros(7 * self.nc, torch.float64)

    def tensor(self, q, x, g, special=False):
        if special and q.index == ZERO:
            x.zero_()
        elif special and q.index == SIGNED_ZERO:
            r = torch.rand(q.shape, device=self.dev, generator=g)
            x = torch.where(r < 0.3, torch.zeros_like(x), torch.where(r < 0.6, -torch.zeros_like(x), x))
        if special and q.index == INF:
            x = physical(x)
            flat(x)[1234] = float("inf")
        return x

    def encode(self, w, residual=0, stats=False):
        C, pl = self.C, self.plan
        gptr = self.gptr(w)
        t0, nt = pl.enc_range[0]
        C.v2_fp8_encode(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr,
                        self.t_arena_peer.data_ptr(), self.t_sig_peer.data_ptr(), 1, pl.arena_floats, w, 0,
                        self.ctrl.data_ptr(), self.counter(), 0, False, residual)
        if stats:
            C.v2_fp8_code_stats(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr,
                                self.t_arena_peer.data_ptr(), 1, pl.arena_floats, w, self.spart.data_ptr(),
                                self.counters.data_ptr(), self.acc.data_ptr())
        torch.cuda.synchronize()

    def slot(self, u, w):
        """(stamps, scales, bytes [buckets, 8 L] uint8) of unit u in worker w's slot."""
        base = self.arena[w * self.plan.arena_floats + u.slot_off:]
        stamps = base[:u.n_ps].view(torch.int32).clone()
        so, wo = P.qsgd_norms_off(u.n_ps), P.qsgd_words_off(u.n_ps, u.rows)
        scales = base[so:so + u.rows].clone()
        byts = base[wo:wo + 2 * u.rows * u.cols].view(torch.uint8).view(u.rows, 8 * u.cols).clone()
        return stamps, scales, byts

    def oracle(self, u, x, w):
        """The oracle's encode of unit u's physical-order gradient x by worker w at the current step."""
        return _coder(self.bucket, self.seed).encode(x.cpu(), unit=u.index, step=self.step, worker=w)


def _decoded_sum(h, phys_by_worker):
    """sum over workers (in worker order, fp32, CPU) of the oracle's decodes, physical order."""
    est = torch.zeros(h.plan.w_total)
    for w, phys in enumerate(phys_by_worker):
        for u in h.plan.units:
            if u.kind == P.KIND_FP8:
                est[u.w_off:u.w_off + u.numel] += _coder(h.bucket).decode_flat(h.oracle(u, phys[u.param], w))
    return est


# ---------------------------------------------------------------------------------------------------- GPU: encode
@pytest.mark.gpu
@pytest.mark.parametrize("bucket", BUCKETS)
def test_v2_fp8_encode_matches_oracle_bitwise(bucket):
    h = HF(ORACLE_SHAPES, bucket)
    h.set_step(3)
    phys = h.fill(0, 11, special=True)
    h.encode(0)
    first = h.arena.clone()
    for u in h.plan.units:
        if u.kind != P.KIND_FP8:
            continue
        ref = h.oracle(u, phys[u.param], 0)
        stamps, scales, byts = h.slot(u, 0)
        assert bool((stamps == 3).all()), u.param
        assert torch.equal(scales.cpu().view(torch.int32), ref["scales"].view(torch.int32)), u.param
        assert torch.equal(byts.cpu(), ref["bytes"]), u.param
        if u.param == ZERO:
            assert bool((scales == 0).all()) and bool((byts == 0).all())
        if u.param == INF:          # only the bucket holding the Inf is non-finite
            bad = (~torch.isfinite(scales)).nonzero().flatten().tolist()
            assert bad == [1234 // u.K]
    assert int(h.signals[0]) == 3
    h.arena.zero_()                  # a second encode of the same gradient and step: the same bits
    h.encode(0)
    assert torch.equal(h.arena.view(torch.int32), first.view(torch.int32))
    u = next(u for u in h.plan.units if u.kind == P.KIND_FP8 and u.param == 2)
    ref3 = h.oracle(u, phys[u.param], 0)["bytes"]
    h.set_step(4)                    # the next step draws afresh, still the oracle's draws
    h.encode(0)
    assert torch.equal(h.slot(u, 0)[2].cpu(), h.oracle(u, phys[u.param], 0)["bytes"])
    assert not torch.equal(h.slot(u, 0)[2].cpu(), ref3)


# ---------------------------------------------------------------------------------------------------- GPU: PS
@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 2])
@pytest.mark.parametrize("bucket", [64, 512])
def test_v2_ps_fp8_decoded_mean_is_bitwise_the_oracles(W, bucket):
    """lr = 1, no momentum, a zero master: the PS writes -(oracle decodes summed in worker order) * fp32(1 / W)."""
    h = HF(NET_SHAPES, bucket, W=W, lr=1.0)
    phys = []
    for w in range(W):
        phys.append(h.fill(w, 70 + w))
        h.encode(w)
    want = (_decoded_sum(h, phys) * torch.tensor(1.0 / W, dtype=torch.float32)).to(h.dev)
    h.master.zero_()
    h.ps()
    assert int(h.ctrl.view(torch.int32)[1]) == 0
    used, _ = h.used()
    assert torch.equal(-h.master[used], want[used])


@pytest.mark.gpu
@pytest.mark.parametrize("momentum,nesterov,wd,opt", [(0.0, False, 0.0, 0), (0.9, True, 1e-3, 0), (0.9, False, 0.0, 0),
                                                      (0.0, False, 0.0, 1), (0.0, False, 1e-3, 2)])
def test_v2_ps_fp8_matches_reference(momentum, nesterov, wd, opt):
    W, lr = 3, 0.05
    h = HF(NET_SHAPES, 512, W=W, lr=lr, momentum=momentum, wd=wd, nesterov=nesterov, opt=opt)
    used, vused = h.used()
    for step in (1, 2):
        h.set_step(step)
        phys = []
        for w in range(W):
            phys.append(h.fill(w, 10 * step + w))
            h.encode(w)
        gw = _decoded_sum(h, phys).to(h.dev) / W
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
def test_v2_ps_fp8_num_aggregate_and_stale_slots():
    """num_aggregate = 2 of 3 workers, worker 1 never pushes: only {0, 2} are averaged.  Then a slot whose stamp is of
    another step is skipped and flagged with ERR2_SLOT_STEP."""
    lr = 0.1
    h = HF(NET_SHAPES, 512, W=3, lr=lr, num_aggregate=2)
    phys = [None, None, None]
    for w in (0, 2):
        phys[w] = h.fill(w, 40 + w)
        h.encode(w)
    h.vgrads[1].fill_(1e6)                         # garbage a skipped worker may hold
    assert int(h.signals[0]) == 1 and int(h.signals[1]) == 0 and int(h.signals[2]) == 1
    est = torch.zeros(h.plan.w_total)
    for w in (0, 2):
        for u in h.plan.units:
            if u.kind == P.KIND_FP8:
                est[u.w_off:u.w_off + u.numel] += _coder(512).decode_flat(h.oracle(u, phys[w][u.param], w))
    est = est.to(h.dev)
    p0, v0 = h.master.clone(), h.vparams.clone()
    h.ps()
    assert int(h.ctrl.view(torch.int32)[1]) == 0 and int(h.signals[256]) == 2
    assert int(h.signals[320]) == 0b101 and int(h.signals[321]) == 1
    used, vused = h.used()
    assert torch.allclose(h.master[used], (p0 - lr * est / 2)[used], rtol=3e-4, atol=3e-5)
    assert torch.allclose(h.vparams[vused], (v0 - lr * (h.vgrads[0] + h.vgrads[2]) / 2)[vused], rtol=3e-4, atol=3e-5)

    hs = HF(NET_SHAPES, 512, W=2, lr=lr)            # worker 1's slot holds step 0 while its flag claims step 1
    hs.fill(0, 1)
    hs.encode(0)
    hs.signals[1] = 1
    hs.ps()
    assert int(hs.ctrl.view(torch.int32)[1]) & 4          # ERR2_SLOT_STEP


# ---------------------------------------------------------------------------------------------------- GPU: stats
@pytest.mark.gpu
@pytest.mark.parametrize("bucket", BUCKETS)
def test_v2_fp8_code_stats_match_fp64(bucket):
    h = HF(ORACLE_SHAPES, bucket)
    h.set_step(2)
    phys = h.fill(0, 21, special=True)
    h.encode(0, stats=True)
    acc = h.acc.view(-1, 7).tolist()
    from atomo_b200.codings.sign import bf16_flushed
    for u in h.plan.units:
        if u.kind != P.KIND_FP8:
            continue
        gsq, mse, ex, bias, real, real4, n = acc[u.ts_index]
        if u.param == INF:
            assert math.isnan(mse)
            continue
        x = torch.from_numpy(bf16_flushed(phys[u.param].cpu())).double()
        assert n == 1 and bias == 0 and ex == real == real4 == u.numel
        assert gsq == pytest.approx(float(x.square().sum()), rel=1e-12, abs=0)
        assert mse == pytest.approx(_coder(bucket).expected_error_sq(phys[u.param].cpu()), rel=1e-12, abs=1e-300)
        if u.param != ZERO:
            assert 0 < mse < 3e-3 * gsq


@pytest.mark.gpu
def test_v2_fp8_code_stats_agree_with_sampled_error():
    """The closed-form expected error against the error of 400 encodes (steps 1..400) decoded on the GPU."""
    h = HF([(64, 32, 3, 3), (300, 200), (7, 20)], 512)
    phys = h.fill(0, 5)
    sq = torch.zeros(h.plan.w_total, dtype=torch.float64, device=h.dev)
    T = 400
    per_step = []
    for step in range(1, T + 1):
        h.set_step(step)
        h.encode(0, stats=True)
        tot = 0.0
        for u in h.plan.units:
            if u.kind != P.KIND_FP8:
                continue
            _, scales, byts = h.slot(u, 0)
            dec = (byts[:, :u.K].contiguous().view(torch.float8_e4m3fn).float() * scales[:, None]).reshape(-1)
            e = (dec[:u.numel].double() - phys[u.param].double()).square()
            tot += float(e.sum())
        per_step.append(tot)
    acc = h.acc.view(-1, 7)
    assert float(acc[0, 6]) == T
    want = float(acc[:, 1].sum()) / T
    per = torch.tensor(per_step, dtype=torch.float64)
    assert abs(float(per.mean()) - want) <= 5 * float(per.std()) / math.sqrt(T), (float(per.mean()), want)


# ---------------------------------------------------------------------------------------------------- GPU: feedback
@pytest.mark.gpu
@pytest.mark.parametrize("bucket", BUCKETS)
def test_error_feedback_identity(bucket):
    h = Loopback("fp8", ef_grads(1), bucket_size=bucket)
    try:
        g, e_old = h.g, h.residual()
        for _ in range(4):
            A = g + e_old
            ghat, e_new = h.step()
            scale = g.abs() + e_old.abs() + ghat.abs() + e_new.abs()
            assert bool(((A - (ghat + e_new)).abs() <= 1e-6 * scale + 1e-7 * float(scale.max())).all())
            assert 0 < float(e_new.norm()) <= 0.2 * float(A.norm())
            e_old = e_new
    finally:
        h.close()


@pytest.mark.gpu
def test_error_feedback_residual_stays_bounded():
    """A fixed gradient for 200 steps: every step leaves at most one e4m3 step of each element (||e_{t+1}|| <= rho
    ||g + e_t||, rho < 1), so ||e|| stays below rho / (1 - rho) ||g||; the pushed sum misses 200 g by exactly the
    final residual."""
    h = Loopback("fp8", ef_grads(2), bucket_size=512)
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
        assert rho < 0.2
        assert max(norms) <= rho / (1 - rho) * float(h.g.norm()) * (1 + 1e-4)
        assert torch.allclose(s - 200 * h.g, -e, rtol=0, atol=200 * 1e-6 * (float(h.g.abs().max()) + float(e.abs().max())))
    finally:
        h.close()


@pytest.mark.gpu
def test_code_stats_bytes_follow_the_plan():
    h = Loopback("fp8", ef_grads(4), bucket_size=256, code_stats=True)
    try:
        h.step()
        st = h.eng.code_stats()
        pl = h.eng.plan
        assert st["code"] == "fp8" and st["steps"] == 1
        names = {id(p): n for n, p in h.eng.model.named_parameters()}
        for u in pl.units:
            t = st["tensors"][names[id(h.eng.params[u.param])]]
            if u.kind == P.KIND_FP8:
                assert t["bytes"] == 8 * u.rows * u.cols + 4 * u.rows
                assert t["atoms"] == t["exp_atoms"] == u.numel and 0 < t["rel_var"] < 3e-3
        assert st["model"]["bytes"] == pl.qsgd_bytes() + pl.dense_bytes()
    finally:
        h.close()


# ---------------------------------------------------------------------------------------------------- GPU: engine
_train = functools.partial(train, code="fp8", bucket_size=512)


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
    """lr 0.05 / momentum 0.9: the setting where the unbiased codes with a large variance diverge under error
    feedback."""
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
        return ShadowEngine(build_model("VGG11", 10), 0, 1, code="fp8", bucket_size=256, lr=0.05, momentum=0.9,
                            use_graph=False)
    a = mk()
    a.prepare(x.pin_memory(), y.pin_memory(), warmup=0)
    for _ in range(3):
        a.train_step(x, y)
    path = a.save_checkpoint(str(tmp_path) + "/")
    side = torch.load(path + "_optim", weights_only=False)
    assert side["code"] == "fp8" and side["bucket_size"] == 256
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
def test_launcher_fp8_writes_ef_norm_and_code_stats(tmp_path, monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    args = add_fit_args(argparse.ArgumentParser(), [
        "--network", "ResNet18", "--dataset", "Cifar10", "--synthetic", "1", "--train-len", "512", "--test-len", "64",
        "--batch-size", "32", "--test-batch-size", "64", "--backend", "p2p", "--dtype", "bf16", "--max-steps", "6",
        "--log-interval", "2", "--eval-freq", "100", "--train-dir", str(tmp_path) + "/",
        "--metrics-file", str(tmp_path / "m"), "--code", "fp8", "--bucket-size", "512", "--error-feedback", "1",
        "--code-stats", "1"])
    L.run_p2p_training(args)
    recs = [json.loads(l) for l in open(str(tmp_path / "m") + ".rank0.jsonl")]
    assert recs and all(r["ef_norm"] > 0 and math.isfinite(r["ef_norm"]) for r in recs)
    m = recs[-1]["code_stats"]["model"]
    assert m["atoms"] > 0 and 0 < m["rel_var"] < 3e-3


@pytest.mark.gpu
@pytest.mark.multigpu
def test_shadow_engine_fp8_multi_gpu_replicas_identical():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 8 else (8 if os.environ.get("ATOMO_TEST_WORLD8") else 2)
    res = run_mp(world, {"code": "fp8", "ps_mode": "sharded", "net": "VGG11"}, 29812)
    for rank, err, same, l0, l1, mode, mc, _ in res:
        assert err == 0 and same, res

"""Scaled sign on the bf16 engine (``code="sign"``, csrc/v2_sign.cu): the ``codings.sign`` oracle, the planner, the
refusals and the launcher routing (CPU); the encode against the oracle bit for bit, the PS, error feedback and
``--code-stats`` (GPU loopback harness); and the engine end to end (GPU)."""
import argparse
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

NET_SHAPES = [(64, 3, 3, 3), (64,), (64,), (128, 64, 3, 3), (128,), (256, 128, 3, 3), (512, 256, 1, 1), (300, 200),
              (10, 512), (7, 20), (10,)]
# the 1728-element stem, 3x3 convs (one a multiple of the 4096-element tile, one not), fc layers, a tensor smaller than
# a bucket, a vector, an all-zero tensor (ZERO), one with zeros and -0 (SIGNED_ZERO), one with an Inf (INF)
ORACLE_SHAPES = [(64, 3, 3, 3), (64, 32, 3, 3), (128, 64, 3, 3), (96, 64, 3, 3), (10, 512), (300, 200), (7, 20), (5, 3),
                 (64,), (32, 16, 3, 3), (40, 30), (48, 16, 3, 3)]
ZERO, SIGNED_ZERO, INF = 9, 10, 11
BUCKETS = [64, 512, 4096]


def _coder(bucket):
    from atomo_b200.codings.sign import ScaledSign
    return ScaledSign(bucket)


# ---------------------------------------------------------------------------------------------------- CPU: coder
def test_coder_bit_layout_and_signed_zero():
    x = torch.tensor([1.0, -2.0, 0.0, -0.0, 3.0] + [-1.0] * 59 + [0.5, -0.5, -0.0])
    code = _coder(64).encode(x)
    assert code["words"].shape == (2, 1) and code["scales"].shape == (2,)
    w0 = int(code["words"][0, 0]) & (2 ** 64 - 1)
    assert w0 == sum(1 << i for i in [1] + list(range(5, 64)))    # bit i of word j = element 64 j + i < 0
    assert int(code["words"][1, 0]) == 0b10                       # tail bucket: -0 is not negative, padding is 0
    assert float(code["scales"][0]) == np.float32((1 + 2 + 3 + 59) / 64)
    assert float(code["scales"][1]) == np.float32(1.0 / 3)          # divided by the real length 3
    dec = _coder(64).decode(code)
    assert dec[2] > 0 and dec[3] > 0 and dec[66] > 0                # +0 and -0 decode to +scale
    assert torch.equal(dec[:64].abs(), torch.full((64,), float(code["scales"][0])))
    assert _coder(64).encode(torch.zeros(100))["scales"].abs().sum() == 0   # all zero: scale 0, decodes to 0
    assert bool((_coder(64).decode(_coder(64).encode(torch.zeros(100))) == 0).all())


@pytest.mark.parametrize("bucket", BUCKETS)
def test_coder_tail_bucket_and_small_tensor(bucket):
    g = torch.Generator().manual_seed(bucket)
    for n in (1, 40, bucket - 1, bucket, bucket + 3, 3 * bucket + 70):
        x = torch.randn(n, generator=g).bfloat16().float()
        c = _coder(bucket)
        code = c.encode(x)
        b = min(bucket, n)
        nb = -(-n // b)
        assert code["bucket_size"] == b and code["words"].shape == (nb, -(-b // 64))
        for k in range(nb):
            seg = x[k * b:(k + 1) * b].double()
            assert float(code["scales"][k]) == pytest.approx(float(seg.abs().sum() / seg.numel()), rel=1e-7)
        dec = c.decode(code)
        assert dec.shape == x.shape
        assert torch.equal(torch.signbit(dec), x < 0)


@pytest.mark.parametrize("bucket", BUCKETS)
@pytest.mark.parametrize("kind", ["random", "tied", "spiky"])
def test_coder_error_identity_and_contraction(bucket, kind):
    g = torch.Generator().manual_seed(7)
    n = 5 * bucket + 37
    x = torch.randn(n, generator=g)
    if kind == "tied":
        x = (x * 2).round() / 4
    elif kind == "spiky":
        x = x * 1e-3
        x[torch.randperm(n, generator=g)[:5]] = 50.0
    c = _coder(bucket)
    xb = x.bfloat16().double()
    want, bound = 0.0, 0.0
    for k in range(0, n, bucket):
        seg = xb[k:k + bucket]
        want += float(seg.square().sum() - seg.abs().sum() ** 2 / seg.numel())
        bound += (1 - 1 / seg.numel()) * float(seg.square().sum())
    err = c.error_sq(x)
    assert err == pytest.approx(want, rel=1e-9, abs=1e-12)
    assert err <= bound * (1 + 1e-12)
    assert err < float(xb.square().sum())


def test_coder_refuses_bucket_sizes():
    for b in (0, 32, 100, 4160, 8192):
        with pytest.raises(ValueError):
            _coder(b)


# ---------------------------------------------------------------------------------------------------- CPU: planner
@pytest.mark.parametrize("bucket,owners", [(64, 1), (512, 3), (4096, 2), (256, 4), (1024, 1)])
def test_plan2_sign_units_tiles_and_slots(bucket, owners):
    pl = P.build_plan2(NET_SHAPES, "sign", n_owners=owners, n_groups=3, bucket_size=bucket)
    for p in pl.params:
        units = [u for u in pl.units if u.param == p.index]
        assert len(units) == 1
        u = units[0]
        if not p.is_w:
            assert u.kind == P.KIND_VEC
            continue
        b = min(bucket, p.numel)
        bpt = max(1, 4096 // b)
        assert u.kind == P.KIND_SIGN and (u.K, u.numel, u.w_off, u.I, u.rs) == (b, p.numel, p.off, 0, 0)
        assert u.rows == -(-p.numel // b) and u.cols == -(-b // 64) and u.cs == bpt and u.ps_rows == bpt * b
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
        if u.kind == P.KIND_SIGN:
            wo = u.slot_off + P.qsgd_words_off(u.n_ps, u.rows)
            assert u.slot_off % 4 == 0 and wo % 4 == 0
            assert P.qsgd_norms_off(u.n_ps) >= u.n_ps and P.qsgd_words_off(u.n_ps, u.rows) >= P.qsgd_norms_off(u.n_ps) + u.rows
            spans.append((u.slot_off, u.slot_off + P.qsgd_slot_floats(u.n_ps, u.rows, u.cols)))
            assert wo + 2 * u.rows * u.cols <= spans[-1][1]
    spans.sort()
    assert all(a1 >= b0 for (a0, b0), (a1, b1) in zip(spans, spans[1:])) and spans[-1][1] <= pl.arena_floats
    c = _coder(bucket)
    want = 0
    for s in NET_SHAPES:
        if len(s) >= 2:
            code = c.encode(torch.zeros(s))
            want += 8 * code["words"].numel() + 4 * code["scales"].numel()
    assert pl.qsgd_bytes() == want and pl.expected_factor_bytes() == want
    assert pl.dense_bytes() == 4 * sum(p.numel for p in pl.params if not p.is_w)


def test_plan2_sign_refuses_bucket_sizes():
    for b in (0, 32, 100, 4160, 8192):
        with pytest.raises(ValueError, match="multiple of 64"):
            P.build_plan2(NET_SHAPES, "sign", bucket_size=b)


def test_plan2_other_codes_unchanged_by_the_new_code():
    """Digests of the plans of the existing codes, taken from the planner before the sign code was added."""
    want = {"svd": "917543867e0167683f770150a43eaf4c129e4d461aa989111b2a491e5eeca388",
            "qsvd": "6ea73c4cd4a95d51288ea6c2a2053f66ff7800fc277120bdccfda766e92e3cf9",
            "sgd": "6d3fd294b9211300d2945b4d3f20d6bf9615e56c5dfa3bab6b294fa9370a37d8",
            "qsgd": "1f34b0853ed1349c3ede1baad5eecd6d7a8e9d4bd571740ec8e531cedbfe275c",
            "terngrad": "5ab388e54d2c51d29226927eaa996c37b3173a968114dce188b5cb8121895e57",
            "entrywise": "5ec97d1b33d12cee3ed4b7b6466f49526420e0442c54d8d8aa9634e1cfe73dcf",
            "topk": "0fed82b9ada85f2510d5f1e0b047978d4124c2a1bd1557bba9353e0d7fae72f0"}
    for code, digest in want.items():
        pl = P.build_plan2(NET_SHAPES, code, 3, n_owners=2, n_groups=3, entry_budget=0.05)
        b = pl.units_bytes() + P.Plan2.tiles_bytes(pl.enc_tiles) + P.Plan2.tiles_bytes(pl.ps_tiles) + \
            repr((pl.enc_range, pl.ps_range, pl.arena_floats, pl.n_coded)).encode()
        assert hashlib.sha256(b).hexdigest() == digest, code


@pytest.mark.parametrize("bucket", [0, 32, 100, 4160])
def test_shadow_engine_sign_refuses_before_cuda(bucket, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S

    def no_cuda(*a, **k):
        raise AssertionError("refused only after CUDA work started")
    monkeypatch.setattr(S, "load_ext", no_cuda)
    with pytest.raises(ValueError, match="multiple of 64"):
        S.ShadowEngine(None, 0, 1, code="sign", bucket_size=bucket)
    with pytest.raises(ValueError, match="num_aggregate"):     # the error-feedback rule applies unchanged
        S.ShadowEngine(None, 0, 4, code="sign", error_feedback=True, num_aggregate=2)


# ---------------------------------------------------------------------------------------------------- CPU: launcher
def _args(tmp_path, *extra):
    return add_fit_args(argparse.ArgumentParser(), [
        "--network", "LeNet", "--dataset", "MNIST", "--synthetic", "1", "--train-len", "512", "--test-len", "128",
        "--batch-size", "32", "--test-batch-size", "64", "--lr", "0.05", "--log-interval", "1", "--eval-freq", "100",
        "--train-dir", str(tmp_path) + "/", *extra])


def test_launcher_routes_sign(tmp_path, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    seen = []

    class Fake:
        def __init__(self, model, rank, world, **kw):
            seen.append(kw)
    monkeypatch.setattr(S, "ShadowEngine", Fake)
    model = torch.nn.Linear(4, 4)
    for engine in ("auto", "shadow"):
        _, kind = L._build_engine(_args(tmp_path, "--code", "sign", "--dtype", "bf16", "--engine", engine,
                                        "--bucket-size", "256", "--error-feedback", "1", "--code-stats", "1"),
                                  model, 0, 1)
        assert kind == "shadow" and seen[-1]["code"] == "sign" and seen[-1]["bucket_size"] == 256
        assert seen[-1]["error_feedback"] is True and seen[-1]["code_stats"] is True
    n = len(seen)
    for extra in (("--dtype", "fp32"), ("--dtype", "bf16", "--engine", "fused")):
        with pytest.raises(SystemExit, match="sign"):
            L._build_engine(_args(tmp_path, "--code", "sign", *extra), model, 0, 1)
    assert len(seen) == n


def test_role_paths_refuse_sign(monkeypatch, tmp_path):
    from atomo_b200 import distributed_nn
    from atomo_b200.runtime.master import build_coder
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    with pytest.raises(SystemExit, match="p2p bf16 engine"):
        distributed_nn.run_rank(_args(tmp_path, "--code", "sign", "--backend", "gloo"))
    with pytest.raises(ValueError, match="p2p bf16 engine"):
        build_coder({"code": "sign", "bucket_size": 512}, worker_side=True)


# ---------------------------------------------------------------------------------------------------- GPU harness
def _ext():
    from atomo_b200.ops._ext import load
    return load()


class HS:
    """Loopback harness (the QSGD tests' style): one rank that is worker 0..W-1 (virtual) and the only owner."""

    def __init__(self, shapes, bucket=512, W=1, lr=0.1, momentum=0.0, wd=0.0, nesterov=False, opt=0, seed=7,
                 num_aggregate=0):
        self.C = _ext()
        dev = self.dev = torch.device("cuda", 0)
        self.W, self.bucket = W, bucket
        self.plan = pl = P.build_plan2(shapes, "sign", n_owners=1, n_groups=1, bucket_size=bucket)
        u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)
        self.t_units = u8(pl.units_bytes())
        self.t_enc = u8(P.Plan2.tiles_bytes(pl.enc_tiles))
        self.t_ps = u8(P.Plan2.tiles_bytes(pl.ps_tiles))
        nc = self.nc = max(pl.n_coded, 1)
        z = lambda n, dt=torch.float32: torch.zeros(n, dtype=dt, device=dev)
        self.counters = z(nc + 32, torch.int32)
        self.spart = z(5 * max(len(pl.enc_tiles), 1), torch.float64)
        self.acc = z(7 * nc, torch.float64)
        self.arena = z(pl.arena_floats * W)
        self.signals = z(1024, torch.int32)
        self.signals[256] = 1
        self.ctrl = u8(P.pack_ctrl2(step=1, lr=lr, momentum=momentum, weight_decay=wd, nesterov=nesterov, seed=seed,
                                    opt=opt, num_aggregate=num_aggregate))
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.master = torch.randn(pl.w_total, device=dev, generator=g)
        self.wshadow = self.master.to(torch.bfloat16)
        self.vparams = torch.randn(pl.v_total, device=dev, generator=g)
        self.mom, self.vmom = z(pl.w_total), z(pl.v_total)
        self.sq, self.vsq, self.sqmax, self.vsqmax = z(pl.w_total), z(pl.v_total), z(pl.w_total), z(pl.v_total)
        self.vgrads = [z(pl.v_total) for _ in range(W)]
        self.wgrads = [None] * W
        i64 = lambda xs: torch.tensor(list(xs), dtype=torch.int64, device=dev)
        self.t_arena_peer = i64([self.arena.data_ptr()])
        self.t_sig_peer = i64([self.signals.data_ptr()])
        self.t_wshadow_peer = i64([self.wshadow.data_ptr()])
        self.t_vparams_peer = i64([self.vparams.data_ptr()])
        self.t_vgrads_peer = i64([t.data_ptr() for t in self.vgrads])
        self.tstats = z(32, torch.int64)

    def set_step(self, step):
        self.ctrl.view(torch.int32)[0] = step

    def fill(self, w, seed, special=False):
        """Random bf16 gradients of virtual worker w ({param index: fp32 physical-order flat tensor}); with
        ``special`` the ZERO / SIGNED_ZERO / INF tensors of ORACLE_SHAPES get their content."""
        pl, dev = self.plan, self.dev
        g = torch.Generator(device="cuda").manual_seed(seed)
        grads, phys = [], {}
        for q in pl.params:
            if q.is_w:
                x = torch.randn(q.shape, device=dev, generator=g)
                if special and q.index == ZERO:
                    x.zero_()
                elif special and q.index == SIGNED_ZERO:
                    r = torch.rand(q.shape, device=dev, generator=g)
                    x = torch.where(r < 0.3, torch.zeros_like(x), torch.where(r < 0.6, -torch.zeros_like(x), x))
                x = x.to(torch.bfloat16)
                t = x.contiguous(memory_format=torch.channels_last) if x.dim() == 4 else x.contiguous()
                if special and q.index == INF:
                    (t.permute(0, 2, 3, 1) if t.dim() == 4 else t).view(-1)[1234] = float("inf")
                grads.append(t)
                phys[q.index] = (t.permute(0, 2, 3, 1) if t.dim() == 4 else t).reshape(-1).float()
            else:
                v = torch.randn(q.numel, device=dev, generator=g)
                self.vgrads[w][q.off:q.off + q.numel] = v
                phys[q.index] = v
        self.wgrads[w] = grads
        return phys

    def encode(self, w, residual=0, stats=False):
        C, pl = self.C, self.plan
        gptr = torch.tensor([t.data_ptr() for t in self.wgrads[w]], dtype=torch.int64, device=self.dev)
        self._gptr = gptr
        t0, nt = pl.enc_range[0]
        C.v2_sign_encode(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr.data_ptr(),
                         self.t_arena_peer.data_ptr(), self.t_sig_peer.data_ptr(), 1, pl.arena_floats, w, 0,
                         self.ctrl.data_ptr(), self.counters.data_ptr() + 4 * (self.nc + 8), 0, False, residual)
        if stats:
            C.v2_sign_code_stats(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr.data_ptr(),
                                 self.t_arena_peer.data_ptr(), 1, pl.arena_floats, w, self.spart.data_ptr(),
                                 self.counters.data_ptr(), self.acc.data_ptr())
        torch.cuda.synchronize()

    def ps(self, grid=64):
        C, pl = self.C, self.plan
        t0, nt = pl.ps_range[0][0]
        C.v2_ps_sign(self.t_units.data_ptr(), self.t_ps.data_ptr(), t0, nt, self.W, 1, 0, True, 0,
                     self.master.data_ptr(), self.mom.data_ptr(), self.sq.data_ptr(), self.sqmax.data_ptr(),
                     self.vmom.data_ptr(), self.vsq.data_ptr(), self.vsqmax.data_ptr(), 0,
                     self.t_wshadow_peer.data_ptr(), self.vparams.data_ptr(), 0, self.t_vparams_peer.data_ptr(), 0,
                     self.t_vgrads_peer.data_ptr(), self.arena.data_ptr(), pl.arena_floats, self.signals.data_ptr(),
                     self.t_sig_peer.data_ptr(), self.ctrl.data_ptr(), self.counters.data_ptr() + 4 * (self.nc + 16),
                     int(5e9), self.tstats.data_ptr(), 1.0 / self.W, grid)
        torch.cuda.synchronize()

    def slot(self, u, w):
        """(stamps, scales, words [buckets, L] int64) of unit u in worker w's slot."""
        base = self.arena[w * self.plan.arena_floats + u.slot_off:]
        stamps = base[:u.n_ps].view(torch.int32).clone()
        so, wo = P.qsgd_norms_off(u.n_ps), P.qsgd_words_off(u.n_ps, u.rows)
        scales = base[so:so + u.rows].clone()
        words = base[wo:wo + 2 * u.rows * u.cols].view(torch.int64).view(u.rows, u.cols).clone()
        return stamps, scales, words

    def used(self):
        mw = torch.zeros(self.plan.w_total, dtype=torch.bool, device=self.dev)
        mv = torch.zeros(self.plan.v_total, dtype=torch.bool, device=self.dev)
        for q in self.plan.params:
            (mw if q.is_w else mv)[q.off:q.off + q.numel] = True
        return mw, mv


def _decoded_sum(h, phys_by_worker):
    """sum over workers (in worker order, fp32, CPU) of the oracle's decodes, physical order, times fp32(1 / W)."""
    est = torch.zeros(h.plan.w_total)
    for phys in phys_by_worker:
        for u in h.plan.units:
            if u.kind == P.KIND_SIGN:
                c = _coder(h.bucket)
                est[u.w_off:u.w_off + u.numel] += c.decode(c.encode(phys[u.param].cpu())).reshape(-1)
    return est


# ---------------------------------------------------------------------------------------------------- GPU: encode
@pytest.mark.gpu
@pytest.mark.parametrize("bucket", BUCKETS)
def test_v2_sign_encode_matches_oracle_bitwise(bucket):
    h = HS(ORACLE_SHAPES, bucket)
    h.set_step(3)
    phys = h.fill(0, 11, special=True)
    h.encode(0)
    first = h.arena.clone()
    for u in h.plan.units:
        if u.kind != P.KIND_SIGN:
            continue
        ref = _coder(bucket).encode(phys[u.param].cpu())
        stamps, scales, words = h.slot(u, 0)
        assert bool((stamps == 3).all()), u.param
        assert torch.equal(scales.cpu().view(torch.int32), ref["scales"].view(torch.int32)), u.param
        assert torch.equal(words.cpu(), ref["words"]), u.param
        if u.param == ZERO:
            assert bool((scales == 0).all()) and bool((words == 0).all())
        if u.param == INF:          # only the bucket holding the Inf is non-finite
            bad = (~torch.isfinite(scales)).nonzero().flatten().tolist()
            assert bad == [1234 // u.K]
    assert int(h.signals[0]) == 3
    h.arena.zero_()                  # a second encode of the same gradient: the same bits
    h.encode(0)
    assert torch.equal(h.arena.view(torch.int32), first.view(torch.int32))


# ---------------------------------------------------------------------------------------------------- GPU: PS
@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 2])
@pytest.mark.parametrize("bucket", [64, 512])
def test_v2_ps_sign_decoded_mean_is_bitwise_the_oracles(W, bucket):
    """lr = 1, no momentum, a zero master: the PS writes -(oracle decodes summed in worker order) * fp32(1 / W)."""
    h = HS(NET_SHAPES, bucket, W=W, lr=1.0)
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
def test_v2_ps_sign_matches_reference(momentum, nesterov, wd, opt):
    from test_gpu_shadow_qsgd import _opt_ref
    W, lr = 3, 0.05
    h = HS(NET_SHAPES, 512, W=W, lr=lr, momentum=momentum, wd=wd, nesterov=nesterov, opt=opt)
    used, vused = h.used()
    for step in (1, 2):
        h.set_step(step)
        phys = []
        for w in range(W):
            phys.append(h.fill(w, 10 * step + w))
            h.encode(w)
        gw = _decoded_sum(h, phys).to(h.dev) / W
        gv = sum(h.vgrads) / W
        rp, _ = _opt_ref(h.master.clone(), gw, h.mom.clone(), h.sq.clone(), h.sqmax.clone(), step, lr, momentum,
                         nesterov, wd, opt)
        rv, _ = _opt_ref(h.vparams.clone(), gv, h.vmom.clone(), h.vsq.clone(), h.vsqmax.clone(), step, lr, momentum,
                         nesterov, wd, opt)
        h.ps()
        assert int(h.ctrl.view(torch.int32)[1]) == 0
        assert int(h.signals[256]) == step + 1
        tol = dict(rtol=3e-4, atol=3e-5) if opt == 0 else dict(rtol=2e-3, atol=2e-4)
        assert torch.allclose(h.master[used], rp[used], **tol), float((h.master - rp)[used].abs().max())
        assert torch.allclose(h.vparams[vused], rv[vused], **tol)
        assert torch.equal(h.wshadow[used], h.master.to(torch.bfloat16)[used])


@pytest.mark.gpu
def test_v2_ps_sign_num_aggregate_and_stale_slots():
    """num_aggregate = 2 of 3 workers, worker 1 never pushes: only {0, 2} are averaged.  Then a slot whose stamp is of
    another step is skipped and flagged with ERR2_SLOT_STEP."""
    lr = 0.1
    h = HS(NET_SHAPES, 512, W=3, lr=lr, num_aggregate=2)
    phys = []
    for w in (0, 2):
        phys.append(h.fill(w, 40 + w))
        h.encode(w)
    h.vgrads[1].fill_(1e6)                         # garbage a skipped worker may hold
    assert int(h.signals[0]) == 1 and int(h.signals[1]) == 0 and int(h.signals[2]) == 1
    est = _decoded_sum(h, phys).to(h.dev)
    p0, v0 = h.master.clone(), h.vparams.clone()
    h.ps()
    assert int(h.ctrl.view(torch.int32)[1]) == 0 and int(h.signals[256]) == 2
    assert int(h.signals[320]) == 0b101 and int(h.signals[321]) == 1
    used, vused = h.used()
    assert torch.allclose(h.master[used], (p0 - lr * est / 2)[used], rtol=3e-4, atol=3e-5)
    assert torch.allclose(h.vparams[vused], (v0 - lr * (h.vgrads[0] + h.vgrads[2]) / 2)[vused], rtol=3e-4, atol=3e-5)

    hs = HS(NET_SHAPES, 512, W=2, lr=lr)            # worker 1's slot holds step 0 while its flag claims step 1
    hs.fill(0, 1)
    hs.encode(0)
    hs.signals[1] = 1
    hs.ps()
    assert int(hs.ctrl.view(torch.int32)[1]) & 4          # ERR2_SLOT_STEP


# ---------------------------------------------------------------------------------------------------- GPU: stats
@pytest.mark.gpu
@pytest.mark.parametrize("bucket", BUCKETS)
def test_v2_sign_code_stats_match_fp64(bucket):
    h = HS(ORACLE_SHAPES, bucket)
    h.set_step(2)
    phys = h.fill(0, 21, special=True)
    h.encode(0, stats=True)
    acc = h.acc.view(-1, 7).tolist()
    from atomo_b200.codings.sign import bf16_flushed
    for u in h.plan.units:
        if u.kind != P.KIND_SIGN or u.param == INF:
            continue
        gsq, mse, ex, bias, real, real4, n = acc[u.ts_index]
        x = torch.from_numpy(bf16_flushed(phys[u.param].cpu())).double()
        assert n == 1 and bias == 0 and ex == real == real4 == u.numel
        assert gsq == pytest.approx(float(x.square().sum()), rel=1e-12, abs=0)
        assert mse == pytest.approx(_coder(bucket).error_sq(phys[u.param].cpu()), rel=1e-12, abs=1e-300)
        if u.param != ZERO:
            assert mse < gsq


# ---------------------------------------------------------------------------------------------------- GPU: feedback
def _grads(seed=0):
    from test_gpu_error_feedback import SHAPES
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(s, generator=g) * (0.01 * (1 + i))).bfloat16().float().cuda() for i, s in enumerate(SHAPES)]


@pytest.mark.gpu
@pytest.mark.parametrize("bucket", BUCKETS)
def test_error_feedback_identity_and_contraction(bucket):
    from test_gpu_error_feedback import Loopback
    h = Loopback("sign", _grads(1), bucket_size=bucket)
    try:
        g, e_old = h.g, h.residual()
        for _ in range(4):
            A = g + e_old
            ghat, e_new = h.step()
            scale = g.abs() + e_old.abs() + ghat.abs() + e_new.abs()
            assert bool(((A - (ghat + e_new)).abs() <= 1e-6 * scale + 1e-7 * float(scale.max())).all())
            for q in h.w:
                sl = slice(q.off, q.off + q.numel)
                assert float(e_new[sl].norm()) <= float(A[sl].norm())
            assert float(e_new.norm()) > 0
            e_old = e_new
    finally:
        h.close()


@pytest.mark.gpu
def test_error_feedback_residual_stays_bounded():
    """A fixed gradient for 200 steps: every step contracts (||e_{t+1}|| <= rho ||g + e_t||, rho < 1), so ||e|| stays
    below rho / (1 - rho) ||g||; the pushed sum misses 200 g by exactly the final residual."""
    from test_gpu_error_feedback import Loopback
    h = Loopback("sign", _grads(2), bucket_size=512)
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
        assert rho < 1
        assert max(norms) <= rho / (1 - rho) * float(h.g.norm()) * (1 + 1e-4)
        assert torch.allclose(s - 200 * h.g, -e, rtol=0, atol=200 * 1e-6 * (float(h.g.abs().max()) + float(e.abs().max())))
    finally:
        h.close()


@pytest.mark.gpu
def test_code_stats_bytes_follow_the_plan():
    from test_gpu_error_feedback import Loopback
    h = Loopback("sign", _grads(4), bucket_size=256, code_stats=True)
    try:
        h.step()
        st = h.eng.code_stats()
        pl = h.eng.plan
        assert st["code"] == "sign" and st["steps"] == 1
        names = {id(p): n for n, p in h.eng.model.named_parameters()}
        for u in pl.units:
            t = st["tensors"][names[id(h.eng.params[u.param])]]
            if u.kind == P.KIND_SIGN:
                assert t["bytes"] == 8 * u.rows * u.cols + 4 * u.rows
                assert t["atoms"] == t["exp_atoms"] == u.numel and 0 < t["rel_var"] < 1
        assert st["model"]["bytes"] == pl.qsgd_bytes() + pl.dense_bytes()
    finally:
        h.close()


# ---------------------------------------------------------------------------------------------------- GPU: engine
def _train(net, graph, ef, steps=6, bucket=512, lr=0.05, seed=3):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model, input_shape
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    x, y = SyntheticImageDataset(input_shape(net), 10, 4096, seed=0).materialize(32)
    eng = ShadowEngine(build_model(net, 10), 0, 1, code="sign", bucket_size=bucket, lr=lr, momentum=0.9,
                       use_graph=graph, overlap=graph, seed=seed, error_feedback=ef)
    eng.prepare(x.pin_memory(), y.pin_memory(), warmup=2)
    losses, norms = [], []
    for _ in range(steps):
        losses.append(float(eng.train_step(x, y)[0]))
        if ef:
            norms.append(eng.error_feedback_norm()["model"])
    torch.cuda.synchronize()
    assert eng.error_code() == 0
    m = eng.gather_fp32("master").clone()
    eng.close()
    return m, losses, norms


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
def test_error_feedback_training_stays_finite(net):
    """lr 0.05 / momentum 0.9: the setting where the unbiased codes with error feedback diverge."""
    _, losses, norms = _train(net, True, True, steps=30)
    assert all(math.isfinite(v) for v in losses + norms)
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
        return ShadowEngine(build_model("VGG11", 10), 0, 1, code="sign", bucket_size=256, lr=0.05, momentum=0.9,
                            use_graph=False)
    a = mk()
    a.prepare(x.pin_memory(), y.pin_memory(), warmup=0)
    for _ in range(3):
        a.train_step(x, y)
    path = a.save_checkpoint(str(tmp_path) + "/")
    side = torch.load(path + "_optim", weights_only=False)
    assert side["code"] == "sign" and side["bucket_size"] == 256
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
def test_launcher_sign_writes_ef_norm_and_code_stats(tmp_path, monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    args = add_fit_args(argparse.ArgumentParser(), [
        "--network", "ResNet18", "--dataset", "Cifar10", "--synthetic", "1", "--train-len", "512", "--test-len", "64",
        "--batch-size", "32", "--test-batch-size", "64", "--backend", "p2p", "--dtype", "bf16", "--max-steps", "6",
        "--log-interval", "2", "--eval-freq", "100", "--train-dir", str(tmp_path) + "/",
        "--metrics-file", str(tmp_path / "m"), "--code", "sign", "--bucket-size", "512", "--error-feedback", "1",
        "--code-stats", "1"])
    L.run_p2p_training(args)
    recs = [json.loads(l) for l in open(str(tmp_path / "m") + ".rank0.jsonl")]
    assert recs and all(r["ef_norm"] > 0 and math.isfinite(r["ef_norm"]) for r in recs)
    m = recs[-1]["code_stats"]["model"]
    assert m["atoms"] > 0 and 0 < m["rel_var"] < 1


@pytest.mark.gpu
@pytest.mark.multigpu
def test_shadow_engine_sign_multi_gpu_replicas_identical():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    from test_gpu_v2 import _run_mp
    world = 2 if n < 8 else (8 if os.environ.get("ATOMO_TEST_WORLD8") else 2)
    res = _run_mp(world, {"code": "sign", "ps_mode": "sharded", "net": "VGG11"}, 29810)
    for rank, err, same, l0, l1, mode, mc, _ in res:
        assert err == 0 and same, res

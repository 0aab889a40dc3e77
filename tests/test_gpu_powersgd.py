"""PowerSGD on the bf16 engine (``code="powersgd"``, csrc/v2_powersgd.cu): the ``codings.powersgd`` oracle, the planner,
the refusals and the launcher routing (CPU); the encode, the warm state and the PS against the oracle, error feedback
and ``--code-stats`` (GPU loopback harness); and the engine end to end (GPU).

The kernels sum in fp32 in a fixed order that differs from the oracle's fp64 products, so factors are compared within
``TOL`` of the largest magnitude of the compared array; repeated encodes are compared bit for bit."""
import argparse
import functools
import hashlib
import json
import math
import os

import numpy as np
import pytest
import torch

from atomo_b200.codings import powersgd as PS
from atomo_b200.ops import plan2 as P
from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils.flags import add_fit_args

from shadow_harness import (LoopbackPS, Loopback, ef_grads, fit_args, flat, forbid_cuda, opt_ref, physical, run_mp,
                            train)

TOL = 2e-4
NET_SHAPES = [(64, 3, 3, 3), (64,), (64,), (128, 64, 3, 3), (128,), (256, 128, 3, 3), (512, 256, 1, 1), (300, 200),
              (10, 512), (7, 20), (5, 3), (10,)]
# the 27-column stem, 3x3 convs, an fc layer, odd sizes, a vector, an all-zero tensor (ZERO), an exactly rank-1 tensor
# (RANK1), one with an Inf (INF), the largest ResNet-18 layer shape
ORACLE_SHAPES = [(64, 3, 3, 3), (64, 32, 3, 3), (128, 64, 3, 3), (10, 512), (300, 200), (7, 20), (33, 17, 3, 3), (64,),
                 (32, 16, 3, 3), (40, 30), (48, 16, 3, 3), (512, 512, 3, 3)]
ZERO, RANK1, INF = 8, 9, 10


# ---------------------------------------------------------------------------------------------------- CPU: oracle
def _lowrank(o, c, k, seed):
    g = np.random.default_rng(seed)
    return (g.standard_normal((o, k)) @ g.standard_normal((k, c))).astype(np.float32)


@pytest.mark.parametrize("r", [1, 2, 4])
def test_oracle_orthonormal_factors_and_error_identity(r):
    M = np.random.default_rng(r).standard_normal((96, 150)).astype(np.float32)
    st = PS.power_step(M, PS.normals(1, 3, 150, r, 0))
    assert st["mask"] == (1 << r) - 1 and not st["nonfinite"]
    ph = st["phat"].astype(np.float64)
    assert np.allclose(ph.T @ ph, np.eye(r), atol=1e-5)
    c = PS.PowerSGD(r)
    grad = torch.from_numpy(M)
    bound, exact = c.error_sq(grad)
    assert bound == pytest.approx(exact, rel=1e-4)
    assert 0 < exact < float((M.astype(np.float64) ** 2).sum())


@pytest.mark.parametrize("r,k", [(1, 1), (2, 2), (4, 2), (4, 4)])
def test_oracle_exact_when_rank_at_most_r(r, k):
    M = _lowrank(40, 70, k, 7 + r)
    st = PS.power_step(M, PS.normals(5, 0, 70, r, 0))
    assert bin(st["mask"]).count("1") == k                 # the surplus columns are degenerate (zero)
    ghat = st["phat"].astype(np.float64) @ st["qnew"].astype(np.float64).T
    assert np.abs(ghat - M).max() <= 1e-5 * np.abs(M).max()


def test_oracle_degenerate_cases():
    qw = PS.normals(1, 2, 30, 4, 0)
    z = PS.power_step(np.zeros((20, 30), np.float32), qw)          # zero tensor: nothing pushed, every column re-drawn
    assert z["mask"] == 0 and not z["nonfinite"] and not z["phat"].any() and not z["qnew"].any()
    q1, d1 = PS.next_warm_state(z, qw, 1, 2, 0)
    assert d1 == 1 and np.array_equal(q1, PS.normals(1, 2, 30, 4, 1))
    u = np.array([1.0, -2.0, 0.5, 4.0] * 5, np.float32)[:, None]
    v = np.random.default_rng(0).standard_normal((1, 30)).astype(np.float32)
    one = PS.power_step(u @ v, qw)                                  # rank 1 at r = 4: one column, three re-drawn
    assert one["mask"] == 1
    q2, d2 = PS.next_warm_state(one, qw, 1, 2, 0)
    assert d2 == 1 and np.array_equal(q2[:, 0], one["qnew"][:, 0])
    assert np.array_equal(q2[:, 1:], PS.normals(1, 2, 30, 4, 1)[:, 1:])
    M = np.ones((20, 30), np.float32)
    M[3, 4] = np.inf
    bad = PS.power_step(M, qw)                                      # an Inf: zeros pushed, warm state kept
    assert bad["nonfinite"] and bad["mask"] == 0 and not bad["phat"].any() and not bad["qnew"].any()
    q3, d3 = PS.next_warm_state(bad, qw, 1, 2, 0)
    assert d3 == 0 and np.array_equal(q3, qw)


def test_oracle_warm_start_converges_to_svd_tail():
    g = np.random.default_rng(3)
    U, _ = np.linalg.qr(g.standard_normal((64, 64)))
    V, _ = np.linalg.qr(g.standard_normal((90, 64)))
    s = 0.7 ** np.arange(64)
    M = ((U * s) @ V.T).astype(np.float32)
    sv = torch.linalg.svdvals(torch.from_numpy(M).double()).numpy()
    for r in (1, 2, 4):
        tail = float((sv[r:] ** 2).sum())
        c = PS.PowerSGD(r, seed=9)
        errs = []
        for _ in range(40):
            errs.append(c.error_sq(torch.from_numpy(M))[1])
            c.encode(torch.from_numpy(M))
        assert errs[-1] == pytest.approx(tail, rel=1e-3)
        assert errs[0] > errs[-1]


def test_oracle_normals_and_refusals():
    z = PS.normals(1, 0, 20000, 4, 0)
    assert abs(float(z.mean())) < 0.02 and abs(float(z.std()) - 1) < 0.02
    assert not np.array_equal(PS.normals(1, 0, 8, 1, 0), PS.normals(1, 1, 8, 1, 0))
    assert not np.array_equal(PS.normals(1, 0, 8, 1, 0), PS.normals(1, 0, 8, 1, 1))
    for r in (0, 5, -1):
        with pytest.raises(ValueError, match="svd_rank"):
            PS.PowerSGD(r)


def test_oracle_philox_matches_the_reference_vector():
    # Philox4x32-10 known-answer test (Salmon et al. 2011, counter 0, key 0)
    w = PS.philox(0, 0, 0, 0, 0)
    assert [int(x) for x in w] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]


# ---------------------------------------------------------------------------------------------------- CPU: planner
@pytest.mark.parametrize("r,owners", [(1, 1), (2, 3), (4, 2), (3, 4)])
def test_plan2_powersgd_units_tiles_and_slots(r, owners):
    pl = P.build_plan2(NET_SHAPES, "powersgd", r, n_owners=owners, n_groups=3)
    want_bytes = 0
    for p in pl.params:
        units = [u for u in pl.units if u.param == p.index]
        assert len(units) == 1
        u = units[0]
        if not p.is_w:
            assert u.kind == P.KIND_VEC
            continue
        o, c = p.shape[0], p.numel // p.shape[0]
        if not PS.coded(p.shape, r):
            assert u.kind == P.KIND_DENSE16
            continue
        assert u.kind == P.KIND_POWER and (u.rows, u.cols, u.rcap, u.w_off, u.numel) == (o, c, r, p.off, p.numel)
        enc = [(a, n, j) for (ui, a, n, j) in pl.enc_tiles if ui == u.index]
        assert enc == [(a, min(P.PW_ENC_ROWS, o - a), j) for j, a in enumerate(range(0, o, P.PW_ENC_ROWS))]
        assert u.n_enc == len(enc)
        pw = [(a, n, j) for (ui, a, n, j) in pl.pw_tiles if ui == u.index]
        assert pw == [(a, min(P.PW_COL_BLOCK, c - a), j) for j, a in enumerate(range(0, c, P.PW_COL_BLOCK))]
        assert u.K == len(pw)
        ps = sorted((a, n, ow) for (ui, a, n, ow) in pl.ps_tiles if ui == u.index)
        assert [a for a, _, _ in ps] == list(range(0, o, P.PW_PS_ROWS)) and len(ps) == u.n_ps
        assert [ow for _, _, ow in ps] == [u.own0] * u.n_ps and 0 <= u.own0 < owners   # one owner: Q' sent once
        want_bytes += 4 * r * (o + c)
    spans = sorted((u.slot_off, u.slot_off + P.pw_slot_floats(u.n_ps, u.rows, u.cols, u.rcap))
                   for u in pl.units if u.kind == P.KIND_POWER)
    assert all(a1 >= b0 for (a0, b0), (a1, b1) in zip(spans, spans[1:])) and spans[-1][1] <= pl.arena_floats
    scr = sorted((u.gpart_off, u.gpart_off + P.pw_scratch_floats(u.rows, u.cols, u.rcap))
                 for u in pl.units if u.kind == P.KIND_POWER)
    assert all(a1 >= b0 for (a0, b0), (a1, b1) in zip(scr, scr[1:])) and scr[-1][1] <= pl.gpart_floats
    assert pl.powersgd_bytes() == want_bytes
    assert [n for _, n in pl.pw_range] and sum(n for _, n in pl.pw_range) == len(pl.pw_tiles)
    for g in range(pl.n_groups):        # a group's units go to the owner with the fewest PowerSGD elements so far
        load = [0] * owners
        for ui in pl.group_units[g]:
            u = pl.units[ui]
            if u.kind == P.KIND_POWER:
                assert u.own0 == min(range(owners), key=lambda k: (load[k], k))
                load[u.own0] += u.numel


def test_plan2_powersgd_bytes_and_bounded_scratch():
    # the issue's shape-derived figures: ResNet-18 / VGG-11 push 4 r (O + C) bytes per coded tensor on one owner
    from atomo_b200.models import build_model
    for net, want in (("ResNet18", (0.1453, 0.2906, 0.5812)), ("VGG11", (0.1020, 0.2041, 0.4081))):
        shapes = [tuple(p.shape) for p in build_model(net, 10).parameters()]
        for r, mb in zip((1, 2, 4), want):
            for owners in (1, 2, 8):            # Q' travels once whatever the owner count
                pl = P.build_plan2(shapes, "powersgd", r, n_owners=owners)
                assert pl.powersgd_bytes() / 1e6 == pytest.approx(mb, abs=1e-4)
            # worker-local factors + warm state: 2 x the pushed floats; Gram partials: 16 doubles per 8-row tile
            assert 4 * pl.gpart_floats <= 2.2 * pl.powersgd_bytes()
            assert 8 * P.PW_GRAM * len(pl.enc_tiles) < 0.2e6
    big = P.build_plan2([(512, 512, 3, 3)], "powersgd", 4)          # no per-tile Q' partials exist
    assert 4 * big.gpart_floats == 4 * 2 * 4 * (512 + 4608)


def test_plan2_powersgd_refuses_ranks():
    for r in (0, 5, -2):
        with pytest.raises(ValueError, match="svd_rank"):
            P.build_plan2(NET_SHAPES, "powersgd", r)


def test_plan2_other_codes_unchanged_by_the_new_code():
    """Digests of the plans of the existing codes, taken from the planner before PowerSGD was added."""
    want = {"svd": "917543867e0167683f770150a43eaf4c129e4d461aa989111b2a491e5eeca388",
            "qsvd": "6ea73c4cd4a95d51288ea6c2a2053f66ff7800fc277120bdccfda766e92e3cf9",
            "sgd": "6d3fd294b9211300d2945b4d3f20d6bf9615e56c5dfa3bab6b294fa9370a37d8",
            "qsgd": "1f34b0853ed1349c3ede1baad5eecd6d7a8e9d4bd571740ec8e531cedbfe275c",
            "terngrad": "5ab388e54d2c51d29226927eaa996c37b3173a968114dce188b5cb8121895e57",
            "entrywise": "5ec97d1b33d12cee3ed4b7b6466f49526420e0442c54d8d8aa9634e1cfe73dcf",
            "topk": "0fed82b9ada85f2510d5f1e0b047978d4124c2a1bd1557bba9353e0d7fae72f0",
            "sign": "81b324f24294287fe7a390c33fc80496d4e05e4f6e2236d722a14a87cc73cb97"}
    shapes = NET_SHAPES[:10] + NET_SHAPES[11:]
    for code, digest in want.items():
        pl = P.build_plan2(shapes, code, 3, n_owners=2, n_groups=3, entry_budget=0.05)
        b = pl.units_bytes() + P.Plan2.tiles_bytes(pl.enc_tiles) + P.Plan2.tiles_bytes(pl.ps_tiles) + \
            repr((pl.enc_range, pl.ps_range, pl.arena_floats, pl.n_coded)).encode()
        assert hashlib.sha256(b).hexdigest() == digest, code
        assert pl.pw_tiles == [] and pl.powersgd_bytes() == 0


@pytest.mark.parametrize("r", [0, 5])
def test_shadow_engine_powersgd_refuses_before_cuda(r, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    forbid_cuda(monkeypatch)
    with pytest.raises(ValueError, match="svd_rank"):
        S.ShadowEngine(None, 0, 1, code="powersgd", svd_rank=r)
    with pytest.raises(ValueError, match="num_aggregate"):     # the error-feedback rule applies unchanged
        S.ShadowEngine(None, 0, 4, code="powersgd", svd_rank=2, error_feedback=True, num_aggregate=2)


# ---------------------------------------------------------------------------------------------------- CPU: launcher
def test_launcher_routes_powersgd(tmp_path, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    seen = []

    class Fake:
        def __init__(self, model, rank, world, **kw):
            seen.append(kw)
    monkeypatch.setattr(S, "ShadowEngine", Fake)
    model = torch.nn.Linear(4, 4)
    for engine in ("auto", "shadow"):
        _, kind = L._build_engine(fit_args(tmp_path, "--code", "powersgd", "--dtype", "bf16", "--engine", engine,
                                        "--svd-rank", "2", "--error-feedback", "1", "--code-stats", "1"),
                                  model, 0, 1)
        assert kind == "shadow" and seen[-1]["code"] == "powersgd" and seen[-1]["svd_rank"] == 2
        assert seen[-1]["error_feedback"] is True and seen[-1]["code_stats"] is True
    n = len(seen)
    for extra in (("--dtype", "fp32", "--svd-rank", "2"), ("--dtype", "bf16", "--engine", "fused", "--svd-rank", "2"),
                  ("--dtype", "bf16"), ("--dtype", "bf16", "--svd-rank", "5")):
        with pytest.raises(SystemExit, match="powersgd"):
            L._build_engine(fit_args(tmp_path, "--code", "powersgd", *extra), model, 0, 1)
    assert len(seen) == n


def test_role_paths_refuse_powersgd(monkeypatch, tmp_path):
    from atomo_b200 import distributed_nn
    from atomo_b200.runtime.master import build_coder
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    with pytest.raises(SystemExit, match="p2p bf16 engine"):
        distributed_nn.run_rank(fit_args(tmp_path, "--code", "powersgd", "--svd-rank", "2", "--backend", "gloo"))
    with pytest.raises(ValueError, match="p2p bf16 engine"):
        build_coder({"code": "powersgd", "svd_rank": 2}, worker_side=True)


# ---------------------------------------------------------------------------------------------------- GPU harness
class HP(LoopbackPS):
    """PowerSGD, with per-worker warm state and staging copies; owners are virtual too."""

    PS = "v2_ps_powersgd"

    def __init__(self, shapes, r=2, W=1, lr=0.1, momentum=0.0, wd=0.0, nesterov=False, opt=0, seed=7,
                 num_aggregate=0, n_owners=1):
        super().__init__(shapes, "powersgd", W, lr, momentum, wd, nesterov, opt, seed, num_aggregate,
                         n_owners=n_owners, stage=True, rank=r)
        self.r = r
        pl, z, nc = self.plan, self.zeros, self.nc
        self.t_pw = torch.frombuffer(bytearray(P.Plan2.tiles_bytes(pl.pw_tiles)), dtype=torch.uint8).to(self.dev)
        self.spart = z(5 * max(len(pl.enc_tiles), 1), torch.float64)
        self.acc = z(7 * nc, torch.float64)
        # per virtual worker: warm state + factors, Gram partials, unit state
        self.scratch = [z(pl.gpart_floats) for _ in range(W)]
        self.gram = [z(P.PW_GRAM * max(len(pl.enc_tiles), 1), torch.float64) for _ in range(W)]
        self.state = [z(nc * self.C.v2_powersgd_state_bytes(), torch.uint8) for _ in range(W)]
        for w in range(W):
            self.C.v2_powersgd_init(self.t_units.data_ptr(), len(pl.units), self.scratch[w].data_ptr(),
                                    self.ctrl.data_ptr())
        torch.cuda.synchronize()

    def tensor(self, q, x, g, special=False):
        if special and q.index == ZERO:
            x.zero_()
        elif special and q.index == RANK1:     # powers of two times bf16 values: exactly rank 1 in bf16
            u = 2.0 ** torch.randint(-2, 3, (q.shape[0],), device=self.dev, generator=g).float()
            v = torch.randn(q.numel // q.shape[0], device=self.dev, generator=g).bfloat16().float()
            x = (u[:, None] * v[None, :])
            x = x.view(q.shape[0], q.shape[2], q.shape[3], q.shape[1]).permute(0, 3, 1, 2) \
                if len(q.shape) == 4 else x.view(q.shape)
        elif special and q.index == INF:
            x = physical(x)
            flat(x)[1234] = float("inf")
        return x

    def fill(self, w, seed, special=False):
        """Random bf16 gradients of virtual worker w ({param index: fp32 [O][C] matrix in physical order, or the
        fp32 vector}); with ``special`` the ZERO / RANK1 / INF tensors of ORACLE_SHAPES get their content."""
        phys = super().fill(w, seed, special=special)
        return {i: v.reshape(self.plan.params[i].shape[0], -1) if self.plan.params[i].is_w else v
                for i, v in phys.items()}

    def encode(self, w, residual=0, stats=False):
        C, pl = self.C, self.plan
        gptr = self.gptr(w)
        t0, nt = pl.enc_range[0]
        p0, npw = pl.pw_range[0]
        C.v2_powersgd_encode(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, self.t_pw.data_ptr(), p0, npw,
                             gptr, self.scratch[w].data_ptr(), self.gram[w].data_ptr(),
                             self.state[w].data_ptr(), self.stage[w].data_ptr(), self.t_arena_peer.data_ptr(),
                             self.t_sig_peer.data_ptr(), self.n_owners, pl.arena_floats, w, 0, self.ctrl.data_ptr(),
                             self.counter(), 0, False, residual)
        if stats:
            C.v2_powersgd_code_stats(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr,
                                     self.scratch[w].data_ptr(), self.state[w].data_ptr(), self.spart.data_ptr(),
                                     self.counters.data_ptr(), self.acc.data_ptr())
        torch.cuda.synchronize()

    def slot(self, u, w, owner=None):
        """(stamps, P_hat [O][r], Q' [C][r]) of unit u in worker w's slot in an owner's arena (default: the unit's)."""
        base = self.arenas[u.own0 if owner is None else owner][w * self.plan.arena_floats + u.slot_off:]
        r, op, cp = u.rcap, -(-u.rows // 4) * 4, -(-u.cols // 4) * 4
        stamps = base[:u.n_ps].view(torch.int32).clone()
        ph = base[P.pw_phat_off(u.n_ps):][:r * op].view(r, op)[:, :u.rows].T.cpu()
        q = base[P.pw_q_off(u.n_ps, u.rows, r):][:r * cp].view(r, cp)[:, :u.cols].T.cpu()
        return stamps, ph, q

    def warm(self, u, w):
        """The warm Q_w [C][r] of unit u on worker w."""
        r, op, cp = u.rcap, -(-u.rows // 4) * 4, -(-u.cols // 4) * 4
        base = self.scratch[w][u.gpart_off + 2 * r * op + r * cp:]
        return base[:r * cp].view(r, cp)[:, :u.cols].T.cpu()

    def draw(self, u, w):
        st = self.state[w].view(-1, self.C.v2_powersgd_state_bytes())[u.ts_index]
        return int(st[128:].view(torch.int32)[2])


def _close(a, b, what):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    scale = max(float(b.abs().max()) if b.numel() else 0.0, 1e-30)
    err = float((a - b).abs().max()) if b.numel() else 0.0
    assert err <= TOL * scale, (what, err, scale)


def _oracle_sum(h, phys_by_worker, qw_by_worker):
    """sum over workers (fp64, CPU, physical order) of the oracle's P_hat Q'^T."""
    est = torch.zeros(h.plan.w_total, dtype=torch.float64)
    for phys, qws in zip(phys_by_worker, qw_by_worker):
        for u in h.plan.units:
            if u.kind == P.KIND_POWER:
                st = PS.power_step(phys[u.param].cpu().numpy(), qws[u.index])
                est[u.w_off:u.w_off + u.numel] += torch.from_numpy(
                    st["phat"].astype(np.float64) @ st["qnew"].astype(np.float64).T).reshape(-1)
            elif u.kind == P.KIND_DENSE16:
                est[u.w_off:u.w_off + u.numel] += phys[u.param].cpu().reshape(-1).double()
    return est


# ---------------------------------------------------------------------------------------------------- GPU: encode
@pytest.mark.gpu
@pytest.mark.parametrize("r", [1, 2, 4])
def test_v2_powersgd_encode_matches_oracle(r):
    h = HP(ORACLE_SHAPES, r)
    h.set_step(3)
    phys = h.fill(0, 11, special=True)
    qw0 = {}
    for u in h.plan.units:
        if u.kind == P.KIND_POWER:
            qw0[u.index] = PS.normals(h.seed, u.index, u.cols, r, 0)
            _close(h.warm(u, 0), qw0[u.index], ("init", u.param))
    h.encode(0)
    first = (h.arena.clone(), [s.clone() for s in h.scratch])
    for u in h.plan.units:
        if u.kind != P.KIND_POWER:
            continue
        ref = PS.power_step(phys[u.param].cpu().numpy(), qw0[u.index])
        stamps, ph, q = h.slot(u, 0)
        assert bool((stamps == 3).all()), u.param
        _close(ph, ref["phat"], ("phat", u.param))
        _close(q, ref["qnew"], ("qnew", u.param))
        nq, ndraw = PS.next_warm_state(ref, qw0[u.index], h.seed, u.index, 0)
        assert h.draw(u, 0) == ndraw, u.param
        _close(h.warm(u, 0), nq, ("warm", u.param))
        if u.param == ZERO:
            assert not ph.any() and not q.any() and ndraw == 1
        elif u.param == RANK1:
            assert ref["mask"] == 1 and (ndraw == 1 or r == 1)
        elif u.param == INF:
            assert ref["nonfinite"] and not ph.any() and not q.any() and torch.equal(h.warm(u, 0), torch.from_numpy(qw0[u.index]))
        else:
            assert ref["mask"] == (1 << r) - 1
            phd = ph.double()
            assert torch.allclose(phd.T @ phd, torch.eye(r, dtype=torch.float64), atol=1e-4)
    assert int(h.signals[0]) == 3
    # a second encode of the same gradient from the same warm state: the same bits
    h2 = HP(ORACLE_SHAPES, r)
    h2.set_step(3)
    h2.fill(0, 11, special=True)
    h2.encode(0)
    assert torch.equal(h2.arena.view(torch.int32), first[0].view(torch.int32))
    assert torch.equal(h2.scratch[0].view(torch.int32), first[1][0].view(torch.int32))


@pytest.mark.gpu
def test_v2_powersgd_warm_state_follows_the_oracle_over_steps():
    h = HP(ORACLE_SHAPES[:7], 2)
    c = {u.index: PS.normals(h.seed, u.index, u.cols, 2, 0) for u in h.plan.units if u.kind == P.KIND_POWER}
    phys = h.fill(0, 5)
    for step in range(1, 6):
        h.set_step(step)
        h.encode(0)
        for u in h.plan.units:
            if u.kind == P.KIND_POWER:
                ref = PS.power_step(phys[u.param].cpu().numpy(), c[u.index])
                c[u.index], _ = PS.next_warm_state(ref, c[u.index], h.seed, u.index, 0)
                _close(h.warm(u, 0), c[u.index], ("warm", step, u.param))


# ---------------------------------------------------------------------------------------------------- GPU: PS
@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 2])
@pytest.mark.parametrize("r", [1, 4])
def test_v2_ps_powersgd_mean_matches_the_oracle(W, r):
    """lr = 1, no momentum, a zero master: the PS writes -(sum of the workers' P_hat Q'^T) * fp32(1 / W)."""
    h = HP(NET_SHAPES, r, W=W, lr=1.0)
    phys, qws = [], []
    for w in range(W):
        phys.append(h.fill(w, 70 + w))
        qws.append({u.index: h.warm(u, w).numpy().copy() for u in h.plan.units if u.kind == P.KIND_POWER})
        h.encode(w)
    want = _oracle_sum(h, phys, qws) / W
    h.master.zero_()
    h.ps()
    assert int(h.ctrl.view(torch.int32)[1]) == 0
    used, _ = h.used()
    got = -h.master.cpu()
    for u in h.plan.units:
        if u.kind in (P.KIND_POWER, P.KIND_DENSE16):
            sl = slice(u.w_off, u.w_off + u.numel)
            _close(got[sl], want[sl], ("ps", u.param))


@pytest.mark.gpu
@pytest.mark.parametrize("momentum,nesterov,wd,opt", [(0.0, False, 0.0, 0), (0.9, True, 1e-3, 0), (0.0, False, 0.0, 1),
                                                      (0.0, False, 1e-3, 2)])
def test_v2_ps_powersgd_optimizer_epilogues(momentum, nesterov, wd, opt):
    W, lr = 2, 0.05
    h = HP(NET_SHAPES, 2, W=W, lr=lr, momentum=momentum, wd=wd, nesterov=nesterov, opt=opt)
    used, vused = h.used()
    for step in (1, 2):
        h.set_step(step)
        phys, qws = [], []
        for w in range(W):
            phys.append(h.fill(w, 10 * step + w))
            qws.append({u.index: h.warm(u, w).numpy().copy() for u in h.plan.units if u.kind == P.KIND_POWER})
            h.encode(w)
        gw = (_oracle_sum(h, phys, qws) / W).float().to(h.dev)
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
def test_v2_ps_powersgd_num_aggregate_and_stale_slots():
    """num_aggregate = 2 of 3 workers, worker 1 never pushes: only {0, 2} are averaged.  Then a slot whose stamp is of
    another step is skipped and flagged with ERR2_SLOT_STEP."""
    lr = 0.1
    h = HP(NET_SHAPES, 2, W=3, lr=lr, num_aggregate=2)
    phys, qws = [], []
    for w in (0, 2):
        phys.append(h.fill(w, 40 + w))
        qws.append({u.index: h.warm(u, w).numpy().copy() for u in h.plan.units if u.kind == P.KIND_POWER})
        h.encode(w)
    h.vgrads[1].fill_(1e6)
    assert int(h.signals[0]) == 1 and int(h.signals[1]) == 0 and int(h.signals[2]) == 1
    est = _oracle_sum(h, phys, qws).float().to(h.dev)
    p0, v0 = h.master.clone(), h.vparams.clone()
    h.ps()
    assert int(h.ctrl.view(torch.int32)[1]) == 0 and int(h.signals[256]) == 2
    assert int(h.signals[320]) == 0b101 and int(h.signals[321]) == 1
    used, vused = h.used()
    assert torch.allclose(h.master[used], (p0 - lr * est / 2)[used], rtol=3e-4, atol=3e-5)
    assert torch.allclose(h.vparams[vused], (v0 - lr * (h.vgrads[0] + h.vgrads[2]) / 2)[vused], rtol=3e-4, atol=3e-5)

    hs = HP(NET_SHAPES, 2, W=2, lr=lr)            # worker 1's slot holds step 0 while its flag claims step 1
    hs.fill(0, 1)
    hs.encode(0)
    hs.signals[1] = 1
    hs.ps()
    assert int(hs.ctrl.view(torch.int32)[1]) & 4          # ERR2_SLOT_STEP


@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 2])
def test_v2_powersgd_two_owners_route_and_reconstruct(W):
    """Two (virtual) owners: each unit's stamps, P_hat and Q' land in its owner's arena only, and the two owners' PS
    launches together reconstruct the oracle mean on every weight."""
    h = HP(NET_SHAPES, 2, W=W, lr=1.0, n_owners=2)
    assert {u.own0 for u in h.plan.units if u.kind == P.KIND_POWER} == {0, 1}
    h.set_step(2)
    phys, qws = [], []
    for w in range(W):
        phys.append(h.fill(w, 90 + w))
        qws.append({u.index: h.warm(u, w).numpy().copy() for u in h.plan.units if u.kind == P.KIND_POWER})
        h.encode(w)
    for o in range(2):
        assert [int(h.sigs[o][w]) for w in range(W)] == [2] * W        # the push flag reaches both owners
    for w in range(W):
        for u in h.plan.units:
            if u.kind != P.KIND_POWER:
                continue
            ref = PS.power_step(phys[w][u.param].cpu().numpy(), qws[w][u.index])
            stamps, ph, q = h.slot(u, w)
            assert bool((stamps == 2).all())
            _close(ph, ref["phat"], ("phat", u.param))
            _close(q, ref["qnew"], ("qnew", u.param))
            other = h.slot(u, w, owner=1 - u.own0)
            assert not other[0].any() and not other[1].any() and not other[2].any()
    want = _oracle_sum(h, phys, qws) / W
    h.master.zero_()
    h.ps()
    for o in range(2):
        assert int(h.sigs[o][256 + o]) == 3
    assert int(h.ctrl.view(torch.int32)[1]) == 0
    got = -h.master.cpu()
    for u in h.plan.units:
        if u.kind in (P.KIND_POWER, P.KIND_DENSE16):
            sl = slice(u.w_off, u.w_off + u.numel)
            _close(got[sl], want[sl], ("ps", u.param))


# ---------------------------------------------------------------------------------------------------- GPU: stats
@pytest.mark.gpu
@pytest.mark.parametrize("r", [1, 4])
def test_v2_powersgd_code_stats_match_fp64(r):
    h = HP(ORACLE_SHAPES, r)
    h.set_step(2)
    phys = h.fill(0, 21, special=True)
    h.encode(0, stats=True)
    acc = h.acc.view(-1, 7).tolist()
    for u in h.plan.units:
        if u.kind != P.KIND_POWER or u.param == INF:
            continue
        gsq, mse, ex, bias, real, real4, n = acc[u.ts_index]
        _, ph, q = h.slot(u, 0)
        A = phys[u.param].cpu().double()
        ghat = (ph.double() @ q.double().T).float().double()
        assert n == 1 and bias == 0 and ex == real == real4
        assert real == bin(PS.power_step(A.float().numpy(), PS.normals(h.seed, u.index, u.cols, r, 0))["mask"]).count("1")
        assert gsq == pytest.approx(float(A.square().sum()), rel=1e-12, abs=0)
        assert mse == pytest.approx(float((A - ghat).square().sum()), rel=1e-3, abs=1e-30)
        if u.param != ZERO:
            assert mse < gsq


# ---------------------------------------------------------------------------------------------------- GPU: feedback
@pytest.mark.gpu
@pytest.mark.parametrize("r", [1, 2, 4])
def test_error_feedback_identity_and_contraction(r):
    h = Loopback("powersgd", ef_grads(1), svd_rank=r)
    try:
        g, e_old = h.g, h.residual()
        for _ in range(4):
            A = g + e_old
            ghat, e_new = h.step()
            scale = g.abs() + e_old.abs() + ghat.abs() + e_new.abs()
            assert bool(((A - (ghat + e_new)).abs() <= 1e-6 * scale + 1e-7 * float(scale.max())).all())
            for q in h.w:
                sl = slice(q.off, q.off + q.numel)
                assert float(e_new[sl].norm()) <= float(A[sl].norm()) * (1 + 1e-6)
            assert float(e_new.norm()) > 0
            e_old = e_new
    finally:
        h.close()


@pytest.mark.gpu
def test_error_feedback_residual_stays_bounded():
    """A fixed gradient for 200 steps: every step contracts (||e_{t+1}|| <= rho ||g + e_t||, rho < 1), so ||e|| stays
    below rho / (1 - rho) ||g||; the pushed sum misses 200 g by exactly the final residual."""
    h = Loopback("powersgd", ef_grads(2), svd_rank=2)
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
    h = Loopback("powersgd", ef_grads(4), svd_rank=2, code_stats=True)
    try:
        h.step()
        st = h.eng.code_stats()
        pl = h.eng.plan
        assert st["code"] == "powersgd" and st["steps"] == 1
        names = {id(p): n for n, p in h.eng.model.named_parameters()}
        for u in pl.units:
            t = st["tensors"][names[id(h.eng.params[u.param])]]
            if u.kind == P.KIND_POWER:
                assert t["bytes"] == 4 * u.rcap * (u.rows + u.cols)
                assert t["atoms"] == t["exp_atoms"] == 2 and 0 < t["rel_var"] < 1
        assert st["model"]["bytes"] == pl.powersgd_bytes() + pl.dense_bytes()
    finally:
        h.close()


# ---------------------------------------------------------------------------------------------------- GPU: engine
_train = functools.partial(train, code="powersgd", svd_rank=2)


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
        return ShadowEngine(build_model("VGG11", 10), 0, 1, code="powersgd", svd_rank=2, lr=0.05, momentum=0.9,
                            use_graph=False)
    a = mk()
    a.prepare(x.pin_memory(), y.pin_memory(), warmup=0)
    for _ in range(3):
        a.train_step(x, y)
    path = a.save_checkpoint(str(tmp_path) + "/")
    side = torch.load(path + "_optim", weights_only=False)
    assert side["code"] == "powersgd" and side["svd_rank"] == 2
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
def test_launcher_powersgd_writes_ef_norm_and_code_stats(tmp_path, monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    args = add_fit_args(argparse.ArgumentParser(), [
        "--network", "ResNet18", "--dataset", "Cifar10", "--synthetic", "1", "--train-len", "512", "--test-len", "64",
        "--batch-size", "32", "--test-batch-size", "64", "--backend", "p2p", "--dtype", "bf16", "--max-steps", "6",
        "--log-interval", "2", "--eval-freq", "100", "--train-dir", str(tmp_path) + "/",
        "--metrics-file", str(tmp_path / "m"), "--code", "powersgd", "--svd-rank", "2", "--error-feedback", "1",
        "--code-stats", "1"])
    L.run_p2p_training(args)
    recs = [json.loads(l) for l in open(str(tmp_path / "m") + ".rank0.jsonl")]
    assert recs and all(r["ef_norm"] > 0 and math.isfinite(r["ef_norm"]) for r in recs)
    m = recs[-1]["code_stats"]["model"]
    assert m["atoms"] > 0 and 0 < m["rel_var"] < 1


@pytest.mark.gpu
@pytest.mark.multigpu
def test_shadow_engine_powersgd_multi_gpu_replicas_identical():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 8 else (8 if os.environ.get("ATOMO_TEST_WORLD8") else 2)
    res = run_mp(world, {"code": "powersgd", "ps_mode": "sharded", "net": "VGG11"}, 29812)
    for rank, err, same, l0, l1, mode, mc, _ in res:
        assert err == 0 and same, res

"""Signum with majority vote on the bf16 engine (``code="signum"``): the refusals of the engine and the launcher before
any CUDA work, the planner's units, slots and byte accounting, and the ``codings.signum`` oracle on hand-made cases."""
import math

import numpy as np
import pytest
import torch

from atomo_b200.codings import signum as S
from atomo_b200.ops import plan2 as P
from atomo_b200.runtime import p2p_launcher as L

from shadow_harness import fit_args, forbid_cuda, model_shapes

REFUSALS = [
    (dict(optimizer="adam"), "optimizer='sgd'"),
    (dict(optimizer="adamw"), "optimizer='sgd'"),
    (dict(optimizer="lars"), "optimizer='sgd'"),
    (dict(nesterov=True), "nesterov"),
    (dict(dampening=0.1), "dampening"),
    (dict(momentum=1.0), r"\[0, 1\)"),
    (dict(momentum=-0.1), r"\[0, 1\)"),
    (dict(momentum=True), r"\[0, 1\)"),
    (dict(momentum=math.nan), r"\[0, 1\)"),
    (dict(error_feedback=True), "error_feedback"),
    (dict(code_stats=True), "code_stats"),
    (dict(clip_grad_norm=1.0), "clip_grad_norm"),
    (dict(momentum_correction=True), "momentum_correction"),
    (dict(weight_decay=-1e-4), "weight_decay"),
    (dict(weight_decay=math.inf), "weight_decay"),
]


@pytest.mark.parametrize("kw,match", REFUSALS)
def test_engine_refuses_before_cuda(kw, match, monkeypatch):
    from atomo_b200.runtime import shadow_engine as SE
    forbid_cuda(monkeypatch)
    with pytest.raises(ValueError, match=match):
        SE.ShadowEngine(None, 0, 1, **{"code": "signum", "momentum": 0.9, **kw})


@pytest.mark.parametrize("kw", [dict(momentum=0.0), dict(momentum=0.9, weight_decay=5e-4), dict(accumulate_steps=2),
                                dict(ema_decay=0.99), dict(num_aggregate=1, momentum=0.5)])
def test_engine_accepts_and_reaches_cuda(kw, monkeypatch):
    """Accepted settings get past every check to the first CUDA work."""
    from atomo_b200.runtime import shadow_engine as SE
    forbid_cuda(monkeypatch)
    with pytest.raises(AssertionError, match="after CUDA work"):
        SE.ShadowEngine(None, 0, 1, **{"code": "signum", **kw})


LAUNCHER_REFUSALS = [
    (("--optimizer", "adam"), "optimizer='sgd'"),
    (("--nesterov", "1"), "nesterov"),
    (("--momentum", "1.0"), r"\[0, 1\)"),
    (("--error-feedback", "1"), "error_feedback"),
    (("--code-stats", "1"), "code_stats"),
    (("--clip-grad-norm", "1.0"), "clip_grad_norm"),
    (("--momentum-correction", "1"), "momentum_correction"),
]


@pytest.mark.parametrize("extra,match", LAUNCHER_REFUSALS)
def test_launcher_refuses_before_cuda(extra, match, tmp_path, monkeypatch):
    forbid_cuda(monkeypatch)
    args = fit_args(tmp_path, "--code", "signum", "--dtype", "bf16", "--backend", "p2p", *extra)
    with pytest.raises(ValueError, match=match):
        L._build_engine(args, torch.nn.Linear(4, 4), 0, 1)


def test_launcher_routes_signum(tmp_path, monkeypatch):
    from atomo_b200.runtime import shadow_engine as SE
    seen = []

    class Fake:
        def __init__(self, model, rank, world, **kw):
            seen.append(kw)
    monkeypatch.setattr(SE, "ShadowEngine", Fake)
    model = torch.nn.Linear(4, 4)
    for engine in ("auto", "shadow"):
        _, kind = L._build_engine(fit_args(tmp_path, "--code", "signum", "--dtype", "bf16", "--engine", engine,
                                        "--momentum", "0.9", "--weight-decay", "1e-4"), model, 0, 1)
        assert kind == "shadow" and seen[-1]["code"] == "signum"
        assert seen[-1]["momentum"] == 0.9 and seen[-1]["weight_decay"] == 1e-4
    n = len(seen)
    for extra in (("--dtype", "fp32"), ("--dtype", "bf16", "--engine", "fused")):
        with pytest.raises(SystemExit, match="signum runs on the bf16 engine only"):
            L._build_engine(fit_args(tmp_path, "--code", "signum", *extra), model, 0, 1)
    assert len(seen) == n


def test_role_paths_refuse_signum(monkeypatch, tmp_path):
    from atomo_b200 import distributed_nn
    from atomo_b200.runtime.master import build_coder
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    with pytest.raises(SystemExit, match="p2p bf16 engine"):
        distributed_nn.run_rank(fit_args(tmp_path, "--code", "signum", "--backend", "gloo"))
    with pytest.raises(ValueError, match="p2p bf16 engine"):
        build_coder({"code": "signum"}, worker_side=True)


# ---------------------------------------------------------------------------------------------------- planner
LENET_SHAPES = [(20, 1, 5, 5), (20,), (50, 20, 5, 5), (50,), (500, 800), (500,), (10, 500), (10,)]


def _shapes(net):
    return LENET_SHAPES if net == "LeNet" else model_shapes(net)


@pytest.mark.parametrize("net", ["ResNet18", "VGG11", "LeNet"])
@pytest.mark.parametrize("owners,groups", [(1, 1), (2, 3), (3, 5)])
def test_plan_units_slots_and_bytes(net, owners, groups):
    shapes = _shapes(net) + [(7, 20), (5, 3)]       # tensors whose size is not a multiple of 64
    pl = P.build_plan2(shapes, "signum", n_owners=owners, n_groups=groups, bucket_size=512)
    ref = P.build_plan2(shapes, "sign", n_owners=owners, n_groups=groups, bucket_size=4096)
    spans = []
    for p in pl.params:
        us = [u for u in pl.units if u.param == p.index]
        assert len(us) == 1
        u = us[0]
        if not p.is_w:
            assert u.kind == P.KIND_VEC
            continue
        b = min(4096, p.numel)                          # one bucket per PS tile, whatever --bucket-size says
        assert u.kind == P.KIND_SIGNUM and (u.K, u.ps_rows, u.cs, u.I, u.rs) == (b, b, 1, 0, 0)
        assert u.rows == -(-p.numel // b) == u.n_ps and u.cols == -(-b // 64)
        tiles = sorted((a, n, o) for (ui, a, n, o) in pl.ps_tiles if ui == u.index)
        assert [a for a, _, _ in tiles] == list(range(0, p.numel, 4096))
        assert all(n == min(4096, p.numel - a) for a, n, _ in tiles)
        assert [o for _, _, o in tiles] == [(u.own0 + j) % owners for j in range(u.n_ps)]
        assert [(a, n, j) for (ui, a, n, j) in pl.enc_tiles if ui == u.index] == \
            [(a, n, j) for j, (a, n, _) in enumerate(tiles)]
        spans.append((u.slot_off, u.slot_off + P.qsgd_slot_floats(u.n_ps, u.rows, u.cols)))
        assert (u.slot_off + P.qsgd_words_off(u.n_ps, u.rows)) % 4 == 0     # 16-byte aligned words
    spans.sort()
    assert all(a1 >= b0 for (a0, b0), (a1, b1) in zip(spans, spans[1:])) and spans[-1][1] <= pl.arena_floats
    # the geometry of sign with 4096-element buckets: same tiles, owners, ranges and slots
    assert (pl.enc_tiles, pl.ps_tiles, pl.enc_range, pl.ps_range, pl.arena_floats) == \
        (ref.enc_tiles, ref.ps_tiles, ref.enc_range, ref.ps_range, ref.arena_floats)
    assert [(u.slot_off, u.rows, u.cols, u.own0) for u in pl.units] == [(u.slot_off, u.rows, u.cols, u.own0)
                                                                         for u in ref.units]
    # bytes: ceil(numel / 64) uint64 words per weight tensor, fp32 vectors
    want_bits = sum(8 * -(-p.numel // 64) for p in pl.params if p.is_w)
    assert pl.signum_bytes() == want_bits
    assert pl.dense_bytes() == sum(4 * p.numel for p in pl.params if not p.is_w)
    assert pl.qsgd_bytes() == 0 and pl.expected_factor_bytes() == want_bits
    assert P.build_plan2(shapes, "signum", bucket_size=64).units_bytes() == \
        P.build_plan2(shapes, "signum", bucket_size=4096).units_bytes()


def test_plan_bytes_pinned():
    """The byte accounting of the three models, pinned: a 140-element tensor takes 3 words."""
    got = {net: P.build_plan2(_shapes(net), "signum").signum_bytes() for net in ("ResNet18", "VGG11", "LeNet")}
    for net, v in got.items():
        assert v == sum(8 * -(-math.prod(s) // 64) for s in _shapes(net) if len(s) >= 2)
    assert got["LeNet"] == 8 * (8 + 391 + 6250 + 79)
    assert P.build_plan2([(7, 20)], "signum").signum_bytes() == 24


# ---------------------------------------------------------------------------------------------------- oracle
def test_vote_ties_majorities_and_no_worker():
    # workers x elements: 1 = negative
    bits = [[1, 0, 1, 0, 1],
            [1, 0, 0, 0, 1],
            [0, 0, 1, 1, 1],
            [0, 1, 0, 1, 1]]
    assert S.vote(bits, 5).tolist() == [0.0, 1.0, 0.0, 0.0, -1.0]          # even W: exact ties vote 0
    assert S.vote(bits[:3], 5).tolist() == [-1.0, 1.0, -1.0, 1.0, -1.0]
    assert S.vote(bits[:1], 5).tolist() == [-1.0, 1.0, -1.0, 1.0, -1.0]
    assert S.vote([], 5).tolist() == [0.0] * 5                             # nobody counted: no step
    # one worker flipped: wherever 3 of the other 4 agree, the vote stays
    honest = np.array(bits + [[1, 1, 0, 0, 1]])
    v = S.vote(honest, 5)
    flipped = honest.copy()
    flipped[4] = 1 - flipped[4]
    vf = S.vote(flipped, 5)
    agree = np.abs(honest[:4].sum(axis=0) - 2) >= 1
    assert np.array_equal(v[agree], vf[agree])


def test_zeros_take_the_coin_and_nonfinite_makes_nan():
    u = np.array([1.0, -1.0, 0.0, -0.0, 1e-40, -1e-40, np.inf, -np.inf, np.nan], dtype=np.float32)
    lo = np.full(u.size, 0.25, dtype=np.float32)
    hi = np.full(u.size, 0.75, dtype=np.float32)
    assert S.bits(u, lo).tolist()[:6] == [0, 1, 1, 1, 1, 1]       # zeros and subnormals: coin 1 below one half
    assert S.bits(u, hi).tolist()[:6] == [0, 1, 0, 0, 0, 0]
    assert S.bits(u, hi).tolist()[6:8] == [0, 1]                    # Inf: its sign
    assert not S.nonfinite(u[:6]) and S.nonfinite(u[6:7]) and S.nonfinite(u[8:])
    v = S.vote([S.bits(u[:6], lo[:6]), S.bits(u[:6], hi[:6])], 6, bad=[False, True])
    assert np.isnan(v).all()
    assert np.isnan(S.step(np.ones(6, np.float32), v, 0.1)).all()
    assert S.step(np.float32([1.0, 1.0, 1.0]), np.float32([1, 0, -1]), 0.5).tolist() == [0.5, 1.0, 1.5]


def test_coin_is_fair_and_keyed():
    e = np.arange(40000)
    a = S.coin_uniforms(7, 3, e, 2, 0)
    assert abs(float((a < 0.5).mean()) - 0.5) < 0.01
    for other in (S.coin_uniforms(8, 3, e, 2, 0), S.coin_uniforms(7, 4, e, 2, 0), S.coin_uniforms(7, 3, e, 3, 0),
                  S.coin_uniforms(7, 3, e, 2, 1)):
        assert (other != a).mean() > 0.99


def test_momentum_and_pack():
    u = np.zeros(3, np.float32)
    g = np.float32([1.0, -2.0, 0.0])
    u = S.momentum_step(u, g, 0.9)
    assert u.tolist() == [1.0, -2.0, 0.0]
    u = S.momentum_step(u, np.float32([-1.0, 1.0, 0.0]), 0.9)
    assert u.tolist() == [np.float32(np.float32(0.9) * 1) - 1, np.float32(np.float32(0.9) * -2) + 1, 0.0]
    assert S.momentum_step(np.float32([1e-38]), np.float32([0.0]), 0.01)[0] == 0   # flushed like the kernels
    b = np.zeros(140, np.int64)
    b[[0, 63, 64, 139]] = 1
    w = S.pack(b)
    assert w.size == 3 and int(w[0]) == (1 | (1 << 63)) and int(w[1]) == 1 and int(w[2]) == 1 << 11
    assert np.array_equal(S.unpack(w, 140), b)

"""Distributed Lion on the bf16 engine (``code="dlion"``): the refusals of the engine and the launcher before any CUDA
work, the launcher's routing and flags, the role paths' refusals, the planner's bytes against Signum's, and the
``codings.dlion`` oracle on hand-made cases."""
import argparse
import math

import numpy as np
import pytest
import torch

from atomo_b200.codings import dlion as D
from atomo_b200.codings import signum as S
from atomo_b200.ops import plan2 as P
from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils.flags import add_fit_args

from shadow_harness import fit_args, forbid_cuda, model_shapes

REFUSALS = [
    (dict(optimizer="adam"), "optimizer='sgd'"),
    (dict(optimizer="adamw"), "optimizer='sgd'"),
    (dict(optimizer="lars"), "optimizer='sgd'"),
    (dict(optimizer="lion"), "owners step by the aggregate"),
    (dict(nesterov=True), "nesterov"),
    (dict(dampening=0.1), "dampening"),
    (dict(betas=(1.0, 0.99)), "dlion: betas"),
    (dict(betas=(0.9, -0.1)), "dlion: betas"),
    (dict(betas=(0.9, math.nan)), "dlion: betas"),
    (dict(betas=(0.9, math.inf)), "dlion: betas"),
    (dict(betas=(True, 0.5)), "dlion: betas"),
    (dict(betas=(0.9,)), "dlion: betas"),
    (dict(error_feedback=True), "error_feedback"),
    (dict(code_stats=True), "code_stats"),
    (dict(clip_grad_norm=1.0), "clip_grad_norm"),
    (dict(momentum_correction=True), "momentum_correction"),
    (dict(dlion_aggregate="median"), "dlion_aggregate"),
    (dict(weight_decay=-1e-4), "weight_decay"),
    (dict(weight_decay=math.inf), "weight_decay"),
]


@pytest.mark.parametrize("kw,match", REFUSALS)
def test_engine_refuses_before_cuda(kw, match, monkeypatch):
    from atomo_b200.runtime import shadow_engine as SE
    forbid_cuda(monkeypatch)
    with pytest.raises(ValueError, match=match):
        SE.ShadowEngine(None, 0, 1, **{"code": "dlion", **kw})


@pytest.mark.parametrize("kw", [dict(), dict(betas=(0.0, 0.99)), dict(momentum=0.5), dict(momentum=1.5),
                                dict(weight_decay=5e-4), dict(accumulate_steps=2), dict(ema_decay=0.99),
                                dict(num_aggregate=1), dict(dlion_aggregate="mean"), dict(ps_mode="dedicated")])
def test_engine_accepts_and_reaches_cuda(kw, monkeypatch):
    """Accepted settings get past every check to the first CUDA work; --momentum is ignored, whatever its value."""
    from atomo_b200.runtime import shadow_engine as SE
    forbid_cuda(monkeypatch)
    with pytest.raises(AssertionError, match="after CUDA work"):
        SE.ShadowEngine(None, 0, 1, **{"code": "dlion", **kw})


def test_engine_default_betas(monkeypatch):
    from atomo_b200.runtime import shadow_engine as SE
    forbid_cuda(monkeypatch)
    e = SE.ShadowEngine.__new__(SE.ShadowEngine)
    with pytest.raises(AssertionError, match="after CUDA work"):
        e.__init__(None, 0, 1, code="dlion", momentum=0.5, weight_decay=1e-3)
    assert e.betas == (0.9, 0.99) and e.dlion and e.signum and not e.lion
    assert e.dlion_aggregate == "vote" and e.adamw_wd == 1e-3 and e.decay_on


LAUNCHER_REFUSALS = [
    (("--optimizer", "adam"), "optimizer='sgd'"),
    (("--optimizer", "lion"), "owners step by the aggregate"),
    (("--nesterov", "1"), "nesterov"),
    (("--lion-betas", "1.0", "0.99"), "dlion: betas"),
    (("--error-feedback", "1"), "error_feedback"),
    (("--code-stats", "1"), "code_stats"),
    (("--clip-grad-norm", "1.0"), "clip_grad_norm"),
    (("--momentum-correction", "1"), "momentum_correction"),
]


@pytest.mark.parametrize("extra,match", LAUNCHER_REFUSALS)
def test_launcher_refuses_before_cuda(extra, match, tmp_path, monkeypatch):
    forbid_cuda(monkeypatch)
    args = fit_args(tmp_path, "--code", "dlion", "--dtype", "bf16", "--backend", "p2p", *extra)
    with pytest.raises(ValueError, match=match):
        L._build_engine(args, torch.nn.Linear(4, 4), 0, 1)


def test_flags():
    a = add_fit_args(argparse.ArgumentParser(), ["--code", "dlion"])
    assert a.dlion_aggregate == "vote" and a.lion_betas == [0.9, 0.99] and a.momentum == 0.5
    a = add_fit_args(argparse.ArgumentParser(), ["--code", "dlion", "--dlion-aggregate", "mean", "--lion-betas", "0.95",
                                                 "0.98"])
    assert a.dlion_aggregate == "mean" and a.lion_betas == [0.95, 0.98]
    with pytest.raises(SystemExit):
        add_fit_args(argparse.ArgumentParser(), ["--dlion-aggregate", "median"])


def test_launcher_routes_dlion(tmp_path, monkeypatch):
    from atomo_b200.runtime import shadow_engine as SE
    seen = []

    class Fake:
        def __init__(self, model, rank, world, **kw):
            seen.append(kw)
    monkeypatch.setattr(SE, "ShadowEngine", Fake)
    model = torch.nn.Linear(4, 4)
    for engine in ("auto", "shadow"):
        for agg in ("vote", "mean"):
            _, kind = L._build_engine(fit_args(tmp_path, "--code", "dlion", "--dtype", "bf16", "--engine", engine,
                                               "--lion-betas", "0.95", "0.98", "--dlion-aggregate", agg,
                                               "--weight-decay", "1e-4"), model, 0, 1)
            assert kind == "shadow" and seen[-1]["code"] == "dlion" and seen[-1]["dlion_aggregate"] == agg
            assert seen[-1]["betas"] == (0.95, 0.98) and seen[-1]["weight_decay"] == 1e-4
    # the launcher's default --momentum 0.5 reaches the engine, which ignores it
    L._build_engine(fit_args(tmp_path, "--code", "dlion", "--dtype", "bf16"), model, 0, 1)
    assert seen[-1]["momentum"] == 0.5 and seen[-1]["betas"] == (0.9, 0.99) and seen[-1]["dlion_aggregate"] == "vote"
    # other codes get no dlion_aggregate
    L._build_engine(fit_args(tmp_path, "--code", "signum", "--dtype", "bf16"), model, 0, 1)
    assert "dlion_aggregate" not in seen[-1] and "betas" not in seen[-1]
    n = len(seen)
    for extra in (("--dtype", "fp32"), ("--dtype", "bf16", "--engine", "fused")):
        with pytest.raises(SystemExit, match="dlion runs on the bf16 engine only"):
            L._build_engine(fit_args(tmp_path, "--code", "dlion", *extra), model, 0, 1)
    assert len(seen) == n


def test_role_paths_refuse_dlion(monkeypatch, tmp_path):
    from atomo_b200 import distributed_nn
    from atomo_b200.runtime.master import build_coder
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    for backend in ("gloo", "nccl"):
        with pytest.raises(SystemExit, match="--code dlion runs on the --backend p2p bf16 engine"):
            distributed_nn.run_rank(fit_args(tmp_path, "--code", "dlion", "--backend", backend))
    with pytest.raises(ValueError, match="--code dlion runs on the --backend p2p bf16 engine"):
        build_coder({"code": "dlion"}, worker_side=True)


# ---------------------------------------------------------------------------------------------------- planner
@pytest.mark.parametrize("net", ["ResNet18", "VGG11"])
def test_plan_bytes_equal_signum(net):
    """The engine plans dlion as signum: same units, tiles and slots, so the same bytes per push."""
    pl = P.build_plan2(model_shapes(net), "signum")
    assert pl.signum_bytes() == sum(8 * -(-math.prod(s) // 64) for s in model_shapes(net) if len(s) >= 2)
    assert pl.dense_bytes() == sum(4 * math.prod(s) for s in model_shapes(net) if len(s) < 2)
    if net == "ResNet18":
        assert (pl.signum_bytes(), pl.dense_bytes()) == (1395544, 38440)
        assert P.build_plan2(model_shapes(net), "sgd").dense_bytes() == 22367144


# ---------------------------------------------------------------------------------------------------- oracle
def _rule(m, g, b1, b2):
    """The hand-written rule in fp32 scalars, every operation rounded on its own."""
    f = np.float32
    c = f(f(f(b1) * f(m)) + f(f(f(1) - f(b1)) * f(g)))
    return c, f(f(f(b2) * f(m)) + f(f(f(1) - f(b2)) * f(g)))


@pytest.mark.parametrize("b1,b2", [(0.9, 0.99), (0.95, 0.98), (0.5, 0.0), (0.0, 0.99)])
def test_worker_step_matches_the_hand_written_rule(b1, b2):
    rng = np.random.default_rng(3)
    m = np.zeros(257, np.float32)
    for _ in range(4):
        g = rng.standard_normal(257).astype(np.float32)
        c, m2 = D.worker_step(m, g, b1, b2)
        want = [_rule(mi, gi, b1, b2) for mi, gi in zip(m, g)]
        assert np.array_equal(c, np.float32([w[0] for w in want]))
        assert np.array_equal(m2, np.float32([w[1] for w in want]))
        m = m2
    assert D.worker_step(np.float32([1e-38]), np.float32([0.0]), 0.01, 0.01)[0][0] == 0   # flushed like the kernels


def test_b1_zero_is_the_sign_of_g():
    """b1 == 0: c == g bit for bit (the direction of --code signum --momentum 0), whatever m and b2 are."""
    rng = np.random.default_rng(5)
    g = rng.standard_normal(4096).astype(np.float32)
    g[:8] = [0.0, -0.0, 1e-40, -1e-40, np.inf, -np.inf, 1.0, -1.0]
    m = rng.standard_normal(4096).astype(np.float32)
    c, _ = D.worker_step(m, g, 0.0, 0.99)
    assert np.array_equal(c.view(np.uint32), S.ftz(g).view(np.uint32))
    un = rng.random(4096).astype(np.float32)
    assert np.array_equal(S.bits(c, un), S.bits(g, un))
    # with b1 == b2 the direction is Signum's momentum up to the scale (1 - b): the same sign away from rounding
    m0 = np.zeros(4096, np.float32)
    u = S.momentum_step(m0, g, 0.9)
    c1, _ = D.worker_step(m0, g, 0.9, 0.9)
    fin = np.isfinite(g) & (np.abs(g) > 1e-30)
    assert np.array_equal(np.sign(c1[fin]), np.sign(u[fin]))


def test_mean_values_for_every_k_and_n():
    """n counted workers, k of them negative: (n - 2k) / n rounded once in fp32; n = 0 gives 0."""
    for n in range(0, 17):
        for k in range(0, n + 1):
            rows = [[1] * 3 if w < k else [0] * 3 for w in range(n)]
            v = D.mean(rows, 3)
            want = np.float32(0) if n == 0 else np.float32(np.float32(n - 2 * k) / np.float32(n))
            assert v.dtype == np.float32 and (v == want).all(), (n, k, v, want)
            assert (np.abs(np.float64(v) - ((n - 2 * k) / n if n else 0.0)) <= 2.0 ** -24).all()
            assert np.array_equal(D.aggregate("vote", rows, 3), S.vote(rows, 3))
    assert np.isnan(D.mean([[0, 1], [1, 1]], 2, bad=[False, True])).all()
    assert D.mean([], 5).tolist() == [0.0] * 5
    with pytest.raises(ValueError):
        D.aggregate("median", [[0]], 1)


def test_mean_equals_vote_for_one_worker_and_step_rounds_once():
    rows = [[0, 1, 1, 0]]
    assert np.array_equal(D.mean(rows, 4), S.vote(rows, 4))
    p = np.float32([1.0, 1.0, 3.0, np.nan])
    v = np.float32([1.0 / 3.0, -1.0, 0.0, 1.0])
    got = D.step(p, v, 0.1)
    want = [np.float32(np.float64(p[i]) + np.float64(np.float32(-0.1)) * np.float64(v[i])) for i in range(3)]
    assert got[:3].tolist() == want and np.isnan(got[3])
    # with a vote in {-1, 0, 1} the fused step is Signum's
    vv = np.float32([1, 0, -1])
    assert np.array_equal(D.step(p[:3], vv, 0.1), S.step(p[:3], vv, 0.1))

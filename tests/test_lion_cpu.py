"""Lion without a GPU: ``optim/lion.py`` against a hand-written fp32 rule, the ``--optimizer lion`` and
``--lion-betas`` flags, the engine's default betas and its refusals (each before any CUDA work), the fp32-flat engine's
refusal, and the gloo role path's update against ``optim/lion.py``, with a 2-process run that trains and resumes."""
import argparse
import os

import numpy as np
import pytest
import torch

from atomo_b200.optim import Lion
from atomo_b200.optim.lion import lion_sign
from atomo_b200.runtime import master as M
from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils.flags import add_fit_args

from shadow_harness import fit_args, forbid_cuda, role_master, role_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def _rule(p, m, g, lr, b1, b2, wd):
    """The Lion rule element by element in numpy float32 scalars: every operation rounded on its own."""
    p, m, g = p.copy(), m.copy(), g.copy()
    om1, om2 = f32(1) - f32(b1), f32(1) - f32(b2)
    fac = f32(1.0 - lr * wd)
    for i in np.ndindex(p.shape):
        if p.ndim >= 2 and wd:
            p[i] = f32(p[i] * fac)
        c = f32(f32(f32(b1) * m[i]) + f32(om1 * g[i]))
        s = f32(np.sign(c))                           # numpy: NaN for NaN, 0 for +-0
        p[i] = f32(p[i] - f32(f32(lr) * s))
        m[i] = f32(f32(f32(b2) * m[i]) + f32(om2 * g[i]))
    return p, m


@pytest.mark.parametrize("wd", [0.0, 0.1])
@pytest.mark.parametrize("betas", [(0.9, 0.99), (0.5, 0.95), (0.0, 0.0)])
def test_matches_the_hand_written_fp32_rule(betas, wd):
    g = torch.Generator().manual_seed(3)
    shapes = [(4, 3, 2, 2), (5,), (6, 7)]
    params = [torch.randn(s, generator=g) for s in shapes]
    ref = [p.numpy().copy() for p in params]
    mom = [np.zeros(s, np.float32) for s in shapes]
    opt = Lion(params, lr=0.01, betas=betas, weight_decay=wd)
    with np.errstate(invalid="ignore"):
        for step in range(4):
            grads = [torch.randn(s, generator=g) for s in shapes]
            grads[0].view(-1)[:5] = 0.0              # c == 0 while m is 0 there: p stays
            if step == 3:
                grads[2][0, 0] = float("nan")         # NaN propagates into p and m
            opt.step(grads=grads)
            for i, x in enumerate(grads):
                ref[i], mom[i] = _rule(ref[i], mom[i], x.numpy(), 0.01, betas[0], betas[1], wd)
            for p, r in zip(params, ref):
                assert np.array_equal(p.numpy().view(np.int32), r.view(np.int32)) or \
                    np.array_equal(p.numpy(), r, equal_nan=True)
    assert torch.isnan(params[2][0, 0]) and not torch.isnan(params[2][0, 1])
    assert torch.isnan(opt.state[params[2]]["exp_avg"][0, 0])


def test_zero_interpolation_leaves_the_weight_and_only_weights_decay():
    w, b = torch.randn(3, 4), torch.randn(4)
    w0, b0 = w.clone(), b.clone()
    opt = Lion([w, b], lr=0.5, weight_decay=0.2)
    opt.step(grads=[torch.zeros(3, 4), torch.zeros(4)])
    assert torch.equal(w, w0 * float(f32(1 - 0.5 * 0.2))) and torch.equal(b, b0)   # c == 0: the decay only


def test_sign_keeps_nan_and_zeros():
    c = torch.tensor([2.0, -3.0, 0.0, -0.0, float("nan"), 1e-30])
    s = lion_sign(c)
    assert s[:4].tolist() == [1.0, -1.0, 0.0, 0.0] and torch.isnan(s[4]) and s[5] == 1.0
    assert torch.sign(torch.tensor(float("nan"))) == 0          # why lion_sign is not torch.sign


@pytest.mark.parametrize("kw", [dict(lr=-1.0), dict(betas=(1.0, 0.9)), dict(betas=(0.9, -0.1)),
                                dict(weight_decay=float("inf"))])
def test_oracle_refuses_bad_settings(kw):
    with pytest.raises(ValueError, match="Lion"):
        Lion([torch.zeros(2, 2)], **kw)


def test_flags_parse():
    a = add_fit_args(argparse.ArgumentParser(), [])
    assert a.lion_betas == [0.9, 0.99]
    a = add_fit_args(argparse.ArgumentParser(), ["--optimizer", "lion", "--lion-betas", "0.95", "0.98",
                                                 "--weight-decay", "0.1"])
    assert a.optimizer == "lion" and a.lion_betas == [0.95, 0.98] and a.weight_decay == 0.1


def _engine(monkeypatch, **kw):
    from atomo_b200.runtime import shadow_engine as S
    forbid_cuda(monkeypatch)
    return S.ShadowEngine(None, 0, 1, **dict(dict(optimizer="lion"), **kw))


@pytest.mark.parametrize("kw, msg", [
    (dict(nesterov=True), "lion takes no Nesterov"),
    (dict(amsgrad=True), "lion keeps no second moment"),
    (dict(code="signum"), "owners step by the vote"),
    (dict(code="topk", error_feedback=True, momentum_correction=True), "plain SGD"),
    (dict(clip_grad_norm=1.0), "clip_grad_norm"),
    (dict(betas=(1.0, 0.99)), "lion: betas"),
    (dict(betas=(0.9, float("nan"))), "lion: betas"),
    (dict(betas=(0.9, -0.5)), "lion: betas"),
    (dict(betas=(True, 0.5)), "lion: betas"),
    (dict(betas=(0.9,)), "lion: betas"),
    (dict(weight_decay=-0.1), "lion: weight_decay"),
    (dict(weight_decay=float("nan")), "lion: weight_decay"),
])
def test_engine_refusals_come_before_cuda_work(kw, msg, monkeypatch):
    with pytest.raises(ValueError, match=msg):
        _engine(monkeypatch, **kw)


def test_engine_default_betas_and_ignored_momentum(monkeypatch):
    """The defaults are resolved before the first CUDA work: Lion (0.9, 0.99), Adam (0.9, 0.999); the launcher's
    --momentum 0.5 is no refusal for Lion."""
    from atomo_b200.runtime import shadow_engine as S
    seen = {}

    def stop(*a, **k):
        raise RuntimeError("stop")
    monkeypatch.setattr(S, "load_ext", stop)
    for opt in ("lion", "adam"):
        eng = S.ShadowEngine.__new__(S.ShadowEngine)
        with pytest.raises(RuntimeError, match="stop"):
            S.ShadowEngine.__init__(eng, None, 0, 1, optimizer=opt, momentum=0.5, weight_decay=0.1)
        seen[opt] = eng
    assert seen["lion"].lion and seen["lion"].adamw_wd == 0.1 and seen["lion"].decay_on
    assert seen["lion"].betas == (0.9, 0.99) and seen["adam"].betas == (0.9, 0.999)
    assert not seen["adam"].lion and seen["adam"].adamw_wd == 0.0


def test_fp32_flat_engine_refuses(tmp_path):
    model = torch.nn.Linear(4, 4)
    for extra in (("--engine", "fused", "--dtype", "bf16"), ("--dtype", "fp32")):
        with pytest.raises(SystemExit, match="--optimizer lion runs on the bf16 engine.*--engine shadow"):
            L._build_engine(fit_args(tmp_path, "--code", "svd", "--optimizer", "lion", *extra), model, 0, 1)


# ---------------------------------------------------------------------------------------------------- role path
def _master(tmp_path, wd=0.1, betas=(0.9, 0.99)):
    return role_master(tmp_path, learning_rate=0.01, optimizer="lion", weight_decay=wd, lion_betas=betas)


def test_role_path_update_is_lion(tmp_path):
    m = _master(tmp_path, betas=(0.8, 0.95))
    assert isinstance(m.optimizer, Lion) and m.optimizer.param_groups[0]["betas"] == (0.8, 0.95)
    params = [p.detach().clone() for p in m.network.parameters()]
    ref = Lion(params, lr=0.01, betas=(0.8, 0.95), weight_decay=0.1)
    g = torch.Generator().manual_seed(1)
    for step in range(4):
        if step == 2:
            m.lr = 0.004
            m.optimizer.set_lr(m.lr)
            ref.set_lr(m.lr)
        grads = [torch.randn(v.shape, generator=g, dtype=torch.float64) for v in m.grad_accumulator.gradient_aggregator]
        for v, x in zip(m.grad_accumulator.gradient_aggregator, grads):
            v.copy_(x)
        m._model_update(1)
        ref.step(grads=grads)
        assert all(torch.equal(a, b) for a, b in zip(m.network.parameters(), params))


ROLE_FLAGS = ("--optimizer", "lion", "--weight-decay", "0.1", "--lion-betas", "0.9", "0.99")


def test_gloo_role_path_matches_the_oracle_and_resumes(tmp_path):
    """Two processes (PS and one worker) for 3 steps, then a resume to 5.  Each saved step follows from the one
    before by ``optim/lion.py`` on the gradient the momenta imply: with b2 = 0.99 the stored momenta give g exactly
    enough to fix the sign of every c that is not tiny, and the step is then checked bit for bit."""
    d = str(tmp_path) + "/"
    role_run(d, 29591, 3, *ROLE_FLAGS)
    out = role_run(d, 29592, 5, *ROLE_FLAGS, "--resume", "1")
    assert "Master: Step: 5" in out and "Master: Step: 1," not in out
    load = lambda s: torch.load(d + "model_step_%d_optim" % s, map_location="cpu", weights_only=False)
    net = M.build_model("LeNet", 10, "MNIST")
    pnames = [n for n, _ in net.named_parameters()]
    b1, b2, lr, wd = f32(0.9), f32(0.99), f32(0.01), 0.1
    checked = 0
    for s in range(2, 6):
        m_prev, m_next = (torch.load(d + "model_step_%d" % k, map_location="cpu") for k in (s - 1, s))
        o_prev, o_next = load(s - 1)["optimizer"], load(s)["optimizer"]
        assert o_next["param_groups"][0]["betas"] == (0.9, 0.99)
        for i, n in enumerate(pnames):
            mp, mn = o_prev["state"][i]["exp_avg"].double(), o_next["state"][i]["exp_avg"].double()
            g = (mn - float(b2) * mp) / float(f32(1) - b2)
            c = float(b1) * mp + float(f32(1) - b1) * g
            sure = c.abs() > 1e-3 * (mp.abs() + g.abs() + 1e-12)
            p = m_prev[n].clone()
            if p.dim() >= 2:
                p = p * float(f32(1.0 - 0.01 * wd))
            p = p - torch.sign(c).float() * lr
            assert torch.equal(p[sure], m_next[n][sure]), (s, n)
            checked += int(sure.sum())
    assert checked > 1000

"""AdamW without a GPU: ``optim/adamw.py`` against ``torch.optim.AdamW`` with two parameter groups in fp64, the
``--optimizer adamw`` flag and its refusals (fp32-flat engine, a negative or non-finite decay before any CUDA work),
``Ctrl2.decay_factor`` at offset 68 and its rewrite by ``set_lr``, and the gloo role path's update against
``optim/adamw.py``, with a resume."""
import argparse
import os
import struct

import numpy as np
import pytest
import torch

from atomo_b200.ops import plan2 as P2
from atomo_b200.optim import AdamW
from atomo_b200.runtime import master as M
from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils.flags import add_fit_args

from shadow_harness import fit_args, forbid_cuda, role_master, role_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(6, 3, 3, 3), (6,), (10, 24), (10,), (4, 5)]


def _torch_adamw(params, lr, wd, amsgrad):
    """torch.optim.AdamW with the two groups: weights decayed, 1-D parameters not."""
    return torch.optim.AdamW([{"params": [p for p in params if p.dim() >= 2]},
                              {"params": [p for p in params if p.dim() < 2], "weight_decay": 0.0}],
                             lr=lr, weight_decay=wd, amsgrad=amsgrad)


@pytest.mark.parametrize("amsgrad", [False, True], ids=["adamw", "amsgrad"])
@pytest.mark.parametrize("wd", [0.0, 0.05, 0.5])
def test_matches_torch_adamw_in_fp64(wd, amsgrad):
    g = torch.Generator().manual_seed(3)
    init = [torch.randn(s, generator=g, dtype=torch.float64) for s in SHAPES]
    ours = [p.clone() for p in init]
    ref = [torch.nn.Parameter(p.clone()) for p in init]
    opt, topt = AdamW(ours, lr=0.02, weight_decay=wd, amsgrad=amsgrad), _torch_adamw(ref, 0.02, wd, amsgrad)
    for step in range(8):
        if step == 4:       # an LR change mid-run: the decay follows it
            opt.set_lr(0.005)
            for group in topt.param_groups:
                group["lr"] = 0.005
        grads = [torch.randn(s, generator=g, dtype=torch.float64) * (1 + step) for s in SHAPES]
        opt.step(grads=grads)
        for p, x in zip(ref, grads):
            p.grad = x.clone()
        topt.step()
        for a, b in zip(ours, ref):
            # fp64, one rounding per operation on both sides; torch forms the moments with lerp
            assert torch.allclose(a, b.detach(), rtol=1e-13, atol=1e-15)
    # the same run without decay: 1-D parameters end bit for bit where they did, every weight elsewhere
    g = torch.Generator().manual_seed(3)
    plain = [torch.randn(s, generator=g, dtype=torch.float64) for s in SHAPES]
    popt = AdamW(plain, lr=0.02, weight_decay=0.0, amsgrad=amsgrad)
    for step in range(8):
        if step == 4:
            popt.set_lr(0.005)
        popt.step(grads=[torch.randn(s, generator=g, dtype=torch.float64) * (1 + step) for s in SHAPES])
    for a, b in zip(ours, plain):
        assert torch.equal(a, b) == (a.dim() < 2 or wd == 0)


def test_decay_comes_before_the_moments():
    """One step on a zero gradient: the weight is only decayed, the vector untouched."""
    w, v = torch.full((3, 2), 2.0, dtype=torch.float64), torch.full((3,), 2.0, dtype=torch.float64)
    AdamW([w, v], lr=0.1, weight_decay=0.5).step(grads=[torch.zeros(3, 2, dtype=torch.float64),
                                                        torch.zeros(3, dtype=torch.float64)])
    assert torch.equal(w, torch.full((3, 2), 2.0 * (1 - 0.1 * 0.5), dtype=torch.float64))
    assert torch.equal(v, torch.full((3,), 2.0, dtype=torch.float64))


def test_optimizer_refuses_bad_settings():
    for kw in (dict(lr=-1.0), dict(weight_decay=-0.1), dict(weight_decay=float("inf")),
               dict(weight_decay=float("nan")), dict(betas=(1.0, 0.999))):
        with pytest.raises(ValueError, match="AdamW"):
            AdamW([torch.zeros(2, 2)], **kw)


def test_flag_parses():
    assert add_fit_args(argparse.ArgumentParser(), []).optimizer == "sgd"
    args = add_fit_args(argparse.ArgumentParser(), ["--optimizer", "adamw", "--weight-decay", "0.05"])
    assert args.optimizer == "adamw" and args.weight_decay == 0.05


@pytest.mark.parametrize("bad", [-0.1, -1e-12, float("nan"), float("inf"), -float("inf"), True, "0.1"])
def test_engine_refuses_a_bad_decay_before_cuda_work(bad, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    forbid_cuda(monkeypatch)
    with pytest.raises(ValueError, match="adamw: weight_decay"):
        S.ShadowEngine(None, 0, 1, optimizer="adamw", weight_decay=bad)


def test_engine_refuses_momentum_correction_with_adamw(monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    forbid_cuda(monkeypatch)
    with pytest.raises(ValueError, match="optimizer='sgd' only"):
        S.ShadowEngine(None, 0, 1, code="topk", error_feedback=True, momentum_correction=True, optimizer="adamw",
                       weight_decay=0.01)


def test_fp32_flat_engine_refuses(tmp_path):
    model = torch.nn.Linear(4, 4)
    for extra in (("--engine", "fused", "--dtype", "bf16"), ("--dtype", "fp32"),
                  ("--dtype", "bf16", "--code", "entrywise")):        # auto sends these to the fp32-flat engine
        with pytest.raises(SystemExit, match="--optimizer adamw runs on the bf16 engine.*--engine shadow"):
            L._build_engine(fit_args(tmp_path, "--code", "svd", "--optimizer", "adamw", *extra), model, 0, 1)
    with pytest.raises(SystemExit, match="--optimizer adam on the p2p backend"):      # unchanged for adam
        L._build_engine(fit_args(tmp_path, "--code", "svd", "--optimizer", "adam", "--dtype", "fp32"), model, 0, 1)


def test_ctrl2_carries_the_decay_factor_at_offset_68():
    assert struct.calcsize(P2.CTRL2_FMT) == P2.CTRL2_BYTES == 72
    f = float(np.float32(1.0 - 0.01 * 0.05))
    kw = dict(step=3, lr=0.01, opt=P2.OPT_ADAM, num_aggregate=2, trust_coefficient=0.5, clip_grad_norm=1.5)
    off, on = P2.pack_ctrl2(**kw), P2.pack_ctrl2(decay_factor=f, **kw)
    assert off[:68] == on[:68]                                          # no other field moves
    assert struct.unpack_from("<f", off, 68)[0] == 0.0 and struct.unpack_from("<f", on, 68)[0] == f
    assert struct.unpack_from("<ii", on, 56) == (P2.OPT_ADAM, 2) and struct.unpack_from("<f", on, 64)[0] == 0.5


def _host_engine(lr, wd):
    """The parts of a ShadowEngine that set_lr touches, with Ctrl2 in host memory."""
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    eng = ShadowEngine.__new__(ShadowEngine)
    eng.adamw_wd, eng.decay_on = wd, wd > 0
    eng.ctrl = torch.frombuffer(bytearray(P2.pack_ctrl2(lr=lr, opt=P2.OPT_ADAM,
                                                        decay_factor=eng.decay_factor(lr) if wd else 0.0)),
                                dtype=torch.uint8)
    eng.ctrl_f32 = eng.ctrl.view(torch.float32)
    return eng


def test_set_lr_rewrites_the_decay_factor():
    eng = _host_engine(0.01, 0.05)
    assert struct.unpack_from("<f", eng.ctrl.numpy().tobytes(), 68)[0] == np.float32(1 - 0.01 * 0.05)
    for lr in (0.1, 3e-4, 0.0):
        eng.set_lr(lr)
        b = eng.ctrl.numpy().tobytes()
        assert struct.unpack_from("<f", b, 8)[0] == np.float32(lr)
        assert struct.unpack_from("<f", b, 68)[0] == np.float32(1.0 - lr * 0.05)    # in double, rounded once
    # without decay the word stays 0 and set_lr leaves it alone
    eng = _host_engine(0.01, 0.0)
    eng.set_lr(0.5)
    assert struct.unpack_from("<f", eng.ctrl.numpy().tobytes(), 68)[0] == 0.0


# ---------------------------------------------------------------------------------------------------- role path
def _master(tmp_path, wd=0.05, resume=False):
    return role_master(tmp_path, learning_rate=0.01, optimizer="adamw", weight_decay=wd, resume=resume)


def test_role_path_update_is_adamw(tmp_path):
    m = _master(tmp_path)
    assert isinstance(m.optimizer, AdamW) and m.optimizer.param_groups[0]["weight_decay"] == 0.05
    params = [p.detach().clone() for p in m.network.parameters()]
    ref = AdamW(params, lr=0.01, weight_decay=0.05)
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


ROLE_FLAGS = ("--optimizer", "adamw", "--weight-decay", "0.05")


def test_gloo_role_path_trains_and_resumes_adamw(tmp_path):
    d = str(tmp_path) + "/"
    role_run(d, 29581, 3, *ROLE_FLAGS)
    out = role_run(d, 29582, 5, *ROLE_FLAGS, "--resume", "1")
    assert "Master: Step: 5" in out and "Master: Step: 1," not in out
    load = lambda s: torch.load(d + "model_step_%d_optim" % s, map_location="cpu", weights_only=False)
    for s in range(1, 6):
        opt = load(s)["optimizer"]
        assert opt["param_groups"][0]["weight_decay"] == 0.05
        assert all(st["step"] == s for st in opt["state"].values())       # the resumed run kept counting
    # the weights of step 4 follow from those of step 3 by one AdamW step from the saved moments: with the moments of
    # step 4 known, the decay and the step size are checked exactly where the gradient drops out (m4 = b1 m3 + ...)
    m3, m4 = (torch.load(d + "model_step_%d" % s, map_location="cpu") for s in (3, 4))
    o3, o4 = load(3)["optimizer"], load(4)["optimizer"]
    names = list(m3.keys())
    net = M.build_model("LeNet", 10, "MNIST")
    pnames = [n for n, _ in net.named_parameters()]
    for i, n in enumerate(pnames):
        p = m3[n].double()
        s4 = o4["state"][i]
        bc1, sbc2 = 1 - 0.9 ** 4, (1 - 0.999 ** 4) ** 0.5
        if p.dim() >= 2:
            p = p * (1 - 0.01 * 0.05)
        p = p - 0.01 / bc1 * s4["exp_avg"].double() / (s4["exp_avg_sq"].double().sqrt() / sbc2 + 1e-8)
        assert torch.allclose(p, m4[n].double(), rtol=1e-5, atol=1e-6), n
    assert set(pnames) <= set(names) and o3["state"][0]["step"] == 3

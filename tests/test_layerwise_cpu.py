"""LARS and LAMB without a GPU: the ``optim/`` classes against a hand-written numpy fp64 step, the refusals of the
engine and the launcher, the ``Ctrl2`` packing, a gloo role-path run with ``--optimizer lamb`` and the launcher loop
with the new flags on a stand-in engine."""
import argparse
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

from atomo_b200.ops import plan2 as P2
from atomo_b200.optim import LAMB, LARS
from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils.flags import add_fit_args

from shadow_harness import SVD3, StandInEngine, fit_args, forbid_cuda

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ratio(num, den, wn):
    return num / den if wn > 0 and den > 0 else 1.0


def _np_lars(ws, gs, ms, lr, mu, wd, eta, first):
    out_w, out_m = [], []
    for w, g, m in zip(ws, gs, ms):
        if w.ndim >= 2:
            wn, gn = np.sqrt((w * w).sum()), np.sqrt((g * g).sum())
            x = _ratio(eta * wn, gn + wd * wn, wn) * (g + wd * w)
        else:
            x = g
        m = x.copy() if first else mu * m + x
        out_w.append(w - lr * m)
        out_m.append(m)
    return out_w, out_m


def _np_lamb(ws, gs, ms, vs, t, lr, wd, b1=0.9, b2=0.999, eps=1e-8):
    out = []
    for w, g, m, v in zip(ws, gs, ms, vs):
        m = b1 * m + (1 - b1) * g
        v = b2 * v + (1 - b2) * g * g
        a = (m / (1 - b1 ** t)) / (np.sqrt(v) / np.sqrt(1 - b2 ** t) + eps)
        if w.ndim >= 2:
            u = a + wd * w
            wn, un = np.sqrt((w * w).sum()), np.sqrt((u * u).sum())
            w = w - lr * _ratio(wn, un, wn) * u
        else:
            w = w - lr * a
        out.append((w, m, v))
    return out


def _tensors(seed, zero_w=False, zero_g=False):
    rng = np.random.default_rng(seed)
    shapes = [(4, 3, 3, 3), (10, 6), (6,)]
    ws = [rng.standard_normal(s) for s in shapes]
    gs = [rng.standard_normal(s) * 0.1 for s in shapes]
    if zero_w:
        ws[0][:] = 0
    if zero_g:
        gs[1][:] = 0
    return ws, gs


@pytest.mark.parametrize("zero_w,zero_g", [(False, False), (True, False), (False, True)])
def test_lars_matches_numpy(zero_w, zero_g):
    ws, gs0 = _tensors(1, zero_w, zero_g)
    ps = [torch.nn.Parameter(torch.tensor(w)) for w in ws]
    o = LARS(ps, lr=0.3, momentum=0.9, weight_decay=0.0 if zero_g else 1e-3, trust_coefficient=0.01)
    nw, nm = [w.copy() for w in ws], [np.zeros_like(w) for w in ws]
    for k in range(3):
        gs = [g * (k + 1) for g in gs0]
        o.step([torch.tensor(g) for g in gs])
        nw, nm = _np_lars(nw, gs, nm, 0.3, 0.9, 0.0 if zero_g else 1e-3, 0.01, k == 0)
        for p, w in zip(ps, nw):
            assert p.dtype == torch.float64 and np.allclose(p.detach().numpy(), w, rtol=1e-13, atol=1e-15)
        if zero_w and k == 0:        # ||w|| = 0 before the first step
            assert o.state[ps[0]]["ratio"] == 1.0
    assert all(np.isfinite(p.detach().numpy()).all() for p in ps)
    if zero_g:
        assert o.state[ps[1]]["ratio"] == 1.0


@pytest.mark.parametrize("zero_w,zero_g", [(False, False), (True, False), (False, True)])
def test_lamb_matches_numpy(zero_w, zero_g):
    ws, gs0 = _tensors(2, zero_w, zero_g)
    ps = [torch.nn.Parameter(torch.tensor(w)) for w in ws]
    wd = 0.0 if zero_g else 0.01
    o = LAMB(ps, lr=0.01, weight_decay=wd)
    st = [(w.copy(), np.zeros_like(w), np.zeros_like(w)) for w in ws]
    for k in range(3):
        gs = [g * (k + 1) for g in gs0]
        o.step([torch.tensor(g) for g in gs])
        st = _np_lamb([s[0] for s in st], gs, [s[1] for s in st], [s[2] for s in st], k + 1, 0.01, wd)
        for p, s in zip(ps, st):
            assert np.allclose(p.detach().numpy(), s[0], rtol=1e-13, atol=1e-15)
    assert all(np.isfinite(p.detach().numpy()).all() for p in ps)
    if zero_g:       # u = 0 (m = 0 and no weight decay): ratio 1, no NaN
        assert o.state[ps[1]]["ratio"] == 1.0


def test_optimizers_refuse_what_they_do_not_define():
    p = [torch.nn.Parameter(torch.zeros(2, 2))]
    with pytest.raises(ValueError, match="nesterov"):
        LARS(p, momentum=0.9, nesterov=True)
    with pytest.raises(ValueError, match="dampening"):
        LARS(p, momentum=0.9, dampening=0.1)
    with pytest.raises(ValueError, match="AMSGrad"):
        LAMB(p, amsgrad=True)


@pytest.mark.parametrize("kw,match", [(dict(optimizer="lars", momentum=0.9, nesterov=True), "nesterov"),
                                      (dict(optimizer="lars", dampening=0.5), "dampening"),
                                      (dict(optimizer="lars", trust_coefficient=0.0), "trust_coefficient"),
                                      (dict(optimizer="lamb", amsgrad=True), "AMSGrad"),
                                      (dict(optimizer="rmsprop"), "optimizers")])
def test_engine_refuses_before_cuda_work(kw, match, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    forbid_cuda(monkeypatch)
    with pytest.raises(ValueError, match=match):
        S.ShadowEngine(None, 0, 1, **kw)


def test_flags_parse():
    a = add_fit_args(argparse.ArgumentParser(), ["--optimizer", "lars", "--trust-coefficient", "0.02"])
    assert a.optimizer == "lars" and a.trust_coefficient == 0.02
    assert add_fit_args(argparse.ArgumentParser(), []).trust_coefficient == 0.001


@pytest.mark.parametrize("opt", ["lars", "lamb"])
def test_fp32_flat_engine_refuses(opt, tmp_path):
    model = torch.nn.Linear(4, 4)
    for extra in (("--engine", "fused", "--dtype", "bf16"), ("--dtype", "fp32"),
                  ("--dtype", "bf16", "--code", "entrywise")):        # auto sends these to the fp32-flat engine
        with pytest.raises(SystemExit, match="--engine shadow"):
            L._build_engine(fit_args(tmp_path, *SVD3, "--optimizer", opt, *extra), model, 0, 1)


def test_ctrl2_packing_keeps_every_offset():
    assert struct.calcsize(P2.CTRL2_FMT) == P2.CTRL2_BYTES == 72
    b = P2.pack_ctrl2(step=5, lr=0.25, momentum=0.9, opt=P2.OPT_LAMB, num_aggregate=3, trust_coefficient=0.125)
    assert struct.unpack_from("<i", b, 0)[0] == 5 and struct.unpack_from("<f", b, 8)[0] == 0.25
    assert struct.unpack_from("<ii", b, 56) == (P2.OPT_LAMB, 3)         # opt, num_aggregate where they were
    assert struct.unpack_from("<f", b, 64)[0] == 0.125                  # the former pad1
    assert struct.unpack_from("<i", b, 68)[0] == 0
    # with trust_coefficient 0 the bytes are those of the former layout
    assert P2.pack_ctrl2(opt=P2.OPT_ADAM) == struct.pack("<iiffffiiQffffiiii", 1, 0, 0.01, 0.0, 0.0, 0.0, 0, 1, 1,
                                                         0.9, 0.999, 1e-8, 0.0, 1, 0, 0, 0)
    assert (P2.OPT_LARS, P2.OPT_LAMB) == (3, 4)


def test_layerwise_tables():
    shapes = [(8, 3, 3, 3), (8,), (8,), (16, 8, 3, 3), (16,), (10, 16), (10,)]
    pl = P2.build_plan2(shapes, "svd", 3, n_owners=2, n_groups=2)
    tile_layer, per_group = P2.layerwise_tables(pl)
    assert len(tile_layer) == len(pl.ps_tiles) and sum(per_group) == 3
    for (ui, _a, _b, _o), l in zip(pl.ps_tiles, tile_layer):
        u = pl.units[ui]
        assert (l == -1) == (u.kind == P2.KIND_VEC)
        if l >= 0:
            q = pl.params[u.param]
            ws = [p.index for p in pl.params if p.is_w and p.group == q.group]
            assert ws[l] == q.index


def test_gloo_role_path_trains_with_lamb(tmp_path):
    d = str(tmp_path) + "/"
    cmd = [sys.executable, "-m", "atomo_b200.distributed_nn", "--synthetic", "1", "--train-len", "512",
           "--test-len", "128", "--batch-size", "32", "--lr", "0.01", "--test-batch-size", "64", "--nproc", "2",
           "--network", "LeNet", "--dataset", "MNIST", "--code", "sgd", "--optimizer", "lamb", "--max-steps", "6",
           "--eval-freq", "3", "--train-dir", d, "--master-port", "29547"]
    env = dict(os.environ, ATOMO_HANG_DUMP_S="400", PYTHONPATH=ROOT, OMP_NUM_THREADS="2", MKL_NUM_THREADS="2")
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=420)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "Master: Step: 6" in r.stdout and os.path.isfile(d + "model_step_6")


def test_launcher_loop_with_the_new_flags(tmp_path, monkeypatch, capsys):
    StandInEngine.instances.clear()
    monkeypatch.setattr(L, "_build_engine", lambda args, model, rank, world: (StandInEngine(model, args), "shadow"))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    L.run_p2p_training(fit_args(tmp_path, *SVD3, "--max-steps", "4", "--optimizer", "lars", "--trust-coefficient", "0.02",
                             "--dtype", "bf16"), device="cpu")
    eng = StandInEngine.instances[-1]
    assert eng.args.optimizer == "lars" and eng.args.trust_coefficient == 0.02 and eng.step == 5
    assert sum(l.startswith("Worker: 0, Step:") for l in capsys.readouterr().out.splitlines()) >= 2

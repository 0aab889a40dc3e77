"""Signum with majority vote on the bf16 engine (``code="signum"``, csrc/v2_signum.cu) on one H100: the encode and the
vote against the ``codings.signum`` oracle bit for bit through the loopback harness (virtual workers and owners), and
the engine end to end: graph replay, reruns, ``set_lr``, resume, weight decay, gradient accumulation, the weight
average, the launcher and training."""
import argparse
import json
import math

import numpy as np
import pytest
import torch

from atomo_b200.codings import signum as S
from atomo_b200.utils.flags import add_fit_args

from shadow_harness import HSG, NAN, SIGNUM_SHAPES, ZERO, Linear, SignumOracle, ef_grads, run_mp, signum_check_ps, \
    signum_check_push, train


def _run(h, steps, special=False, pushers=None, coin=False, negate=None):
    o = SignumOracle(h)
    if coin:
        h.ps_tail = (0, 0)          # the owners draw the vectors' coins from Philox too
    for s in range(1, steps + 1):
        h.set_step(s)
        ws = pushers(s) if pushers else list(range(h.W))
        phys = {}
        for w in ws:
            phys[w] = h.fill(w, 1000 * s + w, special=special, who=w)
            if negate is not None and w == negate[0]:           # this worker pushes the negated bits of another
                src = negate[1]
                h.wgrads[w] = [-t for t in h.wgrads[src]]
                h.vgrads[w].copy_(-h.vgrads[src])
                phys[w] = {k: -v for k, v in phys[src].items()}
            o.push(w, phys[w], coin)
            h.encode(w, coin)
            signum_check_push(h, o, w)
        h.ps()
        o.ps(ws, coin)
        signum_check_ps(h, o)
    return h, o


# ---------------------------------------------------------------------------------------------------- kernels
@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("owners", [1, 2])
@pytest.mark.parametrize("groups", [1, 3])
@pytest.mark.parametrize("beta", [0.0, 0.9])
def test_encode_and_vote_match_oracle_bitwise(W, owners, groups, beta):
    h = HSG(SIGNUM_SHAPES[:10], W=W, beta=beta, n_groups=groups, n_owners=owners, seed=W + 10 * owners)
    _run(h, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("W,beta", [(2, 0.0), (4, 0.9), (3, 0.9)])
def test_designed_zeros_ties_nan_and_tails(W, beta):
    h = HSG(SIGNUM_SHAPES, W=W, beta=beta, n_owners=2, n_groups=2)
    init = h.master.cpu().numpy().copy()
    _, o = _run(h, 3, special=True)
    # the NaN of worker 0 makes its tile's vote NaN on every step; its momentum keeps it with beta > 0
    q = h.plan.params[NAN]
    assert np.isnan(o.master[q.off:q.off + 4096]).all() and np.isfinite(o.master[q.off + 4096:q.off + q.numel]).all()
    z = h.plan.params[ZERO]
    d = o.master[z.off:z.off + z.numel] - init[z.off:z.off + z.numel]
    assert (d > 0).any() and (d < 0).any()     # all-zero gradients vote by the coins, not all one way


@pytest.mark.gpu
@pytest.mark.parametrize("beta", [0.0, 0.9])
def test_philox_coin_matches_oracle(beta):
    h = HSG(SIGNUM_SHAPES, W=3, beta=beta, n_owners=2)
    _run(h, 2, special=True, coin=True)


@pytest.mark.gpu
def test_nonfinite_vector_makes_its_tile_nan():
    h = HSG(SIGNUM_SHAPES[:10], W=3, beta=0.0)
    o = SignumOracle(h)
    h.set_step(1)
    q = h.plan.params[1]
    for w in range(3):
        phys = h.fill(w, 7 + w)
        if w == 1:
            h.vgrads[w][q.off + 3] = float("inf")
            phys[1] = h.vgrads[w][q.off:q.off + q.numel].clone()
        o.push(w, phys)
        h.encode(w)
    h.ps()
    o.ps([0, 1, 2])
    signum_check_ps(h, o)
    v = h.vparams.cpu().numpy()
    assert np.isnan(v[q.off:q.off + q.numel]).all() and np.isfinite(v[h.plan.params[4].off]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("beta", [0.0, 0.9])
def test_num_aggregate_counts_only_fresh_workers(beta):
    """W = 3, --num-aggregate 2: worker 2 pushes at step 1 only, then goes stale; the owners vote with 0 and 1."""
    h = HSG(SIGNUM_SHAPES[:10], W=3, beta=beta, num_aggregate=2, n_owners=2)
    _run(h, 3, pushers=lambda s: [0, 1, 2] if s == 1 else [0, 1])


@pytest.mark.gpu
def test_one_negated_worker_cannot_move_a_three_of_four_majority():
    h = HSG(SIGNUM_SHAPES[:10], W=5, beta=0.0)
    before = h.master.cpu().numpy().copy()
    _, o = _run(h, 1, negate=(4, 0))
    x = np.stack([o.x[w] for w in range(4)])
    neg = (x < 0).sum(axis=0)
    pos = (x > 0).sum(axis=0)
    strong = (neg >= 3) | (pos >= 3)
    used = np.zeros_like(strong)
    for q in h.plan.params:
        if q.is_w:
            used[q.off:q.off + q.numel] = True
    sel = strong & used
    want = np.where(pos[sel] >= 3, -1.0, 1.0).astype(np.float32) * np.float32(0.0625)
    assert np.array_equal(o.master[sel], (before[sel] + want).astype(np.float32))
    assert np.array_equal(h.master.cpu().numpy()[sel], o.master[sel])


# ---------------------------------------------------------------------------------------------------- engine
def _linear_engine(grads, beta=0.9, **kw):
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.cuda.set_device(0)
    eng = ShadowEngine(Linear(grads), 0, 1, code="signum", lr=0.0625, momentum=beta, use_graph=kw.pop("graph", False),
                       overlap=False, criterion=lambda lg, y: lg[0, 0], seed=5, **kw)
    x, y = torch.zeros(4, 2), torch.zeros(4, dtype=torch.long)
    eng.prepare(x, y, warmup=0)
    return eng, x, y


def _linear_oracle(eng, grads, steps, beta, lr=0.0625, wd=0.0, ema=0.0):
    """numpy Signum of a single worker fed fixed gradients: master, vparams (and their average)."""
    pl = eng.plan
    m, v = eng.gather_fp32("master").cpu().numpy().copy(), eng.vparams.cpu().numpy().copy()
    e, ev = m.copy(), v.copy()
    u, uv = np.zeros_like(m), np.zeros_like(v)
    g, gv = np.zeros_like(m), np.zeros_like(v)
    for q in pl.params:
        t = grads[q.index].float()
        t = (t.permute(0, 2, 3, 1) if t.dim() == 4 else t).reshape(-1).cpu().numpy()
        (g if q.is_w else gv)[q.off:q.off + q.numel] = t
    wmask = np.zeros(m.size, bool)
    for q in pl.params:
        if q.is_w:
            wmask[q.off:q.off + q.numel] = True
    f, w_ema = S.decay_factor(lr, wd), np.float32(1 - ema)
    for _ in range(steps):
        if beta > 0:
            u, uv = S.momentum_step(u, g, beta), S.momentum_step(uv, gv, beta)
            x, xv = u, uv
        else:
            x, xv = g, gv
        assert (S.classify(x[wmask]) < 2).all() and (S.classify(xv) < 2).all()   # no coins in this oracle
        if wd:
            m = np.where(wmask, (m * f).astype(np.float32), m)
        m = np.where(wmask, S.step(m, np.where(x < 0, -1.0, 1.0), lr), m)
        vv = np.zeros(v.size, bool)
        for q in pl.params:
            if not q.is_w:
                vv[q.off:q.off + q.numel] = True
        v = np.where(vv, S.step(v, np.where(xv < 0, -1.0, 1.0), lr), v)
        if ema:
            e = (e + w_ema * (m - e)).astype(np.float32)
            ev = (ev + w_ema * (v - ev)).astype(np.float32)
    return m, v, e, ev, wmask


@pytest.mark.gpu
@pytest.mark.parametrize("beta", [0.0, 0.9])
@pytest.mark.parametrize("kw", [{}, {"accumulate_steps": 2}, {"ema_decay": 0.75}, {"weight_decay": 0.5}])
def test_engine_matches_oracle(beta, kw):
    grads = ef_grads(3)
    eng, x, y = _linear_engine(grads, beta, **kw)
    want = _linear_oracle(eng, grads, 4, beta, wd=kw.get("weight_decay", 0.0), ema=kw.get("ema_decay", 0.0))
    for _ in range(4):
        eng.train_step(x, y)
    torch.cuda.synchronize()
    assert eng.error_code() == 0
    m, v, e, ev, wmask = want
    assert np.array_equal(eng.gather_fp32("master").cpu().numpy()[wmask], m[wmask])
    assert np.array_equal(eng.vparams.cpu().numpy(), v)
    if kw.get("ema_decay"):
        assert np.array_equal(eng.gather_fp32("ema").cpu().numpy()[wmask], e[wmask])
        assert np.array_equal(eng.gather_fp32("vema").cpu().numpy(), ev)
    assert (eng.mc_mom is None) == (beta == 0)
    eng.close()


@pytest.mark.gpu
def test_beta_zero_allocates_no_momentum():
    eng, x, y = _linear_engine(ef_grads(1), 0.0)
    assert eng.mc_mom is None and eng.mc_vmom is None
    with pytest.raises(RuntimeError):
        eng.momentum_correction_norm()
    eng.close()
    eng, x, y = _linear_engine(ef_grads(1), 0.9)
    eng.train_step(x, y)
    assert eng.momentum_correction_norm()["model"] > 0
    eng.close()


@pytest.mark.gpu
def test_weight_decay_equals_torch_mul():
    grads = ef_grads(4)
    a, x, y = _linear_engine(grads, 0.9, weight_decay=0.25)
    b, _, _ = _linear_engine(grads, 0.9)
    a.train_step(x, y)
    f = np.float32(1.0 - 0.0625 * 0.25)
    wmask = torch.zeros_like(b.master, dtype=torch.bool)
    for q in b.plan.params:
        if q.is_w:
            wmask[q.off:q.off + q.numel] = True
    b.master.copy_(torch.where(wmask, b.master.mul(float(f)), b.master))
    b.train_step(x, y)
    torch.cuda.synchronize()
    assert torch.equal(a.master, b.master) and torch.equal(a.vparams, b.vparams)
    a.close()
    b.close()


def _train(net, graph, steps=6):
    """``steps`` steps of ``shadow_harness.train`` (momentum 0.9 on the workers, no error feedback)."""
    return train(net, graph, False, steps=steps, lr=1e-3, code="signum")


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["ResNet18", "VGG11"])
def test_graph_replay_equals_eager_and_reruns(net, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    mg, lg, _ = _train(net, True)
    me, le, _ = _train(net, False)
    assert torch.equal(mg, me) and lg == le
    mg2, _, _ = _train(net, True)
    assert torch.equal(mg, mg2)


def _engine(net, graph, **kw):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model, input_shape
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    x, y = SyntheticImageDataset(input_shape(net), 10, 4096, seed=0).materialize(32)
    eng = ShadowEngine(build_model(net, 10), 0, 1, code="signum", lr=1e-3, momentum=kw.pop("momentum", 0.9),
                       use_graph=graph, overlap=graph, seed=3, **kw)
    eng.prepare(x.pin_memory(), y.pin_memory(), warmup=1)
    return eng, x, y


@pytest.mark.gpu
def test_set_lr_between_replays_as_in_eager(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    out = []
    for graph in (True, False):
        eng, x, y = _engine("ResNet18", graph, weight_decay=1e-2)
        for i in range(4):
            eng.set_lr([1e-3, 5e-4, 2e-3, 1e-4][i])
            eng.train_step(x, y)
        torch.cuda.synchronize()
        assert eng.error_code() == 0
        out.append(eng.gather_fp32("master").clone())
        eng.close()
    assert torch.equal(out[0], out[1])


@pytest.mark.gpu
def test_resume_is_bitwise(tmp_path, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    a, x, y = _engine("ResNet18", False, weight_decay=1e-3)
    for _ in range(3):
        a.train_step(x, y)
    k = a.step - 1
    path = a.save_checkpoint(str(tmp_path) + "/")
    side = torch.load(path + "_optim", weights_only=False)
    assert side["code"] == "signum" and side["signum_momentum"] == 0.9
    for _ in range(3):
        a.train_step(x, y)
    want, want_u = a.gather_fp32("master").clone(), a.mc_mom.clone()
    a.close()
    b, _, _ = _engine("ResNet18", False, weight_decay=1e-3)
    b.load_checkpoint(str(tmp_path) + "/", k)
    for _ in range(3):
        b.train_step(x, y)
    torch.cuda.synchronize()
    assert b.error_code() == 0
    assert torch.equal(b.gather_fp32("master"), want) and torch.equal(b.mc_mom, want_u)
    b.close()


@pytest.mark.gpu
def test_launcher_runs_signum_with_gpu_data(tmp_path, monkeypatch):
    from atomo_b200.runtime import p2p_launcher as L
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    args = add_fit_args(argparse.ArgumentParser(), [
        "--network", "ResNet18", "--dataset", "Cifar10", "--synthetic", "1", "--train-len", "512", "--test-len", "64",
        "--batch-size", "32", "--test-batch-size", "64", "--backend", "p2p", "--dtype", "bf16", "--max-steps", "6",
        "--log-interval", "2", "--eval-freq", "100", "--train-dir", str(tmp_path) + "/", "--gpu-data", "1",
        "--metrics-file", str(tmp_path / "m"), "--code", "signum", "--momentum", "0.9", "--lr", "0.001"])
    L.run_p2p_training(args)
    recs = [json.loads(l) for l in open(str(tmp_path / "m") + ".rank0.jsonl")]
    assert recs and all(math.isfinite(r["loss"]) and r["mom_norm"] > 0 for r in recs)


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["ResNet18", "LeNet"])
def test_loss_falls_within_100_steps(net):
    _, losses, _ = train(net, True, False, steps=100, lr=1e-3, code="signum")
    assert all(math.isfinite(v) for v in losses)
    assert sum(losses[-10:]) / 10 < 0.8 * losses[0], losses


@pytest.mark.gpu
@pytest.mark.multigpu
def test_multi_gpu_replicas_identical():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    res = run_mp(2, {"code": "signum", "ps_mode": "sharded", "net": "VGG11"}, 29830)
    for rank, err, same, l0, l1, mode, mc, _ in res:
        assert err == 0 and same, res

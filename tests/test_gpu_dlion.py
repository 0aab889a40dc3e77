"""Distributed Lion on the bf16 engine (``code="dlion"``, csrc/v2_signum.cu) on one H100: the encode and the vote / mean
against the ``codings.dlion`` oracle bit for bit through Signum's loopback harness (virtual workers and owners), the
cross-check against ``code="signum"``, and the engine end to end: graph replay, reruns, ``set_lr``, resume, weight
decay, gradient accumulation, the weight average, the launcher and training."""
import argparse
import json
import math

import numpy as np
import pytest
import torch

from atomo_b200.codings import dlion as D
from atomo_b200.codings import signum as S
from atomo_b200.ops import plan2 as P
from atomo_b200.utils.flags import add_fit_args

from shadow_harness import HSG, NAN, SIGNUM_SHAPES, ZERO, Linear, SignumOracle, ef_grads, run_mp, signum_check_ps, \
    signum_check_push, train

BETAS = [(0.0, 0.99), (0.9, 0.99), (0.95, 0.98)]


class HDL(HSG):
    """Distributed Lion: Signum's harness with Lion's worker rule (b1, b2) and the owners' vote or mean."""

    def __init__(self, shapes, betas=(0.9, 0.99), agg="vote", **kw):
        super().__init__(shapes, beta=betas[0], **kw)
        self.betas, self.agg = betas, agg
        self.ps_tail = self.ps_tail + (agg == "mean",)

    def encode(self, w, coin=False):
        C, pl = self.C, self.plan
        gptr = self.gptr(w)
        for g in range(pl.n_groups):
            t0, nt = pl.enc_range[g]
            v0, nv = self.vec_range[g]
            if self.beta == 0:
                nv = 0
            C.v2_dlion_encode(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr,
                              self.t_vchunks.data_ptr() + 24 * v0, nv, self.vgrads[w].data_ptr(),
                              self.wmom[w].data_ptr() if self.wmom else 0,
                              self.vmom_w[w].data_ptr() if self.vmom_w else 0, self.betas[0], self.betas[1],
                              self.t_arena_peer.data_ptr(), self.t_sig_peer.data_ptr(), self.n_owners,
                              pl.arena_floats, w, g, self.ctrl.data_ptr(), self.counter(g), 0,
                              g == pl.n_groups - 1, 0 if coin else self.unif[w].data_ptr())
        torch.cuda.synchronize()


class DOracle(SignumOracle):
    """Signum's oracle with the Lion worker step (``u`` holds m, ``x`` the pushed direction c) and the aggregate."""

    def push(self, w, phys, coin=False):
        pl, (b1, b2) = self.plan, self.h.betas
        x, xv = np.zeros(pl.w_total, np.float32), np.zeros(pl.v_total, np.float32)
        for q in pl.params:
            g = phys[q.index].cpu().numpy().astype(np.float32)
            sl = slice(q.off, q.off + q.numel)
            st, dst = (self.u[w], x) if q.is_w else (self.uv[w], xv)
            if b1 > 0:
                dst[sl], st[sl] = D.worker_step(st[sl], g, b1, b2)
            else:
                dst[sl] = g
        self.x[w], self.xv[w] = x, xv
        if coin:
            self.unif[w] = np.zeros(pl.w_total, np.float32)
            for u in pl.units:
                if u.kind == P.KIND_SIGNUM:
                    self.unif[w][u.w_off:u.w_off + u.numel] = S.coin_uniforms(self.h.seed, u.index,
                                                                               np.arange(u.numel), self.h.step, w)

    def ps(self, counted, coin=False):
        pl, lr = self.plan, np.float32(self.h_lr())
        for (ui, a, b, o) in pl.ps_tiles:
            u = pl.units[ui]
            rows, bad = [], []
            for w in counted:
                r, nf = self.vec_bits(w, u, a, b, coin) if u.kind == P.KIND_VEC else self.tile_bits(w, u, a, b)
                rows.append(r)
                bad.append(nf)
            v = D.aggregate(self.h.agg, rows, b, bad)
            dst = self.vparams if u.kind == P.KIND_VEC else self.master
            dst[u.w_off + a:u.w_off + a + b] = D.step(dst[u.w_off + a:u.w_off + a + b], v, lr)


def _run(h, steps, special=False, pushers=None, coin=False):
    o = DOracle(h)
    if coin:
        h.ps_tail = (0, 0, h.agg == "mean")      # the owners draw the vectors' coins from Philox too
    for s in range(1, steps + 1):
        h.set_step(s)
        ws = pushers(s) if pushers else list(range(h.W))
        for w in ws:
            phys = h.fill(w, 1000 * s + w, special=special, who=w)
            o.push(w, phys, coin)
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
@pytest.mark.parametrize("betas", BETAS)
@pytest.mark.parametrize("agg", ["vote", "mean"])
def test_encode_and_aggregate_match_oracle_bitwise(W, owners, groups, betas, agg):
    h = HDL(SIGNUM_SHAPES[:10], betas=betas, agg=agg, W=W, n_groups=groups, n_owners=owners, seed=W + 10 * owners)
    _run(h, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("W,betas", [(2, (0.0, 0.99)), (4, (0.9, 0.99)), (3, (0.95, 0.98))])
@pytest.mark.parametrize("agg", ["vote", "mean"])
def test_designed_zeros_ties_nan_and_tails(W, betas, agg):
    h = HDL(SIGNUM_SHAPES, betas=betas, agg=agg, W=W, n_owners=2, n_groups=2)
    init = h.master.cpu().numpy().copy()
    _, o = _run(h, 3, special=True)
    # the NaN of worker 0 makes its tile NaN under either aggregate, on every step
    q = h.plan.params[NAN]
    assert np.isnan(o.master[q.off:q.off + 4096]).all() and np.isfinite(o.master[q.off + 4096:q.off + q.numel]).all()
    z = h.plan.params[ZERO]
    d = o.master[z.off:z.off + z.numel] - init[z.off:z.off + z.numel]
    assert (d > 0).any() and (d < 0).any()     # all-zero gradients move by the coins, not all one way


@pytest.mark.gpu
@pytest.mark.parametrize("agg", ["vote", "mean"])
def test_even_w_ties_step_zero(agg):
    """W = 2, worker 1 pushes the negated gradient of worker 0 (b1 == 0): every nonzero element ties and stays."""
    h = HDL(SIGNUM_SHAPES[:10], betas=(0.0, 0.99), agg=agg, W=2)
    before = h.master.cpu().numpy().copy()
    o = DOracle(h)
    h.set_step(1)
    phys0 = h.fill(0, 11)
    h.wgrads[1] = [-t for t in h.wgrads[0]]
    h.vgrads[1].copy_(-h.vgrads[0])
    for w, ph in ((0, phys0), (1, {k: -v for k, v in phys0.items()})):
        o.push(w, ph)
        h.encode(w)
        signum_check_push(h, o, w)
    h.ps()
    o.ps([0, 1])
    signum_check_ps(h, o)
    x = o.x[0]
    tie = np.zeros(x.size, bool)
    for q in h.plan.params:
        if q.is_w:
            tie[q.off:q.off + q.numel] = S.classify(x[q.off:q.off + q.numel]) < 2
    assert tie.sum() > 1000 and np.array_equal(h.master.cpu().numpy()[tie], before[tie])


@pytest.mark.gpu
@pytest.mark.parametrize("betas", [(0.0, 0.99), (0.9, 0.99)])
@pytest.mark.parametrize("agg", ["vote", "mean"])
def test_philox_coin_matches_oracle(betas, agg):
    h = HDL(SIGNUM_SHAPES, betas=betas, agg=agg, W=3, n_owners=2)
    _run(h, 2, special=True, coin=True)


@pytest.mark.gpu
@pytest.mark.parametrize("betas", [(0.0, 0.99), (0.9, 0.99)])
@pytest.mark.parametrize("agg", ["vote", "mean"])
def test_num_aggregate_counts_only_fresh_workers(betas, agg):
    """W = 3, --num-aggregate 2: worker 2 pushes at step 1 only, then goes stale; the owners count 0 and 1."""
    h = HDL(SIGNUM_SHAPES[:10], betas=betas, agg=agg, W=3, num_aggregate=2, n_owners=2)
    _run(h, 3, pushers=lambda s: [0, 1, 2] if s == 1 else [0, 1])


# ---------------------------------------------------------------------------------------------------- engine
def _linear_engine(grads, betas=(0.9, 0.99), agg="vote", **kw):
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.cuda.set_device(0)
    eng = ShadowEngine(Linear(grads), 0, 1, code="dlion", lr=0.0625, momentum=0.5, betas=betas, dlion_aggregate=agg,
                       use_graph=kw.pop("graph", False), overlap=False, criterion=lambda lg, y: lg[0, 0], seed=5, **kw)
    x, y = torch.zeros(4, 2), torch.zeros(4, dtype=torch.long)
    eng.prepare(x, y, warmup=0)
    return eng, x, y


def _linear_oracle(eng, grads, steps, betas, lr=0.0625, wd=0.0, ema=0.0):
    """numpy Distributed Lion of a single worker fed fixed gradients: master, vparams (and their average)."""
    pl = eng.plan
    m, v = eng.gather_fp32("master").cpu().numpy().copy(), eng.vparams.cpu().numpy().copy()
    e, ev = m.copy(), v.copy()
    u, uv = np.zeros_like(m), np.zeros_like(v)
    g, gv = np.zeros_like(m), np.zeros_like(v)
    for q in pl.params:
        t = grads[q.index].float()
        t = (t.permute(0, 2, 3, 1) if t.dim() == 4 else t).reshape(-1).cpu().numpy()
        (g if q.is_w else gv)[q.off:q.off + q.numel] = t
    wmask, vmask = np.zeros(m.size, bool), np.zeros(v.size, bool)
    for q in pl.params:
        (wmask if q.is_w else vmask)[q.off:q.off + q.numel] = True
    f, w_ema = S.decay_factor(lr, wd), np.float32(1 - ema)
    for _ in range(steps):
        if betas[0] > 0:
            x, u = D.worker_step(u, g, *betas)
            xv, uv = D.worker_step(uv, gv, *betas)
        else:
            x, xv = g, gv
        assert (S.classify(x[wmask]) < 2).all() and (S.classify(xv) < 2).all()   # no coins in this oracle
        if wd:
            m = np.where(wmask, (m * f).astype(np.float32), m)
        m = np.where(wmask, D.step(m, np.where(x < 0, -1.0, 1.0), lr), m)
        v = np.where(vmask, D.step(v, np.where(xv < 0, -1.0, 1.0), lr), v)
        if ema:
            e = (e + w_ema * (m - e)).astype(np.float32)
            ev = (ev + w_ema * (v - ev)).astype(np.float32)
    return m, v, e, ev, wmask, u


@pytest.mark.gpu
@pytest.mark.parametrize("betas", BETAS)
@pytest.mark.parametrize("agg", ["vote", "mean"])
@pytest.mark.parametrize("kw", [{}, {"accumulate_steps": 2}, {"ema_decay": 0.75}, {"weight_decay": 0.5}])
def test_engine_matches_oracle(betas, agg, kw):
    grads = ef_grads(3)
    eng, x, y = _linear_engine(grads, betas, agg, **kw)
    assert eng.plan.code == "signum"
    want = _linear_oracle(eng, grads, 4, betas, wd=kw.get("weight_decay", 0.0), ema=kw.get("ema_decay", 0.0))
    for _ in range(4):
        eng.train_step(x, y)
    torch.cuda.synchronize()
    assert eng.error_code() == 0
    m, v, e, ev, wmask, u = want
    assert np.array_equal(eng.gather_fp32("master").cpu().numpy()[wmask], m[wmask])
    assert np.array_equal(eng.vparams.cpu().numpy(), v)
    if kw.get("ema_decay"):
        assert np.array_equal(eng.gather_fp32("ema").cpu().numpy()[wmask], e[wmask])
        assert np.array_equal(eng.gather_fp32("vema").cpu().numpy(), ev)
    assert (eng.mc_mom is None) == (betas[0] == 0)
    if betas[0] > 0:
        assert np.array_equal(eng.mc_mom.cpu().numpy()[wmask], u[wmask])
        assert eng.momentum_correction_norm()["model"] > 0
    else:
        with pytest.raises(RuntimeError):
            eng.momentum_correction_norm()
    eng.close()


def _engine(net, graph, **kw):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model, input_shape
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    x, y = SyntheticImageDataset(input_shape(net), 10, 4096, seed=0).materialize(32)
    kw.setdefault("code", "dlion")
    eng = ShadowEngine(build_model(net, 10), 0, 1, lr=1e-3, use_graph=graph, overlap=graph, seed=3, **kw)
    eng.prepare(x.pin_memory(), y.pin_memory(), warmup=1)
    return eng, x, y


def _steps(eng, x, y, n):
    for _ in range(n):
        eng.train_step(x, y)
    torch.cuda.synchronize()
    assert eng.error_code() == 0
    m = eng.gather_fp32("master").clone()
    eng.close()
    return m


@pytest.mark.gpu
def test_b1_zero_vote_equals_signum_momentum_zero_and_w1_mean_equals_vote(monkeypatch):
    """ResNet-18, graph replay: dlion with b1 = 0 and the vote is --code signum --momentum 0 bit for bit, and at
    W = 1 the mean equals the vote (with b1 = 0.9 too)."""
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    a = _steps(*_engine("ResNet18", True, betas=(0.0, 0.99), weight_decay=1e-2), 5)
    b = _steps(*_engine("ResNet18", True, code="signum", momentum=0.0, weight_decay=1e-2), 5)
    assert torch.equal(a, b)
    c = _steps(*_engine("ResNet18", True, betas=(0.0, 0.99), weight_decay=1e-2, dlion_aggregate="mean"), 5)
    assert torch.equal(a, c)
    d = _steps(*_engine("ResNet18", True, dlion_aggregate="vote"), 5)
    e = _steps(*_engine("ResNet18", True, dlion_aggregate="mean"), 5)
    assert torch.equal(d, e)


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["ResNet18", "VGG11"])
@pytest.mark.parametrize("agg", ["vote", "mean"])
def test_graph_replay_equals_eager_and_reruns(net, agg, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    mg, lg, _ = train(net, True, False, steps=6, lr=1e-3, code="dlion", dlion_aggregate=agg)
    me, le, _ = train(net, False, False, steps=6, lr=1e-3, code="dlion", dlion_aggregate=agg)
    assert torch.equal(mg, me) and lg == le
    mg2, _, _ = train(net, True, False, steps=6, lr=1e-3, code="dlion", dlion_aggregate=agg)
    assert torch.equal(mg, mg2)


@pytest.mark.gpu
def test_set_lr_between_replays_as_in_eager(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    out = []
    for graph in (True, False):
        eng, x, y = _engine("ResNet18", graph, weight_decay=1e-2, dlion_aggregate="mean")
        for i in range(4):
            eng.set_lr([1e-3, 5e-4, 2e-3, 1e-4][i])
            eng.train_step(x, y)
        torch.cuda.synchronize()
        assert eng.error_code() == 0
        out.append(eng.gather_fp32("master").clone())
        eng.close()
    assert torch.equal(out[0], out[1])


@pytest.mark.gpu
def test_resume_is_bitwise_and_other_betas_start_fresh(tmp_path, monkeypatch, capsys):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    a, x, y = _engine("ResNet18", False, weight_decay=1e-3, dlion_aggregate="mean")
    for _ in range(3):
        a.train_step(x, y)
    k = a.step - 1
    path = a.save_checkpoint(str(tmp_path) + "/")
    side = torch.load(path + "_optim", weights_only=False)
    assert side["code"] == "dlion" and tuple(side["dlion_betas"]) == (0.9, 0.99)
    assert side["dlion_aggregate"] == "mean" and side["weight_decay"] == 1e-3
    for _ in range(3):
        a.train_step(x, y)
    want, want_u = a.gather_fp32("master").clone(), a.mc_mom.clone()
    a.close()
    b, _, _ = _engine("ResNet18", False, weight_decay=1e-3, dlion_aggregate="mean")
    b.load_checkpoint(str(tmp_path) + "/", k)
    for _ in range(3):
        b.train_step(x, y)
    torch.cuda.synchronize()
    assert b.error_code() == 0
    assert torch.equal(b.gather_fp32("master"), want) and torch.equal(b.mc_mom, want_u)
    b.close()
    capsys.readouterr()
    c, _, _ = _engine("ResNet18", False, weight_decay=1e-3, betas=(0.95, 0.98))
    c.load_checkpoint(str(tmp_path) + "/", k)
    assert "not restored (dlion_betas)" in capsys.readouterr().out
    assert not c.mc_mom.any()
    c.close()


@pytest.mark.gpu
def test_launcher_runs_dlion_with_gpu_data(tmp_path, monkeypatch):
    from atomo_b200.runtime import p2p_launcher as L
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    args = add_fit_args(argparse.ArgumentParser(), [
        "--network", "ResNet18", "--dataset", "Cifar10", "--synthetic", "1", "--train-len", "512", "--test-len", "64",
        "--batch-size", "32", "--test-batch-size", "64", "--backend", "p2p", "--dtype", "bf16", "--max-steps", "6",
        "--log-interval", "2", "--eval-freq", "100", "--train-dir", str(tmp_path) + "/", "--gpu-data", "1",
        "--metrics-file", str(tmp_path / "m"), "--code", "dlion", "--dlion-aggregate", "mean", "--lr", "0.001"])
    L.run_p2p_training(args)
    recs = [json.loads(l) for l in open(str(tmp_path / "m") + ".rank0.jsonl")]
    assert recs and all(math.isfinite(r["loss"]) and r["mom_norm"] > 0 for r in recs)


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["ResNet18", "LeNet"])
@pytest.mark.parametrize("agg", ["vote", "mean"])
def test_loss_falls_within_100_steps(net, agg):
    _, losses, _ = train(net, True, False, steps=100, lr=1e-3, code="dlion", dlion_aggregate=agg)
    assert all(math.isfinite(v) for v in losses)
    assert sum(losses[-10:]) / 10 < 0.8 * losses[0], losses


@pytest.mark.gpu
@pytest.mark.multigpu
def test_multi_gpu_replicas_identical():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    res = run_mp(2, {"code": "dlion", "ps_mode": "sharded", "net": "VGG11"}, 29840)
    for rank, err, same, l0, l1, mode, mc, _ in res:
        assert err == 0 and same, res

"""Lion on the bf16 engine (``ShadowEngine(optimizer="lion")``): the Lion instantiation of every PS kernel
(``v2_ps_lion``), after the decay pass ``v2_decay`` of csrc/v2_ema.cu when ``weight_decay > 0``.

* Loopback, every PS family (slab and matrix units of svd, dense-16 tiles of the dense code and the stem, vector tiles,
  QSGD, TernGrad, entry-wise, top-k, sign, fp8, hadamard, PowerSGD): 2 virtual workers over 3 steps.  Per step the
  family's gather instantiation (``v2_ps_gather``) first stores the mean gradient ``g`` of the same pushes, exactly
  the value the Lion epilogue steps with; then ``optim/lion.py`` on ``g`` must give ``master``, ``mom``, ``vparams``,
  ``vmom`` and the broadcast bf16 copy bit for bit.  Zeroed gradients give elements with ``c == 0`` exactly; ``sq``
  and ``vsq`` keep a sentinel.  Also 2 owners (PowerSGD), 2 groups (svd) and ``num_aggregate=1`` of 2 (sign).
* Engine: a step with weight decay is bit for bit "torch ``master.mul_(f)``, then the Lion step without decay";
  eager = graph and run = rerun; ``set_lr`` between replays; ``accumulate_steps=2``; the weight average follows the
  Lion weights; top-k with error feedback; resume is bitwise (svd, top-k + EF); cross-optimizer loads are refused;
  the launcher trains, checkpoints and resumes.  The two-GPU test checks that two owners keep identical replicas.
"""
import functools

import numpy as np
import pytest
import torch

from atomo_b200.ops import plan2 as P2
from atomo_b200.optim import Lion

from shadow_harness import H2, HE, SHAPES, deterministic_cudnn, differs, engine_batch, make_engine, nccl_init, spawn, \
    state, step  # noqa: F401

LR, WD, BETAS = 1e-3, 0.1, (0.9, 0.99)
FAMILY = {"svd": 0, "sgd": 0, "qsgd": 1, "terngrad": 1, "entrywise": 2, "topk": 2, "sign": 3, "fp8": 4,
          "hadamard": 5, "powersgd": 6}
LOOP_SHAPES = SHAPES + [(10,)]
ZERO_SHAPES = ((7, 20), (32, 16, 3, 3))     # weight gradients zeroed in every push: c == 0 at every step


def _harness(code, W=2, **kw):
    if code in ("svd", "sgd"):
        return H2(LOOP_SHAPES, code=code, rank=3, W=W, **kw)
    if code in ("qsgd", "terngrad"):
        from test_gpu_shadow_qsgd import HQ
        return HQ(LOOP_SHAPES, code=code, q=4, bucket=512, W=W, **kw)
    if code == "entrywise":
        return HE(LOOP_SHAPES, 0.05, W=W, **kw)
    if code == "topk":
        from test_gpu_topk import HT
        return HT(LOOP_SHAPES, 0.05, W=W, **kw)
    if code == "sign":
        from test_gpu_sign import HS
        return HS(LOOP_SHAPES, 512, W=W, **kw)
    if code == "fp8":
        from test_gpu_fp8 import HF
        return HF(LOOP_SHAPES, 512, W=W, **kw)
    if code == "hadamard":
        from test_gpu_hadamard import HH
        return HH(LOOP_SHAPES, 4, 256, W=W, **kw)
    from test_gpu_powersgd import HP
    return HP(LOOP_SHAPES, 2, W=W, **kw)


def _tail(h):
    return (h.maxq, h.maxb) if hasattr(h, "maxq") else (0, 0)


def _launch(h, kind, grad, vgrad, part, grid=64):
    """Per group and owner: the gather launch (g into grad / vgrad), then the Lion launch on the same pushes."""
    C, pl = h.C, h.plan
    stage = h.t_stage_peer.data_ptr() if h.t_stage_peer is not None else 0
    for g in range(pl.n_groups):
        for o in range(h.n_owners):
            t0, nt = pl.ps_range[g][o]
            common = (h.arenas[o].data_ptr(), pl.arena_floats, h.sigs[o].data_ptr(), h.t_sig_own[o].data_ptr(),
                      h.ctrl.data_ptr(), h.counter(g, o), int(5e9), h.tstats.data_ptr(), 1.0 / h.W)
            C.v2_ps_gather(kind, h.t_units.data_ptr(), h.t_ps.data_ptr(), t0, nt, h.W, 1, g, o, 0,
                           h.t_vgrads_peer.data_ptr(), stage, *common, grad.data_ptr(), vgrad.data_ptr(),
                           part.data_ptr() + 8 * t0, grid, *_tail(h))
            C.v2_ps_lion(kind, h.t_units.data_ptr(), h.t_ps.data_ptr(), t0, nt, h.W, 1, g, g == pl.n_groups - 1, o,
                         h.master.data_ptr(), h.mom.data_ptr(), h.vmom.data_ptr(), 0, h.t_wshadow_peer.data_ptr(),
                         h.vparams.data_ptr(), 0, h.t_vparams_peer.data_ptr(), 0, h.t_vgrads_peer.data_ptr(), stage,
                         *common, grid, *_tail(h))
    torch.cuda.synchronize()


def _loopback(code, W=2, steps=3, pushers=None, **kw):
    h = _harness(code, W=W, **kw)
    kind = FAMILY[code]
    cv = h.ctrl.view(torch.float32)
    cv[10], cv[11] = BETAS                                    # Ctrl2 beta1 / beta2
    cv[2] = LR
    h.ctrl.view(torch.int32)[14] = P2.OPT_LION               # bookkeeping only: the Lion launch never reads it
    pl = h.plan
    for t in (h.sq, h.vsq, h.sqmax, h.vsqmax):
        t.fill_(7.0)
    grad, vgrad = h.zeros(pl.w_total), h.zeros(pl.v_total)
    part = h.zeros(2 * max(len(pl.ps_tiles), 1))
    zero = [q.widx for q in pl.params if q.is_w and tuple(q.shape) in ZERO_SHAPES]
    vec0 = next(q for q in pl.params if not q.is_w)
    # the oracle: optim/lion.py on the whole fp32 arrays (1-D, so no decay), with its own fp32 momenta
    ref_p, ref_v = h.master.clone(), h.vparams.clone()
    opt = Lion([ref_p, ref_v], lr=LR, betas=BETAS)
    mw, mv = h.used()
    czero_w = czero_v = 0
    for s in range(1, steps + 1):
        h.set_step(s)
        for w in (range(W) if pushers is None else pushers):
            h.fill(w, seed=100 * s + w)
            for k in zero:
                h.wgrads[w][k].zero_()
            h.vgrads[w][vec0.off:vec0.off + 8] = 0.0
            h.encode(w)
        _launch(h, kind, grad, vgrad, part)
        assert int(h.ctrl.view(torch.int32)[1]) == 0, "device error"
        st = opt.state
        mw_prev = st[ref_p]["exp_avg"] if ref_p in st else torch.zeros_like(ref_p)
        mv_prev = st[ref_v]["exp_avg"] if ref_v in st else torch.zeros_like(ref_v)
        b1, om1 = float(np.float32(BETAS[0])), float(np.float32(1) - np.float32(BETAS[0]))
        czero_w += int(((torch.add(mw_prev * b1, grad * om1) == 0) & mw).sum())
        czero_v += int(((torch.add(mv_prev * b1, vgrad * om1) == 0) & mv).sum())
        opt.step(grads=[grad.clone(), vgrad.clone()])
        assert torch.equal(h.master, ref_p), (code, s, "master")
        assert torch.equal(h.mom, opt.state[ref_p]["exp_avg"]), (code, s, "mom")
        assert torch.equal(h.vparams, ref_v), (code, s, "vparams")
        assert torch.equal(h.vmom, opt.state[ref_v]["exp_avg"]), (code, s, "vmom")
        assert torch.equal(h.wshadow[mw], ref_p[mw].to(torch.bfloat16)), (code, s, "bf16 broadcast")
    for t in (h.sq, h.vsq, h.sqmax, h.vsqmax):
        assert bool((t == 7.0).all()), (code, "second moments touched")
    assert czero_v > 0 and czero_w > 0, (code, czero_w, czero_v)
    assert bool((h.mom[mw] != 0).any()) and bool((h.vmom[mv] != 0).any())
    return h


@pytest.mark.gpu
@pytest.mark.parametrize("code", list(FAMILY))
def test_loopback_family_matches_the_oracle(code):
    _loopback(code)


@pytest.mark.gpu
def test_loopback_two_owners():
    h = _loopback("powersgd", n_owners=2)
    assert h.n_owners == 2 and all(nt > 0 for _, nt in h.plan.ps_range[0])


@pytest.mark.gpu
def test_loopback_two_groups():
    h = _loopback("svd", groups=2)
    assert h.plan.n_groups == 2


@pytest.mark.gpu
def test_loopback_num_aggregate_one_of_two():
    """Only worker 0 pushes: both launches count it alone (inv_w = 1)."""
    _loopback("sign", num_aggregate=1, pushers=[0])


# ---------------------------------------------------------------------------------------------------- engine
CODES = {
    "svd": dict(code="svd", svd_rank=3), "sgd": dict(code="sgd"), "qsgd": dict(code="qsgd"),
    "topk": dict(code="topk", entry_budget=0.05, error_feedback=True), "sign": dict(code="sign"),
    "powersgd": dict(code="powersgd", svd_rank=2), "fp8": dict(code="fp8"),
    "hadamard": dict(code="hadamard", quantization_level=4, bucket_size=256),
}
DATA_SEED = 900
_state = functools.partial(state, keys=("master", "vparams", "mom", "vmom", "wshadow"))


def _engine(graph=False, optimizer="lion", lr=LR, weight_decay=WD, **kw):
    kw = dict(CODES["svd"], **kw) if "code" not in kw else kw
    return make_engine(use_graph=graph, overlap=graph, optimizer=optimizer, lr=lr, weight_decay=weight_decay,
                       prepare_n=32 * kw.get("accumulate_steps", 1), data_seed=DATA_SEED, **kw)


def _step(eng):
    return step(eng, engine_batch("ResNet18", eng.step, 32 * eng.accum, DATA_SEED))


@pytest.mark.gpu
@pytest.mark.parametrize("code", list(CODES))
def test_decay_is_the_torch_multiply_before_the_lion_step(code, deterministic_cudnn):
    a = _engine(**CODES[code])
    b = _engine(weight_decay=0.0, **CODES[code])
    assert a.sq is None and a.vsq is None and a.sqmax is None and b.sq is None
    f = float(np.float32(1.0 - LR * WD))
    for _ in range(3):
        _step(a)
        b.master.mul_(f)          # weights only: vectors live in vparams
        _step(b)
        assert not differs(_state(a), _state(b)), (code, differs(_state(a), _state(b)))
    assert a.launches_per_step == b.launches_per_step + a.G      # one decay launch per group
    assert bool((a.mom != 0).any()) and bool((a.vmom != 0).any())
    a.close()
    b.close()


def _run(graph, steps=4, lr_at=None, **kw):
    eng = _engine(graph=graph, **kw)
    for s in range(steps):
        if lr_at is not None and s == lr_at:
            eng.set_lr(LR / 4)
        _step(eng)
    out = _state(eng)
    if eng.ema is not None:
        out["ema"], out["vema"] = eng.ema.clone(), eng.vema.clone()
    eng.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("code", ["svd", "sgd", "topk"])
def test_eager_equals_graph_and_reruns(code, deterministic_cudnn):
    e1, e2, g1 = _run(False, **CODES[code]), _run(False, **CODES[code]), _run(True, **CODES[code])
    assert not differs(e1, e2) and not differs(e1, g1), (differs(e1, e2), differs(e1, g1))


@pytest.mark.gpu
def test_set_lr_between_replays(deterministic_cudnn):
    eager, graph, plain = _run(False, lr_at=2), _run(True, lr_at=2), _run(True)
    assert not differs(eager, graph)
    assert differs(graph, plain)        # both the step and the decay factor changed


@pytest.mark.gpu
def test_set_lr_rewrites_the_decay_factor():
    eng = _engine()
    eng.set_lr(0.02)
    assert float(eng.ctrl_f32[17]) == float(np.float32(1.0 - 0.02 * WD)) and float(eng.ctrl_f32[2]) == np.float32(0.02)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_accumulate_steps_two(graph, deterministic_cudnn):
    eng = _engine(graph=graph, accumulate_steps=2)
    m0 = eng.master.clone()
    losses = [_step(eng) for _ in range(3)]
    assert all(np.isfinite(losses)) and not torch.equal(eng.master, m0)
    # every weight element steps by lr (or 0) per step, on top of the decay: |p - p0 f^3| <= 3 lr (+ rounding)
    f = float(np.float32(1.0 - LR * WD))
    assert float((eng.master - m0 * f ** 3).abs().max()) <= 3 * LR * 1.001
    eng.close()


@pytest.mark.gpu
def test_weight_average_follows_the_lion_weights():
    eng = _engine(ema_decay=0.9)
    w = float(np.float32(1.0 - 0.9))
    e, ev = eng.master.clone(), eng.vparams.clone()
    for _ in range(3):
        _step(eng)
        e = e + w * (eng.master - e)
        ev = ev + w * (eng.vparams - ev)
    assert torch.equal(eng.ema, e) and torch.equal(eng.vema, ev)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("code", ["svd", "topk"])
def test_resume_is_bitwise(code, tmp_path, deterministic_cudnn):
    d = str(tmp_path) + "/"
    ref = _engine(**CODES[code])
    for _ in range(4):
        _step(ref)
    want = _state(ref)
    ref.close()
    a = _engine(**CODES[code])
    for _ in range(2):
        _step(a)
    a.save_checkpoint(d)
    side = torch.load(d + "model_step_2_optim", map_location="cpu", weights_only=False)
    assert side["optimizer"] == "lion" and side["lion_betas"] == BETAS and side["weight_decay"] == WD
    assert "sq_w" not in side
    a.close()
    b = _engine(**CODES[code])
    b.load_checkpoint(d, 2)
    for _ in range(2):
        _step(b)
    assert not differs(_state(b), want), differs(_state(b), want)
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("other", ["sgd", "adam", "adamw"])
def test_cross_optimizer_loads_are_refused(other, tmp_path):
    d = str(tmp_path) + "/"
    kw = dict(momentum=0.9, weight_decay=0.0) if other == "sgd" else {}
    a = _engine(optimizer=other, **kw)
    _step(a)
    a.save_checkpoint(d)
    a.close()
    b = _engine()
    with pytest.raises(ValueError, match="written by optimizer %s; this engine runs lion" % other):
        b.load_checkpoint(d, 1)
    _step(b)
    b.save_checkpoint(d, 5)
    b.close()
    c = _engine(optimizer=other, **kw)
    with pytest.raises(ValueError, match="written by optimizer lion; this engine runs %s" % other):
        c.load_checkpoint(d, 5)
    c.close()


@pytest.mark.gpu
def test_launcher_trains_checkpoints_and_resumes(tmp_path, monkeypatch, capsys):
    import argparse
    from atomo_b200.runtime import p2p_launcher as L
    from atomo_b200.utils.flags import add_fit_args
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    d = str(tmp_path) + "/"
    argv = ["--network", "ResNet18", "--dataset", "Cifar10", "--synthetic", "1", "--train-len", "1024", "--test-len",
            "256", "--batch-size", "64", "--test-batch-size", "128", "--engine", "shadow", "--dtype", "bf16", "--code",
            "svd", "--svd-rank", "3", "--lr", "1e-4", "--optimizer", "lion", "--weight-decay", "0.1",
            "--lion-betas", "0.9", "0.98", "--eval-freq", "4", "--log-interval", "4", "--train-dir", d]
    L.run_p2p_training(add_fit_args(argparse.ArgumentParser(), argv + ["--max-steps", "4"]))
    L.run_p2p_training(add_fit_args(argparse.ArgumentParser(), argv + ["--max-steps", "8", "--resume", "1"]))
    out = capsys.readouterr().out
    for s in (4, 8):
        assert "Test set: Step: %d," % s in out, out
        side = torch.load(d + "model_step_%d_optim" % s, map_location="cpu", weights_only=False)
        assert side["optimizer"] == "lion" and side["step"] == s and side["lion_betas"] == (0.9, 0.98)
    assert "device error" not in out


# ---------------------------------------------------------------------------------------------------- two GPUs
def _mp(rank, world, port, out):
    import torch.distributed as dist
    nccl_init(rank, world, port)
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    eng = ShadowEngine(build_model("ResNet18", 10), rank, world, use_graph=True, seed=7, ps_mode="sharded",
                       optimizer="lion", lr=LR, weight_decay=WD, **CODES["svd"])
    x, y = engine_batch("ResNet18", rank, seed=DATA_SEED)
    eng.prepare(x, y, warmup=0)
    for s in range(4):
        x, y = engine_batch("ResNet18", 1 + s + rank, seed=DATA_SEED)
        eng.train_step(x, y)
    torch.cuda.synchronize()
    dist.barrier()
    torch.cuda.synchronize()
    out.put((rank, eng.error_code(), eng.wshadow.cpu(), eng.vparams.cpu(), eng.gather_fp32("master").cpu()))
    eng.close()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_owners_keep_identical_replicas():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    res = spawn(2, _mp, 29740)
    assert all(r[1] == 0 for r in res)
    a, b = res
    assert torch.equal(a[2], b[2]) and torch.equal(a[3], b[3]) and torch.equal(a[4], b[4])

"""Momentum correction for top-k on the bf16 engine (``ShadowEngine(momentum_correction=True)``,
``--momentum-correction``, csrc/v2_momentum.cu and the masking epilogue of the top-k encode).

CPU: the flag, the refusals before any CUDA work, the launcher routing, the fp32-flat and gloo refusals, and the fp32
oracle (``optim/momentum_correction.py``) against a float64 evaluation of its formulas.
GPU: the apply pass and the masked encode equal the oracle bit for bit; the momentum is zero exactly where this
worker's arena words say an entry was sent; ``m = 0, wd = 0`` is top-k + error feedback bit for bit; a resume is
bitwise; ResNet-18 trains; two ranks stay replicas.
"""
import argparse
import functools
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

from atomo_b200.codings.topk import TopK
from atomo_b200.optim import momentum_correction as MC
from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils.flags import add_fit_args

from shadow_harness import deterministic_cudnn, differs, engine_batch, fit_args, forbid_cuda, make_engine, nccl_init, \
    spawn  # noqa: F401


# ---------------------------------------------------------------------------------------------------- CPU
def test_flag_parses():
    parse = lambda *a: add_fit_args(argparse.ArgumentParser(), list(a))
    assert parse().momentum_correction is False
    assert parse("--momentum-correction", "1").momentum_correction is True
    assert parse("--momentum-correction", "0").momentum_correction is False
    a = parse("--momentum", "0.9", "--momentum-correction", "1")      # the full name still wins over the prefix
    assert a.momentum == 0.9 and a.momentum_correction is True


BASE = dict(code="topk", error_feedback=True, momentum=0.9)


@pytest.mark.parametrize("kw,match", [
    (dict(code="svd"), "topk"), (dict(code="entrywise"), "topk"), (dict(code="sign"), "topk"),
    (dict(error_feedback=False), "error_feedback"), (dict(optimizer="adam"), "sgd"), (dict(optimizer="lars"), "sgd"),
    (dict(dampening=0.1), "dampening"), (dict(momentum=-0.1), "momentum"), (dict(momentum=float("nan")), "momentum"),
    (dict(momentum=float("inf")), "momentum"), (dict(clip_grad_norm=1.0), "clip_grad_norm"),
    (dict(accumulate_steps=2), "accumulate_steps")])
def test_engine_refuses_before_cuda(kw, match, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    forbid_cuda(monkeypatch)
    with pytest.raises(ValueError, match=match):
        S.ShadowEngine(None, 0, 1, momentum_correction=True, **dict(BASE, **kw))


def test_launcher_passes_the_kwarg_only_when_on(tmp_path, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    seen = []

    class Fake:
        def __init__(self, model, rank, world, **kw):
            seen.append(kw)
    monkeypatch.setattr(S, "ShadowEngine", Fake)
    topk = ("--code", "topk", "--dtype", "bf16", "--entry-budget", "0.01", "--error-feedback", "1")
    L._build_engine(fit_args(tmp_path, *topk), nn.Linear(4, 4), 0, 1)
    assert "momentum_correction" not in seen[-1]
    L._build_engine(fit_args(tmp_path, *topk, "--momentum-correction", "0"), nn.Linear(4, 4), 0, 1)
    assert "momentum_correction" not in seen[-1]
    L._build_engine(fit_args(tmp_path, *topk, "--momentum-correction", "1", "--momentum", "0.9"), nn.Linear(4, 4), 0, 1)
    assert seen[-1]["momentum_correction"] is True and seen[-1]["momentum"] == 0.9


def test_fp32_flat_engine_refuses_the_flag(tmp_path):
    for extra in (("--dtype", "fp32"), ("--dtype", "bf16", "--engine", "fused")):
        with pytest.raises(SystemExit, match="--momentum-correction"):
            L._build_engine(fit_args(tmp_path, "--code", "svd", "--momentum-correction", "1", *extra), nn.Linear(4, 4),
                            0, 1)


def test_gloo_refuses_the_flag(monkeypatch, tmp_path):
    from atomo_b200 import distributed_nn
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    with pytest.raises(SystemExit, match="--momentum-correction"):
        distributed_nn.run_rank(fit_args(tmp_path, "--code", "svd", "--momentum-correction", "1", "--backend", "gloo"))


def _f32(rng, n, scale):
    return (rng.standard_normal(n) * scale).astype(np.float32)


@pytest.mark.parametrize("nesterov", [False, True])
@pytest.mark.parametrize("wd", [0.0, 5e-4])
def test_oracle_against_float64(nesterov, wd):
    """Each fp32 operation of the oracle is the float64 value of the formula on the same fp32 operands, rounded once;
    b = bf16(A) and b + e == A exactly; kept entries get u = 0 and e = A - b, the others keep u and get e = A."""
    rng = np.random.default_rng(3)
    n, m = 1000, 0.9
    g = torch.from_numpy(_f32(rng, n, 1e-2)).bfloat16().float().numpy()
    w = torch.from_numpy(_f32(rng, n, 1e-1)).bfloat16().float().numpy()
    u, e = _f32(rng, n, 1e-2), _f32(rng, n, 1e-3)
    b, u1, e1 = MC.mc_apply(g, w, u, e, m, wd, nesterov)
    r = lambda x: np.asarray(x, dtype=np.float64).astype(np.float32)           # one rounding of a float64 value
    d = r(g.astype(np.float64) + r(np.float32(wd) * w.astype(np.float64))) if wd > 0 else g
    assert np.array_equal(u1, r(r(np.float64(np.float32(m)) * u) + d.astype(np.float64)))
    s = r(d.astype(np.float64) + r(np.float64(np.float32(m)) * u1)) if nesterov else u1
    a = r(s.astype(np.float64) + e)
    assert np.array_equal(b, torch.from_numpy(a).bfloat16().float().numpy())
    assert np.array_equal(b.astype(np.float64) + e1.astype(np.float64), a.astype(np.float64))
    coder = TopK(0.05)
    kept, u2, e2 = MC.mc_encode(b, u1, e1, coder)
    assert len(kept) == coder.k_for(n)
    mask = np.zeros(n, dtype=bool)
    mask[kept] = True
    assert np.all(u2[mask] == 0) and np.array_equal(u2[~mask], u1[~mask])
    assert np.array_equal(e2[mask], e1[mask])
    assert np.array_equal(e2[~mask], r(e1[~mask].astype(np.float64) + b[~mask]))
    v, p, uv = _f32(rng, 64, 1e-2), _f32(rng, 64, 1.0), _f32(rng, 64, 1e-2)
    v1, uv1 = MC.mc_apply_vector(v, p, uv, m, wd, nesterov)
    dv = r(v.astype(np.float64) + r(np.float32(wd) * p.astype(np.float64))) if wd > 0 else v
    assert np.array_equal(uv1, r(r(np.float64(np.float32(m)) * uv) + dv.astype(np.float64)))
    want_v = r(dv.astype(np.float64) + r(np.float64(np.float32(m)) * uv1)) if nesterov else uv1
    assert np.array_equal(v1, want_v)


def test_oracle_without_momentum_is_the_error_feedback_apply():
    """m = 0, wd = 0: A = g + e exactly as the error-feedback apply forms it, whatever the momentum held."""
    rng = np.random.default_rng(5)
    g = torch.from_numpy(_f32(rng, 4096, 1e-2)).bfloat16().float().numpy()
    g[:16] = 0.0
    e, u = _f32(rng, 4096, 1e-3), _f32(rng, 4096, 1.0)
    b, u1, e1 = MC.mc_apply(g, None, u, e, 0.0)
    a = g + e
    want_b = torch.from_numpy(a).bfloat16().float().numpy()
    assert np.array_equal(b, want_b) and np.array_equal(e1, a - want_b) and np.array_equal(u1, g)
    v = _f32(rng, 64, 1.0)
    v1, _ = MC.mc_apply_vector(v, None, _f32(rng, 64, 1.0), 0.0)
    assert np.array_equal(v1, v)


# ---------------------------------------------------------------------------------------------------- GPU harness
# a 3x3 conv (a multiple of 8 elements, several encode tiles), a length that is not a multiple of 8, a large fc
# matrix, a tensor of few distinct magnitudes (ties at the threshold), an all-zero tensor, two vectors
SHAPES = [(64, 32, 3, 3), (7, 20), (300, 200), (16, 8, 3, 3), (32, 16), (64,), (10,)]
TIES, ZERO = 3, 4
BUDGET = 0.05


def _grads(step):
    g = torch.Generator().manual_seed(100 + step)
    out = []
    for i, s in enumerate(SHAPES):
        t = torch.randn(s, generator=g) * (0.01 * (1 + i))
        if i == TIES:
            t = torch.randint(-3, 4, s, generator=g).float() * 2.0 ** -7
        if i == ZERO:
            t = torch.zeros(s)
        out.append(t.bfloat16().float().cuda())
    return out


class Linear(nn.Module):
    """loss = sum_p <p, G_p>: the gradient of every parameter is G_p whatever the weights are.  The weights start
    non-zero, so that weight decay has something to act on."""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(9)
        self.ps = nn.ParameterList([nn.Parameter(torch.randn(s, generator=g) * 0.1) for s in SHAPES])
        self.gs = _grads(0)

    def forward(self, x):
        s = sum((p.float() * g).sum() for p, g in zip(self.ps, self.gs))
        return s.reshape(1, 1).expand(x.shape[0], 2)


def _raw(t, n):
    """The n elements of a gradient buffer in memory order: what the kernels read through the pointer table."""
    return t.as_strided((n,), (1,)).float().clone()


class Spy:
    """Stands in for the engine's native module: keeps the inputs and outputs of the apply launch.  With overlap=False
    every launch and copy runs on the backward's stream in order."""

    def __init__(self, eng):
        self.C, self.eng = eng.C, eng
        self.before = self.after = None

    def __getattr__(self, name):
        return getattr(self.C, name)

    def _grab(self):
        e, ws = self.eng, [(q, p) for p, q in zip(self.eng.params, self.eng.plan.params) if q.is_w]
        return {"g": {q.index: _raw(p.grad, q.numel) for q, p in ws}, "w": e.wshadow.float().clone(),
                "u": e.mc_mom.clone(), "e": e.residual.clone(), "v": e.vgrads.clone(), "p": e.vparams.clone(),
                "uv": e.mc_vmom.clone()}

    def v2_mc_apply(self, *a):
        self.before = self._grab()
        r = self.C.v2_mc_apply(*a)
        self.after = self._grab()
        return r


def _bits(t):
    t = torch.as_tensor(t).float().cpu()
    return t.view(torch.int32)


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _sent(eng, q):
    """Element indices (physical order) of the entries this worker's arena words carry for weight q."""
    from atomo_b200.ops import plan2 as P
    pl = eng.plan
    u = next(u for u in pl.units if u.kind == P.KIND_ENTRY and u.param == q.index)
    assert u.w_off == q.off and u.numel == q.numel
    base = eng.heap.tensor("arena")[eng.worker_index * pl.arena_floats + u.slot_off:]
    idx = []
    for j in range(u.n_ps):
        count = int(base[P.entry_hdr_off(j):P.entry_hdr_off(j) + 4].view(torch.int32)[1])
        wo = P.entry_words_off(u.n_ps, j, u.ps_rows)
        words = base[wo:wo + count].view(torch.int32).cpu()
        idx += [j * u.ps_rows + (int(x) & 0xFFF) for x in words.tolist()]
    return np.array(sorted(idx), dtype=np.int64)


# ---------------------------------------------------------------------------------------------------- GPU: kernels
@pytest.mark.gpu
@pytest.mark.parametrize("nesterov", [False, True])
@pytest.mark.parametrize("wd", [0.0, 5e-4])
def test_apply_and_masked_encode_equal_the_oracle_bitwise(nesterov, wd):
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.cuda.set_device(0)
    m = 0.9
    model = Linear()
    eng = ShadowEngine(model, 0, 1, code="topk", entry_budget=BUDGET, lr=0.1, momentum=m, weight_decay=wd,
                       nesterov=nesterov, use_graph=False, overlap=False, criterion=lambda lg, y: lg[0, 0],
                       error_feedback=True, momentum_correction=True, seed=5)
    try:
        x, y = torch.zeros(4, 2), torch.zeros(4, dtype=torch.long)
        eng.prepare(x, y, warmup=0)
        coder = TopK(BUDGET)
        ws = [q for q in eng.plan.params if q.is_w]
        vs = [q for q in eng.plan.params if not q.is_w]
        assert {SHAPES[q.index] for q in vs} == {(64,), (10,)}
        kept_some = ties_cut = False
        for step in range(5):
            model.gs = _grads(step % 3)
            spy = eng.C = Spy(eng)
            eng.train_step(x, y)
            torch.cuda.synchronize()
            eng.C = spy.C
            assert eng.error_code() == 0
            bf, af = spy.before, spy.after
            for q in ws:
                sl = slice(q.off, q.off + q.numel)
                b, u1, e1 = MC.mc_apply(bf["g"][q.index].cpu().numpy(), bf["w"][sl].cpu().numpy(),
                                        bf["u"][sl].cpu().numpy(), bf["e"][sl].cpu().numpy(), m, wd, nesterov)
                assert _same(af["g"][q.index], b), (step, q.index)
                assert _same(af["u"][sl], u1) and _same(af["e"][sl], e1), (step, q.index)
                kept, u2, e2 = MC.mc_encode(b, u1, e1, coder)
                assert _same(eng.mc_mom[sl], u2) and _same(eng.residual[sl], e2), (step, q.index)
                sent = _sent(eng, q)
                assert np.array_equal(sent, kept), (step, q.index)
                mom = eng.mc_mom[sl].cpu()
                assert bool((mom[torch.from_numpy(sent)] == 0).all())
                if q.index == ZERO and wd == 0:
                    assert len(sent) == 0 and not bool(mom.ne(0).any())
                elif len(sent):
                    kept_some = True
                    if q.index == TIES:
                        mag = np.abs(b)
                        T = mag[sent].min()
                        ties_cut = ties_cut or int((mag == T).sum()) > int((mag[sent] == T).sum())
            for q in vs:
                sl = slice(q.off, q.off + q.numel)
                v1, uv1 = MC.mc_apply_vector(bf["v"][sl].cpu().numpy(), bf["p"][sl].cpu().numpy(),
                                             bf["uv"][sl].cpu().numpy(), m, wd, nesterov)
                assert _same(af["v"][sl], v1) and _same(af["uv"][sl], uv1), (step, q.index)
                assert _same(eng.mc_vmom[sl], uv1), (step, q.index)
        assert kept_some and ties_cut        # the tie at the threshold was really cut inside the tensor
        assert eng.momentum_correction_norm()["model"] > 0
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------- GPU: engine
_batch = functools.partial(engine_batch, seed=300)


def _engine(net, **kw):
    return make_engine(net, **dict(dict(code="topk", entry_budget=0.01, error_feedback=True, lr=0.05, momentum=0.9),
                                   **kw))


def _state(eng, losses) -> dict:
    out = {"master": eng.master.clone(), "vparams": eng.vparams.clone(), "wshadow": eng.wshadow.clone(),
           "mom": eng.mom.clone(), "vmom": eng.vmom.clone(), "loss": torch.tensor(losses)}
    for name, b in eng.model.named_buffers():
        out["buffer:" + name] = b.clone()
    for name, t in eng._worker_tensors().items():
        out["worker:" + name] = t.clone()
    return out


def _run(net, steps, batch=32, warmup=2, load=None, save=None, **kw):
    eng = _engine(net, **kw)
    x, y = _batch(net, 0, batch)
    eng.prepare(x, y, warmup=warmup)
    if load is not None:
        eng.load_checkpoint(save, load)
    losses = []
    for _ in range(steps):
        x, y = _batch(net, eng.step, batch)
        losses.append(float(eng.train_step(x, y)[0]))
    torch.cuda.synchronize()
    assert eng.error_code() == 0
    st, n = _state(eng, losses), eng.launches_per_step
    if save is not None and load is None:
        eng.save_checkpoint(save)
    eng.close()
    return st, n


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["LeNet", "ResNet18"])
def test_without_momentum_it_is_top_k_with_error_feedback(net, deterministic_cudnn):
    """m = 0, wd = 0, graph + overlap: the corrected engine is the top-k + EF engine with PS momentum 0, bit for bit,
    with the same launches per step (the apply takes the place of the error-feedback apply)."""
    a, na = _run(net, 20, momentum=0.0, momentum_correction=True)
    b, nb = _run(net, 20, momentum=0.0)
    assert na == nb
    assert differs(a, b, ["master", "vparams", "wshadow", "worker:residual", "loss"]) == []
    assert math.isfinite(float(a["loss"][-1]))


@pytest.mark.gpu
def test_resume_is_bitwise(tmp_path, deterministic_cudnn, capsys):
    K, net = 3, "ResNet18"
    kw = dict(momentum_correction=True, weight_decay=5e-4, nesterov=True)
    d = str(tmp_path) + "/"
    a, _ = _run(net, 2 * K, **kw)
    assert differs(a, _run(net, 2 * K, **kw)[0]) == [], "control: two uninterrupted runs differ"
    _run(net, K, save=d, **kw)
    c, _ = _run(net, K, load=2 + K, save=d, **kw)
    assert "not restored" not in capsys.readouterr().out
    assert differs(dict(a, loss=a["loss"][K:]), c) == []
    assert bool(a["worker:mom"].ne(0).any()) and bool(a["worker:vmom_w"].ne(0).any())
    eng = _engine(net, **dict(kw, momentum_correction=False))       # the sidecar refuses another setting
    try:
        x, y = _batch(net, 0, 32)
        eng.prepare(x, y, warmup=0)
        with pytest.raises(ValueError, match="momentum_correction"):
            eng.load_checkpoint(d, 2 + K)
    finally:
        eng.close()


@pytest.mark.gpu
def test_resnet18_trains(deterministic_cudnn):
    eng = _engine("ResNet18", momentum_correction=True, weight_decay=5e-4, lr=0.05)
    try:
        x, y = _batch("ResNet18", 0, 128)
        eng.prepare(x, y, warmup=2)
        losses = [float(eng.train_step(x, y)[0]) for _ in range(40)]
        torch.cuda.synchronize()
        assert eng.error_code() == 0
        n = eng.momentum_correction_norm()
        ef = eng.error_feedback_norm()
        print("ResNet-18 top-k 1%% + momentum correction: loss %.3f -> %.3f, ||u|| %.3g, ||e|| %.3g"
              % (losses[0], losses[-1], n["model"], ef["model"]))
        assert all(math.isfinite(v) for v in losses) and math.isfinite(n["model"]) and math.isfinite(ef["model"])
        assert sum(losses[-5:]) < 0.5 * sum(losses[:5])
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------- two GPUs
def _mp_replicas(rank, world, port, out):
    import torch.distributed as dist
    nccl_init(rank, world, port)
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    eng = ShadowEngine(build_model("ResNet18", 10), rank, world, code="topk", entry_budget=0.01, lr=0.05,
                       momentum=0.9, weight_decay=5e-4, seed=7, ps_mode="sharded", error_feedback=True,
                       momentum_correction=True, timeout_s=20.0)
    x, y = SyntheticImageDataset((3, 32, 32), 10, 4096, seed=400 + rank).materialize(32)
    x, y = x.cuda(), y.cuda()
    eng.prepare(x, y, warmup=2)
    for _ in range(8):
        eng.train_step(x, y)
    torch.cuda.synchronize()
    w = [torch.empty_like(eng.wshadow) for _ in range(world)]
    v = [torch.empty_like(eng.vparams) for _ in range(world)]
    dist.all_gather(w, eng.wshadow.clone())
    dist.all_gather(v, eng.vparams.clone())
    same = all(torch.equal(w[0], t) for t in w) and all(torch.equal(v[0], t) for t in v)
    mom = eng.momentum_correction_norm()["model"]
    out.put((rank, eng.error_code(), same, mom))
    eng.close()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_ranks_stay_replicas():
    """Each worker corrects its own gradient with its own momentum; the owners' published weights are the same on
    every rank."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    res = spawn(2, _mp_replicas, 29870, timeout=300)
    for rank, err, same, mom in res:
        assert err == 0 and same and mom > 0, res

"""Gradient-norm clipping on the bf16 engine (``ShadowEngine(clip_grad_norm=MAX)``, csrc/v2_clip.cu).

Above the norm the engine is the unclipped engine: bitwise for momentum-SGD, Nesterov, Adam and AMSGrad on every code,
over three steps.  For LARS and LAMB the per-tile (w^2, x^2) partials are reduced in the clip launch's element order
instead of the PS kernel's, so the trust ratios, and through them the weights, differ by fp32 reassociation (within
the ratio bound of test_gpu_layerwise.py times the step); the moments and vectors of that step stay bitwise, and the
next forward sees the weight difference, so the comparison covers one step.  Below the norm the step is coef times the
unclipped step and ``grad_norm()`` is the norm of the whole gradient, vectors and dense tensors included.  On the
dense code the whole step matches ``clip_grad_norm_`` followed by the fp64 ``optim/`` class (momentum-SGD, LARS, LAMB;
``optim/adam.py`` places eps unscaled by the bias correction, unlike the engine's Adam, so Adam is covered by the
bitwise comparison with the unclipped engine instead).  Runs are repeatable,
graph replay equals eager, accumulation clips the step's mean once, error feedback is untouched, a resume is bitwise,
and a non-finite norm raises the sticky error.  The two-GPU test exercises the cross-owner exchange.
"""
import functools
import math

import numpy as np
import pytest
import torch

from atomo_b200.optim import LAMB, LARS, SGD

from shadow_harness import deterministic_cudnn, engine_batch, make_engine, nccl_init, spawn, state, step  # noqa: F401

EPS32 = 2.0 ** -24
TILE = 4608
RATIO_RTOL = (TILE + 64) * EPS32 * 4      # fp32 tile partials, fp32 sqrt and division (test_gpu_layerwise.py)
ERR2_NONFINITE = 8

CODES = {
    "svd": dict(code="svd"), "qsvd": dict(code="qsvd"), "sgd": dict(code="sgd"), "qsgd": dict(code="qsgd"),
    "terngrad": dict(code="terngrad"), "entrywise": dict(code="entrywise", entry_budget=0.05),
    "topk": dict(code="topk", entry_budget=0.05), "sign": dict(code="sign"), "powersgd": dict(code="powersgd", svd_rank=2),
    "fp8": dict(code="fp8"), "hadamard": dict(code="hadamard", quantization_level=4, bucket_size=512),
}
OPTS = {
    "momentum": dict(optimizer="sgd", lr=0.05, momentum=0.9, weight_decay=5e-4),
    "nesterov": dict(optimizer="sgd", lr=0.05, momentum=0.9, nesterov=True, weight_decay=5e-4),
    "adam": dict(optimizer="adam", lr=1e-3, weight_decay=1e-4),
    "amsgrad": dict(optimizer="adam", lr=1e-3, amsgrad=True),
    "lars": dict(optimizer="lars", lr=0.5, momentum=0.9, weight_decay=5e-4, trust_coefficient=0.02),
    "lamb": dict(optimizer="lamb", lr=0.02, weight_decay=0.01),
}
HUGE = 1e30       # far above any norm: coef = 1
TINY = 1e-3       # far below the norm of a ResNet-18 gradient: coef < 1

DATA_SEED = 500
_batch = functools.partial(engine_batch, "ResNet18", seed=DATA_SEED)


def _engine(kw, graph=False, **extra):
    return make_engine(use_graph=graph, prepare_n=32, data_seed=DATA_SEED, **dict(kw, **extra))


def _step(eng, check=True):
    step(eng, _batch(eng.step), check)


STATE = ("master", "mom", "sq", "sqmax", "vparams", "vmom", "vsq", "vsqmax", "wshadow")
_state = functools.partial(state, keys=STATE)


def _phys(t):
    return t.permute(0, 2, 3, 1).reshape(-1) if t.dim() == 4 else t.reshape(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("code", list(CODES))
def test_above_the_norm_is_the_unclipped_engine(code, opt):
    kw = dict(OPTS[opt], **CODES[code])
    layerwise = opt in ("lars", "lamb")
    a, b = _engine(kw), _engine(kw, clip_grad_norm=HUGE)
    w0 = a.master.double().clone()
    # LARS / LAMB: one step, since the next forward already sees the (reassociation-sized) weight difference
    for _ in range(1 if layerwise else 3):
        _step(a)
        _step(b)
        total, coef = b.grad_norm()
        assert math.isfinite(total) and total > 0 and coef == 1.0
    sa, sb = _state(a), _state(b)
    assert sa.keys() == sb.keys()
    if not layerwise:
        assert [k for k in sa if not torch.equal(sa[k], sb[k])] == []
    else:
        bitwise = ["vparams", "vmom"] + (["mom", "sq", "vsq"] if opt == "lamb" else [])
        assert [k for k in bitwise if not torch.equal(sa[k], sb[k])] == []
        # the trust ratios differ by fp32 reassociation of the tile partials: within RATIO_RTOL of the step
        disp = (sa["master"].double() - w0).abs()
        tol = 4 * EPS32 * sa["master"].double().abs() + 2 * RATIO_RTOL * disp + 1e-38
        assert ((sa["master"].double() - sb["master"].double()).abs() <= tol).all()
        wa, wb = sa["wshadow"].float(), sb["wshadow"].float()
        assert ((wa - wb).abs() <= wa.abs() * 2.0 ** -7 + 1e-38).all()      # at most one bf16 ulp apart
    assert b.launches_per_step == a.launches_per_step + 1      # the clip launch
    a.close()
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("code", list(CODES))
def test_below_the_norm_scales_the_step(code):
    kw = dict(optimizer="sgd", lr=1.0, momentum=0.0, **CODES[code])
    a, b = _engine(kw), _engine(kw, clip_grad_norm=TINY)
    w0, v0 = a.master.double().clone(), a.vparams.double().clone()
    assert torch.equal(a.master, b.master)
    _step(a)
    _step(b)
    total, coef = b.grad_norm()
    # the norm b's owner computed is the norm of what it gathered (every weight element and every vector)
    g = torch.cat([b.clip_grad.double(), b.clip_vgrad.double()])
    gn = g.norm().item()
    assert abs(total - gn) <= RATIO_RTOL * gn, (total, gn)
    assert coef < 1 and coef == pytest.approx(TINY / (total + 1e-6), rel=4 * EPS32)
    # ... and of the unclipped engine's step / lr (vectors and dense tensors included)
    da = torch.cat([a.master.double() - w0, a.vparams.double() - v0])
    ref = da.norm().item()
    slack = 2 * EPS32 * torch.cat([w0, v0]).abs().norm().item()       # the rounding of w1 in each delta
    assert abs(total - ref) <= RATIO_RTOL * ref + slack, (total, ref)
    # the clipped step is coef times the unclipped one, element by element
    db = torch.cat([b.master.double() - w0, b.vparams.double() - v0])
    tol = 2 * EPS32 * (torch.cat([w0, v0]).abs() + da.abs()) + 1e-38
    assert ((db - coef * da).abs() <= tol).all()
    a.close()
    b.close()


def f32(v):
    return float(np.float32(v))


def _oracle(eng, pre, kw, max_norm, t):
    """The dense code, one worker: clip_grad_norm_ on the workers' bf16 gradient, then the fp64 optim/ class from
    the engine's pre-step state."""
    params = []
    for p, q in zip(eng.params, eng.plan.params):
        src = pre["master"] if q.is_w else pre["vparams"]
        w = torch.nn.Parameter(src[q.off:q.off + q.numel].double().clone().view(-1, 1) if q.is_w else
                               src[q.off:q.off + q.numel].double().clone())
        w.grad = (_phys(p.grad.double()) if q.is_w else eng.vgrads[q.off:q.off + q.numel].double()).view_as(w).clone()
        params.append((q, w))
    ts = [w for _, w in params]
    total = float(torch.nn.utils.clip_grad_norm_(ts, max_norm))
    name = kw["optimizer"]
    if name == "sgd":
        o = SGD(ts, lr=f32(kw["lr"]), momentum=f32(kw["momentum"]), weight_decay=f32(kw["weight_decay"]))
        if t > 0:
            for q, w in params:
                src = pre["mom"] if q.is_w else pre["vmom"]
                o.state[w]["momentum_buffer"] = src[q.off:q.off + q.numel].double().view_as(w).clone()
    elif name == "lars":
        o = LARS(ts, lr=f32(kw["lr"]), momentum=f32(kw["momentum"]), weight_decay=f32(kw["weight_decay"]),
                 trust_coefficient=f32(kw["trust_coefficient"]))
        if t > 0:
            for q, w in params:
                src = pre["mom"] if q.is_w else pre["vmom"]
                o.state[w]["momentum_buffer"] = src[q.off:q.off + q.numel].double().view_as(w).clone()
    else:
        o = LAMB(ts, lr=f32(kw["lr"]), weight_decay=f32(kw["weight_decay"]))
    if name == "lamb":
        for q, w in params:
            m, v = (pre["mom"], pre["sq"]) if q.is_w else (pre["vmom"], pre["vsq"])
            o.state[w].update(step=t, exp_avg=m[q.off:q.off + q.numel].double().view_as(w).clone(),
                              exp_avg_sq=v[q.off:q.off + q.numel].double().view_as(w).clone())
    o.step([w.grad for w in ts])
    return params, total


@pytest.mark.gpu
@pytest.mark.parametrize("opt", ["momentum", "lars", "lamb"])
@pytest.mark.parametrize("max_norm", [HUGE, 0.05])
def test_dense_code_matches_the_fp64_oracle(opt, max_norm):
    kw = dict(OPTS[opt], weight_decay=OPTS[opt].get("weight_decay", 0.0))
    eng = _engine(dict(kw, code="sgd"), clip_grad_norm=max_norm)
    for t in range(3):
        pre = {k: getattr(eng, k).clone() for k in ("master", "mom", "vparams", "vmom")}
        if eng.sq is not None:
            pre.update(sq=eng.sq.clone(), vsq=eng.vsq.clone())
        _step(eng)
        params, total = _oracle(eng, pre, kw, max_norm, t)
        got_total, coef = eng.grad_norm()
        assert abs(got_total - total) <= RATIO_RTOL * total
        assert (coef == 1.0) == (max_norm > total)
        for q, ref in params:
            got = (eng.master if q.is_w else eng.vparams)[q.off:q.off + q.numel].double()
            w0 = (pre["master"] if q.is_w else pre["vparams"])[q.off:q.off + q.numel].double()
            r = ref.detach().view(-1)
            # fp32 roundings of w and of each term of the update; the coefficient's and the ratios' own error; the
            # fp32 bias corrections of Adam / LAMB (powf near 1, as in test_gpu_layerwise.py)
            mag = (r - w0).abs() + kw["lr"] * ref.grad.view(-1).abs()
            src = pre["mom"] if q.is_w else pre["vmom"]
            mag = mag + kw["lr"] * kw.get("momentum", 0.0) * src[q.off:q.off + q.numel].double().abs()
            tt = t + 1
            bias = 8 * EPS32 * (0.5 / (1 - 0.999 ** tt) + 1 / (1 - 0.9 ** tt)) if opt == "lamb" else 0.0
            tol = 4 * EPS32 * w0.abs() + mag * (2 * RATIO_RTOL + 64 * EPS32 + bias) + 1e-30
            assert (got - r).abs().le(tol).all(), (q.index, (got - r).abs().max().item())
    eng.close()


def _run(kw, graph, steps=4, **extra):
    eng = _engine(kw, graph=graph, **extra)
    norms = []
    for _ in range(steps):
        _step(eng)
        norms.append(eng.grad_norm())
    out = {k: v.cpu() for k, v in _state(eng).items()}
    eng.close()
    return out, norms


@pytest.mark.gpu
@pytest.mark.parametrize("opt,code", [("momentum", "svd"), ("lamb", "topk")])
def test_bitwise_repeatable_and_graph_equals_eager(opt, code, deterministic_cudnn):
    kw = dict(OPTS[opt], **CODES[code])
    (a, na), (b, nb) = _run(kw, False, clip_grad_norm=0.5), _run(kw, False, clip_grad_norm=0.5)
    assert [k for k in a if not torch.equal(a[k], b[k])] == [] and na == nb
    c, nc = _run(kw, True, clip_grad_norm=0.5)
    assert [k for k in a if not torch.equal(a[k], c[k])] == [] and na == nc
    assert all(coef < 1 for _, coef in na)


@pytest.mark.gpu
def test_accumulation_clips_the_mean_once():
    kw = dict(optimizer="sgd", lr=0.5, momentum=0.0, code="svd")
    eng = _engine(kw, accumulate_steps=4, clip_grad_norm=TINY)
    for _ in range(2):
        w0 = eng.master.double().clone()
        _step(eng)
        total, coef = eng.grad_norm()
        g = eng.clip_grad.double()
        assert abs(total - torch.cat([g, eng.clip_vgrad.double()]).norm().item()) <= RATIO_RTOL * total
        assert coef < 1
        d = eng.master.double() - w0
        tol = 2 * EPS32 * (w0.abs() + 0.5 * g.abs()) + 1e-38
        assert ((d + 0.5 * coef * g).abs() <= tol).all()
    eng.close()


@pytest.mark.gpu
def test_error_feedback_residual_is_the_unclipped_runs():
    kw = dict(OPTS["momentum"], code="topk", entry_budget=0.01, error_feedback=True)
    a, b = _engine(kw), _engine(kw, clip_grad_norm=TINY)
    _step(a)
    _step(b)
    assert b.grad_norm()[1] < 1
    assert torch.equal(a.residual, b.residual)
    assert not torch.equal(a.master, b.master)
    a.close()
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("opt,extra", [("momentum", dict(code="svd")),
                                       ("lamb", dict(code="topk", entry_budget=0.01, error_feedback=True))])
def test_resume_is_bitwise(opt, extra, tmp_path, deterministic_cudnn):
    kw = dict(OPTS[opt], clip_grad_norm=0.5, **extra)
    d = str(tmp_path) + "/"
    a, na = _run(kw, True, steps=4)
    eng = _engine(kw, graph=True)
    for _ in range(2):
        _step(eng)
    eng.save_checkpoint(d)
    eng.close()
    eng = _engine(kw, graph=True)
    eng.load_checkpoint(d, 2)
    nc = []
    for _ in range(2):
        _step(eng)
        nc.append(eng.grad_norm())
    c = {k: v.cpu() for k, v in _state(eng).items()}
    eng.close()
    assert [k for k in a if not torch.equal(a[k], c[k])] == [] and na[2:] == nc


@pytest.mark.gpu
def test_a_non_finite_norm_sets_the_sticky_error():
    eng = _engine(dict(OPTS["momentum"], code="sgd"), clip_grad_norm=1.0)
    x, y = _batch(eng.step)
    x = x.clone()
    x.view(-1)[0] = float("inf")
    eng.train_step(x, y)
    torch.cuda.synchronize()
    assert eng.error_code() & ERR2_NONFINITE
    assert not math.isfinite(eng.grad_norm()[0])
    eng.close()


# ---------------------------------------------------------------------------------------------------- two GPUs
def _mp(rank, world, port, mode, out):
    import torch.distributed as dist
    nccl_init(rank, world, port)
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    eng = ShadowEngine(build_model("ResNet18", 10), rank, world, use_graph=True, seed=7, ps_mode=mode,
                       clip_grad_norm=0.5, **dict(OPTS["momentum"], code="svd"))
    x, y = _batch(rank)
    eng.prepare(x, y, warmup=0)
    x, y = _batch(1 + rank)
    eng.train_step(x, y)
    torch.cuda.synchronize()
    out.put((rank, mode, eng.error_code(), eng.clip_norm.cpu(), eng.wshadow.cpu()))
    eng.close()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_owners_agree_on_the_norm():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    res = {}
    for i, mode in enumerate(("sharded", "colocated")):
        for r, m, e, n, w in spawn(2, _mp, 29690 + i, mode):
            assert e == 0
            res[(m, r)] = (n, w)
    (n0, w0), (n1, w1) = res[("sharded", 0)], res[("sharded", 1)]
    assert torch.equal(n0, n1) and torch.equal(w0, w1)
    nc = res[("colocated", 0)][0]
    assert abs(float(n0[0]) - float(nc[0])) <= 4 * EPS32 * float(nc[0])

"""LARS and LAMB on the bf16 engine (``ShadowEngine(optimizer='lars' | 'lamb')``, csrc/v2_layerwise.cu).

For every code: after a few steps, the new ``master`` equals an fp64 evaluation of the rule from the engine's own
pre-step ``master`` / ``mom`` and the direction phase 1 left in ``lw_dir``, and each trust ratio matches the fp64 norms.
On the dense code, where the PS's gradient is the worker's bf16 gradient exactly, the whole step (weights and vectors)
matches the fp64 ``optim/`` oracle.  Zero tensors give ratio 1; runs are bitwise repeatable and graph replay equals
eager; accumulation, error feedback and a resume work.  The two-GPU test exercises the cross-owner exchange.
"""
import functools
import math

import numpy as np
import pytest
import torch

from atomo_b200.optim import LAMB, LARS
from atomo_b200.utils import checkpoint as ckpt

from shadow_harness import deterministic_cudnn, engine_batch, make_engine, nccl_init, spawn, step  # noqa: F401

EPS32 = 2.0 ** -24
TILE = 4608            # the largest PS tile (elements): fp32 partial sums of at most this many terms
RATIO_RTOL = (TILE + 64) * EPS32 * 4     # fp32 tile partials, fp32 sqrt and division of the ratio

LARS_KW = dict(optimizer="lars", lr=0.5, momentum=0.9, weight_decay=5e-4, trust_coefficient=0.02)
LAMB_KW = dict(optimizer="lamb", lr=0.02, weight_decay=0.01)
CODES = {
    "svd": dict(code="svd"), "qsvd": dict(code="qsvd"), "sgd": dict(code="sgd"), "qsgd": dict(code="qsgd"),
    "terngrad": dict(code="terngrad"), "entrywise": dict(code="entrywise", entry_budget=0.05),
    "topk": dict(code="topk", entry_budget=0.05), "sign": dict(code="sign"), "powersgd": dict(code="powersgd", svd_rank=2),
    "fp8": dict(code="fp8"), "hadamard": dict(code="hadamard", quantization_level=4, bucket_size=512),
}

DATA_SEED = 300
_batch = functools.partial(engine_batch, "ResNet18", seed=DATA_SEED)


def _engine(kw, graph=False, **extra):
    return make_engine(use_graph=graph, prepare_n=32, data_seed=DATA_SEED, **dict(kw, **extra))


def _step(eng):
    step(eng, _batch(eng.step))


def _weights(eng):
    """(name, Param2) of every weight tensor, in parameter order."""
    names = {id(p): n for n, p in eng.model.named_parameters()}
    return [(names[id(p)], q) for p, q in zip(eng.params, eng.plan.params) if q.is_w]


def _phys(t):
    return t.permute(0, 2, 3, 1).reshape(-1) if t.dim() == 4 else t.reshape(-1)


def _check_rule(eng, pre, kw):
    """master / mom after the step against fp64 of the rule on the engine's own pre-step state and direction."""
    lr, ratios = kw["lr"], eng.trust_ratios()
    d64 = eng.lw_dir.double()
    for name, q in _weights(eng):
        sl = slice(q.off, q.off + q.numel)
        w0, x = pre["master"][sl].double(), d64[sl]
        wn = w0.norm().item()
        if kw["optimizer"] == "lars":
            g = x - kw["weight_decay"] * w0            # d = fma(wd, w, g): g to within one rounding of d
            den = g.norm().item() + kw["weight_decay"] * wn
            want = kw["trust_coefficient"] * wn / den if wn > 0 and den > 0 else 1.0
        else:
            un = x.norm().item()
            want = wn / un if wn > 0 and un > 0 else 1.0
        r = ratios[name]
        assert math.isfinite(r) and abs(r - want) <= RATIO_RTOL * abs(want) + 1e-30, (name, r, want)
        if kw["optimizer"] == "lars":
            m0 = pre["mom"][sl].double()
            m = r * x if pre["first"] else kw["momentum"] * m0 + r * x
            ref = w0 - lr * m
            m1 = eng.mom[sl].double()
            mag = kw["momentum"] * m0.abs() + (r * x).abs()
            assert (m1 - m).abs().le(4 * EPS32 * mag + 1e-38).all(), name
            step = lr * mag
        else:
            ref = w0 - lr * r * x
            step = lr * r * x.abs()
        w1 = eng.master[sl].double()
        assert (w1 - ref).abs().le(4 * EPS32 * (w0.abs() + step) + 1e-38).all(), name


def _snapshot(eng):
    return {"master": eng.master.clone(), "mom": eng.mom.clone(), "first": eng.step == 1}


@pytest.mark.gpu
@pytest.mark.parametrize("opt", ["lars", "lamb"])
@pytest.mark.parametrize("code", list(CODES))
def test_step_follows_the_rule(code, opt):
    kw = LARS_KW if opt == "lars" else LAMB_KW
    eng = _engine(dict(kw, **CODES[code]))
    for _ in range(3):
        pre = _snapshot(eng)
        _step(eng)
        _check_rule(eng, pre, kw)
    assert eng.launches_per_step > 0
    r = list(eng.trust_ratios().values())
    assert all(math.isfinite(v) and v > 0 for v in r) and any(v != 1.0 for v in r)
    eng.close()


def f32(v):
    return float(np.float32(v))


def _oracle_step(eng, pre, kw):
    """The dense code, one worker: the PS's g is the worker's bf16 gradient; the fp64 optim/ class from the engine's
    pre-step state gives the whole step."""
    params, grads = [], []
    for p, q in zip(eng.params, eng.plan.params):
        if q.is_w:
            w = pre["master"][q.off:q.off + q.numel].double().clone()
            g = _phys(p.grad.double())
        else:
            w = pre["vparams"][q.off:q.off + q.numel].double().clone()
            g = eng.vgrads[q.off:q.off + q.numel].double()
        t = torch.nn.Parameter(w.view(-1, 1) if q.is_w else w)      # 2-D stands for "weight"
        params.append((q, t))
        grads.append(g.view_as(t))
    ts = [t for _, t in params]
    # the hyperparameters as the engine holds them (fp32 in Ctrl2), so that only the arithmetic differs
    if kw["optimizer"] == "lars":
        o = LARS(ts, lr=f32(kw["lr"]), momentum=f32(kw["momentum"]), weight_decay=f32(kw["weight_decay"]),
                 trust_coefficient=f32(kw["trust_coefficient"]))
        if not pre["first"]:
            for q, t in params:
                src = pre["mom"] if q.is_w else pre["vmom"]
                o.state[t]["momentum_buffer"] = src[q.off:q.off + q.numel].double().view_as(t).clone()
    else:
        o = LAMB(ts, lr=f32(kw["lr"]), betas=(f32(0.9), f32(0.999)), eps=f32(1e-8), weight_decay=f32(kw["weight_decay"]))
        for q, t in params:
            m, v = (pre["mom"], pre["sq"]) if q.is_w else (pre["vmom"], pre["vsq"])
            o.state[t].update(step=pre["t"], exp_avg=m[q.off:q.off + q.numel].double().view_as(t).clone(),
                              exp_avg_sq=v[q.off:q.off + q.numel].double().view_as(t).clone())
    o.step(grads)
    return params, grads, o


@pytest.mark.gpu
@pytest.mark.parametrize("opt", ["lars", "lamb"])
def test_dense_code_matches_the_fp64_oracle(opt):
    kw = LARS_KW if opt == "lars" else LAMB_KW
    eng = _engine(dict(kw, code="sgd"))
    for t in range(3):
        pre = _snapshot(eng)
        pre.update(vparams=eng.vparams.clone(), vmom=eng.vmom.clone(), t=t,
                   sq=eng.sq.clone() if eng.sq is not None else None,
                   vsq=eng.vsq.clone() if eng.vsq is not None else None)
        _step(eng)
        params, grads, o = _oracle_step(eng, pre, kw)
        for (q, ref), g in zip(params, grads):
            got = (eng.master if q.is_w else eng.vparams)[q.off:q.off + q.numel].double()
            w0 = (pre["master"] if q.is_w else pre["vparams"])[q.off:q.off + q.numel].double()
            st, g = o.state[ref], g.reshape(-1).abs()
            r, bias = st.get("ratio", 1.0), 0.0
            # per element, the update's terms in magnitude (momentum and moment sums may cancel): fp32 roundings of
            # each term, and the ratio's own error for the weights
            if kw["optimizer"] == "lars":
                src = pre["mom"] if q.is_w else pre["vmom"]
                m0 = 0.0 if pre["first"] else src[q.off:q.off + q.numel].double().abs()
                wd = kw["weight_decay"] if q.is_w else 0.0
                mag = kw["lr"] * (kw["momentum"] * m0 + r * (g + wd * w0.abs()))
            else:
                src = pre["mom"] if q.is_w else pre["vmom"]
                m0 = src[q.off:q.off + q.numel].double().abs()
                tt = st["step"]
                bc1, sbc2 = 1 - 0.9 ** tt, math.sqrt(1 - 0.999 ** tt)
                den = st["exp_avg_sq"].reshape(-1).sqrt() / sbc2 + 1e-8
                wd = kw["weight_decay"] if q.is_w else 0.0
                mag = kw["lr"] * r * ((0.9 * m0 + 0.1 * g) / bc1 / den + wd * w0.abs())
                # the engine takes 1 - b^t in fp32 from powf (ps_opt_consts): its rounding near 1 grows by 1 / (1 - b^t)
                bias = mag * 8 * EPS32 * (0.5 / (1 - 0.999 ** tt) + 1 / (1 - 0.9 ** tt))
            tol = 4 * EPS32 * w0.abs() + mag * (RATIO_RTOL if q.is_w else 64 * EPS32) + bias + 1e-38
            assert (got - ref.detach().view(-1)).abs().le(tol).all(), q.index
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("opt", ["lars", "lamb"])
def test_zero_weight_and_zero_gradient_give_ratio_one(opt):
    kw = LARS_KW if opt == "lars" else LAMB_KW
    eng = _engine(dict(kw, code="sgd"))
    names = [n for n, _ in _weights(eng)]
    q0 = _weights(eng)[0][1]
    eng.master[q0.off:q0.off + q0.numel].zero_()       # ||w|| = 0: ratio 1 and no NaN
    eng.wshadow[q0.off:q0.off + q0.numel].zero_()
    _step(eng)
    r = eng.trust_ratios()
    assert r[names[0]] == 1.0
    assert all(math.isfinite(v) for v in r.values())
    assert torch.isfinite(eng.master).all()
    eng.close()
    # the first BN's gamma at 0 makes the first convolution's gradient exactly 0: with wd = 0, LARS' denominator
    # ||g|| + wd ||w|| and LAMB's u are 0, and the ratio is 1
    eng = _engine(dict(kw, code="sgd", weight_decay=0.0))
    gamma = next(p for n, p in eng.model.named_parameters() if p.dim() == 1 and n.endswith("weight"))
    with torch.no_grad():
        gamma.zero_()
    _step(eng)
    assert not bool(eng.params[0].grad.ne(0).any())
    r = eng.trust_ratios()
    assert r[names[0]] == 1.0
    assert all(math.isfinite(v) for v in r.values())
    assert torch.isfinite(eng.master).all()
    eng.close()


def _run(kw, graph, steps=4, **extra):
    eng = _engine(kw, graph=graph, **extra)
    for _ in range(steps):
        _step(eng)
    out = {"master": eng.master.cpu(), "mom": eng.mom.cpu(), "wshadow": eng.wshadow.cpu(),
           "vparams": eng.vparams.cpu(), "ratio": eng.lw_ratio.cpu()}
    if eng.sq is not None:
        out["sq"] = eng.sq.cpu()
    eng.close()
    return out


def _equal(a, b):
    return [k for k in a if not torch.equal(a[k], b[k])]


@pytest.mark.gpu
@pytest.mark.parametrize("opt,code", [("lars", "svd"), ("lamb", "topk")])
def test_bitwise_repeatable_and_graph_equals_eager(code, opt, deterministic_cudnn):
    kw = dict(LARS_KW if opt == "lars" else LAMB_KW, **CODES[code])
    a, b = _run(kw, False), _run(kw, False)
    assert _equal(a, b) == []
    c = _run(kw, True)
    assert _equal(a, c) == []


@pytest.mark.gpu
@pytest.mark.parametrize("opt", ["lars", "lamb"])
@pytest.mark.parametrize("extra", [dict(code="svd", accumulate_steps=2),
                                   dict(code="topk", entry_budget=0.01, error_feedback=True)])
def test_accumulation_and_error_feedback(opt, extra):
    kw = LARS_KW if opt == "lars" else LAMB_KW
    eng = _engine(dict(kw, **extra))
    for _ in range(3):
        pre = _snapshot(eng)
        _step(eng)
        _check_rule(eng, pre, kw)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("opt,extra", [("lars", dict(code="svd")),
                                       ("lamb", dict(code="topk", entry_budget=0.01, error_feedback=True))])
def test_resume_is_bitwise(opt, extra, tmp_path, deterministic_cudnn):
    kw = dict(LARS_KW if opt == "lars" else LAMB_KW, **extra)
    d = str(tmp_path) + "/"
    a = _run(kw, True, steps=4)
    eng = _engine(kw, graph=True)
    for _ in range(2):
        _step(eng)
    eng.save_checkpoint(d)
    eng.close()
    side = torch.load(ckpt.model_path(d, 2) + "_optim", weights_only=False)
    assert side["optimizer"] == opt and ("sq_w" in side) == (opt == "lamb")
    eng = _engine(kw, graph=True)
    eng.load_checkpoint(d, 2)
    for _ in range(2):
        _step(eng)
    c = {"master": eng.master.cpu(), "mom": eng.mom.cpu(), "wshadow": eng.wshadow.cpu(),
         "vparams": eng.vparams.cpu(), "ratio": eng.lw_ratio.cpu()}
    if eng.sq is not None:
        c["sq"] = eng.sq.cpu()
    eng.close()
    assert _equal(a, c) == []
    # another optimizer's checkpoint is refused, both ways
    other = _engine(dict(extra, lr=0.05, momentum=0.9), graph=False)
    with pytest.raises(ValueError, match="written by optimizer %s" % opt):
        other.load_checkpoint(d, 2)
    other.close()


# ---------------------------------------------------------------------------------------------------- two GPUs
def _mp_sharded(rank, world, port, opt, out):
    import torch.distributed as dist
    nccl_init(rank, world, port)
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    kw = dict(LARS_KW if opt == "lars" else LAMB_KW, code="svd")
    eng = ShadowEngine(build_model("ResNet18", 10), rank, world, use_graph=True, seed=7, ps_mode="sharded", **kw)
    x, y = _batch(rank)
    eng.prepare(x, y, warmup=0)
    for _ in range(3):
        x, y = _batch(eng.step + rank)
        eng.train_step(x, y)
    torch.cuda.synchronize()
    out.put((rank, eng.error_code(), eng.lw_ratio.cpu(), eng.wshadow.cpu()))
    eng.close()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("opt", ["lars", "lamb"])
def test_two_owners_agree_on_the_ratios(opt):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    port = 29680 + (opt == "lamb")
    res = spawn(2, _mp_sharded, port, opt)
    (_, e0, r0, w0), (_, e1, r1, w1) = res
    assert e0 == 0 and e1 == 0
    assert torch.equal(r0, r1) and torch.equal(w0, w1)

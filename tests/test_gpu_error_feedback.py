"""Error feedback on the bf16 engine (``ShadowEngine(error_feedback=True)``, csrc/v2_feedback.cu and the encoders'
residual epilogues): the refusals and the launcher flag (CPU); the per-step identity ``g + e_old == g_hat + e_new``,
telescoping over many steps, "off means off", training under graph replay, ``--code-stats`` on the coded input and
the launcher's metrics record (GPU)."""
import argparse
import json
import math

import pytest
import torch

from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils.flags import add_fit_args

from shadow_harness import SVD3, Loopback, ef_grads, fit_args, forbid_cuda


# ---------------------------------------------------------------------------------------------------- CPU
def test_error_feedback_flag_parses():
    assert add_fit_args(argparse.ArgumentParser(), []).error_feedback is False
    assert add_fit_args(argparse.ArgumentParser(), ["--error-feedback", "1"]).error_feedback is True
    assert add_fit_args(argparse.ArgumentParser(), ["--error-feedback", "0"]).error_feedback is False


@pytest.mark.parametrize("kw,match", [(dict(code="qsvd"), "QSVD"), (dict(code="terngrad"), "TernGrad"),
                                      (dict(code="sgd"), "nothing to feed back"),
                                      (dict(code="svd", world=4, num_aggregate=2), "num_aggregate"),
                                      (dict(code="qsgd", world=3, ps_mode="dedicated", num_aggregate=1),
                                       "num_aggregate")])
def test_shadow_engine_refuses_codes_without_feedback(kw, match, monkeypatch):
    """Checked before any CUDA work, so a bad setting fails the same way on every machine."""
    from atomo_b200.runtime import shadow_engine as S
    forbid_cuda(monkeypatch)
    kw = dict(kw)
    world = kw.pop("world", 1)
    with pytest.raises(ValueError, match=match):
        S.ShadowEngine(None, 0, world, error_feedback=True, **kw)


def test_fused_engine_refuses_the_flag(tmp_path):
    model = torch.nn.Linear(4, 4)
    for extra in (("--engine", "fused", "--dtype", "bf16"), ("--dtype", "fp32")):
        with pytest.raises(SystemExit, match="--error-feedback"):
            L._build_engine(fit_args(tmp_path, *SVD3, "--error-feedback", "1", *extra), model, 0, 1)


def test_role_backends_refuse_the_flag(monkeypatch, tmp_path):
    from atomo_b200 import distributed_nn
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    with pytest.raises(SystemExit, match="--error-feedback"):
        distributed_nn.run_rank(fit_args(tmp_path, *SVD3, "--error-feedback", "1", "--backend", "gloo"))


# ---------------------------------------------------------------------------------------------------- GPU harness
CODES = [("svd", dict(svd_rank=3)), ("svd", dict(svd_rank=1, random_sample=False)),
         ("svd", dict(svd_rank=2, random_sample=False)), ("entrywise", dict(entry_budget=0.05)),
         ("entrywise", dict(entry_budget=0.01)), ("qsgd", dict(quantization_level=2)),
         ("qsgd", dict(quantization_level=4, bucket_size=128))]


# ---------------------------------------------------------------------------------------------------- GPU: kernels
@pytest.mark.gpu
@pytest.mark.parametrize("code,kw", CODES)
def test_per_step_identity(code, kw):
    """g + e_old == g_hat + e_new for every weight element, step after step: what is not pushed stays owed."""
    h = Loopback(code, ef_grads(1), **kw)
    try:
        g = h.g
        e_old = h.residual()
        for _ in range(4):
            ghat, e_new = h.step()
            lhs, rhs = g + e_old, ghat + e_new
            # fp32 rounding of the terms: A = g + e, the reconstruction's products and sums, e += A - g_hat
            scale = g.abs() + e_old.abs() + ghat.abs() + e_new.abs()
            tol = 1e-6 * scale + 1e-7 * float(scale.max())
            bad = (lhs - rhs).abs() > tol
            assert not bool(bad.any()), ((lhs - rhs).abs().max().item(), int(bad.sum()))
            assert float(e_new.norm()) > 0        # every code here drops something
            e_old = e_new
        n = h.eng.error_feedback_norm()
        assert n["model"] == pytest.approx(float(e_old.norm()), rel=1e-5)
        assert len(n["tensors"]) == len(h.w)
    finally:
        h.close()


@pytest.mark.gpu
def test_telescoping_topk_rank1():
    """A fixed gradient for T = 200 steps: the pushed sum misses T g by exactly the final residual (the sum
    telescopes), which stays bounded; without error feedback the same top-k code misses by T ||g - g_hat||."""
    T = 200
    grads = ef_grads(2)
    sums, norms = {}, {}
    for ef in (True, False):
        h = Loopback("svd", grads, ef=ef, svd_rank=1, random_sample=False)
        try:
            s = torch.zeros_like(h.g)
            for _ in range(T):
                ghat, e = h.step()
                s += ghat
            sums[ef], norms[ef] = s - T * h.g, e
            if not ef:
                miss_one = float((ghat - h.g).norm())
        finally:
            h.close()
    e_T = norms[True]
    assert torch.allclose(sums[True], -e_T, rtol=0, atol=T * 1e-6 * (float(h.g.abs().max()) + float(e_T.abs().max())))
    assert float(sums[True].norm()) == pytest.approx(float(e_T.norm()), rel=1e-3)
    # bounded: rank-1 top-k keeps at least 1/cols of ||A||^2 on every unit (cols <= 64), a contraction with
    # ||e|| <= sqrt(1 - d) / (1 - sqrt(1 - d)) ||g||; in practice far below
    d = 1.0 / 64
    bound = math.sqrt(1 - d) / (1 - math.sqrt(1 - d)) * float(h.g.norm())
    assert float(e_T.norm()) <= bound
    assert float(sums[False].norm()) == pytest.approx(T * miss_one, rel=1e-4)
    assert float(sums[False].norm()) > 3 * float(e_T.norm())


@pytest.mark.gpu
@pytest.mark.parametrize("code,kw", CODES)
def test_off_means_off(code, kw):
    """With e = 0 the apply pass writes the gradient back unchanged and the epilogues only touch the residual: the
    first step pushes the same bits with the option on as with it off (arena, gradient buffers, reconstructed master)."""
    out = {}
    for ef in (False, True):
        h = Loopback(code, ef_grads(3), ef=ef, **kw)
        try:
            ghat, _ = h.step()
            arena = h.eng.heap.tensor("arena").clone()
            gb = [p.grad.clone() for p in h.eng.w_params]
            out[ef] = (ghat, arena, gb)
        finally:
            h.close()
    assert torch.equal(out[False][0], out[True][0])
    assert torch.equal(out[False][1], out[True][1])
    assert all(torch.equal(a, b) for a, b in zip(out[False][2], out[True][2]))


# ---------------------------------------------------------------------------------------------------- GPU: engine
def _train(net, code, graph, overlap, steps=6, **kw):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model, input_shape
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    x, y = SyntheticImageDataset(input_shape(net), 10, 4096, seed=0).materialize(32)
    eng = ShadowEngine(build_model(net, 10), 0, 1, code=code, lr=0.05, momentum=0.9, use_graph=graph, overlap=overlap,
                       seed=3, error_feedback=True, **kw)
    eng.prepare(x.pin_memory(), y.pin_memory(), warmup=2)
    losses = []
    for _ in range(steps):
        losses.append(float(eng.train_step(x, y)[0]))
    torch.cuda.synchronize()
    assert eng.error_code() == 0
    m = eng.gather_fp32("master").clone()
    r = eng.residual.clone()
    eng.close()
    return m, r, losses


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["ResNet18", "VGG11"])
@pytest.mark.parametrize("code,kw", [("svd", dict(svd_rank=3)), ("entrywise", dict(entry_budget=0.01)),
                                     ("qsgd", dict(quantization_level=2))])
def test_graph_replay_equals_eager(net, code, kw, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    mg, rg, _ = _train(net, code, True, True, **kw)
    me, re_, _ = _train(net, code, False, False, **kw)
    assert torch.equal(mg, me) and torch.equal(rg, re_)
    assert float(rg.norm()) > 0


@pytest.mark.gpu
def test_loss_falls_on_a_fixed_batch():
    # top-k rank 1: a contraction, so the residual stays bounded (an unbiased code whose relative variance exceeds 1
    # makes the residual grow step after step; profiles/README.md)
    _, _, losses = _train("ResNet18", "svd", True, True, steps=30, svd_rank=1, random_sample=False)
    assert all(math.isfinite(l) for l in losses)
    assert losses[-1] < losses[0], losses


@pytest.mark.gpu
@pytest.mark.parametrize("code,kw", [("svd", dict(svd_rank=3)), ("entrywise", dict(entry_budget=0.05)),
                                     ("qsgd", dict(quantization_level=2))])
def test_code_stats_describe_the_coded_input(code, kw):
    """With error feedback the encoders read bf16(g + e): --code-stats' gsq is ||bf16(A)||^2."""
    h = Loopback(code, ef_grads(4), code_stats=True, **kw)
    try:
        h.step()                        # e != 0 from here on
        h.eng.code_stats(reset=True)
        h.step()
        st = h.eng.code_stats()
        names = {id(p): n for n, p in h.eng.model.named_parameters()}
        checked = 0
        for p in h.eng.w_params:       # after an eager step the gradient buffers hold bf16(A)
            t = st["tensors"][names[id(p)]]
            if t["gsq"] is None:
                continue
            want = float(p.grad.double().square().sum())
            assert t["gsq"] == pytest.approx(want, rel=1e-6)
            checked += 1
        assert checked >= 4
        assert float(h.residual().norm()) > 0
    finally:
        h.close()


@pytest.mark.gpu
def test_launcher_writes_ef_norm(tmp_path, monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    args = add_fit_args(argparse.ArgumentParser(), [
        "--network", "ResNet18", "--dataset", "Cifar10", "--synthetic", "1", "--train-len", "512", "--test-len", "64",
        "--batch-size", "32", "--test-batch-size", "64", "--code", "svd", "--svd-rank", "3", "--backend", "p2p",
        "--dtype", "bf16", "--max-steps", "6", "--log-interval", "2", "--eval-freq", "100", "--error-feedback", "1",
        "--train-dir", str(tmp_path) + "/", "--metrics-file", str(tmp_path / "m")])
    L.run_p2p_training(args)
    recs = [json.loads(l) for l in open(str(tmp_path / "m") + ".rank0.jsonl")]
    assert recs and all(r["ef_norm"] > 0 and math.isfinite(r["ef_norm"]) for r in recs)

"""Estimator statistics of the bf16 engine (``ShadowEngine(code_stats=True)``, csrc/v2_stats.cu) on the GPU: the
kernel against an fp64 evaluation of the closed forms on seeded bf16 gradients, the closed form against the engine's
own sampled decodes, realized atom counts against the slot headers / selcount, training bits unchanged, and the
launcher's metrics record."""
import argparse
import json
import math

import numpy as np
import pytest
import torch

from atomo_b200.ops import plan2 as P

from shadow_harness import Linear, nccl_init, spawn

pytestmark = pytest.mark.gpu

# stem, 3x3 convs (one a multiple of 4096 elements, one not, one with a spike), fc layers, a tensor smaller than an
# absolute budget, a coded conv that is all zero, a vector
SHAPES = [(64, 3, 3, 3), (64, 32, 3, 3), (128, 64, 3, 3), (10, 512), (300, 200), (7, 20), (32, 16, 3, 3), (64,)]
SPIKE, ZERO = 1, 6


def _grads(seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i, s in enumerate(SHAPES):
        x = torch.randn(s, generator=g) * (0.01 * (1 + i))
        if i == SPIKE:
            x.view(-1)[123] = 5.0
        if i == ZERO:
            x.zero_()
        out.append(x.bfloat16().float().cuda())     # bf16-representable: the engine's gradient is exactly this
    return out


def _engine(code, grads, lr=0.0, **kw):
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.cuda.set_device(0)
    eng = ShadowEngine(Linear(grads), 0, 1, code=code, lr=lr, momentum=0.0, use_graph=False, overlap=False,
                       warm_start=False, code_stats=True, criterion=lambda lg, y: lg[0, 0], **kw)
    x, y = torch.zeros(4, 2), torch.zeros(4, dtype=torch.long)
    eng.prepare(x, y, warmup=0)
    return eng, x, y


def _phys(g):
    g = g.cpu()
    return (g.permute(0, 2, 3, 1) if g.dim() == 4 else g).reshape(-1).double()


def _unit_matrix(u, g):
    """The unit's tall matricization in fp64 (singular values do not depend on row / column order)."""
    g = g.cpu()
    if u.kind == P.KIND_SLAB:
        o, i = g.shape[0], g.shape[1]
        w = g.permute(0, 2, 3, 1).reshape(o, u.K, i // 2, 2)
        return w.permute(0, 2, 3, 1).reshape(o * i // 2, 2 * u.K).double()
    m = g.reshape(g.shape[0], -1).double()
    if u.rs == 1:                   # rows = inputs: the transposed matrix
        m = m.t()
    c0 = u.g_off // u.cs
    return m[:, c0:c0 + u.cols]


def _acc(eng):
    return eng.stats_acc.view(-1, eng.C.v2_stats_fields()).cpu().double()


def _close(a, b, rel):
    return abs(a - b) <= rel * max(abs(a), abs(b)) + 1e-300


# ---------------------------------------------------------------------------------------------------- kernel vs closed form
@pytest.mark.parametrize("rule,sampling,random", [("reference", "bernoulli", True), ("waterfill", "bernoulli", True),
                                                  ("reference", "systematic", True), ("waterfill", "systematic", True),
                                                  ("reference", "bernoulli", False)])
@pytest.mark.parametrize("rank", [1, 3])
def test_svd_stats_match_the_closed_form(rule, sampling, random, rank):
    grads = _grads()
    eng, x, y = _engine("svd", grads, svd_rank=rank, prob_rule=rule, sampling=sampling, random_sample=random)
    eng.train_step(x, y)
    torch.cuda.synchronize()
    acc, sig = _acc(eng), eng.sigma.view(-1, P.MAX_COLS).cpu().double()
    sel = eng.selcount.cpu()
    seen = 0
    for u in eng.plan.units:
        if not u.coded:
            continue
        seen += 1
        gsq, mse, ex, bias, real, real4, n = acc[u.ts_index].tolist()
        g = grads[u.param]
        m = _unit_matrix(u, g)
        assert n == 1 and bias == 0 and real == int(sel[u.ts_index])
        assert _close(gsq, float((m * m).sum()), 1e-9)
        if u.param == ZERO:
            assert gsq == 0 and mse == 0
            continue

        def closed(s):
            s = np.sort(np.asarray(s, dtype=np.float64))[::-1]
            n_ = len(s)
            if not random:
                k = min(int(u.budget), n_, u.rcap)
                return float((s[k:] ** 2).sum()), float(k)
            if rule == "reference":
                p = np.minimum(1.0, u.budget * s / s.sum())
            else:
                bud, rest, pin = min(u.budget, n_), s.sum(), 0
                while pin < n_ and rest > 0 and (bud - pin) * s[pin] >= rest and bud - pin > 0:
                    rest -= s[pin]
                    pin += 1
                p = np.where(np.arange(n_) < pin, 1.0, np.minimum(1.0, (bud - pin) * s / rest) if rest > 0 else 0.0)
            pos = p > 0
            return float((s[pos] ** 2 * (1 / p[pos] - 1)).sum() + (s[~pos] ** 2).sum()), float(p.sum())

        m_sig, e_sig = closed(sig[u.ts_index, :u.cols].numpy())
        assert _close(mse, m_sig, 1e-6) and _close(ex, e_sig, 1e-6), (u.index, mse, m_sig, ex, e_sig)
        # a cold full Jacobi solve (warm_start=False) against LAPACK in fp64
        m_ref, e_ref = closed(torch.linalg.svdvals(m).numpy())
        assert _close(mse, m_ref, 1e-3) and _close(ex, e_ref, 1e-3), (u.index, mse, m_ref, ex, e_ref)
    assert seen >= 5
    eng.close()


@pytest.mark.parametrize("budget", [0.01, 0.05, 0.25, 200.0])
def test_entrywise_stats_match_the_closed_form(budget):
    from atomo_b200.codings.entrywise import EntryWise
    grads = _grads(1)
    eng, x, y = _engine("entrywise", grads, entry_budget=budget)
    eng.train_step(x, y)
    torch.cuda.synchronize()
    acc, l1 = _acc(eng), eng.l1.cpu()
    arena = eng.heap.tensor("arena").view(torch.int32).cpu()
    coder = EntryWise(budget)
    for u in eng.plan.units:
        if u.kind != P.KIND_ENTRY:
            continue
        g = _phys(grads[u.param])
        gsq, mse, ex, bias, real, real4, n = acc[u.ts_index].tolist()
        s = coder.atoms_for(u.numel)
        assert s == u.budget and _close(float(l1[u.ts_index]), float(g.abs().sum()), 1e-12)
        # the unit table carries s as fp32, and the encoder forms k = s / L1 from that value
        s32 = float(np.float32(s))
        k = np.float32(s32 / float(l1[u.ts_index])) if float(l1[u.ts_index]) > 0 else np.float32(0)
        p = np.minimum(np.abs(g.float().numpy()) * k, np.float32(1)).astype(np.float64)
        g2 = g.numpy() ** 2
        pos = p > 0
        want_mse = float((g2[pos] * (1 / p[pos] - 1)).sum() + g2[~pos].sum())
        assert _close(gsq, float(g2.sum()), 1e-9) and _close(mse, want_mse, 1e-9) and _close(ex, float(p.sum()), 1e-9)
        hdr = sum(int(arena[u.slot_off + 4 * j + 1]) for j in range(u.n_ps))
        assert bias == 0 and real == hdr == real4
        if u.param == ZERO:
            assert gsq == mse == ex == real == 0
    eng.close()


@pytest.mark.parametrize("code,q,bucket", [("qsgd", 2, 512), ("qsgd", 4, 512), ("qsgd", 8, 512), ("qsgd", 4, 96),
                                           ("terngrad", 1, 512)])
def test_qsgd_stats_match_the_closed_form(code, q, bucket):
    grads = _grads(2)
    eng, x, y = _engine(code, grads, quantization_level=q, bucket_size=bucket)
    eng.train_step(x, y)
    torch.cuda.synchronize()
    acc = _acc(eng)
    arena = eng.heap.tensor("arena").cpu()
    s = (1 << q) - 1
    for u in eng.plan.units:
        if u.kind != P.KIND_QSGD:
            continue
        g = _phys(grads[u.param])
        v = g
        if code == "terngrad":
            c = float(eng.clip[u.ts_index])
            assert _close(c, 2.5 * float(g.std(unbiased=False)), 1e-6) or u.param == ZERO
            v = g.float().clamp(-c, c).double() if c > 0 else g
        nb = u.rows
        norms = arena[u.slot_off + P.qsgd_norms_off(u.n_ps):][:nb].double()
        pad = torch.zeros(nb * u.K, dtype=torch.float64)
        pad[:u.numel] = v
        w = pad.view(nb, u.K)
        ref_norm = w.abs().amax(1) if code == "terngrad" else w.norm(dim=1)
        assert torch.allclose(norms, ref_norm, rtol=1e-5, atol=0)
        safe = torch.where(norms > 0, norms, torch.ones_like(norms)).unsqueeze(1)
        a = (w.abs() / safe * s).clamp(max=s)
        f = a - a.floor()
        want = float(((norms.unsqueeze(1) / s) ** 2 * f * (1 - f)).sum())
        gsq, mse, ex, bias, real, real4, n = acc[u.ts_index].tolist()
        assert _close(gsq, float((g * g).sum()), 1e-9) and _close(mse, want, 1e-9), (u.index, mse, want)
        assert _close(bias, float(((v - g) ** 2).sum()), 1e-9) and ex == real == u.numel
        if u.param == ZERO:
            assert gsq == mse == bias == 0
    eng.close()


# ---------------------------------------------------------------------------------------------------- closed form vs sampling
@pytest.mark.parametrize("code,kw", [("svd", dict(svd_rank=2)), ("svd", dict(svd_rank=2, sampling="systematic")),
                                     ("entrywise", dict(entry_budget=0.05)), ("qsgd", dict(quantization_level=2)),
                                     ("terngrad", {})])
def test_closed_form_matches_400_sampled_decodes(code, kw):
    """lr = 1, momentum 0, master zeroed before each step: after the step the master is minus the decoded gradient."""
    grads = _grads(3)
    eng, x, y = _engine(code, grads, lr=1.0, **kw)
    eng.code_stats(reset=True)
    names = [n for n, _ in eng.model.named_parameters()]
    errs, atoms, stats = {n: [] for n in names}, {n: [] for n in names}, None
    for _ in range(400):
        eng.master.zero_()
        torch.cuda.synchronize()
        eng.train_step(x, y)
        torch.cuda.synchronize()
        st = eng.code_stats(reset=True)
        stats = st if stats is None else stats
        for q, n in zip(eng.plan.params, names):
            if q.is_w:
                dec = -eng.master[q.off:q.off + q.numel].double().cpu()
                errs[n].append(float(((dec - _phys(grads[q.index])) ** 2).sum()))
                atoms[n].append(st["tensors"][n]["atoms"])
    assert eng.error_code() == 0
    checked = 0
    for n in names:
        t = stats["tensors"][n]
        if t["gsq"] is None or t["gsq"] == 0:
            continue
        e, a = np.array(errs[n]), np.array(atoms[n])
        want = t["mse"] + t["bias_sq"]
        se = e.std(ddof=1) / math.sqrt(len(e))
        assert abs(e.mean() - want) <= 5 * se + 1e-6 * want, (n, e.mean(), want, se)
        # systematic sampling sends floor or ceil of sum(p_i), and sum(p_i) is an fp32 sum: 1e-6 of slack
        ase = a.std(ddof=1) / math.sqrt(len(a))
        assert abs(a.mean() - t["exp_atoms"]) <= 5 * ase + 1e-6 * t["exp_atoms"], (n, a.mean(), t["exp_atoms"], ase)
        checked += 1
    assert checked >= 4
    eng.close()


def test_svd_rel_var_does_not_grow_with_the_rank():
    grads = _grads(4)
    rv = []
    for r in (1, 2, 3, 4, 8):
        eng, x, y = _engine("svd", grads, svd_rank=r)
        eng.train_step(x, y)
        st = eng.code_stats()
        assert all(math.isfinite(v) for v in (st["model"]["mse"], st["model"]["gsq"], st["model"]["rel_var"]))
        rv.append(st["model"]["rel_var"])
        eng.close()
    assert all(b <= a * (1 + 1e-6) for a, b in zip(rv, rv[1:])), rv


# ---------------------------------------------------------------------------------------------------- training unchanged
def _train(net, code, graph, overlap, stats, steps=6, **kw):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model, input_shape
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    x, y = SyntheticImageDataset(input_shape(net), 10, 4096, seed=0).materialize(32)
    eng = ShadowEngine(build_model(net, 10), 0, 1, code=code, lr=0.05, momentum=0.9, use_graph=graph, overlap=overlap,
                       seed=3, code_stats=stats, **kw)
    eng.prepare(x.pin_memory(), y.pin_memory(), warmup=2)
    for _ in range(steps):
        eng.train_step(x, y)
    torch.cuda.synchronize()
    assert eng.error_code() == 0
    m = eng.gather_fp32("master").clone()
    st = eng.code_stats() if stats else None
    eng.close()
    return m, st


@pytest.mark.parametrize("net,code,kw", [("ResNet18", "svd", dict(svd_rank=3)), ("ResNet18", "entrywise", {}),
                                         ("ResNet18", "qsgd", {}), ("VGG11", "terngrad", {})])
@pytest.mark.parametrize("graph,overlap", [(True, True), (False, False)])
def test_code_stats_leave_training_bitwise_unchanged(net, code, kw, graph, overlap, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    off, _ = _train(net, code, graph, overlap, False, **kw)
    on, st = _train(net, code, graph, overlap, True, **kw)
    assert torch.equal(off, on)
    assert st["steps"] == 8
    for t in list(st["tensors"].values()) + [st["model"]]:
        for k in ("mse", "bias_sq", "exp_atoms", "atoms", "bytes"):
            assert math.isfinite(t[k]) and t[k] >= 0, (k, t)
    assert st["model"]["gsq"] > 0 and 0 <= st["model"]["rel_var"] < math.inf


def test_sgd_reports_exact_dense_tensors():
    m, st = _train("ResNet18", "sgd", False, False, True, steps=1)
    assert st["model"]["mse"] == 0 and st["model"]["gsq"] == 0
    assert all(t["gsq"] is None for t in st["tensors"].values())
    assert st["model"]["bytes"] > 0


# ---------------------------------------------------------------------------------------------------- launcher
def test_launcher_writes_code_stats_into_the_metrics_file(tmp_path, monkeypatch, capsys):
    from atomo_b200.runtime import p2p_launcher as L
    from atomo_b200.utils.flags import add_fit_args
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    args = add_fit_args(argparse.ArgumentParser(), [
        "--network", "ResNet18", "--dataset", "Cifar10", "--synthetic", "1", "--train-len", "512", "--test-len", "64",
        "--batch-size", "32", "--test-batch-size", "64", "--code", "svd", "--svd-rank", "3", "--backend", "p2p",
        "--dtype", "bf16", "--max-steps", "6", "--log-interval", "2", "--eval-freq", "100", "--code-stats", "1",
        "--train-dir", str(tmp_path) + "/", "--metrics-file", str(tmp_path / "m")])
    L.run_p2p_training(args)
    recs = [json.loads(l) for l in open(str(tmp_path / "m") + ".rank0.jsonl")]
    assert recs and all("code_stats" in r for r in recs)
    cs = recs[-1]["code_stats"]
    assert cs["code"] == "svd" and cs["steps"] == 2 and cs["model"]["gsq"] > 0
    assert "conv1.weight" in cs["tensors"] or any(k.endswith("weight") for k in cs["tensors"])


# ---------------------------------------------------------------------------------------------------- multi GPU
def _mp_worker(rank, world, port, code, out):
    import torch.distributed as dist
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    nccl_init(rank, world, port)
    torch.manual_seed(0)
    x, y = SyntheticImageDataset((3, 32, 32), 10, 4096, seed=rank).materialize(32)
    eng = ShadowEngine(build_model("VGG11", 10), rank, world, code=code, lr=0.05, momentum=0.9, use_graph=False,
                       seed=3, code_stats=True)
    eng.prepare(x.pin_memory(), y.pin_memory(), warmup=0)
    eng.code_stats(reset=True)
    eng.train_step(x, y)
    torch.cuda.synchronize()
    st = eng.code_stats(reset=False)
    ok = eng.error_code() == 0 and all(math.isfinite(t[k]) for t in st["tensors"].values()
                                       for k in ("mse", "atoms", "bytes"))
    if code == "entrywise":       # realized atoms = this worker's tile headers, summed over every owner's arena
        acc = eng.stats_acc.view(-1, eng.C.v2_stats_fields()).cpu()
        arenas = [eng.heap.tensor("arena", torch.int32, rank=r).cpu() for r in range(world)]
        for u in eng.plan.units:
            if u.kind == P.KIND_ENTRY:
                base = eng.worker_index * eng.plan.arena_floats + u.slot_off
                hdr = sum(int(arenas[(u.own0 + j) % world][base + 4 * j + 1]) for j in range(u.n_ps))
                ok = ok and int(acc[u.ts_index, 4]) == hdr
    dist.barrier()
    eng.close()
    dist.destroy_process_group()
    out.put((rank, ok))


@pytest.mark.multigpu
@pytest.mark.parametrize("code", ["svd", "entrywise"])
def test_code_stats_on_every_rank(code):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    port = 29840 + (3 if code == "entrywise" else 0)
    res = spawn(2, _mp_worker, port, code, timeout=300)
    assert all(ok for _, ok in res), res

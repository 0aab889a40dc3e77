"""Gradient accumulation on the bf16 engine (``ShadowEngine(accumulate_steps=N)``, ``--accumulate-steps``,
csrc/v2_accum.cu).

CPU: the refusals before any CUDA work, and the launcher loop drawing ``N * --batch-size`` samples per step.
GPU: ``N = 1`` is the engine without the option; the buffer each encoder reads equals the fp32 oracle
``bf16(fp32(sum_j g_j) * fp32(1/N) (+ e))`` bit for bit; graph replay equals eager; N micro-batches of b match one
batch of N b; a resume is bitwise; the peak memory falls.
"""
import argparse
import functools
import types

import numpy as np
import pytest
import torch

from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils.flags import add_fit_args

from shadow_harness import SVD3, StandInEngine, deterministic_cudnn, differs, engine_batch, fit_args, forbid_cuda, \
    make_engine, nccl_init, spawn  # noqa: F401

FLT_MIN = float(np.finfo(np.float32).tiny)


# ---------------------------------------------------------------------------------------------------- CPU
def test_accumulate_flag_parses():
    assert add_fit_args(argparse.ArgumentParser(), []).accumulate_steps == 1
    assert add_fit_args(argparse.ArgumentParser(), ["--accumulate-steps", "4"]).accumulate_steps == 4


@pytest.mark.parametrize("n", [0, -1, 1.5, True])
def test_engine_refuses_bad_accumulate_steps(n, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    forbid_cuda(monkeypatch)
    with pytest.raises(ValueError, match="accumulate_steps"):
        S.ShadowEngine(None, 0, 1, accumulate_steps=n)


def test_prepare_refuses_an_indivisible_batch():
    """Checked first thing in prepare(), before any tensor is made on the device."""
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    eng = types.SimpleNamespace(accum=3)
    with pytest.raises(ValueError, match="divisible"):
        ShadowEngine.prepare(eng, torch.zeros(8, 3, 4, 4), torch.zeros(8, dtype=torch.long))


def test_fused_engine_and_fp32_refuse_the_flag(tmp_path):
    model = torch.nn.Linear(4, 4)
    for extra in (("--engine", "fused", "--dtype", "bf16"), ("--dtype", "fp32"),
                  ("--dtype", "bf16", "--code", "entrywise")):        # auto sends entrywise to the fp32-flat engine
        with pytest.raises(SystemExit, match="--accumulate-steps"):
            L._build_engine(fit_args(tmp_path, *SVD3, "--accumulate-steps", "2", *extra), model, 0, 1)


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_role_backends_refuse_the_flag(backend, monkeypatch, tmp_path):
    from atomo_b200 import distributed_nn
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    with pytest.raises(SystemExit, match="--accumulate-steps"):
        distributed_nn.run_rank(fit_args(tmp_path, *SVD3, "--accumulate-steps", "2", "--backend", backend))


class BatchStandIn(StandInEngine):
    """Records the batch sizes it is given."""

    def __init__(self, model, args):
        super().__init__(model, args)
        self.batches = []

    def train_step(self, x, y):
        self.batches.append(x.shape[0])
        return super().train_step(x, y)


def test_launcher_draws_n_micro_batches_per_step(tmp_path, monkeypatch, capsys):
    import re
    StandInEngine.instances.clear()
    monkeypatch.setattr(L, "_build_engine", lambda args, model, rank, world: (BatchStandIn(model, args), "fused"))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    L.run_p2p_training(fit_args(tmp_path, *SVD3, "--max-steps", "6", "--accumulate-steps", "4"), device="cpu")
    eng = StandInEngine.instances[-1]
    assert eng.batches and set(eng.batches) == {4 * 32}
    recs = [re.match(r"Worker: 0, Step: (\d+), Epoch: \d+ \[(\d+)/(\d+)", l)
            for l in capsys.readouterr().out.splitlines() if l.startswith("Worker: 0, Step:")]
    steps = [int(m.group(1)) for m in recs]
    assert steps == [3, 4, 5, 6]        # 2 warm-up steps count as steps
    # the sample position advances by N * --batch-size per step
    assert [int(m.group(2)) for m in recs] == [(s * 4 * 32) % 512 for s in steps]
    assert all(int(m.group(3)) == 512 for m in recs)


# ---------------------------------------------------------------------------------------------------- GPU helpers
CODE_KW = {"svd": dict(svd_rank=3), "qsvd": dict(svd_rank=3), "sgd": {}, "qsgd": dict(quantization_level=2),
           "terngrad": {}, "entrywise": dict(entry_budget=0.05), "topk": dict(entry_budget=0.01), "sign": {},
           "powersgd": dict(svd_rank=2), "fp8": {}, "hadamard": dict(quantization_level=4)}
EF_CODES = ("svd", "qsgd", "entrywise", "topk", "sign", "powersgd", "fp8", "hadamard")

_batch = functools.partial(engine_batch, seed=200)


def _engine(net, **kw):
    return make_engine(net, **dict(dict(lr=0.05, momentum=0.9), **kw))


def _state(eng) -> dict:
    out = {"master": eng.master.clone(), "mom": eng.mom.clone(), "wshadow": eng.wshadow.clone(),
           "vparams": eng.vparams.clone(), "vmom": eng.vmom.clone(), "loss": eng.loss_buf.clone()}
    for name, b in eng.model.named_buffers():
        out["buffer:" + name] = b.clone()
    for name, t in eng._worker_tensors().items():
        out["worker:" + name] = t.clone()
    return out


def _run(net, steps, batch, warmup=2, **kw):
    eng = _engine(net, **kw)
    x, y = _batch(net, 0, batch)
    eng.prepare(x, y, warmup=warmup)
    for _ in range(steps):
        x, y = _batch(net, eng.step, batch)
        eng.train_step(x, y)
    torch.cuda.synchronize()
    assert eng.error_code() == 0
    st, n = _state(eng), eng.launches_per_step
    eng.close()
    return st, n


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("code,ef", [("svd", False), ("topk", True)])
def test_one_micro_batch_is_the_engine_without_the_option(code, ef, graph, deterministic_cudnn):
    kw = dict(code=code, error_feedback=ef, use_graph=graph, **CODE_KW[code])
    a, na = _run("ResNet18", 4, 32, **kw)
    b, nb = _run("ResNet18", 4, 32, accumulate_steps=1, **kw)
    assert na == nb
    assert differs(a, b) == []


def ftz(t):
    """fp32 with subnormals replaced by a zero of the same sign (the kernels are compiled with flush-to-zero)."""
    return torch.where(t.abs() < FLT_MIN, torch.zeros_like(t).copysign(t), t)


def _add(a, b):
    return ftz(ftz(a) + ftz(b))


class Spy:
    """Stands in for the engine's native module: before each accumulate launch it keeps a copy of every weight's bf16
    micro-batch gradient and of vgrads, and around the fold the residual and what the fold wrote.  Used with
    overlap=False, so every launch and copy runs on the backward's stream in order."""

    def __init__(self, eng):
        self.C, self.eng = eng.C, eng
        self.g, self.v, self.e_old, self.out = [], [], None, None

    def __getattr__(self, name):
        return getattr(self.C, name)

    def _grab(self):
        self.g.append([p.grad.clone() for p in self.eng.w_params])
        self.v.append(self.eng.vgrads.clone())

    def v2_accum_add(self, *a):
        self._grab()
        return self.C.v2_accum_add(*a)

    def v2_accum_fold(self, *a):
        self._grab()
        e = self.eng.residual
        self.e_old = e.clone() if e is not None else None
        r = self.C.v2_accum_fold(*a)
        self.out = ([p.grad.clone() for p in self.eng.w_params], self.eng.vgrads.clone(),
                    e.clone() if e is not None else None, self.eng.acc.clone(), self.eng.vacc.clone())
        return r


@pytest.mark.gpu
@pytest.mark.parametrize("ef", [False, True])
@pytest.mark.parametrize("code", ["svd", "qsgd", "sign", "fp8", "hadamard", "powersgd"])
@pytest.mark.parametrize("n", [2, 3, 4])
def test_fold_is_the_fp32_oracle(n, code, ef):
    eng = _engine("ResNet18", code=code, error_feedback=ef, use_graph=False, overlap=False, accumulate_steps=n,
                  **CODE_KW[code])
    try:
        x, y = _batch("ResNet18", 0, 4 * n)
        eng.prepare(x, y, warmup=0)
        inv = torch.tensor(1.0 / n, dtype=torch.float32).item()
        qs = [q for q in eng.plan.params if q.is_w]
        for step in range(2):               # the second step codes with a non-zero residual
            spy = eng.C = Spy(eng)
            x, y = _batch("ResNet18", step + 1, 4 * n)
            eng.train_step(x, y)
            torch.cuda.synchronize()
            assert eng.error_code() == 0
            eng.C = spy.C
            assert len(spy.g) == n
            got_g, got_v, got_e, acc, vacc = spy.out
            assert not bool(acc.any()) and not bool(vacc.any())
            for i, q in enumerate(qs):
                s = spy.g[0][i].float()
                for j in range(1, n):
                    s = _add(s, spy.g[j][i].float())
                a = ftz(s * inv)
                if ef:
                    e = torch.as_strided(spy.e_old, q.shape, q.phys_strides(), q.off)
                    a = _add(a, e)
                want = a.bfloat16()
                assert torch.equal(got_g[i], want), (code, n, i)
                if ef:
                    want_e = ftz(a - want.float())
                    assert torch.equal(torch.as_strided(got_e, q.shape, q.phys_strides(), q.off), want_e)
            vs = spy.v[0]
            for j in range(1, n):
                vs = _add(vs, spy.v[j])
            assert torch.equal(got_v, ftz(vs * inv))
            assert float(got_v.abs().sum()) > 0
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 3])
@pytest.mark.parametrize("code", list(CODE_KW))
def test_graph_replay_equals_eager(code, n, deterministic_cudnn):
    kw = dict(code=code, accumulate_steps=n, error_feedback=code in EF_CODES, **CODE_KW[code])
    if code == "qsvd":
        kw.pop("error_feedback")
    g, _ = _run("ResNet18", 4, 24, use_graph=True, **kw)
    e, _ = _run("ResNet18", 4, 24, use_graph=False, **kw)
    assert differs(g, e) == []


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["LeNet", "FC"])
@pytest.mark.parametrize("n", [2, 4])
def test_micro_batches_match_one_batch(net, n):
    """Dense code, no BN, lr = 1 and no momentum, so the step moves the fp32 master by exactly the pushed gradient.

    * N copies of one micro-batch of b push exactly what one step on those b samples pushes: the forward and backward
      are the same launches, the fp32 sum of N equal bf16 values is exact and so is the scale by a power-of-two 1/N.
      A lost or doubled micro-batch, or a wrong scale, moves the result by a multiple of the gradient.
    * N different micro-batches of b against one batch of N b: the forward runs other GEMM shapes, so activations and
      gradients may round differently, but only by bf16 roundings: the two gradients agree within a few units of
      2^-8 in norm, where dropping one micro-batch would be off by about 1 / N."""
    b = 32
    u = 2.0 ** -8

    def pushed(k, x, y):
        eng = _engine(net, code="sgd", lr=1.0, momentum=0.0, use_graph=False, accumulate_steps=k)
        try:
            eng.prepare(x, y, warmup=0)
            v0 = eng.vparams.clone()
            eng.master.zero_()
            eng.train_step(x, y)
            torch.cuda.synchronize()
            assert eng.error_code() == 0
            return -eng.master.double(), (v0 - eng.vparams).double()
        finally:
            eng.close()

    xb, yb = _batch(net, 0, b)
    g1, v1 = pushed(1, xb, yb)
    gn, vn = pushed(n, xb.repeat(n, *[1] * (xb.dim() - 1)), yb.repeat(n))
    assert float(g1.norm()) > 0
    assert torch.equal(gn, g1)
    assert torch.allclose(vn, v1, rtol=4 * 2.0 ** -24, atol=0)

    x, y = _batch(net, 1, n * b)
    g1, v1 = pushed(1, x, y)
    gn, vn = pushed(n, x, y)
    rel = float((gn - g1).norm() / g1.norm())
    rel_v = float((vn - v1).norm() / v1.norm())
    print("%s N=%d: relative difference %.2e (weights), %.2e (vectors)" % (net, n, rel, rel_v))
    assert rel < 8 * u and rel_v < 8 * u


@pytest.mark.gpu
@pytest.mark.parametrize("code", ["svd", "topk"])
def test_resume_is_bitwise(code, tmp_path, deterministic_cudnn, capsys):
    kw = dict(code=code, error_feedback=True, accumulate_steps=2, **CODE_KW[code])
    K, net, B = 3, "ResNet18", 32

    def run(steps, load=None, save=None, **extra):
        eng = _engine(net, **dict(kw, **extra))
        x, y = _batch(net, 0, B)
        eng.prepare(x, y, warmup=2)
        if load is not None:
            eng.load_checkpoint(save, load)
        for _ in range(steps):
            x, y = _batch(net, eng.step, B)
            eng.train_step(x, y)
        torch.cuda.synchronize()
        assert eng.error_code() == 0
        st = _state(eng)
        if save is not None and load is None:
            eng.save_checkpoint(save)
        eng.close()
        return st

    d = str(tmp_path) + "/"
    a = run(2 * K)
    assert differs(a, run(2 * K)) == [], "control: two uninterrupted runs differ"
    run(K, save=d)
    c = run(K, load=2 + K, save=d)
    assert "not restored" not in capsys.readouterr().out
    assert differs(a, c) == []
    assert bool(a["worker:residual"].ne(0).any())
    run(1, load=2 + K, save=d, accumulate_steps=1)      # the accumulators are scratch: N = 2 state loads at N = 1
    assert "not restored" not in capsys.readouterr().out


@pytest.mark.gpu
def test_peak_memory_falls():
    peak = {}
    for n, b in ((1, 256), (4, 256)):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        eng = _engine("ResNet18", code="svd", svd_rank=3, accumulate_steps=n)
        x, y = _batch("ResNet18", 0, b)
        eng.prepare(x, y, warmup=2)
        for _ in range(2):
            eng.train_step(x, y)
        torch.cuda.synchronize()
        assert eng.error_code() == 0
        peak[n] = torch.cuda.max_memory_allocated() - base
        eng.close()
        del eng
    print("peak allocated, ResNet-18 CIFAR batch 256: N=1 %.1f MiB, N=4 (micro-batch 64) %.1f MiB"
          % (peak[1] / 2 ** 20, peak[4] / 2 ** 20))
    assert peak[4] < peak[1]


# ---------------------------------------------------------------------------------------------------- two GPUs
def _mp_graph_eager(rank, world, port, out):
    import torch.distributed as dist
    nccl_init(rank, world, port)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    res = []
    for graph in (True, False):
        torch.manual_seed(0)
        eng = ShadowEngine(build_model("ResNet18", 10), rank, world, code="topk", entry_budget=0.01, lr=0.05,
                           momentum=0.9, seed=7, use_graph=graph, ps_mode="sharded", error_feedback=True,
                           accumulate_steps=2)
        x, y = _batch("ResNet18", rank, 32)
        eng.prepare(x, y, warmup=2)
        for _ in range(3):
            eng.train_step(x, y)
        torch.cuda.synchronize()
        res.append((eng.gather_fp32("master").cpu(), eng.residual.cpu(), eng.error_code()))
        eng.close()
    out.put((rank, torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]), res[0][2], res[1][2]))
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_gpus_sharded_graph_equals_eager():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    res = spawn(2, _mp_graph_eager, 29680)
    assert all(same and e1 == 0 and e2 == 0 for _, same, e1, e2 in res), res

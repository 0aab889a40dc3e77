"""Bitwise resume of the bf16 engine: save -> a fresh engine -> load continues the interrupted run bit for bit.

Run A trains 2N steps.  Run B trains N steps from the same seed, saves and closes.  Run C is a new engine that
prepares (with or without warm-up steps), loads B's checkpoint and trains N more steps.  A and C must be
``torch.equal`` on the owner state, the bf16 weights, the BN statistics and every worker's own state (error-feedback
residual, Jacobi warm start, PowerSGD's warm factor and unit state, the CUDA generator that VGG's dropout draws
from).  A second uninterrupted run of A is the control:
the step is deterministic (fixed-order sums, Philox draws keyed by seed / step / unit / worker) with cuDNN held to
deterministic algorithms, as ``bench.py`` holds it.

CPU: the worker file's name, contents and matching rules, and ``latest_step`` skipping it.
"""
import os
import shutil

import pytest
import torch

from atomo_b200.utils import checkpoint as ckpt

from shadow_harness import deterministic_cudnn, differs, engine_batch, make_engine, nccl_init, spawn  # noqa: F401

N = 3           # steps before and after the interruption
WARMUP = 2      # eager warm-up steps of runs A and B (they count as steps, as in the launcher)


# ---------------------------------------------------------------------------------------------------- CPU
def test_latest_step_skips_worker_files(tmp_path):
    d = str(tmp_path) + "/"
    for name in ("model_step_5", "model_step_5_optim", "model_step_5_worker0", "model_step_5_worker1",
                 "model_step_9_worker0", "model_step_9_worker0.tmp", "model_step_12_worker3"):
        open(d + name, "w").close()
    assert ckpt.latest_step(d) == 5
    assert ckpt.worker_path(d, 5, 1) == d + "model_step_5_worker1"


def _config(**kw):
    c = {"code": "topk", "plan": "ab" * 32, "error_feedback": True, "warm_start": True, "world": 1,
         "ps_mode": "colocated", "worker": 0}
    c.update(kw)
    return c


def test_worker_file_round_trip_and_matching(tmp_path):
    d = str(tmp_path) + "/"
    res = torch.randn(1000)
    pw = torch.arange(320, dtype=torch.uint8)
    path = ckpt.save_worker_state(d, 7, 2, _config(), {"residual": res, "pw_state": pw})
    assert path == d + "model_step_7_worker2" and not os.path.exists(path + ".tmp")
    st = ckpt.load_worker_state(d, 7, 2)
    assert st["format"] == ckpt.WORKER_STATE_FORMAT and st["step"] == 7 and st["config"] == _config()
    assert torch.equal(st["tensors"]["residual"], res) and torch.equal(st["tensors"]["pw_state"], pw)
    mine = {"residual": torch.zeros(1000), "pw_state": torch.zeros(320, dtype=torch.uint8)}
    assert ckpt.worker_state_mismatch(st, 7, _config(), mine) == []
    assert ckpt.load_worker_state(d, 7, 0) is None and ckpt.load_worker_state(d, 8, 2) is None


@pytest.mark.parametrize("field,value", [("code", "sign"), ("plan", "cd" * 32), ("error_feedback", False),
                                         ("warm_start", False), ("world", 2), ("ps_mode", "sharded"), ("worker", 1)])
def test_worker_file_config_mismatch(field, value):
    st = {"format": ckpt.WORKER_STATE_FORMAT, "step": 3, "config": _config(), "tensors": {"residual": torch.zeros(4)}}
    mine = {"residual": torch.zeros(4)}
    assert ckpt.worker_state_mismatch(st, 3, _config(**{field: value}), mine) == [field]


def test_worker_file_format_step_and_tensor_mismatch():
    st = {"format": ckpt.WORKER_STATE_FORMAT, "step": 3, "config": _config(), "tensors": {"residual": torch.zeros(4)}}
    z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt)
    assert ckpt.worker_state_mismatch(dict(st, format=0), 3, _config(), {"residual": z(4)}) == ["format"]
    assert ckpt.worker_state_mismatch(st, 4, _config(), {"residual": z(4)}) == ["step"]
    assert ckpt.worker_state_mismatch(st, 3, _config(), {"residual": z(5)}) == ["tensors"]
    assert ckpt.worker_state_mismatch(st, 3, _config(), {"residual": z(4, dt=torch.float64)}) == ["tensors"]
    assert ckpt.worker_state_mismatch(st, 3, _config(), {"residual": z(4), "vprev": z(4)}) == ["tensors"]
    assert ckpt.worker_state_mismatch(st, 3, _config(), {}) == ["tensors"]
    extra = dict(_config(), seed=5)
    assert ckpt.worker_state_mismatch(st, 3, extra, {"residual": z(4)}) == ["seed"]


def test_plan_digest_follows_the_unit_table():
    from atomo_b200.models import build_model
    from atomo_b200.ops import plan2 as P2
    shapes = [tuple(p.shape) for p in build_model("ResNet18", 10).parameters()]
    d = lambda *a, **k: P2.plan_digest(P2.build_plan2(shapes, *a, **k))
    assert d("svd", 3) == d("svd", 3)
    assert len({d("svd", 3, n_groups=5), d("svd", 2, n_groups=5), d("qsvd", 3), d("svd", 3, n_groups=3),
                d("topk", 3), d("topk", 3, entry_budget=0.02), d("powersgd", 2), d("powersgd", 1)}) == 8


def test_powersgd_warm_ranges_are_the_tail_of_each_scratch():
    from atomo_b200.models import build_model
    from atomo_b200.ops import plan2 as P2
    shapes = [tuple(p.shape) for p in build_model("VGG11", 10).parameters()]
    pl = P2.build_plan2(shapes, "powersgd", 2)
    units = [u for u in pl.units if u.kind == P2.KIND_POWER]
    ranges = P2.pw_warm_ranges(pl)
    assert len(ranges) == len(units) > 0
    for u, (o, n) in zip(units, ranges):
        assert n == u.rcap * ((u.cols + 3) // 4 * 4)
        assert o + n == u.gpart_off + P2.pw_scratch_floats(u.rows, u.cols, u.rcap) <= pl.gpart_floats
    assert P2.pw_warm_ranges(P2.build_plan2(shapes, "svd", 3)) == []


# ---------------------------------------------------------------------------------------------------- GPU
# name -> (network, CUDA graph, warm-up steps of run C before its load, engine arguments)
SGD = dict(lr=0.05, momentum=0.9)
ADAM = dict(lr=1e-3, optimizer="adam")
CASES = {
    "svd": ("ResNet18", True, WARMUP, dict(code="svd", **SGD)),
    "svd-eager": ("ResNet18", False, 0, dict(code="svd", **SGD)),
    "svd-ef": ("ResNet18", True, WARMUP, dict(code="svd", error_feedback=True, **SGD)),
    "svd-adam": ("ResNet18", True, WARMUP, dict(code="svd", **ADAM)),
    "svd-amsgrad": ("ResNet18", True, WARMUP, dict(code="svd", amsgrad=True, **ADAM)),
    "qsvd": ("VGG11", True, WARMUP, dict(code="qsvd", **SGD)),
    "sgd-nesterov-wd": ("VGG11", False, 0, dict(code="sgd", lr=0.05, momentum=0.9, nesterov=True,
                                                     weight_decay=5e-4)),
    "qsgd-ef": ("VGG11", True, WARMUP, dict(code="qsgd", error_feedback=True, **SGD)),
    "terngrad": ("VGG11", True, WARMUP, dict(code="terngrad", **SGD)),
    "entrywise-ef": ("VGG11", True, WARMUP, dict(code="entrywise", entry_budget=0.05, error_feedback=True, **SGD)),
    "topk-ef": ("ResNet18", True, WARMUP, dict(code="topk", entry_budget=0.01, error_feedback=True, **SGD)),
    "topk-ef-eager": ("ResNet18", False, 0, dict(code="topk", entry_budget=0.01, error_feedback=True, **SGD)),
    "topk-ef-adam": ("ResNet18", True, WARMUP, dict(code="topk", entry_budget=0.01, error_feedback=True, **ADAM)),
    "topk-ef-amsgrad": ("ResNet18", True, WARMUP, dict(code="topk", entry_budget=0.01, error_feedback=True,
                                                       amsgrad=True, **ADAM)),
    "sign-ef": ("VGG11", True, WARMUP, dict(code="sign", error_feedback=True, **SGD)),
    "powersgd": ("ResNet18", True, WARMUP, dict(code="powersgd", svd_rank=2, **SGD)),
    "powersgd-ef": ("ResNet18", True, WARMUP, dict(code="powersgd", svd_rank=2, error_feedback=True, **SGD)),
    "fp8-ef": ("VGG11", True, WARMUP, dict(code="fp8", error_feedback=True, **SGD)),
    "hadamard-ef": ("ResNet18", True, WARMUP, dict(code="hadamard", quantization_level=4, error_feedback=True, **SGD)),
}

def _batch(net, step):
    """The batch of training step ``step``: the same in every run, different from step to step."""
    return engine_batch(net, step, seed=100, period=8)


def _engine(net, graph, kw, rank=0, world=1, **extra):
    return make_engine(net, rank, world, seed=11, use_graph=graph, **dict(kw, **extra))


def _train(eng, net, steps):
    losses = []
    for _ in range(steps):
        x, y = _batch(net, eng.step)
        losses.append(eng.train_step(x, y)[0].clone())
    torch.cuda.synchronize()
    assert eng.error_code() == 0
    return torch.stack(losses).cpu()


def _state(eng) -> dict:
    """Everything a resumed run must reproduce, as host copies (collective on more than one rank)."""
    out = {"master": eng.gather_fp32("master").cpu(), "mom": eng.gather_fp32("mom").cpu()}
    for w in ("sq", "sqmax"):
        if getattr(eng, w, None) is not None:
            out[w] = eng.gather_fp32(w).cpu()
    out["wshadow"] = eng.wshadow.cpu()
    out["vparams"] = eng.vparams.cpu()
    if eng.is_owner:
        for v in ("vmom", "vsq", "vsqmax"):
            if getattr(eng, v, None) is not None:
                out[v] = getattr(eng, v).cpu()
    for name, b in eng.model.named_buffers():
        out["buffer:" + name] = b.cpu()
    for name, t in eng._worker_tensors().items():
        out["worker:" + name] = t.cpu()
    out["device_step"] = torch.tensor(eng.device_step())
    return out


def _run_a(net, graph, kw):
    eng = _engine(net, graph, kw)
    x, y = _batch(net, 0)
    eng.prepare(x, y, warmup=WARMUP)
    losses = _train(eng, net, 2 * N)
    st = _state(eng)
    eng.close()
    return st, losses


def _run_b(net, graph, kw, d):
    eng = _engine(net, graph, kw)
    x, y = _batch(net, 0)
    eng.prepare(x, y, warmup=WARMUP)
    _train(eng, net, N)
    path = eng.save_checkpoint(d)
    eng.close()
    assert path == ckpt.model_path(d, WARMUP + N)
    return WARMUP + N


def _run_c(net, graph, warm_c, kw, d, step, **extra):
    eng = _engine(net, graph, kw, **extra)
    x, y = _batch(net, 0)
    eng.prepare(x, y, warmup=warm_c)
    eng.load_checkpoint(d, step)
    assert eng.device_step() == step + 1
    losses = _train(eng, net, N)
    st = _state(eng)
    eng.close()
    return st, losses


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_resume_is_bitwise(case, tmp_path, deterministic_cudnn, capsys):
    net, graph, warm_c, kw = CASES[case]
    a, la = _run_a(net, graph, kw)
    a2, _ = _run_a(net, graph, kw)
    assert differs(a, a2) == [], "control: two uninterrupted runs differ"
    d = str(tmp_path) + "/"
    step = _run_b(net, graph, kw, d)
    assert os.path.exists(ckpt.worker_path(d, step, 0))
    c, lc = _run_c(net, graph, warm_c, kw, d, step)
    assert "not restored" not in capsys.readouterr().out
    assert differs(a, c) == []
    assert torch.equal(la[N:], lc)
    want = {"svd": ["worker:vprev"], "qsvd": ["worker:vprev"], "powersgd": ["worker:pw_qw", "worker:pw_state"]}
    for k in want.get(kw["code"], []) + (["worker:residual"] if kw.get("error_feedback") else []):
        assert k in a and bool(a[k].ne(0).any()), k          # the state the test is about exists and is not trivial


@pytest.mark.gpu
def test_resume_without_worker_file_differs(tmp_path, deterministic_cudnn, capsys):
    """The check above can fail: without its worker file a top-k + EF run resumes with e = 0 and diverges."""
    net, graph, warm_c, kw = CASES["topk-ef-eager"]
    a, _ = _run_a(net, graph, kw)
    d = str(tmp_path) + "/"
    step = _run_b(net, graph, kw, d)
    os.remove(ckpt.worker_path(d, step, 0))
    c, _ = _run_c(net, graph, warm_c, kw, d, step)
    out = capsys.readouterr().out
    assert out.count("per-worker state of step %d not restored (file missing)" % step) == 1, out
    diff = differs(a, c)
    assert "worker:residual" in diff and "master" in diff, diff


@pytest.mark.gpu
@pytest.mark.parametrize("other", [{"svd_rank": 2}, {"code": "qsvd"}])
def test_mismatched_worker_file_is_not_applied(other, tmp_path, deterministic_cudnn, capsys):
    """A worker file of another rank or code is refused: the resume equals one without a worker file, and the
    warm-up steps before the load leave no trace in the worker state."""
    net, graph, _, kw = CASES["svd"]
    d1, d2 = str(tmp_path / "with") + "/", str(tmp_path / "without") + "/"
    step = _run_b(net, graph, kw, d1)
    shutil.copytree(d1, d2)
    os.remove(ckpt.worker_path(d2, step, 0))
    kw2 = dict(kw, **other)
    eng = _engine(net, graph, kw2)
    fresh = {k: v.cpu() for k, v in eng._worker_tensors().items() if k != "cuda_rng"}
    x, y = _batch(net, 0)
    eng.prepare(x, y, warmup=WARMUP)
    eng.load_checkpoint(d1, step)
    after = {k: v.cpu() for k, v in eng._worker_tensors().items() if k != "cuda_rng"}
    out = capsys.readouterr().out
    assert "per-worker state of step %d not restored (" % step in out and "plan" in out, out
    assert fresh.keys() == after.keys() and all(torch.equal(fresh[k], after[k]) for k in fresh)
    c1 = _state_after(eng, net)
    c2, _ = _run_c(net, graph, WARMUP, kw2, d2, step)
    assert differs(c1, c2) == []


def _state_after(eng, net):
    _train(eng, net, N)
    st = _state(eng)
    eng.close()
    return st


# ---------------------------------------------------------------------------------------------------- two GPUs
def _mp_resume(rank, world, port, case, d, out):
    import torch.distributed as dist
    nccl_init(rank, world, port)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    net, graph, warm_c, kw = CASES[case]
    kw = dict(kw, ps_mode="sharded")

    def run(steps, warm, load=None, save=False):
        eng = _engine(net, graph, kw, rank=rank, world=world)
        x, y = _batch(net, 0)
        eng.prepare(x, y, warmup=warm)
        if load is not None:
            eng.load_checkpoint(d, load)
        _train(eng, net, steps)
        st = _state(eng)
        if save:
            eng.save_checkpoint(d)
        eng.close()
        return st

    a = run(2 * N, WARMUP)
    run(N, WARMUP, save=True)
    c = run(N, warm_c, load=WARMUP + N)
    out.put((rank, differs(a, c), os.path.exists(ckpt.worker_path(d, WARMUP + N, rank))))
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("case", ["svd", "topk-ef"])
def test_resume_is_bitwise_two_gpus_sharded(case, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    port = 29610 + list(CASES).index(case)
    res = spawn(2, _mp_resume, port, case, str(tmp_path) + "/")
    assert all(diff == [] and has_file for _, diff, has_file in res), res

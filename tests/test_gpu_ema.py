"""Exponential moving average of the weights on the bf16 engine (``ShadowEngine(ema_decay=d)``, csrc/v2_ema.cu).

After every step the owner's averages ``ema`` / ``vema`` equal a numpy float32 oracle ``e = e + w (p - e)`` run on the
owner's ``master`` / ``vparams`` from the initial weights, bit for bit, for the svd, dense, top-k with error feedback,
QSGD and PowerSGD codes, with momentum-SGD, Adam, LAMB and clipped momentum-SGD, eager and under graph replay; and
``ema_state_dict()`` is that average in the evaluator's layout.  The average leaves training bitwise untouched and adds
one launch per group.  A resume is bitwise, with and without the ``_ema`` file.  The file loads into ``build_model``
strictly, ``latest_step`` skips it and the evaluator reads it with ``ema=True``; the launcher tests the averaged model
at ``--eval-freq`` and resumes it.  The two-GPU test checks the sharded average against the oracle on the gathered
master.
"""
import functools
import os

import numpy as np
import pytest
import torch

from shadow_harness import deterministic_cudnn, engine_batch, make_engine, nccl_init, spawn, step  # noqa: F401

DECAY = 0.9

CODES = {
    "svd": dict(code="svd", svd_rank=3), "sgd": dict(code="sgd"),
    "topk": dict(code="topk", entry_budget=0.05, error_feedback=True), "qsgd": dict(code="qsgd"),
    "powersgd": dict(code="powersgd", svd_rank=2),
}
OPTS = {
    "momentum": dict(optimizer="sgd", lr=0.05, momentum=0.9, weight_decay=5e-4),
    "adam": dict(optimizer="adam", lr=1e-3, weight_decay=1e-4),
    "lamb": dict(optimizer="lamb", lr=0.02, weight_decay=0.01),
    "momentum+clip": dict(optimizer="sgd", lr=0.05, momentum=0.9, weight_decay=5e-4, clip_grad_norm=0.5),
}

DATA_SEED = 500
_batch = functools.partial(engine_batch, "ResNet18", seed=DATA_SEED)


def _engine(kw, graph=False, ema_decay=DECAY):
    return make_engine(use_graph=graph, overlap=graph, ema_decay=ema_decay, prepare_n=32, data_seed=DATA_SEED, **kw)


def _step(eng):
    return step(eng, _batch(eng.step))


def _oracle(e, p, w):
    """One step of the average in numpy float32: three separately rounded operations."""
    return e + w * (p - e)


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("code", list(CODES))
def test_average_is_the_fp32_oracle(code, opt, graph):
    eng = _engine(dict(CODES[code], **OPTS[opt]), graph=graph)
    w = np.float32(eng.ema_w)
    assert w == np.float32(1.0 - DECAY)
    e, ve = eng.master.cpu().numpy().copy(), eng.vparams.cpu().numpy().copy()
    assert torch.equal(eng.ema.cpu(), torch.from_numpy(e)) and torch.equal(eng.vema.cpu(), torch.from_numpy(ve))
    for _ in range(5):
        _step(eng)
        e = _oracle(e, eng.master.cpu().numpy(), w)
        ve = _oracle(ve, eng.vparams.cpu().numpy(), w)
        assert torch.equal(eng.ema.cpu(), torch.from_numpy(e))
        assert torch.equal(eng.vema.cpu(), torch.from_numpy(ve))
    sd = eng.ema_state_dict()
    ref = eng._state_dict(torch.from_numpy(e).cuda(), torch.from_numpy(ve).cuda())
    live = eng.fp32_state_dict()
    assert sd.keys() == ref.keys() == live.keys()
    assert [k for k in sd if not torch.equal(sd[k], ref[k])] == []
    names = dict(eng.model.named_parameters())
    moved = [k for k in names if not torch.equal(sd[k], live[k])]
    assert len(moved) > len(names) // 2         # the average lags the live weights
    buffers = [k for k in sd if k not in names]
    assert buffers and all(torch.equal(sd[k], live[k]) for k in buffers)      # the live BN statistics
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("code,opt", [("svd", "momentum"), ("sgd", "lamb"), ("topk", "momentum+clip")])
def test_training_is_untouched(code, opt, deterministic_cudnn):
    kw = dict(CODES[code], **OPTS[opt])
    runs = {}
    for decay in (0.0, 0.99):
        eng = _engine(kw, graph=True, ema_decay=decay)
        losses = [_step(eng) for _ in range(6)]
        owned = sum(1 for g in range(eng.G) if eng.plan.ps_range[g][eng.owner_index][1] > 0)
        runs[decay] = (losses, eng.fp32_state_dict(), eng.launches_per_step, owned, eng.ema is None)
        eng.close()
    (l0, s0, n0, g0, none0), (l1, s1, n1, g1, none1) = runs[0.0], runs[0.99]
    assert none0 and not none1
    assert l0 == l1
    assert [k for k in s0 if not torch.equal(s0[k], s1[k])] == []
    assert g0 == g1 > 0 and n1 == n0 + g1


@pytest.mark.gpu
def test_ema_state_dict_needs_the_average():
    eng = _engine(dict(CODES["svd"], **OPTS["momentum"]), ema_decay=0.0)
    with pytest.raises(RuntimeError, match="ema_decay"):
        eng.ema_state_dict()
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("opt", ["momentum", "adam"])
def test_resume_is_bitwise(opt, tmp_path, deterministic_cudnn, capsys):
    from atomo_b200.utils import checkpoint as ckpt
    kw = dict(CODES["svd"], **OPTS[opt])
    d = str(tmp_path) + "/"
    eng = _engine(kw, graph=True)
    for _ in range(6):
        _step(eng)
        if eng.step - 1 == 3:
            eng.save_checkpoint(d)
    want = {k: getattr(eng, k).cpu() for k in ("ema", "vema", "master", "vparams")}
    eng.close()
    assert os.path.isfile(d + "model_step_3_ema") and ckpt.latest_step(d) == 3
    eng = _engine(kw, graph=True)
    eng.load_checkpoint(d, 3)
    for _ in range(3):
        _step(eng)
    got = {k: getattr(eng, k).cpu() for k in want}
    eng.close()
    assert [k for k in want if not torch.equal(want[k], got[k])] == []
    assert "missing" not in capsys.readouterr().out

    # without the file the average starts at the loaded weights, and one line says so
    os.remove(d + "model_step_3_ema")
    eng = _engine(kw, graph=True)
    eng.load_checkpoint(d, 3)
    assert torch.equal(eng.ema, eng.master) and torch.equal(eng.vema, eng.vparams)
    out = capsys.readouterr().out
    assert sum("weight average starts at the loaded weights" in line for line in out.splitlines()) == 1
    eng.close()


@pytest.mark.gpu
def test_file_contract(tmp_path):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model
    from atomo_b200.runtime.evaluator import DistributedEvaluator
    from atomo_b200.utils import checkpoint as ckpt
    d = str(tmp_path) + "/"
    eng = _engine(dict(CODES["svd"], **OPTS["momentum"]))
    for _ in range(2):
        _step(eng)
    eng.save_checkpoint(d)
    sd = eng.ema_state_dict()
    eng.close()
    assert ckpt.latest_step(d) == 2
    saved = torch.load(d + "model_step_2_ema", map_location="cpu")
    assert saved.keys() == sd.keys() and all(torch.equal(saved[k], sd[k].cpu()) for k in sd)
    net = build_model("ResNet18", 10)
    net.load_state_dict(saved, strict=True)
    model = torch.load(d + "model_step_2", map_location="cpu")
    assert any(not torch.equal(model[k], saved[k]) for k in dict(net.named_parameters()))
    os.remove(d + "model_step_2")       # the evaluator must read the average, not the model file
    test = SyntheticImageDataset((3, 32, 32), 10, 64, seed=9)
    loader = torch.utils.data.DataLoader(test, batch_size=32, shuffle=False)
    ev = DistributedEvaluator(model_dir=d, eval_freq=2, network="ResNet18", dataset="Cifar10", device="cuda",
                              poll_seconds=0.01, ema=True)
    res = ev.evaluate(loader, max_evals=1, timeout=5.0)
    assert len(res) == 1 and res[0]["step"] == 2 and np.isfinite(res[0]["loss"])
    got = dict(ev.network.state_dict())
    assert all(torch.equal(got[k].cpu(), saved[k]) for k in saved)


@pytest.mark.gpu
def test_launcher_evaluates_and_resumes_the_average(tmp_path, monkeypatch, capsys):
    import argparse
    from atomo_b200.runtime import p2p_launcher as L
    from atomo_b200.utils.flags import add_fit_args
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    d = str(tmp_path) + "/"
    argv = ["--network", "ResNet18", "--dataset", "Cifar10", "--synthetic", "1", "--train-len", "1024", "--test-len",
            "256", "--batch-size", "64", "--test-batch-size", "128", "--engine", "shadow", "--dtype", "bf16", "--code",
            "svd", "--svd-rank", "3", "--lr", "0.05", "--momentum", "0.9", "--ema-decay", "0.9", "--eval-freq", "4",
            "--log-interval", "4", "--train-dir", d]
    L.run_p2p_training(add_fit_args(argparse.ArgumentParser(), argv + ["--max-steps", "4"]))
    L.run_p2p_training(add_fit_args(argparse.ArgumentParser(), argv + ["--max-steps", "8", "--resume", "1"]))
    out = capsys.readouterr().out
    for s in (4, 8):
        assert "Test set: Step: %d," % s in out and "Test set (EMA): Step: %d," % s in out, out
        assert os.path.isfile(d + "model_step_%d_ema" % s)
    assert "missing" not in out and "device error" not in out


# ---------------------------------------------------------------------------------------------------- two GPUs
def _mp(rank, world, port, out):
    import torch.distributed as dist
    nccl_init(rank, world, port)
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    eng = ShadowEngine(build_model("ResNet18", 10), rank, world, use_graph=True, seed=7, ps_mode="sharded",
                       ema_decay=DECAY, **dict(CODES["svd"], **OPTS["momentum"]))
    x, y = _batch(rank)
    eng.prepare(x, y, warmup=0)
    w = np.float32(eng.ema_w)
    e, ve = eng.gather_fp32("master").cpu().numpy(), eng.gather_fp32("vema").cpu().numpy()
    ok = True
    for s in range(4):
        x, y = _batch(1 + s + rank)
        eng.train_step(x, y)
        torch.cuda.synchronize()
        dist.barrier()
        e = _oracle(e, eng.gather_fp32("master").cpu().numpy(), w)
        ve = _oracle(ve, eng.vparams.cpu().numpy(), w)
        ok = ok and torch.equal(eng.gather_fp32("ema").cpu(), torch.from_numpy(e)) and \
            torch.equal(eng.gather_fp32("vema").cpu(), torch.from_numpy(ve))
    sd = eng.ema_state_dict()
    out.put((rank, eng.error_code(), ok, {k: v.cpu() for k, v in sd.items() if "running" not in k}))
    eng.close()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_owners_average_their_shards():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    res = spawn(2, _mp, 29710)
    assert all(r[1] == 0 and r[2] for r in res)
    a, b = res[0][3], res[1][3]
    assert all(torch.equal(a[k], b[k]) for k in a)

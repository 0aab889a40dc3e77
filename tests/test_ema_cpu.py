"""Exponential moving average of the weights without a GPU: the ``--ema-decay`` flag and its refusals (engine, launcher,
role path), ``latest_step`` skipping ``model_step_<N>_ema``, the evaluator's ``ema`` option, the launcher loop on a
stand-in engine evaluating the averaged model at ``--eval-freq``, and the gloo role path's average against a float32
oracle, written beside each model file and restored on ``--resume``."""
import argparse
import os
import types

import numpy as np
import pytest
import torch

from atomo_b200.runtime import master as M
from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils import checkpoint as ckpt
from atomo_b200.utils.flags import add_fit_args, check_ema_decay

from shadow_harness import StandInEngine, fit_args, forbid_cuda, role_master, role_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAD = [1, 1.0, 1.5, -0.5, -1e-9, float("nan"), float("inf"), -float("inf"), True, False, "0.9"]


def test_flag_parses_and_defaults_to_off():
    assert add_fit_args(argparse.ArgumentParser(), []).ema_decay == 0.0
    assert add_fit_args(argparse.ArgumentParser(), ["--ema-decay", "0.999"]).ema_decay == 0.999
    for ok in (0, 0.0, 1e-9, 0.5, 0.9999, np.float32(0.99)):
        assert check_ema_decay(ok) == float(ok)


@pytest.mark.parametrize("bad", BAD)
def test_bad_values_are_refused(bad):
    with pytest.raises(ValueError, match="ema_decay"):
        check_ema_decay(bad)


@pytest.mark.parametrize("bad", [1.0, -0.1, float("nan"), float("inf"), True])
def test_engine_refuses_before_cuda_work(bad, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    forbid_cuda(monkeypatch)
    with pytest.raises(ValueError, match="ema_decay"):
        S.ShadowEngine(None, 0, 1, ema_decay=bad)


@pytest.mark.parametrize("bad", ["1", "-0.5", "nan", "inf"])
def test_launcher_refuses_bad_values(bad, tmp_path):
    with pytest.raises(SystemExit, match="ema-decay"):
        L._build_engine(fit_args(tmp_path, "--code", "svd", "--ema-decay", bad, "--dtype", "bf16"),
                        torch.nn.Linear(4, 4), 0, 1)


def test_fp32_flat_engine_refuses(tmp_path):
    model = torch.nn.Linear(4, 4)
    for extra in (("--engine", "fused", "--dtype", "bf16"), ("--dtype", "fp32"),
                  ("--dtype", "bf16", "--code", "entrywise")):        # auto sends these to the fp32-flat engine
        with pytest.raises(SystemExit, match="--ema-decay runs on the bf16 engine"):
            L._build_engine(fit_args(tmp_path, "--code", "svd", "--ema-decay", "0.9", *extra), model, 0, 1)


def test_role_path_refuses_a_bad_value():
    with pytest.raises(ValueError, match="ema_decay"):
        M.SyncReplicasMaster_NN(types.SimpleNamespace(world_size=2), learning_rate=0.1, network="LeNet", ema_decay=1.0)


def test_latest_step_skips_the_average(tmp_path):
    d = str(tmp_path) + "/"
    for name in ("model_step_3", "model_step_3_ema", "model_step_5_ema", "model_step_5_ema.tmp", "model_step_4_optim"):
        open(d + name, "wb").close()
    assert ckpt.latest_step(d) == 3


def test_evaluator_reads_the_average(tmp_path):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model
    from atomo_b200.runtime.evaluator import DistributedEvaluator
    d = str(tmp_path) + "/"
    torch.manual_seed(0)
    net = build_model("LeNet", 10)
    torch.save(net.state_dict(), d + "model_step_1_ema")
    torch.save({k: torch.zeros_like(v) for k, v in net.state_dict().items()}, d + "model_step_1")
    loader = torch.utils.data.DataLoader(SyntheticImageDataset((1, 28, 28), 10, 64, seed=3), batch_size=32)
    kw = dict(model_dir=d, eval_freq=1, network="LeNet", dataset="MNIST", poll_seconds=0.01)
    ev = DistributedEvaluator(ema=True, **kw)
    assert len(ev.evaluate(loader, max_evals=1, timeout=2.0)) == 1
    assert all(torch.equal(a, b) for a, b in zip(ev.network.state_dict().values(), net.state_dict().values()))
    plain = DistributedEvaluator(**kw)
    plain.evaluate(loader, max_evals=1, timeout=2.0)
    assert all(not v.any() for v in plain.network.state_dict().values())


class EmaStandIn(StandInEngine):
    """Its average is a model of zeros, so that the averaged model's test loss is exactly log(10)."""

    def __init__(self, model, args):
        super().__init__(model, args)
        self.ema_reads = []

    def ema_state_dict(self):
        self.ema_reads.append(self.step - 1)
        return {k: torch.zeros_like(v) for k, v in self.model.state_dict().items()}


def test_launcher_loop_evaluates_the_average(tmp_path, monkeypatch, capsys):
    StandInEngine.instances.clear()
    monkeypatch.setattr(L, "_build_engine", lambda args, model, rank, world: (EmaStandIn(model, args), "shadow"))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    L.run_p2p_training(fit_args(tmp_path, "--code", "svd", "--dtype", "bf16", "--max-steps", "6", "--eval-freq", "3",
                                "--ema-decay", "0.9"), device="cpu")
    eng = StandInEngine.instances[-1]
    assert eng.args.ema_decay == 0.9 and eng.ema_reads == [3, 6]
    out = capsys.readouterr().out.splitlines()
    live = [line for line in out if line.startswith("Test set: Step:")]
    avg = [line for line in out if line.startswith("Test set (EMA): Step:")]
    assert [line.split(",")[0] for line in live] == ["Test set: Step: 3", "Test set: Step: 6"]
    assert [line.split(",")[0] for line in avg] == ["Test set (EMA): Step: 3", "Test set (EMA): Step: 6"]
    assert all("Average loss: %.4f," % np.log(10) in line for line in avg)
    assert not any("Average loss: %.4f," % np.log(10) in line for line in live)


def test_launcher_loop_without_the_average(tmp_path, monkeypatch, capsys):
    StandInEngine.instances.clear()
    monkeypatch.setattr(L, "_build_engine", lambda args, model, rank, world: (EmaStandIn(model, args), "shadow"))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    L.run_p2p_training(fit_args(tmp_path, "--code", "svd", "--dtype", "bf16", "--max-steps", "3", "--eval-freq", "3"),
                       device="cpu")
    assert StandInEngine.instances[-1].ema_reads == []
    assert "Test set (EMA)" not in capsys.readouterr().out


# ---------------------------------------------------------------------------------------------------- role path
def _master(tmp_path, decay, resume=False):
    return role_master(tmp_path, learning_rate=0.1, momentum=0.9, ema_decay=decay, resume=resume)


def test_role_path_average_is_the_fp32_oracle(tmp_path):
    m = _master(tmp_path, 0.9)
    w = np.float32(1.0 - 0.9)
    assert m._ema_w == w and m.ema.dtype == torch.float32
    e = m.flat_params.numpy().copy()
    assert np.array_equal(m.ema.numpy(), e)
    g = torch.Generator().manual_seed(1)
    for _ in range(4):
        grads = [torch.randn(v.shape, generator=g, dtype=torch.float64) for v in m.grad_accumulator.gradient_aggregator]
        for v, x in zip(m.grad_accumulator.gradient_aggregator, grads):
            v.copy_(x)
        m._model_update(1)
        e = e + w * (m.flat_params.numpy() - e)
        assert np.array_equal(m.ema.numpy(), e)
    assert not np.array_equal(e, m.flat_params.numpy())


def test_role_path_without_the_average_keeps_none(tmp_path):
    assert _master(tmp_path, 0.0).ema is None


ROLE_FLAGS = ("--momentum", "0.9", "--ema-decay", "0.8")


def test_gloo_role_path_writes_and_restores_the_average(tmp_path, capsys):
    d = str(tmp_path) + "/"
    role_run(d, 29571, 3, *ROLE_FLAGS)
    out = role_run(d, 29572, 5, *ROLE_FLAGS, "--resume", "1")
    assert "weight average starts" not in out
    w = np.float32(1.0 - 0.8)
    load = lambda name: torch.load(d + name, map_location="cpu")
    names = [n for n, _ in _master(tmp_path / "x", 0.8).network.named_parameters()]
    for s in range(2, 6):       # the average of step s from the file of step s - 1 and the weights of step s
        e, p, got = load("model_step_%d_ema" % (s - 1)), load("model_step_%d" % s), load("model_step_%d_ema" % s)
        assert got.keys() == p.keys()
        for n in names:
            ref = e[n].numpy() + w * (p[n].numpy() - e[n].numpy())
            assert np.array_equal(got[n].numpy(), ref), (s, n)
        for n in p:
            if n not in names:      # BN running statistics: the live model's
                assert torch.equal(got[n], p[n])

    # build_model(resume) restores the average from the file, or starts it at the loaded weights without it
    m = _master(tmp_path, 0.8, resume=True)
    assert m.cur_step == 6
    assert all(torch.equal(v, load("model_step_5_ema")[n]) for n, v in m._ema_views().items())
    capsys.readouterr()
    os.remove(d + "model_step_5_ema")
    m = _master(tmp_path, 0.8, resume=True)
    assert torch.equal(m.ema, m.flat_params)
    assert capsys.readouterr().out.count("weight average starts at the loaded weights") == 1

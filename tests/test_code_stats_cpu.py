"""`--code-stats` without a GPU: the flag, the refusals (engine settings the closed forms do not cover, and the
engines / backends that do not compute the statistics), and the launcher's metrics record on a stand-in engine."""
import argparse
import json

import pytest
import torch

from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils.flags import add_fit_args

from shadow_harness import SVD3, StandInEngine, fit_args, forbid_cuda


def test_code_stats_flag_parses():
    assert add_fit_args(argparse.ArgumentParser(), []).code_stats is False
    assert add_fit_args(argparse.ArgumentParser(), ["--code-stats", "1"]).code_stats is True
    assert add_fit_args(argparse.ArgumentParser(), ["--code-stats", "0"]).code_stats is False


@pytest.mark.parametrize("kw,match", [(dict(code="qsvd"), "QSVD"), (dict(code="svd", resample_empty=True), "resample")])
def test_shadow_engine_refuses_settings_without_a_closed_form(kw, match, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    forbid_cuda(monkeypatch)
    with pytest.raises(ValueError, match=match):
        S.ShadowEngine(torch.nn.Linear(4, 4), code_stats=True, **kw)


def test_fused_engine_and_qsvd_refuse_the_flag(tmp_path):
    model = torch.nn.Linear(4, 4)
    with pytest.raises(SystemExit, match="fp32-flat engine"):
        L._build_engine(fit_args(tmp_path, *SVD3, "--code-stats", "1", "--dtype", "fp32"), model, 0, 1)
    with pytest.raises(SystemExit, match="QSVD"):
        L._build_engine(fit_args(tmp_path, *SVD3, "--code-stats", "1", "--dtype", "bf16", "--code", "qsvd"), model, 0, 1)


def test_role_backends_refuse_the_flag(monkeypatch, tmp_path):
    from atomo_b200 import distributed_nn
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    with pytest.raises(SystemExit, match="--code-stats"):
        distributed_nn.run_rank(fit_args(tmp_path, *SVD3, "--code-stats", "1", "--backend", "gloo"))


class StandIn(StandInEngine):
    """Reports the loss in place of the accuracies, plus ``code_stats``."""

    def __init__(self, model, args):
        super().__init__(model, args)
        self.stats_calls = 0

    def train_step(self, x, y):
        self.opt.zero_grad()
        out = self.model(x)
        loss = torch.nn.functional.cross_entropy(out, y)
        loss.backward()
        self.opt.step()
        self.step += 1
        return torch.stack([loss.detach(), loss.detach(), loss.detach()])

    def code_stats(self, reset=True):
        self.stats_calls += 1
        return {"code": "svd", "steps": 1, "model": {"mse": 0.5, "gsq": 2.0, "rel_var": 0.25},
                "tensors": {"fc.weight": {"mse": 0.5, "gsq": 2.0, "rel_var": 0.25}}}


def _run(tmp_path, monkeypatch, capsys, *extra):
    monkeypatch.setattr(L, "_build_engine", lambda args, model, rank, world: (StandIn(model, args), "shadow"))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    path = tmp_path / ("m" + "".join(extra).replace("-", ""))
    L.run_p2p_training(fit_args(tmp_path, *SVD3, "--max-steps", "6", "--metrics-file", str(path), *extra), device="cpu")
    lines = [l for l in capsys.readouterr().out.splitlines() if l.startswith(("Worker:", "Master:"))]
    return [json.loads(l) for l in open(str(path) + ".rank0.jsonl")], lines


def test_metrics_record_carries_code_stats_only_with_the_flag(tmp_path, monkeypatch, capsys):
    torch.manual_seed(0)
    off, lines_off = _run(tmp_path, monkeypatch, capsys)
    torch.manual_seed(0)
    on, lines_on = _run(tmp_path, monkeypatch, capsys, "--code-stats", "1")
    assert not any("code_stats" in r for r in off)
    assert len(on) == len(off) and all(r["code_stats"]["model"]["rel_var"] == 0.25 for r in on)
    # the log lines are the same bytes with and without the flag (everything but the measured times)
    strip = lambda ls: [l.split("Time Cost")[0] + l.split("Msg(MB)")[-1] if l.startswith("Worker") else
                        l.split("Decode Cost")[0] for l in ls]
    assert lines_on and strip(lines_on) == strip(lines_off)

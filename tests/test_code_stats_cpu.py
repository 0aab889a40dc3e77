"""`--code-stats` without a GPU: the flag, the refusals (engine settings the closed forms do not cover, and the
engines / backends that do not compute the statistics), and the launcher's metrics record on a stand-in engine."""
import argparse
import json
import types

import pytest
import torch

from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils.flags import add_fit_args

from shadow_harness import fit_args, forbid_cuda


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


def _args(tmp_path, *extra):
    return fit_args(tmp_path, "--code", "svd", "--svd-rank", "3", *extra)


def test_fused_engine_and_qsvd_refuse_the_flag(tmp_path):
    model = torch.nn.Linear(4, 4)
    with pytest.raises(SystemExit, match="fp32-flat engine"):
        L._build_engine(_args(tmp_path, "--code-stats", "1", "--dtype", "fp32"), model, 0, 1)
    with pytest.raises(SystemExit, match="QSVD"):
        L._build_engine(_args(tmp_path, "--code-stats", "1", "--dtype", "bf16", "--code", "qsvd"), model, 0, 1)


def test_role_backends_refuse_the_flag(monkeypatch, tmp_path):
    from atomo_b200 import distributed_nn
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    with pytest.raises(SystemExit, match="--code-stats"):
        distributed_nn.run_rank(_args(tmp_path, "--code-stats", "1", "--backend", "gloo"))


class StandIn:
    """The engine interface the launcher uses, trained with plain SGD on the CPU, plus ``code_stats``."""
    first_worker, W, is_worker, is_ps, is_owner = 0, 1, True, True, True

    def __init__(self, model, args):
        self.model, self.lr, self.step = model, args.lr, 1
        self.opt = torch.optim.SGD(model.parameters(), lr=args.lr)
        self.plan = types.SimpleNamespace(expected_factor_bytes=lambda: 1 << 20, dense_bytes=lambda: 1 << 18)
        self.stats_calls = 0

    def prepare(self, x, y, warmup=3):
        for _ in range(warmup):
            self.train_step(x, y)

    def set_lr(self, lr):
        self.lr = lr

    def train_step(self, x, y):
        self.opt.zero_grad()
        out = self.model(x)
        loss = torch.nn.functional.cross_entropy(out, y)
        loss.backward()
        self.opt.step()
        self.step += 1
        return torch.stack([loss.detach(), loss.detach(), loss.detach()])

    def phase_stats(self, reset=True):
        return {"param_wait_us": 10.0, "encode_us": 300.0, "to_push_us": 1500.0}

    def code_stats(self, reset=True):
        self.stats_calls += 1
        return {"code": "svd", "steps": 1, "model": {"mse": 0.5, "gsq": 2.0, "rel_var": 0.25},
                "tensors": {"fc.weight": {"mse": 0.5, "gsq": 2.0, "rel_var": 0.25}}}

    def error_code(self):
        return 0

    def save_checkpoint(self, train_dir, step):
        pass

    def close(self):
        pass


def _run(tmp_path, monkeypatch, capsys, *extra):
    monkeypatch.setattr(L, "_build_engine", lambda args, model, rank, world: (StandIn(model, args), "shadow"))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    path = tmp_path / ("m" + "".join(extra).replace("-", ""))
    L.run_p2p_training(_args(tmp_path, "--max-steps", "6", "--metrics-file", str(path), *extra), device="cpu")
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

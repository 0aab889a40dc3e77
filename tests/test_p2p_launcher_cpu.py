"""The training loop of `--backend p2p` (runtime/p2p_launcher.py) on a CPU stand-in engine: log lines with the
device-timer columns, LR shrinkage derived from the step (resume-safe), checkpoint cadence + evaluation, error-code
polling, metrics file.  The real engines are exercised by tests/test_gpu_*.py; this pins the host-side logic."""
import argparse
import json
import os

import pytest

from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils import checkpoint as ckpt
from atomo_b200.utils.flags import add_fit_args

import shadow_harness as harness


class StandInEngine(harness.StandInEngine):
    """Records the LR it is set to, its checkpoints and its close; reports device error 4 after step `fail_at`."""

    def __init__(self, model, args, fail_at=0):
        super().__init__(model, args)
        self.fail_at = fail_at
        self.lr_history, self.saved, self.closed, self.loaded = [], [], False, None

    def set_lr(self, lr):
        self.lr = lr
        self.lr_history.append((self.step, lr))
        for g in self.opt.param_groups:
            g["lr"] = lr

    def phase_stats(self, reset=True):
        return {"param_wait_us": 10.0, "encode_us": 300.0, "to_push_us": 1500.0, "to_params_us": 1600.0,
                "ps_work_us": 120.0, "ps_wait_push_us": 40.0}

    def error_code(self):
        return 4 if self.fail_at and self.step > self.fail_at else 0

    def save_checkpoint(self, train_dir, step):
        self.saved.append(step)
        ckpt.save_model(train_dir, step, self.model)
        ckpt.save_sidecar(train_dir, step, None, lr=self.lr, extra={"step": step})

    def load_checkpoint(self, train_dir, step):
        ckpt.load_model(train_dir, step, self.model)
        self.step, self.loaded = step + 1, step

    def close(self):
        self.closed = True


def _args(tmp_path, *extra):
    return add_fit_args(argparse.ArgumentParser(), [
        "--network", "LeNet", "--dataset", "MNIST", "--synthetic", "1", "--train-len", "512", "--test-len", "128",
        "--batch-size", "32", "--test-batch-size", "64", "--lr", "0.05", "--code", "svd", "--svd-rank", "3",
        "--log-interval", "1", "--train-dir", str(tmp_path) + "/", *extra])


@pytest.fixture
def standin(monkeypatch):
    StandInEngine.instances.clear()
    cfg = {"fail_at": 0}
    monkeypatch.setattr(L, "_build_engine", lambda args, model, rank, world: (StandInEngine(model, args, cfg["fail_at"]), "fused"))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    return cfg


def test_loop_logs_checkpoints_evaluates_and_shrinks_the_lr(tmp_path, standin, capsys):
    from atomo_b200.tiny_tuning_parser import parse_line
    args = _args(tmp_path, "--max-steps", "12", "--eval-freq", "5", "--shrinkage-freq", "4", "--lr-shrinkage", "0.5",
                 "--metrics-file", str(tmp_path / "m"))
    L.run_p2p_training(args, device="cpu")
    eng = StandInEngine.instances[-1]
    out = capsys.readouterr().out
    recs = [parse_line(l) for l in out.splitlines() if l.startswith("Worker: 0, Step:")]
    # 3 warm-up steps count as steps (the engine trained on them): the loop logs steps 4..12
    assert [r["step"] for r in recs] == list(range(4, 13))
    assert all(abs(r["encode"] - 300e-6) < 1e-4 and r["comp"] > 0 and r["msg_mb"] == pytest.approx(1.25) for r in recs)
    assert recs[-1]["loss"] < recs[0]["loss"]
    assert "Master: Step: 12, Decode Cost: 0.00012" in out
    assert eng.saved == [5, 10] and "Test set: Step: 5," in out and "Test set: Step: 10," in out
    assert os.path.isfile(str(tmp_path) + "/model_step_10") and eng.closed
    # lr = base * shrinkage ** (completed steps // freq), applied to the engine (the reference only printed it)
    assert eng.lr_history[0] == (4, 0.05)                       # steps 1-3 were the warm-up
    assert (5, 0.025) in eng.lr_history and (9, 0.0125) in eng.lr_history and eng.lr == 0.05 * 0.5 ** 3
    m = [json.loads(l) for l in open(str(tmp_path / "m") + ".rank0.jsonl")]
    assert [r["step"] for r in m] == list(range(4, 13)) and m[-1]["phase_us"]["ps_work_us"] == 120.0


def test_resume_continues_with_the_decayed_lr(tmp_path, standin, capsys):
    common = ("--eval-freq", "4", "--shrinkage-freq", "4", "--lr-shrinkage", "0.5")
    L.run_p2p_training(_args(tmp_path, "--max-steps", "8", *common), device="cpu")
    L.run_p2p_training(_args(tmp_path, "--max-steps", "11", "--resume", "1", *common), device="cpu")
    eng = StandInEngine.instances[-1]
    out = capsys.readouterr().out
    assert eng.loaded == 8 and "Worker: 0, Step: 9," in out and "Worker: 0, Step: 11," in out
    assert eng.lr_history[0] == (9, 0.05 * 0.5 ** 2)            # ADVICE r1: no jump back to the base LR


def test_device_error_aborts_the_run(tmp_path, standin):
    standin["fail_at"] = 6
    with pytest.raises(SystemExit, match="device-side error code 4"):
        L.run_p2p_training(_args(tmp_path, "--max-steps", "20", "--eval-freq", "100"), device="cpu")

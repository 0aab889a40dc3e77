"""Gradient-norm clipping without a GPU: the flag and its refusals (engine, launcher, role path), the planner's owner
tile table, the ``Ctrl2`` packing, the role path's update against ``torch.nn.utils.clip_grad_norm_`` followed by the
same ``optim/`` class, a gloo run with ``--clip-grad-norm`` and the launcher loop on a stand-in engine."""
import argparse
import math
import os
import struct
import subprocess
import sys
import types

import pytest
import torch

from atomo_b200.ops import plan2 as P2
from atomo_b200.optim import LAMB, LARS, SGD, Adam
from atomo_b200.runtime import master as M
from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils.flags import add_fit_args, check_clip_grad_norm

from shadow_harness import SVD3, StandInEngine, fit_args, forbid_cuda

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAD = [-1.0, float("nan"), float("inf"), -float("inf"), True, "1.0"]


def test_flag_parses_and_defaults_to_off():
    assert add_fit_args(argparse.ArgumentParser(), []).clip_grad_norm == 0.0
    assert add_fit_args(argparse.ArgumentParser(), ["--clip-grad-norm", "2.5"]).clip_grad_norm == 2.5
    assert check_clip_grad_norm(0) == 0.0 and check_clip_grad_norm(1) == 1.0 and check_clip_grad_norm(1e30) == 1e30


@pytest.mark.parametrize("bad", BAD)
def test_bad_values_are_refused(bad):
    with pytest.raises(ValueError, match="clip_grad_norm"):
        check_clip_grad_norm(bad)


@pytest.mark.parametrize("bad", BAD[:4])
def test_engine_refuses_before_cuda_work(bad, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    forbid_cuda(monkeypatch)
    with pytest.raises(ValueError, match="clip_grad_norm"):
        S.ShadowEngine(None, 0, 1, clip_grad_norm=bad)


@pytest.mark.parametrize("bad", ["-1", "nan", "inf"])
def test_launcher_refuses_bad_values(bad, tmp_path):
    with pytest.raises(SystemExit, match="clip-grad-norm"):
        L._build_engine(fit_args(tmp_path, *SVD3, "--clip-grad-norm", bad, "--dtype", "bf16"), torch.nn.Linear(4, 4), 0, 1)


def test_fp32_flat_engine_refuses(tmp_path):
    model = torch.nn.Linear(4, 4)
    for extra in (("--engine", "fused", "--dtype", "bf16"), ("--dtype", "fp32"),
                  ("--dtype", "bf16", "--code", "entrywise")):        # auto sends these to the fp32-flat engine
        with pytest.raises(SystemExit, match="--engine shadow"):
            L._build_engine(fit_args(tmp_path, *SVD3, "--clip-grad-norm", "1.0", *extra), model, 0, 1)


@pytest.mark.parametrize("n_groups", [1, 2, 3, 5])
@pytest.mark.parametrize("n_owners", [1, 2, 3, 4])
def test_owner_tiles_cover_each_owners_tiles_once(n_owners, n_groups):
    shapes = [(8, 3, 3, 3), (8,), (8,), (16, 8, 3, 3), (16,), (32, 16, 3, 3), (32,), (64, 32, 3, 3), (64,), (10, 64),
              (10,)]
    pl = P2.build_plan2(shapes, "svd", 3, n_owners=n_owners, n_groups=n_groups)
    seen = []
    for o in range(n_owners):
        tiles = P2.owner_ps_tiles(pl, o)
        assert len(tiles) == len(set(tiles))
        assert all(pl.ps_tiles[t][3] == o for t in tiles)
        assert tiles == sorted(tiles)
        seen += tiles
    assert sorted(seen) == list(range(len(pl.ps_tiles)))
    if n_owners > 1 and n_groups > 1:
        assert any(b - a != 1 for a, b in zip(P2.owner_ps_tiles(pl, 0), P2.owner_ps_tiles(pl, 0)[1:]))


def test_ctrl2_packs_the_norm_in_the_padding_word():
    assert struct.calcsize(P2.CTRL2_FMT) == P2.CTRL2_BYTES == 72
    off = P2.pack_ctrl2(opt=P2.OPT_ADAM, num_aggregate=2, trust_coefficient=0.5)
    on = P2.pack_ctrl2(opt=P2.OPT_ADAM, num_aggregate=2, trust_coefficient=0.5, clip_grad_norm=1.5)
    assert struct.unpack_from("<f", off, 52)[0] == 0.0 and struct.unpack_from("<f", on, 52)[0] == 1.5
    assert off[:52] == on[:52] and off[56:] == on[56:]
    assert struct.unpack_from("<ii", on, 56) == (P2.OPT_ADAM, 2)         # opt, num_aggregate where they were


def _params(seed):
    g = torch.Generator().manual_seed(seed)
    shapes = [(6, 3, 3, 3), (6,), (10, 24), (10,)]
    ws = [torch.randn(s, generator=g, dtype=torch.float64) for s in shapes]
    workers = [[torch.randn(s, generator=g, dtype=torch.float64) for s in shapes] for _ in range(3)]
    return ws, workers


def _make_opt(name, params):
    if name == "sgd":
        return SGD(params, lr=0.1, momentum=0.9, weight_decay=1e-3)
    if name == "adam":
        return Adam(params, lr=0.01)
    if name == "lars":
        return LARS(params, lr=0.5, momentum=0.9, weight_decay=5e-4, trust_coefficient=0.02)
    return LAMB(params, lr=0.02, weight_decay=0.01)


@pytest.mark.parametrize("max_norm", [1e6, 0.5])
@pytest.mark.parametrize("opt", ["sgd", "adam", "lars", "lamb"])
def test_role_path_update_is_clip_grad_norm_then_the_optimizer(opt, max_norm):
    ws, workers = _params(3)
    mean = [sum(w[i] for w in workers) / 3 for i in range(len(ws))]
    # the reference: torch's clip_grad_norm_ on .grad, then the same optim/ class
    ref = [torch.nn.Parameter(w.clone()) for w in ws]
    for p, g in zip(ref, mean):
        p.grad = g.clone()
    total = torch.nn.utils.clip_grad_norm_(ref, max_norm)
    ro = _make_opt(opt, ref)
    # the role path: SyncReplicasMaster_NN._model_update on the workers' summed gradients
    m = M.SyncReplicasMaster_NN.__new__(M.SyncReplicasMaster_NN)
    got = [torch.nn.Parameter(w.clone()) for w in ws]
    m._num_workers, m._enable_gpu, m._clip_grad_norm, m.last_grad_norm = 3, False, max_norm, None
    m.optimizer = _make_opt(opt, got)
    m.grad_accumulator = types.SimpleNamespace(gradient_aggregator=[sum(w[i] for w in workers) for i in range(len(ws))])
    for _ in range(2):
        ro.step([p.grad for p in ref])
        m._model_update(3)
    for a, b in zip(got, ref):
        torch.testing.assert_close(a.data, b.data, rtol=1e-12, atol=1e-14)
    t, coef = m.last_grad_norm
    assert t == pytest.approx(float(total), rel=1e-12)
    assert coef == (1.0 if max_norm > t else pytest.approx(max_norm / (t + 1e-6), rel=1e-12))
    if max_norm < t:
        assert coef < 1.0


def test_role_path_refuses_a_bad_value():
    with pytest.raises(ValueError, match="clip_grad_norm"):
        M.SyncReplicasMaster_NN(types.SimpleNamespace(world_size=2), learning_rate=0.1, network="LeNet",
                                clip_grad_norm=-1.0)


def test_gloo_role_path_trains_with_clipping(tmp_path):
    d = str(tmp_path) + "/"
    cmd = [sys.executable, "-m", "atomo_b200.distributed_nn", "--synthetic", "1", "--train-len", "512",
           "--test-len", "128", "--batch-size", "32", "--lr", "0.01", "--test-batch-size", "64", "--nproc", "2",
           "--network", "LeNet", "--dataset", "MNIST", "--code", "sgd", "--optimizer", "adam", "--clip-grad-norm",
           "0.1", "--max-steps", "4", "--eval-freq", "2", "--train-dir", d, "--master-port", "29553"]
    env = dict(os.environ, ATOMO_HANG_DUMP_S="400", PYTHONPATH=ROOT, OMP_NUM_THREADS="2", MKL_NUM_THREADS="2")
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=420)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "Master: Step: 4" in r.stdout and os.path.isfile(d + "model_step_4")


class ClipStandIn(StandInEngine):
    """Clips with torch's ``clip_grad_norm_`` and counts the reads of the norm."""

    def __init__(self, model, args):
        super().__init__(model, args)
        self.norm_reads, self.last = 0, (0.0, 1.0)

    def train_step(self, x, y):
        self.opt.zero_grad()
        out = self.model(x)
        loss = torch.nn.functional.cross_entropy(out, y)
        loss.backward()
        total = float(torch.nn.utils.clip_grad_norm_(self.model.parameters(), self.args.clip_grad_norm))
        self.last = (total, min(1.0, self.args.clip_grad_norm / (total + 1e-6)))
        self.opt.step()
        self.step += 1
        hit = out.argmax(1).eq(y).float().mean() * 100
        return torch.stack([loss.detach(), hit, hit])

    def grad_norm(self):
        self.norm_reads += 1
        return self.last


def test_launcher_loop_records_the_norm_at_log_steps(tmp_path, monkeypatch, capsys):
    import json
    StandInEngine.instances.clear()
    monkeypatch.setattr(L, "_build_engine", lambda args, model, rank, world: (ClipStandIn(model, args), "shadow"))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    mf = str(tmp_path / "m")
    L.run_p2p_training(fit_args(tmp_path, *SVD3, "--max-steps", "6", "--log-interval", "2", "--clip-grad-norm", "0.05",
                             "--dtype", "bf16", "--metrics-file", mf), device="cpu")
    eng = StandInEngine.instances[-1]
    assert eng.args.clip_grad_norm == 0.05 and eng.step == 7
    recs = [json.loads(l) for l in open(mf + ".rank0.jsonl")]
    assert len(recs) >= 2 and all(r["step"] % 2 == 0 for r in recs)
    assert eng.norm_reads == len(recs)          # read at log steps only
    for r in recs:
        assert math.isfinite(r["grad_norm"]) and r["grad_norm"] > 0 and 0 < r["clip_coef"] <= 1
    assert sum(l.startswith("Worker: 0, Step:") for l in capsys.readouterr().out.splitlines()) == len(recs)

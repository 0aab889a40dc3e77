"""Top-k sparsification on the bf16 engine (``code="topk"``, csrc/v2_topk.cu): the ``codings.topk`` oracle, the planner,
the refusals and the launcher routing (CPU); the selection and encode kernels against the oracle bit for bit, the PS
average, error feedback and ``--code-stats`` (GPU loopback harness); and the engine end to end (GPU)."""
import argparse
import json
import math
import os

import pytest
import torch

from atomo_b200.ops import plan2 as P
from atomo_b200.runtime import p2p_launcher as L
from atomo_b200.utils.flags import add_fit_args

NET_SHAPES = [(64, 3, 3, 3), (64,), (64,), (128, 64, 3, 3), (128,), (256, 128, 3, 3), (512, 256, 1, 1), (300, 200),
              (10, 512), (7, 20), (10,)]
# stem, 3x3 convs (one a multiple of 4096 elements, one not), fc layers, a tensor smaller than an absolute budget,
# a tensor that is all zero (ZERO), a spike (SPIKE), one rounded to a few values (TIES), one with an Inf (INF)
ORACLE_SHAPES = [(64, 3, 3, 3), (64, 32, 3, 3), (128, 64, 3, 3), (10, 512), (300, 200), (7, 20), (5, 3), (64,),
                 (96, 64, 3, 3), (32, 16, 3, 3)]
SPIKE, ZERO, TIES, INF = 1, 6, 8, 9


def _coder(b):
    from atomo_b200.codings.topk import TopK
    return TopK(b)


# ---------------------------------------------------------------------------------------------------- CPU: coder
def _stable_topk(x, k):
    """Reference: stable argsort of the bf16 magnitudes (descending, element order on ties), first min(k, nnz)."""
    mag = [int(v) & 0x7FFF for v in x.to(torch.bfloat16).view(torch.int16).tolist()]
    nz = [i for i, m in enumerate(mag) if m]
    order = sorted(nz, key=lambda i: (-mag[i], i))
    return sorted(order[:k])


@pytest.mark.parametrize("budget", [0.01, 0.05, 0.25, 7.0, 200.0])
def test_coder_keeps_the_stable_top_k(budget):
    g = torch.Generator().manual_seed(3)
    for n in (1, 5, 100, 4096, 5000):
        x = (torch.randn(n, generator=g) * 3).round() / 4        # few distinct values: many ties
        x[torch.rand(n, generator=g) < 0.3] = 0
        c = _coder(budget)
        code = c.encode(x)
        k = c.k_for(n)
        assert k == math.floor(min(max(budget * n if budget < 1 else budget, 1.0), n))
        nnz = int((x != 0).sum())
        assert code["idx"].numel() == min(k, nnz)
        assert code["idx"].tolist() == _stable_topk(x, k)
        dec = c.decode(code)
        assert torch.equal(dec[code["idx"].long()], x[code["idx"].long()])       # exact on kept entries
        kept = torch.zeros(n, dtype=torch.bool)
        kept[code["idx"].long()] = True
        assert bool((dec[~kept] == 0).all())
        # contraction: ||x - topk(x)||^2 <= (1 - k_eff / nnz) ||x||^2
        if nnz:
            lhs = float((x.double() - dec.double()).square().sum())
            assert lhs <= (1 - code["idx"].numel() / nnz) * float(x.double().square().sum()) + 1e-12


def test_coder_edge_cases():
    c = _coder(0.25)
    assert c.encode(torch.zeros(100))["idx"].numel() == 0                   # all zero: nothing
    assert _coder(50.0).encode(torch.arange(1.0, 11.0))["idx"].tolist() == list(range(10))   # numel < s
    eq = c.encode(torch.full((40,), -0.5))                                 # ties everywhere: element order
    assert eq["idx"].tolist() == list(range(10))
    x = torch.randn(64)
    x[7] = float("inf")
    assert c.encode(x)["idx"].numel() == 0                                 # non-finite: nothing
    x[7] = float("nan")
    assert c.encode(x)["idx"].numel() == 0
    sub = torch.tensor([1e-40, 0.0, -2e-40, 0.0]).to(torch.bfloat16).float()   # bf16 subnormals are magnitudes
    assert _coder(2.0).encode(sub)["idx"].tolist() == [0, 2]
    with pytest.raises(ValueError):
        _coder(0.0)


# ---------------------------------------------------------------------------------------------------- CPU: planner
@pytest.mark.parametrize("budget,owners", [(0.05, 1), (0.01, 3), (0.25, 2), (300.0, 4), (5000.0, 1)])
def test_plan2_topk_is_the_entrywise_layout_with_k(budget, owners):
    e = P.build_plan2(NET_SHAPES, "entrywise", n_owners=owners, n_groups=3, entry_budget=budget)
    t = P.build_plan2(NET_SHAPES, "topk", n_owners=owners, n_groups=3, entry_budget=budget)
    assert t.enc_tiles == e.enc_tiles and t.ps_tiles == e.ps_tiles and t.enc_range == e.enc_range
    assert t.ps_range == e.ps_range and t.arena_floats == e.arena_floats and t.n_coded == e.n_coded
    c = _coder(budget)
    for ue, ut in zip(e.units, t.units):
        assert ut.kind == ue.kind
        if ut.kind == P.KIND_ENTRY:
            assert ut.budget == float(math.floor(ue.budget)) == float(c.k_for(ut.numel))
            ut.budget = ue.budget
        assert ut.pack() == ue.pack()           # everything else byte-identical
    t = P.build_plan2(NET_SHAPES, "topk", n_owners=owners, n_groups=3, entry_budget=budget)
    want = sum(4 * c.k_for(u.numel) + 16 * u.n_ps for u in t.units if u.kind == P.KIND_ENTRY)
    assert t.entry_bytes() == want and t.expected_factor_bytes() == want


def test_plan2_other_codes_unchanged_by_the_new_code():
    """Digests of the plans of the existing codes, taken from the planner before top-k was added."""
    import hashlib
    want = {"svd": "917543867e0167683f770150a43eaf4c129e4d461aa989111b2a491e5eeca388",
            "qsvd": "6ea73c4cd4a95d51288ea6c2a2053f66ff7800fc277120bdccfda766e92e3cf9",
            "sgd": "6d3fd294b9211300d2945b4d3f20d6bf9615e56c5dfa3bab6b294fa9370a37d8",
            "qsgd": "1f34b0853ed1349c3ede1baad5eecd6d7a8e9d4bd571740ec8e531cedbfe275c",
            "terngrad": "5ab388e54d2c51d29226927eaa996c37b3173a968114dce188b5cb8121895e57",
            "entrywise": "5ec97d1b33d12cee3ed4b7b6466f49526420e0442c54d8d8aa9634e1cfe73dcf"}
    for code, digest in want.items():
        pl = P.build_plan2(NET_SHAPES, code, 3, n_owners=2, n_groups=3, entry_budget=0.05)
        b = pl.units_bytes() + P.Plan2.tiles_bytes(pl.enc_tiles) + P.Plan2.tiles_bytes(pl.ps_tiles) + \
            repr((pl.enc_range, pl.ps_range, pl.arena_floats, pl.n_coded)).encode()
        assert hashlib.sha256(b).hexdigest() == digest, code


@pytest.mark.parametrize("kw", [{"prob_rule": "waterfill"}, {"sampling": "systematic"}, {"entry_budget": 0.0},
                                {"entry_budget": -2.0}])
def test_shadow_engine_topk_refuses_before_cuda(kw, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S

    def no_cuda(*a, **k):
        raise AssertionError("refused only after CUDA work started")
    monkeypatch.setattr(S, "load_ext", no_cuda)
    with pytest.raises(ValueError):
        S.ShadowEngine(None, 0, 1, code="topk", **kw)
    with pytest.raises(ValueError, match="num_aggregate"):     # the error-feedback rule applies unchanged
        S.ShadowEngine(None, 0, 4, code="topk", error_feedback=True, num_aggregate=2)


# ---------------------------------------------------------------------------------------------------- CPU: launcher
def _args(tmp_path, *extra):
    return add_fit_args(argparse.ArgumentParser(), [
        "--network", "LeNet", "--dataset", "MNIST", "--synthetic", "1", "--train-len", "512", "--test-len", "128",
        "--batch-size", "32", "--test-batch-size", "64", "--lr", "0.05", "--log-interval", "1", "--eval-freq", "100",
        "--train-dir", str(tmp_path) + "/", *extra])


def test_flag_parse():
    a = add_fit_args(argparse.ArgumentParser(), ["--code", "topk", "--entry-budget", "0.01", "--error-feedback", "1"])
    assert a.code == "topk" and a.entry_budget == 0.01 and a.error_feedback is True


def test_launcher_routes_topk(tmp_path, monkeypatch):
    from atomo_b200.runtime import shadow_engine as S
    seen = []

    class Fake:
        def __init__(self, model, rank, world, **kw):
            seen.append(kw)
    monkeypatch.setattr(S, "ShadowEngine", Fake)
    model = torch.nn.Linear(4, 4)
    for engine in ("auto", "shadow"):
        eng, kind = L._build_engine(_args(tmp_path, "--code", "topk", "--dtype", "bf16", "--engine", engine,
                                          "--entry-budget", "0.01", "--error-feedback", "1"), model, 0, 1)
        assert kind == "shadow" and seen[-1]["code"] == "topk" and seen[-1]["entry_budget"] == 0.01
        assert seen[-1]["error_feedback"] is True
    n = len(seen)
    from atomo_b200.runtime import engine as E
    monkeypatch.setattr(E, "FusedEngine", lambda *a, **kw: None)
    _, kind = L._build_engine(_args(tmp_path, "--code", "entrywise", "--dtype", "bf16", "--engine", "auto"), model, 0, 1)
    assert kind == "fused" and len(seen) == n       # --engine auto keeps entrywise on the fp32-flat engine
    for extra in (("--dtype", "fp32"), ("--dtype", "bf16", "--engine", "fused")):
        with pytest.raises(SystemExit, match="topk"):
            L._build_engine(_args(tmp_path, "--code", "topk", *extra), model, 0, 1)
    assert len(seen) == n
    with pytest.raises(SystemExit, match="bf16"):           # --engine shadow still needs bf16 weights
        L._build_engine(_args(tmp_path, "--code", "qsgd", "--dtype", "fp32", "--engine", "shadow"), model, 0, 1)
    assert len(seen) == n


def test_role_paths_refuse_topk(monkeypatch, tmp_path):
    from atomo_b200 import distributed_nn
    from atomo_b200.runtime.master import build_coder
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    with pytest.raises(SystemExit, match="p2p bf16 engine"):
        distributed_nn.run_rank(_args(tmp_path, "--code", "topk", "--backend", "gloo"))
    with pytest.raises(ValueError, match="p2p bf16 engine"):
        build_coder({"code": "topk", "entry_budget": 0.05}, worker_side=True)


# ---------------------------------------------------------------------------------------------------- GPU harness
from test_gpu_shadow_entrywise import HE  # noqa: E402


class HT(HE):
    """The loopback harness of the entry-wise tests (one owner, W virtual workers) on a top-k plan."""

    def __init__(self, shapes, budget=0.05, W=1, **kw):
        super().__init__(shapes, budget, W=W, **kw)
        pl = self.plan = P.build_plan2(shapes, "topk", n_owners=1, n_groups=1, entry_budget=budget)
        u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to(self.dev)
        self.t_units = u8(pl.units_bytes())
        nc = max(pl.n_coded, 1)
        i32 = lambda n: torch.zeros(n, dtype=torch.int32, device=self.dev)
        self.sel, self.hist, self.tcounts = i32(8 * nc), i32(256 * nc), i32(128 * max(len(pl.enc_tiles), 1))
        self.acc = torch.zeros(7 * nc, dtype=torch.float64, device=self.dev)
        self.spart = torch.zeros(5 * len(pl.enc_tiles), dtype=torch.float64, device=self.dev)

    def fill_special(self, w, seed):
        phys = self.fill(w, seed, zero=(ZERO,), spike=(SPIKE,))
        for q in self.plan.params:
            if q.index in (TIES, INF):
                t = self.wgrads[w][q.widx]
                if q.index == TIES:
                    t.copy_((t.float() * 2).round() / 8)        # 7-ish distinct magnitudes: ties across tiles
                else:
                    (t.permute(0, 2, 3, 1) if t.dim() == 4 else t).view(-1)[1234] = float("inf")
                phys[q.index] = (t.permute(0, 2, 3, 1) if t.dim() == 4 else t).reshape(-1).float()
        return phys

    def encode(self, w, residual=0, stats=False):
        C, pl = self.C, self.plan
        gptr = torch.tensor([t.data_ptr() for t in self.wgrads[w]], dtype=torch.int64, device=self.dev)
        self._gptr = gptr
        t0, nt = pl.enc_range[0]
        C.v2_topk_select(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr.data_ptr(),
                         self.hist.data_ptr(), self.tcounts.data_ptr(), self.counters.data_ptr(),
                         self.sel.data_ptr(), 0, 0)
        C.v2_topk_encode(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr.data_ptr(), self.sel.data_ptr(),
                         self.tcounts.data_ptr(), self.t_arena_peer.data_ptr(), self.t_sig_peer.data_ptr(), 1,
                         pl.arena_floats, w, 0, self.ctrl.data_ptr(), self.counters.data_ptr() + 4 * (pl.n_coded + 8),
                         0, False, residual)
        if stats:
            C.v2_topk_code_stats(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr.data_ptr(),
                                 self.sel.data_ptr(), self.tcounts.data_ptr(), self.t_arena_peer.data_ptr(), 1,
                                 pl.arena_floats, w, self.spart.data_ptr(), self.counters.data_ptr(),
                                 self.acc.data_ptr())
        torch.cuda.synchronize()


def _oracle_words(flat, u, budget):
    """Per tile: the int32 words the encoder must write (offset | exact flag | bf16 bits << 16)."""
    idx = _coder(budget).select(flat.cpu()).tolist()
    bits = flat.cpu().to(torch.bfloat16).view(torch.int16).to(torch.int32) & 0xFFFF
    out = [[] for _ in range(u.n_ps)]
    for i in idx:
        j, o = divmod(i, P.ENTRY_TILE_ELEMS)
        w = o | 0x1000 | (int(bits[i]) << 16)
        out[j].append(w - (1 << 32) if w >= 1 << 31 else w)
    return out, len(idx)


# ---------------------------------------------------------------------------------------------------- GPU: kernels
@pytest.mark.gpu
@pytest.mark.parametrize("budget", [0.01, 0.05, 0.25, 200.0])
def test_v2_topk_encode_matches_oracle_bitwise(budget):
    h = HT(ORACLE_SHAPES, budget)
    h.set_step(3)
    phys = h.fill_special(0, 11)
    for rep in range(2):                                       # the state and histograms reset themselves
        h.encode(0)
        for u in h.plan.units:
            if u.kind != P.KIND_ENTRY:
                continue
            want, k_eff = _oracle_words(phys[u.param], u, budget)
            tiles = h.tiles(u, 0)
            assert sum(t[1] for t in tiles) == k_eff, u.param
            for j, (stamp, count, scale, words) in enumerate(tiles):
                assert stamp == 3 and scale == 0.0
                assert count == len(want[j]), (u.param, j)
                assert words[:count].tolist() == want[j], (u.param, j)
                assert bool((words[count:] == 0).all())
            if u.param == INF or u.param == ZERO:
                assert k_eff == 0
        assert int(h.hist.abs().sum()) == 0                     # histograms left zero for the next launch
    assert int(h.signals[0]) == 3
    # the tie case really straddles tiles: the threshold's entries lie in more than one tile, some dropped
    u = next(u for u in h.plan.units if u.param == TIES)
    flat = phys[TIES].cpu()
    idx = _coder(budget).select(flat)
    if idx.numel():
        mag = flat.abs()
        T = float(mag[idx].min())
        assert len({int(i) // P.ENTRY_TILE_ELEMS for i in (mag == T).nonzero().flatten()}) > 1


@pytest.mark.gpu
def test_v2_topk_is_repeatable():
    h = HT(ORACLE_SHAPES, 0.05)
    h.set_step(4)
    h.fill_special(0, 3)
    h.encode(0)
    first = h.arena.clone()
    h.arena.zero_()
    h.set_step(5)
    h.encode(0)
    h.set_step(4)
    h.arena.zero_()
    h.encode(0)
    assert torch.equal(h.arena.view(torch.int32), first.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 2])
def test_v2_ps_entry_averages_topk_bitwise(W):
    """lr = 1, no momentum, a zero master: the PS writes -(sum of the oracle decodes in worker order) / W."""
    h = HT(NET_SHAPES, 0.05, W=W, lr=1.0)
    want = torch.zeros(h.plan.w_total, device=h.dev)
    for w in range(W):
        phys = h.fill(w, 70 + w, spike=(3,))
        h.encode(w)
        for u in h.plan.units:
            if u.kind == P.KIND_ENTRY:
                c = _coder(0.05)
                dec = c.decode(c.encode(phys[u.param].cpu())).to(h.dev)
                want[u.w_off:u.w_off + u.numel] += dec
    want = want * torch.tensor(1.0 / W, dtype=torch.float32)
    h.master.zero_()
    h.ps()
    assert int(h.ctrl.view(torch.int32)[1]) == 0
    used = torch.zeros(h.plan.w_total, dtype=torch.bool, device=h.dev)
    for q in h.plan.params:
        if q.is_w:
            used[q.off:q.off + q.numel] = True
    assert torch.equal(-h.master[used], want[used])


@pytest.mark.gpu
def test_v2_topk_code_stats_match_fp64():
    h = HT(ORACLE_SHAPES, 0.05)
    h.set_step(2)
    phys = h.fill_special(0, 21)
    h.encode(0, stats=True)
    acc = h.acc.view(-1, 7).tolist()
    for u in h.plan.units:
        if u.kind != P.KIND_ENTRY or u.param == INF:
            continue
        flat = phys[u.param].cpu().double()
        c = _coder(0.05)
        dec = c.decode(c.encode(phys[u.param].cpu())).double()
        gsq, mse, ex, bias, real, real4, n = acc[u.ts_index]
        k_eff = int(c.select(phys[u.param].cpu()).numel())
        assert n == 1 and bias == 0 and ex == real == real4 == k_eff
        assert gsq == pytest.approx(float(flat.square().sum()), rel=1e-12, abs=0)
        assert mse == pytest.approx(float((flat - dec).square().sum()), rel=1e-12, abs=1e-300)


# ---------------------------------------------------------------------------------------------------- GPU: feedback
def _grads(seed=0):
    from test_gpu_error_feedback import SHAPES
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(s, generator=g) * (0.01 * (1 + i))).bfloat16().float().cuda() for i, s in enumerate(SHAPES)]


@pytest.mark.gpu
@pytest.mark.parametrize("budget", [0.01, 0.05])
def test_error_feedback_identity_and_contraction(budget):
    from test_gpu_error_feedback import Loopback
    h = Loopback("topk", _grads(1), entry_budget=budget)
    try:
        g, e_old = h.g, h.residual()
        for _ in range(4):
            A = g + e_old
            ghat, e_new = h.step()
            scale = g.abs() + e_old.abs() + ghat.abs() + e_new.abs()
            assert bool(((A - (ghat + e_new)).abs() <= 1e-6 * scale + 1e-7 * float(scale.max())).all())
            for q in h.w:
                a = A[q.off:q.off + q.numel]
                nnz = int((a.float().to(torch.bfloat16) != 0).sum())
                k_eff = min(_coder(budget).k_for(q.numel), nnz)
                drop = float((a - ghat[q.off:q.off + q.numel]).square().sum())
                assert drop <= (1 - k_eff / max(nnz, 1)) * float(a.square().sum()) * (1 + 1e-5) + 1e-30
            e_old = e_new
    finally:
        h.close()


@pytest.mark.gpu
def test_error_feedback_residual_stays_bounded():
    """A fixed gradient for 200 steps: e stays below the contraction bound sqrt(1-d) / (1 - sqrt(1-d)) ||g||."""
    from test_gpu_error_feedback import Loopback
    h = Loopback("topk", _grads(2), entry_budget=0.05)
    try:
        s = torch.zeros_like(h.g)
        for _ in range(200):
            ghat, e = h.step()
            s += ghat
        d = min(_coder(0.05).k_for(q.numel) / q.numel for q in h.w)
        bound = math.sqrt(1 - d) / (1 - math.sqrt(1 - d)) * float(h.g.norm())
        assert float(e.norm()) <= bound
        assert torch.allclose(s - 200 * h.g, -e, rtol=0, atol=200 * 1e-6 * (float(h.g.abs().max()) + float(e.abs().max())))
    finally:
        h.close()


# ---------------------------------------------------------------------------------------------------- GPU: engine
def _train(net, graph, ef, steps=6, budget=0.01, lr=0.05, seed=3):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model, input_shape
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    x, y = SyntheticImageDataset(input_shape(net), 10, 4096, seed=0).materialize(32)
    eng = ShadowEngine(build_model(net, 10), 0, 1, code="topk", entry_budget=budget, lr=lr, momentum=0.9,
                       use_graph=graph, overlap=graph, seed=seed, error_feedback=ef)
    eng.prepare(x.pin_memory(), y.pin_memory(), warmup=2)
    losses, norms = [], []
    for _ in range(steps):
        losses.append(float(eng.train_step(x, y)[0]))
        if ef:
            norms.append(eng.error_feedback_norm()["model"])
    torch.cuda.synchronize()
    assert eng.error_code() == 0
    m = eng.gather_fp32("master").clone()
    eng.close()
    return m, losses, norms


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["ResNet18", "VGG11"])
@pytest.mark.parametrize("ef", [False, True])
def test_graph_replay_equals_eager(net, ef, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    mg, _, _ = _train(net, True, ef)
    me, _, _ = _train(net, False, ef)
    assert torch.equal(mg, me)


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["ResNet18", "VGG11"])
def test_error_feedback_training_stays_finite(net):
    """lr 0.05 / momentum 0.9, 1 %: the setting where entry-wise 1 % with error feedback diverges."""
    _, losses, norms = _train(net, True, True, steps=30)
    assert all(math.isfinite(v) for v in losses + norms)
    assert max(norms[10:]) < 20 * max(norms[:10]), norms
    assert losses[-1] < losses[0], losses


@pytest.mark.gpu
def test_checkpoint_round_trip(tmp_path):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.cuda.set_device(0)
    x, y = SyntheticImageDataset((3, 32, 32), 10, 256).materialize(32)

    def mk():
        torch.manual_seed(0)
        return ShadowEngine(build_model("VGG11", 10), 0, 1, code="topk", entry_budget=0.05, lr=0.05, momentum=0.9,
                            use_graph=False)
    a = mk()
    a.prepare(x.pin_memory(), y.pin_memory(), warmup=0)
    for _ in range(3):
        a.train_step(x, y)
    path = a.save_checkpoint(str(tmp_path) + "/")
    side = torch.load(path + "_optim", weights_only=False)
    assert side["code"] == "topk" and side["entry_budget"] == 0.05
    want = a.gather_fp32("master").clone()
    a.close()
    b = mk()
    b.prepare(x.pin_memory(), y.pin_memory(), warmup=0)
    b.load_checkpoint(str(tmp_path) + "/", 3)
    assert b.device_step() == 4 and torch.equal(b.gather_fp32("master"), want)
    b.train_step(x, y)
    torch.cuda.synchronize()
    assert b.error_code() == 0
    b.close()


def _launch(tmp_path, monkeypatch, *extra):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    args = add_fit_args(argparse.ArgumentParser(), [
        "--network", "ResNet18", "--dataset", "Cifar10", "--synthetic", "1", "--train-len", "512", "--test-len", "64",
        "--batch-size", "32", "--test-batch-size", "64", "--backend", "p2p", "--dtype", "bf16", "--max-steps", "6",
        "--log-interval", "2", "--eval-freq", "100", "--train-dir", str(tmp_path) + "/",
        "--metrics-file", str(tmp_path / "m"), *extra])
    L.run_p2p_training(args)
    return [json.loads(l) for l in open(str(tmp_path / "m") + ".rank0.jsonl")]


@pytest.mark.gpu
def test_launcher_topk_writes_ef_norm_and_code_stats(tmp_path, monkeypatch):
    recs = _launch(tmp_path, monkeypatch, "--code", "topk", "--entry-budget", "0.01", "--error-feedback", "1",
                   "--code-stats", "1")
    assert recs and all(r["ef_norm"] > 0 and math.isfinite(r["ef_norm"]) for r in recs)
    m = recs[-1]["code_stats"]["model"]
    assert m["exp_atoms"] > 0 and 0 < m["rel_var"] < 1


@pytest.mark.gpu
@pytest.mark.multigpu
def test_shadow_engine_topk_multi_gpu_replicas_identical():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    from test_gpu_v2 import _run_mp
    world = 2 if n < 8 else (8 if os.environ.get("ATOMO_TEST_WORLD8") else 2)
    res = _run_mp(world, {"code": "topk", "ps_mode": "sharded", "net": "VGG11"}, 29790)
    for rank, err, same, l0, l1, mode, mc, _ in res:
        assert err == 0 and same, res

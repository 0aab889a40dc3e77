"""QSGD / TernGrad on the overlapped, sharded bf16 engine: planner and launcher (CPU), kernels against the
``codings.qsgd`` oracle and the engine end to end (GPU)."""
import argparse
import os
import sys
import types

import pytest
import torch

from atomo_b200.ops import plan2 as P

from shadow_harness import LoopbackPS, batch, opt_ref, run_mp

NET_SHAPES = [(64, 3, 3, 3), (64,), (64,), (128, 64, 3, 3), (128,), (256, 128, 3, 3), (512, 256, 1, 1), (300, 200),
              (10, 512), (10,)]
ORACLE_SHAPES = [(64, 3, 3, 3), (64, 32, 3, 3), (10, 512), (300, 200), (7, 20), (5, 300), (64,)]


# ---------------------------------------------------------------------------------------------------- planner
@pytest.mark.parametrize("code,q,bucket,owners", [("qsgd", 4, 512, 1), ("terngrad", 2, 256, 3), ("qsgd", 8, 1024, 2),
                                                  ("qsgd", 1, 32, 4)])
def test_plan2_qsgd_units_tiles_and_slots(code, q, bucket, owners):
    from atomo_b200.codings.qsgd import words_per_bucket
    pl = P.build_plan2(NET_SHAPES, code, n_owners=owners, n_groups=3, quantization_level=q, bucket_size=bucket)
    for p in pl.params:
        units = [u for u in pl.units if u.param == p.index]
        if p.is_w:
            assert len(units) == 1 and units[0].kind == P.KIND_QSGD, p.shape
            u = units[0]
            b = min(bucket, p.numel)
            assert (u.K, u.I, u.numel, u.w_off) == (b, q, p.numel, p.off)
            assert u.rows == -(-p.numel // b) and u.cols == words_per_bucket(b, q)
            assert u.rs == (1 if code == "terngrad" else 0)
        else:
            assert len(units) == 1 and units[0].kind == P.KIND_VEC
    assert not any(u.kind == P.KIND_DENSE16 for u in pl.units)
    assert pl.n_coded == sum(1 for p in pl.params if p.is_w)
    # PS tiles: every bucket exactly once, bucket-aligned, <= 4096 elements; owners round-robin inside a group
    for u in pl.units:
        if u.kind != P.KIND_QSGD:
            continue
        tiles = [(a, b, o) for (ui, a, b, o) in pl.ps_tiles if ui == u.index]
        assert len(tiles) == u.n_ps
        covered = []
        for a, b, o in tiles:
            assert a % u.K == 0 and b <= P.QSGD_TILE_ELEMS and (b % u.K == 0 or a + b == u.numel)
            covered.extend(range(a // u.K, -(-(a + b) // u.K)))
        assert sorted(covered) == list(range(u.rows))
        enc = [(a, b) for (ui, a, b, j) in pl.enc_tiles if ui == u.index]
        assert enc == sorted((a, b) for a, b, _ in tiles)
    for g in range(pl.n_groups):
        seq = [(ui, a) for (ui, a, b, o) in pl.ps_tiles if pl.units[ui].group == g]
        by_order = []
        for ui in pl.group_units[g]:
            u = pl.units[ui]
            e = u.ps_rows if u.kind == P.KIND_QSGD else P.DENSE_TILE_ELEMS
            by_order.extend((ui, a) for a in range(0, u.numel, e))
        owner_of = {(ui, a): o for (ui, a, b, o) in pl.ps_tiles}
        assert sorted(seq) == sorted(by_order)
        assert [owner_of[k] for k in by_order] == [j % owners for j in range(len(by_order))]
    # slots: disjoint, 16-byte aligned words, inside the arena
    spans = []
    for u in pl.units:
        if u.kind == P.KIND_QSGD:
            wo = u.slot_off + P.qsgd_words_off(u.n_ps, u.rows)
            assert u.slot_off % 4 == 0 and wo % 4 == 0
            assert u.slot_off + P.qsgd_norms_off(u.n_ps) >= u.slot_off + u.n_ps
            spans.append((u.slot_off, wo + 2 * u.rows * u.cols))
    spans.sort()
    assert all(a1 >= b0 for (a0, b0), (a1, b1) in zip(spans, spans[1:]))
    assert spans[-1][1] <= pl.arena_floats
    # wire bytes == bytes of codings.qsgd words + norms for the same (physical-order) tensors
    from atomo_b200 import codings
    coder = codings.build(code, quantization_level=q, bucket_size=bucket)
    want = 0
    for s in NET_SHAPES:
        if len(s) >= 2:
            c = coder.encode(torch.zeros(s))
            want += c["words"].numel() * 8 + c["norms"].numel() * 4
    assert pl.qsgd_bytes() == want
    assert pl.expected_factor_bytes() == want
    assert pl.dense_bytes() == 4 * sum(p.numel for p in pl.params if not p.is_w)


def test_plan2_qsgd_refuses_unrepresentable_settings():
    with pytest.raises(ValueError):
        P.build_plan2(NET_SHAPES, "qsgd", bucket_size=1028)
    with pytest.raises(ValueError):
        P.build_plan2(NET_SHAPES, "qsgd", bucket_size=100)
    with pytest.raises(ValueError):
        P.build_plan2(NET_SHAPES, "terngrad", quantization_level=0)
    with pytest.raises(ValueError):
        P.build_plan2(NET_SHAPES, "qsgd", quantization_level=15)


def test_plan2_spectral_plans_ignore_the_qsgd_settings():
    for code in ("svd", "qsvd", "sgd"):
        a = P.build_plan2(NET_SHAPES, code, 3, n_owners=2, n_groups=3)
        b = P.build_plan2(NET_SHAPES, code, 3, n_owners=2, n_groups=3, quantization_level=2, bucket_size=64)
        assert a.units_bytes() == b.units_bytes() and a.ps_tiles == b.ps_tiles and a.enc_tiles == b.enc_tiles
        assert a.arena_floats == b.arena_floats and a.qsgd_bytes() == 0


# ---------------------------------------------------------------------------------------------------- launcher
def _fake_engines(monkeypatch):
    made = []

    class Fake:
        def __init__(self, *a, **kw):
            made.append((type(self).__name__, kw))

    shadow = types.ModuleType("atomo_b200.runtime.shadow_engine")
    shadow.ShadowEngine = type("ShadowEngine", (Fake,), {})
    fused = types.ModuleType("atomo_b200.runtime.engine")
    fused.FusedEngine = type("FusedEngine", (Fake,), {})
    monkeypatch.setitem(sys.modules, "atomo_b200.runtime.shadow_engine", shadow)
    monkeypatch.setitem(sys.modules, "atomo_b200.runtime.engine", fused)
    return made


def _args(*argv):
    from atomo_b200.utils.flags import add_fit_args
    return add_fit_args(argparse.ArgumentParser(), list(argv))


def test_p2p_launcher_engine_shadow_runs_qsgd(monkeypatch):
    from atomo_b200.runtime import p2p_launcher as L
    made = _fake_engines(monkeypatch)
    _, kind = L._build_engine(_args("--engine", "shadow", "--dtype", "bf16", "--code", "qsgd", "--quantization-level",
                                    "2", "--bucket-size", "256", "--optimizer", "adam"), None, 0, 2)
    assert kind == "shadow" and made[-1][0] == "ShadowEngine"
    kw = made[-1][1]
    assert kw["code"] == "qsgd" and kw["quantization_level"] == 2 and kw["bucket_size"] == 256
    assert kw["optimizer"] == "adam"
    _, kind = L._build_engine(_args("--engine", "shadow", "--dtype", "bf16", "--code", "terngrad"), None, 0, 2)
    assert kind == "shadow" and made[-1][1]["quantization_level"] == 4 and made[-1][1]["bucket_size"] == 512
    _, kind = L._build_engine(_args("--engine", "shadow", "--dtype", "bf16", "--code", "svd"), None, 0, 2)
    assert kind == "shadow"
    _, kind = L._build_engine(_args("--engine", "fused", "--dtype", "bf16", "--code", "svd"), None, 0, 2)
    assert kind == "fused" and made[-1][0] == "FusedEngine"
    _, kind = L._build_engine(_args("--dtype", "bf16", "--code", "qsgd"), None, 0, 2)      # auto: unchanged
    assert kind == "fused"


def test_p2p_launcher_engine_shadow_refuses_entrywise_and_fp32(monkeypatch):
    from atomo_b200.runtime import p2p_launcher as L
    made = _fake_engines(monkeypatch)
    with pytest.raises(SystemExit, match="entrywise"):
        L._build_engine(_args("--engine", "shadow", "--dtype", "bf16", "--code", "entrywise"), None, 0, 2)
    with pytest.raises(SystemExit, match="bf16"):
        L._build_engine(_args("--engine", "shadow", "--dtype", "fp32", "--code", "qsgd"), None, 0, 2)
    assert not made


# ---------------------------------------------------------------------------------------------------- GPU harness
class HQ(LoopbackPS):
    """QSGD / TernGrad; ``fill`` scales the gradients by ``scale``."""

    PS = "v2_ps_qsgd"

    def __init__(self, shapes, code="qsgd", q=4, bucket=512, W=1, lr=0.1, momentum=0.0, wd=0.0, nesterov=False,
                 opt=0, seed=7, num_aggregate=0):
        super().__init__(shapes, code, W, lr, momentum, wd, nesterov, opt, seed, num_aggregate, quantization_level=q,
                         bucket_size=bucket)
        self.code = code
        pl = self.plan
        self.clip = self.zeros(self.nc)
        self.partials = self.zeros(2 * len(pl.enc_tiles), torch.float64)
        self.maxq = max(u.I for u in pl.units if u.kind == P.KIND_QSGD)
        self.maxb = max(u.K for u in pl.units if u.kind == P.KIND_QSGD)
        self.ps_tail = (self.maxq, self.maxb)

    def tensor(self, q, x, g, scale=1.0):
        return x * scale

    def encode(self, w, uniforms=None):
        C, pl = self.C, self.plan
        gptr = self.gptr(w)
        t0, nt = pl.enc_range[0]
        tern = self.code == "terngrad"
        if tern:
            C.v2_qsgd_stats(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr, self.partials.data_ptr(),
                            self.counters.data_ptr(), self.clip.data_ptr(), 0, 0)
        C.v2_qsgd_encode(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr,
                         self.clip.data_ptr() if tern else 0, self.t_arena_peer.data_ptr(), self.t_sig_peer.data_ptr(),
                         1, pl.arena_floats, w, 0, self.ctrl.data_ptr(), self.counter(),
                         uniforms.data_ptr() if uniforms is not None else 0, 0, False, not tern, self.maxq, self.maxb,
                         tern)
        torch.cuda.synchronize()

    def slot(self, u, w):
        """(stamps, norms, words [buckets, L] int64) of unit u in worker w's slot."""
        base = self.arena[w * self.plan.arena_floats + u.slot_off:]
        stamps = base[:u.n_ps].view(torch.int32).clone()
        no, wo = P.qsgd_norms_off(u.n_ps), P.qsgd_words_off(u.n_ps, u.rows)
        norms = base[no:no + u.rows].clone()
        words = base[wo:wo + 2 * u.rows * u.cols].view(torch.int64).view(u.rows, u.cols).clone()
        return stamps, norms, words

    def code_of(self, u, w):
        q = self.plan.params[u.param]
        _, norms, words = self.slot(u, w)
        return {"words": words, "norms": norms, "quantization_level": u.I, "bucket_size": u.K, "shape": [q.numel],
                "scheme": self.code}


# ---------------------------------------------------------------------------------------------------- GPU: encode
@pytest.mark.gpu
@pytest.mark.parametrize("code", ["qsgd", "terngrad"])
@pytest.mark.parametrize("q,bucket", [(2, 256), (4, 512), (8, 256), (4, 256), (8, 512)])
def test_v2_qsgd_encode_matches_oracle(code, q, bucket):
    from atomo_b200 import codings
    h = HQ(ORACLE_SHAPES, code, q, bucket)
    pl = h.plan
    step = 3
    h.set_step(step)
    phys = h.fill(0, 11 + q)
    uni = torch.rand(pl.w_total + 2048, device=h.dev, generator=torch.Generator(device="cuda").manual_seed(q))
    h.encode(0, uni)
    coder = codings.build(code, quantization_level=q, bucket_size=bucket)
    for u in pl.units:
        if u.kind != P.KIND_QSGD:
            continue
        flat = phys[u.param]
        if code == "terngrad":
            want_clip = 2.5 * float(flat.std(unbiased=False))
            assert abs(float(h.clip[u.ts_index]) - want_clip) <= 1e-4 * want_clip, (u.param, want_clip)
        ref = coder.encode(flat.cpu(), uniforms=uni[u.w_off:u.w_off + u.rows * u.K].cpu())
        stamps, norms, words = h.slot(u, 0)
        assert bool((stamps == step).all())
        assert torch.allclose(norms.cpu(), ref["norms"], rtol=1e-5), u.param
        assert float((words.cpu() != ref["words"]).float().mean()) < 2e-2, u.param
        mine = dict(ref)
        mine["words"], mine["norms"] = words.cpu(), norms.cpu()
        a, b = coder.decode(mine), coder.decode(ref)
        tol = 1e-4 * float(b.abs().max())
        assert float(((a - b).abs() > tol).float().mean()) < 2e-3, u.param
    assert int(h.signals[0]) == step


@pytest.mark.gpu
@pytest.mark.parametrize("code", ["qsgd", "terngrad"])
def test_v2_qsgd_philox_rounding_is_unbiased(code):
    from atomo_b200 import codings
    shapes = [(32, 16, 3, 3), (40, 30)]
    h = HQ(shapes, code, 2, 256)
    phys = h.fill(0, 5)
    coder = codings.build(code, quantization_level=2, bucket_size=256)
    units = [u for u in h.plan.units if u.kind == P.KIND_QSGD]
    acc = {u.index: 0 for u in units}
    T = 1000
    for t in range(T):
        h.set_step(t + 1)
        h.encode(0)
        for u in units:
            d = coder.decode(h.code_of(u, 0)).to(h.dev)
            acc[u.index] = acc[u.index] + d
    for u in units:
        flat = phys[u.param]
        if code == "terngrad":      # the estimator is unbiased for the clipped gradient
            lim = 2.5 * float(flat.std(unbiased=False))
            flat = flat.clamp(-lim, lim)
        mean = acc[u.index] / T
        # one draw is lo or lo + 1 levels (step = norm / levels): its standard deviation is at most step / 2
        step = (h.slot(u, 0)[1] / 3.0).repeat_interleave(u.K)[:u.numel]
        bound = 4 * (step / 2) / T ** 0.5 + 1e-6 * float(flat.abs().max())
        frac_out = float(((mean - flat).abs() > bound).float().mean())
        assert frac_out < 1e-3, (u.param, frac_out)
        assert float((mean - flat).norm() / flat.norm()) < 0.2


# ---------------------------------------------------------------------------------------------------- GPU: PS
def _decoded_sum(h, workers, coder):
    """sum over `workers` (in worker order, fp32) of the codings.qsgd decodes of the words actually in the arena,
    physical order.  Decoded on the CPU: there ``norms / s`` is an IEEE division, as in the PS kernel (on CUDA, torch
    divides by a scalar through its reciprocal, which rounds differently)."""
    pl = h.plan
    est = torch.zeros(pl.w_total)
    for u in pl.units:
        if u.kind != P.KIND_QSGD:
            continue
        codes = []
        for w in workers:
            c = h.code_of(u, w)
            c["words"], c["norms"] = c["words"].cpu(), c["norms"].cpu()
            codes.append(c)
        for c in codes:
            est[u.w_off:u.w_off + u.numel] += coder.decode(c, codes=codes)
    return est.to(h.dev)


@pytest.mark.gpu
@pytest.mark.parametrize("code", ["qsgd", "terngrad"])
def test_v2_ps_qsgd_decoded_mean_is_bitwise_the_coders(code):
    """With lr = 1, no momentum / weight decay and a zero master, the PS writes master = -g exactly, so the kernel's
    averaged gradient can be compared bit for bit with the coder's decodes summed in worker order, times 1/W."""
    from atomo_b200 import codings
    W = 3
    h = HQ(NET_SHAPES, code, 4, 512, W=W, lr=1.0)
    pl = h.plan
    coder = codings.build(code, quantization_level=4, bucket_size=512)
    for w in range(W):
        h.fill(w, 70 + w)
        h.encode(w)
    want = _decoded_sum(h, range(W), coder) * torch.tensor(1.0 / W, dtype=torch.float32)
    h.master.zero_()
    h.ps()
    assert int(h.ctrl.view(torch.int32)[1]) == 0
    used = torch.zeros(pl.w_total, dtype=torch.bool, device=h.dev)
    for q in pl.params:
        if q.is_w:
            used[q.off:q.off + q.numel] = True
    assert torch.equal(-h.master[used], want[used])
    assert int((want[used] == 0).sum()) > 0          # the cancelling sums are part of the comparison


@pytest.mark.gpu
@pytest.mark.parametrize("code", ["qsgd", "terngrad"])
@pytest.mark.parametrize("momentum,nesterov,wd,opt", [(0.0, False, 0.0, 0), (0.9, True, 1e-3, 0), (0.9, False, 0.0, 0),
                                                      (0.0, False, 0.0, 1), (0.0, False, 1e-3, 2)])
def test_v2_ps_qsgd_matches_reference(code, momentum, nesterov, wd, opt):
    from atomo_b200 import codings
    W, lr = 3, 0.05
    h = HQ(NET_SHAPES, code, 4, 512, W=W, lr=lr, momentum=momentum, wd=wd, nesterov=nesterov, opt=opt)
    pl = h.plan
    coder = codings.build(code, quantization_level=4, bucket_size=512)
    used = torch.zeros(pl.w_total, dtype=torch.bool, device=h.dev)
    vused = torch.zeros(pl.v_total, dtype=torch.bool, device=h.dev)
    for q in pl.params:
        (used if q.is_w else vused)[q.off:q.off + q.numel] = True
    for step in (1, 2):
        h.set_step(step)
        for w in range(W):
            h.fill(w, 10 * step + w)
            h.encode(w)
        gw = _decoded_sum(h, range(W), coder) / W
        gv = sum(h.vgrads) / W
        rp, rm = opt_ref(h.master.clone(), gw, h.mom.clone(), h.sq.clone(), h.sqmax.clone(), step, lr, momentum,
                          nesterov, wd, opt)
        rv, _ = opt_ref(h.vparams.clone(), gv, h.vmom.clone(), h.vsq.clone(), h.vsqmax.clone(), step, lr, momentum,
                         nesterov, wd, opt)
        h.ps()
        assert int(h.ctrl.view(torch.int32)[1]) == 0
        assert int(h.signals[256]) == step + 1
        tol = dict(rtol=3e-4, atol=3e-5) if opt == 0 else dict(rtol=2e-3, atol=2e-4)
        assert torch.allclose(h.master[used], rp[used], **tol), float((h.master - rp)[used].abs().max())
        assert torch.allclose(h.vparams[vused], rv[vused], **tol)
        assert torch.equal(h.wshadow[used], h.master.to(torch.bfloat16)[used])


@pytest.mark.gpu
@pytest.mark.parametrize("code", ["qsgd", "terngrad"])
def test_v2_ps_qsgd_num_aggregate_and_stale_slots(code):
    """num_aggregate = 2 of 3 workers, worker 1 never pushes: only {0, 2} are averaged (TernGrad: max norm over
    {0, 2}).  Then a slot whose stamp is of another step is skipped and flagged with ERR2_SLOT_STEP."""
    from atomo_b200 import codings
    lr = 0.1
    h = HQ(NET_SHAPES, code, 4, 512, W=3, lr=lr, num_aggregate=2)
    pl = h.plan
    coder = codings.build(code, quantization_level=4, bucket_size=512)
    for w in (0, 2):
        h.fill(w, 40 + w)
        h.encode(w)
    h.vgrads[1].fill_(1e6)                         # garbage a skipped worker may hold
    assert int(h.signals[0]) == 1 and int(h.signals[1]) == 0 and int(h.signals[2]) == 1
    est = _decoded_sum(h, (0, 2), coder)
    p0, v0 = h.master.clone(), h.vparams.clone()
    h.ps()
    assert int(h.ctrl.view(torch.int32)[1]) == 0 and int(h.signals[256]) == 2
    assert int(h.signals[320]) == 0b101 and int(h.signals[321]) == 1
    used = torch.zeros(pl.w_total, dtype=torch.bool, device=h.dev)
    vused = torch.zeros(pl.v_total, dtype=torch.bool, device=h.dev)
    for q in pl.params:
        (used if q.is_w else vused)[q.off:q.off + q.numel] = True
    assert torch.allclose(h.master[used], (p0 - lr * est / 2)[used], rtol=3e-4, atol=3e-5)
    assert torch.allclose(h.vparams[vused], (v0 - lr * (h.vgrads[0] + h.vgrads[2]) / 2)[vused], rtol=3e-4, atol=3e-5)

    # stale stamp: worker 1's slot still holds step 0 (never written) while its flag claims step 1
    hs = HQ(NET_SHAPES, code, 4, 512, W=2, lr=lr)
    hs.fill(0, 1)
    hs.encode(0)
    hs.signals[1] = 1
    hs.ps()
    assert int(hs.ctrl.view(torch.int32)[1]) & 4          # ERR2_SLOT_STEP


# ---------------------------------------------------------------------------------------------------- GPU: engine
def _engine(net, code, graph, overlap, seed=3):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    return ShadowEngine(build_model(net, 10), 0, 1, code=code, lr=0.05, momentum=0.9, use_graph=graph,
                        overlap=overlap, seed=seed)


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["ResNet18", "VGG11"])
@pytest.mark.parametrize("code", ["qsgd", "terngrad"])
@pytest.mark.parametrize("graph,overlap", [(True, True), (False, False)])
def test_shadow_engine_qsgd_trains_single_gpu(net, code, graph, overlap, tmp_path, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)      # bitwise-reproducible backward
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    x, y = batch(net, 64)
    masters = []
    for rep in range(2):
        eng = _engine(net, code, graph, overlap)
        eng.prepare(x, y, warmup=2)
        first = None
        for _ in range(25):
            stats = eng.train_step(x, y)
            if first is None:
                first = float(stats[0])
        torch.cuda.synchronize()
        last = float(stats[0])
        assert eng.error_code() == 0
        assert eng.device_step() == eng.step == 28
        assert torch.isfinite(torch.tensor(last)) and last < first, (first, last)
        m = eng.gather_fp32("master")
        for q in eng.plan.params:
            if q.is_w:
                assert torch.equal(eng.wshadow[q.off:q.off + q.numel], m[q.off:q.off + q.numel].to(torch.bfloat16))
        masters.append(m.clone())
        if rep == 1 and not graph:
            # checkpoint round trip
            d = str(tmp_path) + "/"
            path = eng.save_checkpoint(d)
            side = torch.load(path + "_optim", weights_only=False)
            assert side["quantization_level"] == 4 and side["bucket_size"] == 512 and side["code"] == code
            want = m.clone()
            eng.close()
            b = _engine(net, code, graph, overlap)
            b.prepare(x, y, warmup=0)
            b.load_checkpoint(d, 27)
            assert b.device_step() == 28
            assert torch.equal(b.gather_fp32("master"), want)
            b.train_step(x, y)
            torch.cuda.synchronize()
            assert b.error_code() == 0
            b.close()
        else:
            eng.close()
    assert torch.equal(masters[0], masters[1])       # same seed, same bits


# ---------------------------------------------------------------------------------------------------- multi GPU
@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("code,ps_mode", [("qsgd", "sharded"), ("qsgd", "colocated"), ("terngrad", "sharded"),
                                          ("terngrad", "colocated")])
def test_shadow_engine_qsgd_multi_gpu_replicas_identical(code, ps_mode):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 8 else (8 if os.environ.get("ATOMO_TEST_WORLD8") else 2)
    port = 29600 + 7 * ["sharded", "colocated"].index(ps_mode) + (3 if code == "terngrad" else 0)
    res = run_mp(world, {"code": code, "ps_mode": ps_mode, "net": "VGG11"}, port)
    for rank, err, same, l0, l1, mode, mc, _ in res:
        assert err == 0 and same, res
    assert all(r[4] < r[3] for r in res), res


@pytest.mark.gpu
@pytest.mark.multigpu
def test_shadow_engine_qsgd_protocol_survives_random_delays():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 8 else (8 if os.environ.get("ATOMO_TEST_WORLD8") else 2)
    res = run_mp(world, {"code": "qsgd", "ps_mode": "sharded", "graph": False, "steps": 8, "warmup": 0,
                          "jitter_us": 300.0}, 29650)
    for r in res:
        assert r[1] == 0 and r[2], res

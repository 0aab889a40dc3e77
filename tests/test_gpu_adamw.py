"""AdamW on the bf16 engine (``ShadowEngine(optimizer="adamw")``): the decay pass ``v2_decay`` of csrc/v2_ema.cu
followed by the engine's Adam with weight decay 0.

* Kernel: over the PS tile ranges of ResNet-18, VGG-11 and LeNet plans (several codes, 1 and 2 owners, 3 groups, an
  aligned and a misaligned base), each launch multiplies exactly the weight elements of its tiles by
  ``Ctrl2.decay_factor``, bit for bit as torch's fp32 ``mul``; vectors and everything outside the range stay.
* Composition: an AdamW step is bit for bit "torch ``master.mul_(f)`` over the group's tiles, then the code's PS launch
  with Adam and weight decay 0", for the PS kernel of every code (engine runs with the decay swapped for the torch
  one), and in the loopback harness with 2 virtual workers and 2 groups over 3 steps (svd and dense, Adam and AMSGrad).
* Engine: ``weight_decay=0`` is ``adam`` bit for bit with the same launches; one dense step against ``optim/adamw.py``
  in fp64 within a bound derived from the fp32 operations; eager = graph and run = rerun; ``set_lr`` between replays;
  clipping above the norm; ``accumulate_steps=2``; the weight average; bitwise resume (Adam and AMSGrad, and across
  ``adam`` / ``adamw``); the launcher.  The two-GPU test checks that the replicas agree.
"""
import functools

import numpy as np
import pytest
import torch

from atomo_b200.ops import plan2 as P2

from shadow_harness import H2, deterministic_cudnn, differs, engine_batch, ext, make_engine, model_shapes, nccl_init, \
    spawn, state, step  # noqa: F401

LR, WD = 2e-3, 0.05
CODES = {
    "svd": dict(code="svd", svd_rank=3), "sgd": dict(code="sgd"), "qsgd": dict(code="qsgd"),
    "entrywise": dict(code="entrywise", entry_budget=0.05),
    "topk": dict(code="topk", entry_budget=0.05, error_feedback=True), "sign": dict(code="sign"),
    "powersgd": dict(code="powersgd", svd_rank=2), "fp8": dict(code="fp8"),
    "hadamard": dict(code="hadamard", quantization_level=4, bucket_size=256),
}

DATA_SEED = 700
_state = functools.partial(state, keys=("master", "vparams", "mom", "vmom", "sq", "vsq", "sqmax", "vsqmax", "wshadow"))


def _engine(graph=False, overlap=None, optimizer="adamw", lr=LR, weight_decay=WD, **kw):
    kw = dict(CODES["svd"], **kw) if "code" not in kw else kw
    return make_engine(use_graph=graph, overlap=graph if overlap is None else overlap, optimizer=optimizer, lr=lr,
                       weight_decay=weight_decay, prepare_n=32 * kw.get("accumulate_steps", 1), data_seed=DATA_SEED,
                       **kw)


def _step(eng):
    return step(eng, engine_batch("ResNet18", eng.step, 32 * eng.accum, DATA_SEED))


def _range_mask(pl, t0, nt, device="cuda"):
    """The weight elements (master indexing) of the PS tiles [t0, t0 + nt), from each unit's tile rule; vector tiles
    contribute nothing."""
    mw = torch.zeros(pl.w_total, dtype=torch.bool, device=device)
    for (ui, a, b, _o) in pl.ps_tiles[t0:t0 + nt]:
        u = pl.units[ui]
        if u.kind == P2.KIND_VEC:
            continue
        if u.kind in (P2.KIND_DENSE16, P2.KIND_QSGD, P2.KIND_ENTRY, P2.KIND_SIGN, P2.KIND_FP8, P2.KIND_HADAMARD):
            mw[u.w_off + a:u.w_off + a + b] = True                    # (first element, count)
        elif u.kind == P2.KIND_POWER:
            mw[u.w_off + a * u.cols:u.w_off + (a + b) * u.cols] = True  # (first row, rows)
        elif u.kind == P2.KIND_SLAB:
            half = u.I // 2
            e0 = u.w_off + (a // half) * u.K * u.I
            mw[e0:e0 + (b // half) * u.K * u.I] = True
        else:                                                          # MAT: rows of a strided block
            torch.as_strided(mw, (b, u.cols), (u.rs, u.cs), u.w_off + a * u.rs).fill_(True)
    return mw


# ---------------------------------------------------------------------------------------------------- kernel
KERNEL_CODES = {"svd": dict(rank=3), "sgd": {}, "qsgd": dict(quantization_level=4, bucket_size=512),
                "entrywise": dict(entry_budget=0.05), "sign": dict(bucket_size=512), "powersgd": dict(rank=2),
                "hadamard": dict(quantization_level=4, bucket_size=256)}


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [0, 1], ids=["aligned", "misaligned"])
@pytest.mark.parametrize("owners", [1, 2])
@pytest.mark.parametrize("code", list(KERNEL_CODES))
@pytest.mark.parametrize("net", ["ResNet18", "VGG11", "LeNet"])
def test_decay_kernel_scales_exactly_the_weight_tiles(net, code, owners, shift):
    C = ext()
    shapes = model_shapes(net, "MNIST" if net == "LeNet" else "")
    pl = P2.build_plan2(shapes, code, n_owners=owners, n_groups=3, **KERNEL_CODES[code])
    f = float(np.float32(1.0 - 0.37 * 0.05))
    dev = torch.device("cuda", 0)
    u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)
    t_units, t_ps = u8(pl.units_bytes()), u8(P2.Plan2.tiles_bytes(pl.ps_tiles))
    ctrl = u8(P2.pack_ctrl2(lr=0.37, opt=P2.OPT_ADAM, decay_factor=f))
    g = torch.Generator(device="cuda").manual_seed(11)
    buf = torch.randn(pl.w_total + 1, device=dev, generator=g)       # shift 1: every float4 path is misaligned
    master = buf[shift:shift + pl.w_total]
    b0 = buf.clone()
    ft = torch.tensor(f, dtype=torch.float32, device=dev)
    seen = torch.zeros(pl.w_total, dtype=torch.int32, device=dev)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for gi in range(pl.n_groups):
        for o in range(owners):
            t0, nt = pl.ps_range[gi][o]
            before = master.clone()
            C.v2_decay(t_units.data_ptr(), t_ps.data_ptr(), t0, nt, master.data_ptr(), ctrl.data_ptr(),
                       [1, 7, 3 * sms][(gi + o) % 3])
            torch.cuda.synchronize()
            mask = _range_mask(pl, t0, nt)
            want = torch.where(mask, before * ft, before)
            assert torch.equal(master, want), (gi, o)
            seen += mask.int()
    # every weight element the plan holds was decayed once (no vector tile wrote into master); the word outside stays
    used = torch.zeros(pl.w_total, dtype=torch.bool, device=dev)
    for q in pl.params:
        if q.is_w:
            used[q.off:q.off + q.numel] = True
    assert torch.equal(seen.bool(), used) and int(seen.max()) == 1
    out = slice(pl.w_total, None) if shift == 0 else slice(0, 1)       # the word of buf outside master
    assert torch.equal(buf[out], b0[out])


@pytest.mark.gpu
def test_decay_binding_checks_its_arguments():
    C = ext()
    with pytest.raises(RuntimeError, match="v2_decay: bad tile range"):
        C.v2_decay(1, 1, 0, -1, 1, 1, 1)
    with pytest.raises(RuntimeError, match="v2_decay: units / tiles / master / ctrl required"):
        C.v2_decay(1, 1, 0, 3, 1, 0, 1)
    C.v2_decay(0, 0, 0, 0, 0, 0, 1)        # an empty range launches nothing


# ---------------------------------------------------------------------------------------------------- composition
def _torch_decay(eng):
    """Swap the engine's decay launch for torch: master.mul_(f) over the group's tiles, in the same stream order."""
    pl = eng.plan
    masks = [_range_mask(pl, *pl.ps_range[g][eng.owner_index]) for g in range(eng.G)]

    def decay(g):
        if not eng.decay_on:
            return
        f = torch.tensor(eng.decay_factor(eng.lr), dtype=torch.float32, device=eng.device)
        eng.master.copy_(torch.where(masks[g], eng.master * f, eng.master))
    eng._launch_decay = decay


@pytest.mark.gpu
@pytest.mark.parametrize("code,amsgrad", [(c, False) for c in CODES] + [(c, True) for c in ("svd", "sgd", "qsgd", "topk")])
def test_step_is_torch_decay_then_the_ps_launch(code, amsgrad, deterministic_cudnn):
    runs = []
    for swap in (False, True):
        eng = _engine(overlap=False, amsgrad=amsgrad, **CODES[code])
        if swap:
            _torch_decay(eng)
        for s in range(3):
            _step(eng)
        runs.append(_state(eng))
        eng.close()
    assert differs(runs[0], runs[1]) == []


@pytest.mark.gpu
@pytest.mark.parametrize("opt", [P2.OPT_ADAM, P2.OPT_AMSGRAD], ids=["adam", "amsgrad"])
@pytest.mark.parametrize("code", ["svd", "sgd"])
def test_loopback_two_workers_two_groups(code, opt):
    """Two identical loopback harnesses, 2 virtual workers and 2 groups: one decays with v2_decay, the other with torch,
    then both run the same PS launches with Adam and weight decay 0."""
    shapes = model_shapes("ResNet18")
    f = float(np.float32(1.0 - 0.01 * 0.1))
    hs = [H2(shapes, code, rank=3, W=2, lr=0.01, wd=0.0, opt=opt, seed=5, groups=2) for _ in range(2)]
    for h in hs:
        h.ctrl.view(torch.float32)[17] = f
    for step in (1, 2, 3):
        for k, h in enumerate(hs):
            h.set_step(step)
            for w in range(2):
                h.fill(w, seed=100 * step + w)
                h.encode(w)
            pl = h.plan
            for g in range(pl.n_groups):
                t0, nt = pl.ps_range[g][0]
                if k == 0:
                    h.C.v2_decay(h.t_units.data_ptr(), h.t_ps.data_ptr(), t0, nt, h.master.data_ptr(),
                                 h.ctrl.data_ptr(), 64)
                else:
                    m = _range_mask(pl, t0, nt)
                    h.master.copy_(torch.where(m, h.master * torch.tensor(f, device="cuda"), h.master))
            h.ps()
            assert int(h.ctrl.view(torch.int32)[1]) == 0
        a, b = hs
        for name in ("master", "vparams", "mom", "sq", "sqmax", "vmom", "vsq", "wshadow"):
            assert torch.equal(getattr(a, name), getattr(b, name)), (step, name)


# ---------------------------------------------------------------------------------------------------- engine
@pytest.mark.gpu
@pytest.mark.parametrize("amsgrad", [False, True], ids=["adam", "amsgrad"])
def test_zero_decay_is_adam(amsgrad, deterministic_cudnn):
    runs = []
    for opt in ("adam", "adamw"):
        eng = _engine(graph=True, optimizer=opt, weight_decay=0.0, amsgrad=amsgrad)
        assert not eng.decay_on
        losses = [_step(eng) for _ in range(5)]
        runs.append((losses, _state(eng), eng.launches_per_step))
        eng.close()
    assert runs[0][0] == runs[1][0] and differs(runs[0][1], runs[1][1]) == [] and runs[0][2] == runs[1][2]


@pytest.mark.gpu
def test_one_dense_step_matches_the_fp64_rule():
    """One step of the dense code (W = 1: the owner decodes the bf16 gradient exactly) against optim/adamw.py in fp64,
    on the engine's fp32 hyperparameters (lr, betas, eps as Ctrl2 holds them).

    Bound per element, in units of u = 2^-24, with p the initial weight, p' the result and d the update:
    * the decay: f = fp32(1 - lr wd) and the product p f round once each, 2 u |p|;
    * the update: the roundings of m, v and the fast-math sqrt, two approximate divisions of at most 2 ulp each, the
      add of eps and two multiplies, 16 u |d| with slack; and the bias corrections, which the kernel forms with the
      fast-math powf (ex2.approx of t lg2.approx(b), absolute error within 2^-21 for b^t <= 1), so bc1 = 1 - b1^t and
      sqrt(1 - b2^t) are off by at most 2^-21 / bc1 and 2^-21 / (2 (1 - b2^t)) relative;
    * the final subtraction rounds once, u |p'|.
    With lr wd = 0.01 the decay moves a weight by |p| / 100, far outside the bound: a missing decay fails."""
    from atomo_b200.optim import AdamW
    f32 = lambda x: float(np.float32(x))
    lr, wd, b1, b2, eps = f32(1e-2), 1.0, f32(0.9), f32(0.999), f32(1e-8)
    eng = _engine(code="sgd", lr=lr, weight_decay=wd)
    pl = eng.plan
    w0, v0 = eng.master.double().clone(), eng.vparams.double().clone()
    _step(eng)
    gw = torch.zeros_like(w0)
    for p, q in zip(eng.params, pl.params):
        if q.is_w:
            t = p.grad.double()
            gw[q.off:q.off + q.numel] = t.permute(0, 2, 3, 1).reshape(-1) if t.dim() == 4 else t.reshape(-1)
    gv = eng.vgrads.double().clone()
    got_w, got_v = eng.master.double(), eng.vparams.double()
    eng.close()

    def oracle(decay):
        ps, gs = [], []
        for q in pl.params:
            src, g = (w0, gw) if q.is_w else (v0, gv)
            shape = (q.numel, 1) if q.is_w else (q.numel,)       # dims decide the group, not the layout
            ps.append(src[q.off:q.off + q.numel].clone().view(shape))
            gs.append(g[q.off:q.off + q.numel].view(shape))
        AdamW(ps, lr=lr, betas=(b1, b2), eps=eps, weight_decay=decay).step(grads=gs)
        rw, rv = w0.clone(), v0.clone()
        for q, p in zip(pl.params, ps):
            (rw if q.is_w else rv)[q.off:q.off + q.numel] = p.reshape(-1)
        return rw, rv

    u = 2.0 ** -24
    e_bc = 2.0 ** -21 * (1 / (1 - b1) + 1 / (2 * (1 - b2)))
    ref_w, ref_v = oracle(wd)
    for got, ref, start, fac in ((got_w, ref_w, w0, 1 - lr * wd), (got_v, ref_v, v0, 1.0)):
        d = (start * fac - ref).abs()
        bound = u * (2 * start.abs() + ref.abs()) + d * (16 * u + e_bc) + 1e-30
        assert bool(((got - ref).abs() <= bound).all()), float(((got - ref).abs() / bound).max())
    plain_w, _ = oracle(0.0)
    d = (w0 - plain_w).abs()
    miss = (got_w - plain_w).abs() > u * (2 * w0.abs() + plain_w.abs()) + d * (16 * u + e_bc)
    assert float(miss.double().mean()) > 0.9       # without the decay the same bound fails almost everywhere


@pytest.mark.gpu
@pytest.mark.parametrize("code", ["svd", "sgd"])
def test_eager_equals_graph_and_reruns(code, deterministic_cudnn):
    runs = []
    for graph in (False, True, False, True):
        eng = _engine(graph=graph, overlap=True, **CODES[code])
        for _ in range(4):
            _step(eng)
        runs.append(_state(eng))
        eng.close()
    assert all(differs(runs[0], r) == [] for r in runs[1:])


@pytest.mark.gpu
def test_set_lr_between_replays_changes_the_decay(deterministic_cudnn):
    runs = []
    for graph, change in ((False, True), (True, True), (True, False)):
        eng = _engine(graph=graph, overlap=True, code="sgd", weight_decay=0.5)
        f0 = float(eng.ctrl_f32[17])
        for s in range(4):
            if s == 2 and change:
                eng.set_lr(5 * LR)
                assert float(eng.ctrl_f32[17]) == np.float32(1 - 5 * LR * 0.5) != f0
            _step(eng)
        runs.append(_state(eng))
        eng.close()
    assert differs(runs[0], runs[1]) == []
    assert "master" in differs(runs[1], runs[2])


@pytest.mark.gpu
@pytest.mark.parametrize("code", ["svd", "sgd"])
def test_clip_above_the_norm_is_unclipped_adamw(code, deterministic_cudnn):
    runs = []
    for clip in (0.0, 1e6):
        eng = _engine(graph=True, clip_grad_norm=clip, **CODES[code])
        for _ in range(4):
            _step(eng)
        if clip:
            total, coef = eng.grad_norm()
            assert 0 < total < clip and coef == 1.0
        runs.append(_state(eng))
        eng.close()
    assert differs(runs[0], runs[1]) == []


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_accumulate_steps_two(graph, deterministic_cudnn):
    runs = {}
    for opt, wd in (("adam", 0.0), ("adamw", WD), ("adamw-torch", WD)):
        eng = _engine(graph=graph and opt != "adamw-torch", overlap=graph and opt != "adamw-torch",
                      optimizer=opt[:5], weight_decay=wd, accumulate_steps=2)
        if opt == "adamw-torch":
            _torch_decay(eng)
        losses = [_step(eng) for _ in range(3)]
        assert all(np.isfinite(losses))
        runs[opt] = (_state(eng), eng.launches_per_step, sum(1 for g in range(eng.G)
                                                              if eng.plan.ps_range[g][eng.owner_index][1] > 0))
        eng.close()
    assert runs["adamw"][1] == runs["adam"][1] + runs["adamw"][2]
    assert "master" in differs(runs["adam"][0], runs["adamw"][0])
    if not graph:
        assert differs(runs["adamw"][0], runs["adamw-torch"][0]) == []


@pytest.mark.gpu
@pytest.mark.parametrize("clip", [0.0, 1.0], ids=["plain", "clip"])
def test_weight_average_follows_the_decayed_weights(clip):
    eng = _engine(graph=True, ema_decay=0.9, clip_grad_norm=clip)
    w = np.float32(eng.ema_w)
    e, ve = eng.master.cpu().numpy().copy(), eng.vparams.cpu().numpy().copy()
    for _ in range(5):
        _step(eng)
        e = e + w * (eng.master.cpu().numpy() - e)
        ve = ve + w * (eng.vparams.cpu().numpy() - ve)
        assert torch.equal(eng.ema.cpu(), torch.from_numpy(e)) and torch.equal(eng.vema.cpu(), torch.from_numpy(ve))
    eng.close()


@pytest.mark.gpu
def test_launches_per_group_and_with_clipping():
    n = {}
    for opt, wd, clip in (("adam", WD, 0.0), ("adamw", WD, 0.0), ("adam", WD, 1.0), ("adamw", WD, 1.0)):
        eng = _engine(graph=True, optimizer=opt, weight_decay=wd, clip_grad_norm=clip)
        _step(eng)
        n[(opt, clip)] = (eng.launches_per_step, sum(1 for g in range(eng.G)
                                                     if eng.plan.ps_range[g][eng.owner_index][1] > 0))
        eng.close()
    for clip in (0.0, 1.0):
        assert n[("adamw", clip)][0] == n[("adam", clip)][0] + n[("adamw", clip)][1] > n[("adam", clip)][0]


@pytest.mark.gpu
@pytest.mark.parametrize("amsgrad", [False, True], ids=["adamw", "amsgrad"])
def test_resume_is_bitwise(amsgrad, tmp_path, deterministic_cudnn):
    d = str(tmp_path) + "/"
    eng = _engine(graph=True, amsgrad=amsgrad)
    for _ in range(6):
        _step(eng)
        if eng.step - 1 == 3:
            eng.save_checkpoint(d)
    want = _state(eng)
    eng.close()
    side = torch.load(d + "model_step_3_optim", map_location="cpu", weights_only=False)
    assert side["optimizer"] == "adamw" and "sq_w" in side and ("sqmax_w" in side) == amsgrad
    eng = _engine(graph=True, amsgrad=amsgrad)
    eng.load_checkpoint(d, 3)
    for _ in range(3):
        _step(eng)
    assert differs(want, _state(eng)) == []
    eng.close()


@pytest.mark.gpu
def test_adam_and_adamw_checkpoints_load_into_each_other(tmp_path):
    for saver, loader in (("adam", "adamw"), ("adamw", "adam")):
        d = str(tmp_path / saver) + "/"
        eng = _engine(optimizer=saver)
        for _ in range(2):
            _step(eng)
        eng.save_checkpoint(d)
        want = _state(eng)
        eng.close()
        eng = _engine(optimizer=loader)
        eng.load_checkpoint(d, 2)
        got = _state(eng)
        assert differs({k: want[k] for k in ("master", "mom", "sq", "vsq")},
                       {k: got[k] for k in ("master", "mom", "sq", "vsq")}) == []
        _step(eng)
        eng.close()


@pytest.mark.gpu
def test_launcher_trains_checkpoints_and_resumes(tmp_path, monkeypatch, capsys):
    import argparse
    from atomo_b200.runtime import p2p_launcher as L
    from atomo_b200.utils.flags import add_fit_args
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    d = str(tmp_path) + "/"
    argv = ["--network", "ResNet18", "--dataset", "Cifar10", "--synthetic", "1", "--train-len", "1024", "--test-len",
            "256", "--batch-size", "64", "--test-batch-size", "128", "--engine", "shadow", "--dtype", "bf16", "--code",
            "svd", "--svd-rank", "3", "--lr", "0.002", "--optimizer", "adamw", "--weight-decay", "0.05",
            "--eval-freq", "4", "--log-interval", "4", "--train-dir", d]
    L.run_p2p_training(add_fit_args(argparse.ArgumentParser(), argv + ["--max-steps", "4"]))
    L.run_p2p_training(add_fit_args(argparse.ArgumentParser(), argv + ["--max-steps", "8", "--resume", "1"]))
    out = capsys.readouterr().out
    for s in (4, 8):
        assert "Test set: Step: %d," % s in out, out
        side = torch.load(d + "model_step_%d_optim" % s, map_location="cpu", weights_only=False)
        assert side["optimizer"] == "adamw" and side["step"] == s
    assert "device error" not in out


# ---------------------------------------------------------------------------------------------------- two GPUs
def _mp(rank, world, port, out):
    import torch.distributed as dist
    nccl_init(rank, world, port)
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    eng = ShadowEngine(build_model("ResNet18", 10), rank, world, use_graph=True, seed=7, ps_mode="sharded",
                       optimizer="adamw", lr=LR, weight_decay=WD, **CODES["svd"])
    x, y = engine_batch("ResNet18", rank, seed=DATA_SEED)
    eng.prepare(x, y, warmup=0)
    for s in range(4):
        x, y = engine_batch("ResNet18", 1 + s + rank, seed=DATA_SEED)
        eng.train_step(x, y)
    torch.cuda.synchronize()
    dist.barrier()
    torch.cuda.synchronize()
    out.put((rank, eng.error_code(), eng.wshadow.cpu(), eng.vparams.cpu(), eng.gather_fp32("master").cpu()))
    eng.close()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_owners_keep_identical_replicas():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    res = spawn(2, _mp, 29730)
    assert all(r[1] == 0 for r in res)
    a, b = res
    assert torch.equal(a[2], b[2]) and torch.equal(a[3], b[3]) and torch.equal(a[4], b[4])

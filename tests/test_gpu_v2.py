"""v2 (overlapped / sharded bf16) kernels and engine vs plain PyTorch fp32 references."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [(64, 32, 3, 3), (32, 64, 3, 3), (48, 16, 5, 5), (10, 512), (128, 64, 1, 1), (64,), (512, 256, 1, 1),
          (64, 3, 3, 3), (300, 200), (10,)]


def _ext():
    from atomo_b200.ops._ext import load
    return load()


class H2:
    """Loopback harness: one rank that is worker 0..W-1 (virtual) and the only owner."""

    def __init__(self, shapes, code="svd", rank=3, W=1, lr=0.1, momentum=0.0, wd=0.0, nesterov=False, opt=0, seed=7,
                 systematic=False, groups=1, warm=False, max_sweeps=0):
        from atomo_b200.ops import plan2 as P
        self.C, self.P = _ext(), P
        dev = self.dev = torch.device("cuda", 0)
        self.W = W
        self.plan = pl = P.build_plan2(shapes, code, rank, systematic, n_owners=1, n_groups=groups)
        u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)
        self.t_units = u8(pl.units_bytes())
        self.t_enc = u8(P.Plan2.tiles_bytes(pl.enc_tiles))
        self.t_ps = u8(P.Plan2.tiles_bytes(pl.ps_tiles))
        nc = max(pl.n_coded, 1)
        z = lambda n, dt=torch.float32: torch.zeros(n, dtype=dt, device=dev)
        self.gpart, self.vsel, self.sigma = z(pl.gpart_floats), z(nc * 64 * 32), z(nc * 64)
        self.selcount = z(nc, torch.int32)
        self.counters = z(nc + 32, torch.int32)
        self.arena = z(pl.arena_floats * W)
        self.signals = z(1024, torch.int32)
        self.signals[256] = 1
        self.ctrl = u8(P.pack_ctrl2(step=1, lr=lr, momentum=momentum, weight_decay=wd, nesterov=nesterov, seed=seed, opt=opt))
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.master = torch.randn(pl.w_total, device=dev, generator=g)
        self.wshadow = self.master.to(torch.bfloat16)
        self.vparams = torch.randn(pl.v_total, device=dev, generator=g)
        self.mom, self.vmom = z(pl.w_total), z(pl.v_total)
        self.sq, self.vsq, self.sqmax, self.vsqmax = z(pl.w_total), z(pl.v_total), z(pl.w_total), z(pl.v_total)
        self.stage = [z(pl.stage_total, torch.bfloat16) for _ in range(W)]
        self.vgrads = [z(pl.v_total) for _ in range(W)]
        self.wgrads = []          # per worker: list of bf16 grad tensors (physical layout), one per W param
        i64 = lambda xs: torch.tensor(list(xs), dtype=torch.int64, device=dev)
        self.t_arena_peer = i64([self.arena.data_ptr()])
        self.t_sig_peer = i64([self.signals.data_ptr()])
        self.t_wshadow_peer = i64([self.wshadow.data_ptr()])
        self.t_vparams_peer = i64([self.vparams.data_ptr()])
        self.t_vgrads_peer = i64([t.data_ptr() for t in self.vgrads])
        self.t_stage_peer = i64([t.data_ptr() for t in self.stage])
        self.tstats = z(32, torch.int64)
        self.max_sweeps = max_sweeps
        self.vprev = None
        if warm:
            self.vprev = z(nc * 64 * 64)
            for u in pl.units:
                if u.coded:
                    self.vprev[u.ts_index * 4096:u.ts_index * 4096 + u.cols * u.cols] = torch.eye(u.cols, device=dev).reshape(-1)

    def fill(self, w, seed, lowrank=True):
        """Random gradients for virtual worker w; returns {param index: fp32 tensor in the logical layout}."""
        pl, dev = self.plan, self.dev
        g = torch.Generator(device="cuda").manual_seed(seed)
        grads, logical = [], {}
        for q in pl.params:
            if q.is_w:
                x = torch.randn(q.shape, device=dev, generator=g)
                if lowrank and len(q.shape) >= 2:
                    m = x.reshape(q.shape[0], -1)
                    k = min(m.shape)
                    a = torch.randn(m.shape[0], k, device=dev, generator=g) * torch.logspace(0, -1.5, k, device=dev)
                    x = (a @ torch.linalg.qr(torch.randn(m.shape[1], k, device=dev, generator=g)).Q.T).reshape(q.shape)
                xb = x.to(torch.bfloat16)
                phys = xb.contiguous(memory_format=torch.channels_last) if xb.dim() == 4 else xb.contiguous()
                grads.append(phys)
                logical[q.index] = phys.float()
            else:
                v = torch.randn(q.numel, device=dev, generator=g)
                self.vgrads[w][q.off:q.off + q.numel] = v
                logical[q.index] = v
        while len(self.wgrads) <= w:
            self.wgrads.append(None)
        self.wgrads[w] = grads
        return logical

    def encode(self, w, random_sample=True, waterfill=False, systematic=False, uniforms=None, resample_empty=False):
        C, pl = self.C, self.plan
        gptr = torch.tensor([t.data_ptr() for t in self.wgrads[w]] or [0], dtype=torch.int64, device=self.dev)
        self._gptr = gptr
        for g in range(pl.n_groups):
            t0, nt = pl.enc_range[g]
            C.v2_encode(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr.data_ptr(), self.gpart.data_ptr(),
                        self.counters.data_ptr(), self.vsel.data_ptr(), self.selcount.data_ptr(), self.sigma.data_ptr(),
                        self.t_arena_peer.data_ptr(), 1, pl.arena_floats, self.stage[w].data_ptr(), self.ctrl.data_ptr(),
                        uniforms.data_ptr() if uniforms is not None else 0,
                        self.vprev.data_ptr() if self.vprev is not None else 0, self.max_sweeps, random_sample,
                        waterfill, systematic, w, resample_empty, 0, 0, g)
            C.v2_project(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr.data_ptr(), self.vsel.data_ptr(),
                         self.selcount.data_ptr(), self.t_arena_peer.data_ptr(), self.t_sig_peer.data_ptr(), 1,
                         pl.arena_floats, w, g, self.ctrl.data_ptr(), self.counters.data_ptr() + 4 * (pl.n_coded + g), 0, 0,
                         False, False)
        torch.cuda.synchronize()

    def ps(self, grid=64):
        C, pl = self.C, self.plan
        for g in range(pl.n_groups):
            t0, nt = pl.ps_range[g][0]
            C.v2_ps(self.t_units.data_ptr(), self.t_ps.data_ptr(), t0, nt, self.W, 1, g, g == pl.n_groups - 1, 0,
                    self.master.data_ptr(), self.mom.data_ptr(), self.sq.data_ptr(), self.sqmax.data_ptr(),
                    self.vmom.data_ptr(), self.vsq.data_ptr(), self.vsqmax.data_ptr(), 0, self.t_wshadow_peer.data_ptr(),
                    self.vparams.data_ptr(), 0, self.t_vparams_peer.data_ptr(), 0, self.t_vgrads_peer.data_ptr(),
                    self.t_stage_peer.data_ptr(), self.arena.data_ptr(), pl.arena_floats, self.signals.data_ptr(),
                    self.t_sig_peer.data_ptr(), self.ctrl.data_ptr(),
                    self.counters.data_ptr() + 4 * (pl.n_coded + 8 + g), int(5e9), self.tstats.data_ptr(), 1.0 / self.W,
                    grid)
        torch.cuda.synchronize()

    # ---- references ---------------------------------------------------------------------------------------
    def unit_matrix(self, u, logical):
        """fp32 tall matrix of a coded unit, in the kernel's row/column convention."""
        q = self.plan.params[u.param]
        t = logical[q.index]
        if u.kind == self.P.KIND_SLAB:
            o, i, kh, kw = q.shape
            return t.contiguous().reshape(o * i // 2, 2 * kh * kw)       # the reference's matricization
        m = t.reshape(q.shape[0], -1)
        tall = m if m.shape[0] >= m.shape[1] else m.t()
        c0 = u.g_off // u.cs if u.cs > 1 else u.g_off
        return tall[:, c0:c0 + u.cols]

    def slot(self, u, w):
        base = self.arena[w * self.plan.arena_floats + u.slot_off:]
        hdr = base[:4].view(torch.int32)
        count = int(hdr[0])
        s = base[4:4 + u.rcap][:count]
        V = base[4 + u.rcap:4 + u.rcap + u.rcap * u.cols].view(u.rcap, u.cols)[:count]
        uo = self.P.slot_u_off(u.rcap, u.cols)
        if u.ubits == 8:      # QSVD: int8 U with one fp32 scale per row
            q = base[uo:uo + u.rows * u.rcap // 4].view(torch.int8).view(u.rows, u.rcap)[:, :count].float()
            so = self.P.slot_scale_off(u.rows, u.cols, u.rcap)
            U = q * (base[so:so + u.rows] / 127.0).unsqueeze(1)
        else:
            U = base[uo:uo + u.rows * u.rcap].view(u.rows, u.rcap)[:, :count]
        return count, s, V, U, int(hdr[1])

    def write_unit(self, u, flat, mat):
        """Scatter a tall unit matrix into a flat fp32 array indexed like wshadow (physical order)."""
        q = self.plan.params[u.param]
        if u.kind == self.P.KIND_SLAB:
            o, i, kh, kw = q.shape
            logical = mat.reshape(o, i, kh, kw)
            flat[q.off:q.off + q.numel] = logical.permute(0, 2, 3, 1).reshape(-1)
        else:
            torch.as_strided(flat, (u.rows, u.cols), (u.rs, u.cs), u.w_off).copy_(mat)


def test_v2_gram_matches_torch():
    h = H2(SHAPES)
    logical = h.fill(0, 1)
    h.encode(0)
    pl = h.plan
    n = 0
    for u in pl.units:
        if not u.coded:
            continue
        A = h.unit_matrix(u, logical).double()
        G = h.gpart[u.gpart_off:u.gpart_off + u.n_enc * u.cols * u.cols].view(u.n_enc, u.cols, u.cols).sum(0)
        ref = (A.T @ A).float()
        assert torch.allclose(G, ref, rtol=2e-4, atol=2e-4 * float(ref.abs().max())), (u.kind, u.rows, u.cols)
        n += 1
    assert n >= 8


@pytest.mark.parametrize("rank", [64, 3])
def test_v2_topk_factors_reconstruct_the_gradient(rank):
    """random_sample=False keeps the top-`rank` atoms: with rank >= cols the factors must reproduce the bf16
    gradient exactly (validates Jacobi, the (b,k) column convention, the projection and the slot layout);
    with rank 3 they must match the best rank-3 approximation."""
    h = H2(SHAPES, rank=rank)
    logical = h.fill(0, 2)
    h.encode(0, random_sample=False)
    for u in h.plan.units:
        if not u.coded:
            continue
        A = h.unit_matrix(u, logical)
        count, s, V, U, step = h.slot(u, 0)
        assert step == 1
        rec = (U * s) @ V
        if rank >= u.cols:
            assert count == min(int(u.budget), u.cols, u.rcap)
            if count == u.cols:
                assert torch.allclose(rec, A, rtol=1e-3, atol=2e-4 * float(A.abs().max())), (u.kind, u.rows, u.cols)
        else:
            sv = torch.linalg.svdvals(A.double()).float()
            k = int(min(u.budget, u.cols))
            best = float(sv[k:].norm())
            assert float((A - rec).norm()) <= 1.02 * best + 1e-3 * float(A.norm()), (u.kind, u.rows, u.cols)
    if rank >= 64:
        return
    # warm start: second encode of a slightly perturbed gradient with a 2-sweep cap must still find the subspace
    hw = H2(SHAPES, rank=rank, warm=True, max_sweeps=2)
    logical = hw.fill(0, 2)
    hw.encode(0, random_sample=False)
    hw.ctrl.view(torch.int32)[0] = 2
    hw.encode(0, random_sample=False)
    for u in hw.plan.units:
        if u.coded:
            A = hw.unit_matrix(u, logical)
            count, s, V, U, step = hw.slot(u, 0)
            assert step == 2
            sv = torch.linalg.svdvals(A.double()).float()
            k = int(min(u.budget, u.cols))
            assert float((A - (U * s) @ V).norm()) <= 1.1 * float(sv[k:].norm()) + 2e-3 * float(A.norm()), (u.kind, u.cols)
            Vfull = hw.vprev[u.ts_index * 4096:u.ts_index * 4096 + u.cols * u.cols].view(u.cols, u.cols)
            eye = torch.eye(u.cols, device=hw.dev)
            assert float((Vfull.T @ Vfull - eye).abs().max()) < 1e-4
    # dense bf16 weights were staged verbatim
    for u in h.plan.units:
        if u.kind == h.P.KIND_DENSE16:
            q = h.plan.params[u.param]
            phys = h.wgrads[0][q.widx].permute(0, 2, 3, 1).reshape(-1) if len(q.shape) == 4 else h.wgrads[0][q.widx].reshape(-1)
            assert torch.equal(h.stage[0][u.rs:u.rs + u.numel], phys)


@pytest.mark.parametrize("warm,max_sweeps", [(False, 0), (True, 2)])
def test_v2_sampled_atoms_are_unbiased(warm, max_sweeps):
    """Also with the production setting (warm-started Jacobi capped at 2 sweeps): eigenvectors are then only
    approximate, but the basis is complete and orthonormal, so the estimator must stay unbiased."""
    shapes = [(32, 16, 3, 3), (64, 48)]
    h = H2(shapes, rank=3, warm=warm, max_sweeps=max_sweeps)
    logical = h.fill(0, 3)
    acc = {u.index: 0 for u in h.plan.units if u.coded}
    cnt = {u.index: 0.0 for u in h.plan.units if u.coded}
    T = 600
    early = {}
    for t in range(T):
        h.ctrl.view(torch.int32)[0] = t + 1
        h.encode(0)
        for u in h.plan.units:
            if u.coded:
                c, s, V, U, _ = h.slot(u, 0)
                acc[u.index] = acc[u.index] + (U * s) @ V
                cnt[u.index] += c
                if t + 1 == T // 6:
                    A = h.unit_matrix(u, logical)
                    early[u.index] = float((acc[u.index] / (t + 1) - A).norm() / A.norm())
    for u in h.plan.units:
        if u.coded:
            A = h.unit_matrix(u, logical)
            err = float((acc[u.index] / T - A).norm() / A.norm())
            # an unbiased estimator's error shrinks like 1/sqrt(T) (x0.41 for 6x the draws); a biased one plateaus
            assert err < 0.25 and err < 0.62 * early[u.index], (u.kind, err, early[u.index])
            assert cnt[u.index] / T <= u.budget + 0.3


@pytest.mark.parametrize("W,momentum,nesterov,wd,opt", [(1, 0.0, False, 0.0, 0), (3, 0.9, True, 1e-3, 0),
                                                         (8, 0.9, False, 0.0, 0), (2, 0.0, False, 0.0, 1),
                                                         (2, 0.0, False, 1e-3, 2)])
def test_v2_ps_matches_reference(W, momentum, nesterov, wd, opt):
    """W virtual workers push; the PS result must equal optimizer(mean of the per-worker decodes / dense grads)
    on the fp32 master, and the bf16 working copy must be its rounding."""
    lr = 0.05
    h = H2(SHAPES, rank=3, W=W, lr=lr, momentum=momentum, wd=wd, nesterov=nesterov, opt=opt)
    pl = h.plan
    for step in (1, 2):
        h.ctrl.view(torch.int32)[0] = step
        est_w = torch.zeros(pl.w_total, device=h.dev)
        est_v = torch.zeros(pl.v_total, device=h.dev)
        for w in range(W):
            logical = h.fill(w, 10 * step + w)
            h.encode(w)
            tmp = torch.zeros(pl.w_total, device=h.dev)
            for u in pl.units:
                q = pl.params[u.param]
                if u.coded:
                    c, s, V, U, st = h.slot(u, w)
                    assert st == step
                    if u.kind == h.P.KIND_SLAB:
                        h.write_unit(u, tmp, (U * s) @ V)
                    else:
                        torch.as_strided(tmp, (u.rows, u.cols), (u.rs, u.cs), u.w_off).copy_((U * s) @ V)
                elif u.kind == h.P.KIND_DENSE16:
                    t = logical[q.index]
                    tmp[u.w_off:u.w_off + u.numel] = t.permute(0, 2, 3, 1).reshape(-1) if t.dim() == 4 else t.reshape(-1)
            est_w += tmp
            est_v += h.vgrads[w]
        assert all(int(h.signals[w]) == step for w in range(W))
        gw, gv = est_w / W, est_v / W
        p0, m0, q0, qm0 = h.master.clone(), h.mom.clone(), h.sq.clone(), h.sqmax.clone()
        v0, vm0, vq0, vqm0 = h.vparams.clone(), h.vmom.clone(), h.vsq.clone(), h.vsqmax.clone()

        def ref(p, g, m, s2, s2m):
            g = g + wd * p
            if opt == 0:
                if momentum:
                    m = g.clone() if step == 1 else momentum * m + g
                    d = g + momentum * m if nesterov else m
                else:
                    d = g
                return p - lr * d, m
            b1, b2, eps = 0.9, 0.999, 1e-8
            m = b1 * m + (1 - b1) * g
            s2 = b2 * s2 + (1 - b2) * g * g
            vv = torch.maximum(s2m, s2) if opt == 2 else s2
            denom = vv.sqrt() / (1 - b2 ** step) ** 0.5 + eps
            return p - lr / (1 - b1 ** step) * m / denom, m
        rp, rm = ref(p0, gw, m0, q0, qm0)
        rv, rvm = ref(v0, gv, vm0, vq0, vqm0)
        h.ps()
        assert int(h.ctrl.view(torch.int32)[1]) == 0
        assert int(h.signals[256]) == step + 1
        used = torch.zeros(pl.w_total, dtype=torch.bool, device=h.dev)
        for q in pl.params:
            if q.is_w:
                used[q.off:q.off + q.numel] = True
        tol = dict(rtol=3e-4, atol=3e-5) if opt == 0 else dict(rtol=2e-3, atol=2e-4)
        assert torch.allclose(h.master[used], rp[used], **tol), float((h.master - rp)[used].abs().max())
        assert torch.equal(h.wshadow[used], h.master.to(torch.bfloat16)[used])
        vused = torch.zeros(pl.v_total, dtype=torch.bool, device=h.dev)
        for q in pl.params:
            if not q.is_w:
                vused[q.off:q.off + q.numel] = True
        assert torch.allclose(h.vparams[vused], rv[vused], **tol)
        if opt == 0 and momentum:
            assert torch.allclose(h.mom[used], rm[used], rtol=3e-4, atol=3e-5)


def test_v2_qsvd_quantized_factors_are_unbiased_and_applied_by_the_ps():
    """--code qsvd on the GPU path: spectral atoms whose left factors travel as int8 with a per-row scale
    (stochastic rounding).  Same atoms as --code svd for the same seed; |U_q - U| <= scale/127; the mean over many
    rounding draws converges to U; the PS applies exactly the de-quantized factors."""
    shapes = [(64, 32, 3, 3), (128, 64, 1, 1), (64,), (10, 512)]
    lr = 0.1
    hq, hf = H2(shapes, code="qsvd", rank=3, lr=lr), H2(shapes, code="svd", rank=3, lr=lr)
    assert hq.plan.arena_floats < 0.6 * hf.plan.arena_floats
    lq, lf = hq.fill(0, 5), hf.fill(0, 5)
    hq.encode(0); hf.encode(0)
    for uq, uf in zip(hq.plan.units, hf.plan.units):
        if not uq.coded:
            continue
        assert uq.ubits == 8 and uf.ubits == 0
        cq, sq, Vq, Uq, _ = hq.slot(uq, 0)
        cf, sf, Vf, Uf, _ = hf.slot(uf, 0)
        assert cq == cf and torch.allclose(sq, sf, rtol=1e-4) and torch.allclose(Vq, Vf, rtol=1e-3, atol=1e-5)
        if cq:
            step = Uf.abs().amax(dim=1, keepdim=True) / 127.0
            assert bool(((Uq - Uf).abs() <= step * 1.001 + 2e-5).all())
    # unbiased rounding: average the de-quantized U over many draws (the step enters the Philox counter of the
    # rounding only through the same atoms when sampling is deterministic)
    ht = H2(shapes, code="qsvd", rank=3)
    ht.fill(0, 5)
    acc, T = {}, 200
    ref = {}
    hr = H2(shapes, code="svd", rank=3)
    hr.fill(0, 5)
    hr.encode(0, random_sample=False)
    for u in hr.plan.units:
        if u.coded:
            ref[u.index] = hr.slot(u, 0)[3].clone()
    for t in range(T):
        ht.ctrl.view(torch.int32)[0] = t + 1
        ht.encode(0, random_sample=False)
        for u in ht.plan.units:
            if u.coded:
                acc[u.index] = acc.get(u.index, 0) + ht.slot(u, 0)[3]
    for u in ht.plan.units:
        if u.coded:
            err = float((acc[u.index] / T - ref[u.index]).abs().max() / ref[u.index].abs().max())
            assert err < 2.5e-3, (u.kind, err)          # one rounding step is 1/127 = 7.9e-3 of the row maximum
    # PS applies the de-quantized factors
    pl = hq.plan
    est = torch.zeros(pl.w_total, device=hq.dev)
    for u in pl.units:
        q = pl.params[u.param]
        if u.coded:
            c, s_, V, U, _ = hq.slot(u, 0)
            if u.kind == hq.P.KIND_SLAB:
                hq.write_unit(u, est, (U * s_) @ V)
            else:
                torch.as_strided(est, (u.rows, u.cols), (u.rs, u.cs), u.w_off).copy_((U * s_) @ V)
    p0 = hq.master.clone()
    hq.ps()
    assert int(hq.ctrl.view(torch.int32)[1]) == 0
    for q in pl.params:
        if q.is_w and any(u.coded and u.param == q.index for u in pl.units):
            sl = slice(q.off, q.off + q.numel)
            assert torch.allclose(hq.master[sl], (p0 - lr * est)[sl], rtol=3e-4, atol=3e-5)


def test_v2_ps_num_aggregate_uses_only_the_workers_that_pushed():
    """--num-aggregate 2 of 3 workers (backup-worker semantics, the reference's unused flag): worker 1 never
    pushes this step; the PS must proceed with workers {0, 2}, average over 2, and ignore worker 1's stale slot."""
    lr = 0.1
    h = H2(SHAPES, rank=3, W=3, lr=lr)
    h.ctrl.copy_(torch.frombuffer(bytearray(h.P.pack_ctrl2(step=1, lr=lr, seed=7, num_aggregate=2)), dtype=torch.uint8).to(h.dev))
    pl = h.plan
    est_w = torch.zeros(pl.w_total, device=h.dev)
    est_v = torch.zeros(pl.v_total, device=h.dev)
    for w in (0, 2):
        logical = h.fill(w, 40 + w)
        h.encode(w)
        tmp = torch.zeros(pl.w_total, device=h.dev)
        for u in pl.units:
            q = pl.params[u.param]
            if u.coded:
                c, s, V, U, st = h.slot(u, w)
                if u.kind == h.P.KIND_SLAB:
                    h.write_unit(u, tmp, (U * s) @ V)
                else:
                    torch.as_strided(tmp, (u.rows, u.cols), (u.rs, u.cs), u.w_off).copy_((U * s) @ V)
            elif u.kind == h.P.KIND_DENSE16:
                t = logical[q.index]
                tmp[u.w_off:u.w_off + u.numel] = t.permute(0, 2, 3, 1).reshape(-1) if t.dim() == 4 else t.reshape(-1)
        est_w += tmp
        est_v += h.vgrads[w]
    h.vgrads[1].fill_(1e6)                      # garbage a skipped worker may hold
    assert int(h.signals[0]) == 1 and int(h.signals[1]) == 0 and int(h.signals[2]) == 1
    p0, v0 = h.master.clone(), h.vparams.clone()
    h.ps()
    assert int(h.ctrl.view(torch.int32)[1]) == 0 and int(h.signals[256]) == 2
    assert int(h.signals[320]) == 0b101 and int(h.signals[321]) == 1     # published aggregation mask, step stamp
    used = torch.zeros(pl.w_total, dtype=torch.bool, device=h.dev)
    vused = torch.zeros(pl.v_total, dtype=torch.bool, device=h.dev)
    for q in pl.params:
        (used if q.is_w else vused)[q.off:q.off + q.numel] = True
    assert torch.allclose(h.master[used], (p0 - lr * est_w / 2)[used], rtol=3e-4, atol=3e-5)
    assert torch.allclose(h.vparams[vused], (v0 - lr * est_v / 2)[vused], rtol=3e-4, atol=3e-5)


def _batch(net, n=32, seed=0):
    from atomo_b200.models import input_shape
    from atomo_b200.data import SyntheticImageDataset
    x, y = SyntheticImageDataset(input_shape(net), 10, 4096, seed=seed).materialize(n)
    return x.pin_memory(), y.pin_memory()


@pytest.mark.parametrize("code,graph,overlap", [("svd", False, False), ("svd", True, True), ("sgd", True, True)])
def test_shadow_engine_trains_single_gpu(code, graph, overlap):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    eng = ShadowEngine(build_model("ResNet18", 10), 0, 1, code=code, svd_rank=3, lr=0.05, momentum=0.9, use_graph=graph,
                       overlap=overlap, seed=3)
    x, y = _batch("ResNet18", 64)
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
    # the bf16 working copy is the rounding of the fp32 master
    m = eng.gather_fp32("master")
    for q in eng.plan.params:
        if q.is_w:
            assert torch.equal(eng.wshadow[q.off:q.off + q.numel], m[q.off:q.off + q.numel].to(torch.bfloat16))
    eng.close()


def test_shadow_engine_dense_code_applies_exactly_its_gradients():
    """--code sgd, eager: after every step the fp32 master must equal momentum-SGD applied to the very bf16
    gradients autograd produced (checks pointer table, staging, NVLS-free dense path, epilogue, layouts)."""
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(1)
    torch.cuda.set_device(0)
    eng = ShadowEngine(build_model("VGG11", 10), 0, 1, code="sgd", lr=0.05, momentum=0.9, use_graph=False, overlap=True)
    x, y = _batch("VGG11", 32)
    eng.prepare(x, y, warmup=0)
    pl = eng.plan
    master = eng.gather_fp32("master").clone()
    vparams = eng.vparams.clone()
    mom, vmom = torch.zeros_like(master), torch.zeros_like(vparams)
    for step in range(1, 4):
        eng.train_step(x, y)
        torch.cuda.synchronize()
        g = torch.zeros_like(master)
        for p, q in zip(eng.params, pl.params):
            if q.is_w:
                t = p.grad.float()
                g[q.off:q.off + q.numel] = t.permute(0, 2, 3, 1).reshape(-1) if t.dim() == 4 else t.reshape(-1)
        gv = eng.vgrads.clone()
        mom = g.clone() if step == 1 else 0.9 * mom + g
        vmom = gv.clone() if step == 1 else 0.9 * vmom + gv
        master = master - 0.05 * mom
        vparams = vparams - 0.05 * vmom
        got = eng.gather_fp32("master")
        assert torch.allclose(got, master, rtol=1e-4, atol=1e-5), (step, float((got - master).abs().max()))
        assert torch.allclose(eng.vparams, vparams, rtol=1e-4, atol=1e-5), step
    assert eng.error_code() == 0
    eng.close()


def test_shadow_engine_checkpoint_roundtrip(tmp_path):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.cuda.set_device(0)
    d = str(tmp_path) + "/"
    x, y = _batch("ResNet18", 32)

    def make():
        torch.manual_seed(0)
        return ShadowEngine(build_model("ResNet18", 10), 0, 1, code="sgd", lr=0.05, momentum=0.9, use_graph=False, seed=5)
    a = make()
    a.prepare(x, y, warmup=0)
    for _ in range(4):
        a.train_step(x, y)
    path = a.save_checkpoint(d)
    sd = torch.load(path, weights_only=False)
    assert sd["conv1.weight"].dtype == torch.float32 and tuple(sd["conv1.weight"].shape) == (64, 3, 3, 3)
    # ADVICE r1: a checkpoint of a BN network must carry TRAINED running statistics
    assert float(sd["bn1.running_mean"].abs().sum()) > 0 and not torch.allclose(sd["bn1.running_var"], torch.ones(64))
    want = a.gather_fp32("master").clone()
    a.close()
    b = make()
    b.prepare(x, y, warmup=0)
    b.load_checkpoint(d, 4)
    assert b.device_step() == 5
    assert torch.allclose(b.gather_fp32("master"), want, rtol=0, atol=0)
    b.train_step(x, y)
    torch.cuda.synchronize()
    assert b.error_code() == 0
    b.close()


# ---------------------------------------------------------------------------------------------------- multi GPU
def _mp_worker(rank, world, port, cfg, out):
    import torch.distributed as dist
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    torch.manual_seed(0)
    net = cfg.get("net", "ResNet18")
    eng = ShadowEngine(build_model(net, 10), rank, world, code=cfg["code"], svd_rank=3, lr=0.05, momentum=0.9,
                       use_graph=cfg.get("graph", True), seed=5, ps_mode=cfg["ps_mode"], timeout_s=20.0,
                       debug_jitter_us=cfg.get("jitter_us", 0.0))
    x, y = _batch(net, 32, seed=rank)
    eng.prepare(x, y, warmup=cfg.get("warmup", 2))
    losses = []
    ref = None
    if cfg.get("check_dense"):
        ref = {"master": eng.gather_fp32("master").clone(), "v": eng.vparams.clone()}
        ref["mom"], ref["vmom"] = torch.zeros_like(ref["master"]), torch.zeros_like(ref["v"])
    ok_dense = True
    for it in range(cfg.get("steps", 12)):
        losses.append(float(eng.train_step(x, y)[0]))
        if ref is not None:
            torch.cuda.synchronize()
            g = torch.zeros_like(ref["master"])
            for p, q in zip(eng.params, eng.plan.params):
                if q.is_w and eng.is_worker:
                    t = p.grad.float()
                    g[q.off:q.off + q.numel] = t.permute(0, 2, 3, 1).reshape(-1) if t.dim() == 4 else t.reshape(-1)
            gv = eng.vgrads.clone() if eng.is_worker else torch.zeros_like(eng.vgrads)
            dist.all_reduce(g); dist.all_reduce(gv)
            g /= eng.W; gv /= eng.W
            first = eng.step - 1 == 1
            ref["mom"] = g.clone() if first else 0.9 * ref["mom"] + g
            ref["vmom"] = gv.clone() if first else 0.9 * ref["vmom"] + gv
            ref["master"] -= 0.05 * ref["mom"]
            ref["v"] -= 0.05 * ref["vmom"]
            got = eng.gather_fp32("master")
            ok_dense = ok_dense and bool(torch.allclose(got, ref["master"], rtol=2e-4, atol=2e-5)) and \
                bool(torch.allclose(eng.vparams, ref["v"], rtol=2e-4, atol=2e-5))
    torch.cuda.synchronize()
    dist.barrier()           # every owner's last PS launch (peer / multicast stores into OUR copy) has completed
    torch.cuda.synchronize()
    ws = [torch.zeros_like(eng.wshadow) for _ in range(world)]
    dist.all_gather(ws, eng.wshadow.clone())
    vs = [torch.zeros_like(eng.vparams) for _ in range(world)]
    dist.all_gather(vs, eng.vparams.clone())
    same = all(torch.equal(ws[0], t) for t in ws) and all(torch.equal(vs[0], t) for t in vs)
    out.put((rank, eng.error_code(), same, losses[0], losses[-1], eng.heap.mode, eng.heap.has_multicast, ok_dense))
    eng.close()
    dist.destroy_process_group()


def _run_mp(world, cfg, port):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    procs = [ctx.Process(target=_mp_worker, args=(r, world, port, cfg, out)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    return sorted(out.get() for _ in range(world))


@pytest.mark.multigpu
@pytest.mark.parametrize("code,ps_mode", [("svd", "sharded"), ("svd", "colocated"), ("sgd", "sharded"),
                                          ("svd", "dedicated")])
def test_shadow_engine_multi_gpu_replicas_identical(code, ps_mode):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 8 else (8 if os.environ.get("ATOMO_TEST_WORLD8") else 2)
    port = 29700 + 7 * ["sharded", "colocated", "dedicated"].index(ps_mode) + (3 if code == "sgd" else 0)
    res = _run_mp(world, {"code": code, "ps_mode": ps_mode}, port)
    for rank, err, same, l0, l1, mode, mc, _ in res:
        assert err == 0 and same, res
    trained = [r for r in res if not (ps_mode == "dedicated" and r[0] == 0)]
    assert all(r[4] < r[3] for r in trained), res


@pytest.mark.multigpu
@pytest.mark.parametrize("ps_mode", ["sharded", "colocated"])
def test_shadow_engine_protocol_survives_random_delays(ps_mode):
    """Protocol fuzzing (VERDICT r1 #5c): every rank sleeps a different random time (0-300 us, device side) before
    each group's push and each PS launch, eager mode so the delays change every step.  The step-stamped flags must
    still order everything: dense code == mean-gradient SGD exactly, replicas identical, no device error."""
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 8 else (8 if os.environ.get("ATOMO_TEST_WORLD8") else 2)
    res = _run_mp(world, {"code": "sgd", "ps_mode": ps_mode, "graph": False, "check_dense": True, "steps": 6,
                          "net": "VGG11", "warmup": 0, "jitter_us": 300.0}, 29870 + (3 if ps_mode == "sharded" else 0))
    for r in res:
        assert r[1] == 0 and r[2] and r[7], res
    res = _run_mp(world, {"code": "svd", "ps_mode": ps_mode, "graph": False, "steps": 8, "jitter_us": 300.0},
                  29890 + (3 if ps_mode == "sharded" else 0))
    for r in res:
        assert r[1] == 0 and r[2], res


@pytest.mark.multigpu
@pytest.mark.parametrize("ps_mode", ["sharded", "colocated"])
def test_shadow_engine_multi_gpu_dense_equals_mean_gradient_sgd(ps_mode):
    """VERDICT r1 #5: W-GPU --code sgd must equal momentum-SGD on the mean of the workers' gradients."""
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 8 else (8 if os.environ.get("ATOMO_TEST_WORLD8") else 2)
    res = _run_mp(world, {"code": "sgd", "ps_mode": ps_mode, "graph": False, "check_dense": True, "steps": 4,
                          "net": "VGG11", "warmup": 0}, 29950 + (7 if ps_mode == "sharded" else 0))
    for r in res:
        assert r[1] == 0 and r[2] and r[7], res

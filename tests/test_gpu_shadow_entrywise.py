"""Entry-wise ATOMO on the overlapped, sharded bf16 engine: planner and argument checks (CPU), kernels against the
``codings.entrywise`` oracle and the engine end to end (GPU)."""
import os

import pytest
import torch

from atomo_b200.ops import plan2 as P

NET_SHAPES = [(64, 3, 3, 3), (64,), (64,), (128, 64, 3, 3), (128,), (256, 128, 3, 3), (512, 256, 1, 1), (300, 200),
              (10, 512), (7, 20), (10,)]
# stem, 3x3 convs (one a multiple of 4096 elements, one not), fc layers, a tensor smaller than an absolute budget,
# a tensor that is all zero in the oracle test, a vector
ORACLE_SHAPES = [(64, 3, 3, 3), (64, 32, 3, 3), (128, 64, 3, 3), (10, 512), (300, 200), (7, 20), (5, 3), (64,)]
ZERO_PARAM, SPIKE_PARAM = 6, 1


def _entry_budget_of(b):
    from atomo_b200.codings.entrywise import EntryWise
    return EntryWise(b)


# ---------------------------------------------------------------------------------------------------- planner
@pytest.mark.parametrize("budget,owners", [(0.05, 1), (0.01, 3), (0.25, 2), (300.0, 4), (5000.0, 1)])
def test_plan2_entry_units_tiles_and_slots(budget, owners):
    pl = P.build_plan2(NET_SHAPES, "entrywise", n_owners=owners, n_groups=3, entry_budget=budget)
    coder = _entry_budget_of(budget)
    for p in pl.params:
        units = [u for u in pl.units if u.param == p.index]
        assert len(units) == 1, p.shape
        u = units[0]
        if p.is_w:
            assert u.kind == P.KIND_ENTRY and (u.numel, u.w_off, u.g_off) == (p.numel, p.off, 0)
            assert u.budget == coder.atoms_for(p.numel)
            assert u.ps_rows == P.ENTRY_TILE_ELEMS
        else:
            assert u.kind == P.KIND_VEC
    assert not any(u.kind == P.KIND_DENSE16 for u in pl.units)
    entry_units = [u for u in pl.units if u.kind == P.KIND_ENTRY]
    assert pl.n_coded == len(entry_units) == sum(1 for p in pl.params if p.is_w)
    assert sorted(u.ts_index for u in entry_units) == list(range(len(entry_units)))
    # tiles: every element exactly once, <= 4096 elements, encode tile == PS tile
    for u in entry_units:
        tiles = sorted((a, b) for (ui, a, b, o) in pl.ps_tiles if ui == u.index)
        assert len(tiles) == u.n_ps == -(-u.numel // P.ENTRY_TILE_ELEMS)
        assert all(a == j * P.ENTRY_TILE_ELEMS and 0 < b <= P.ENTRY_TILE_ELEMS for j, (a, b) in enumerate(tiles))
        assert sum(b for _, b in tiles) == u.numel
        enc = [(a, b, j) for (ui, a, b, j) in pl.enc_tiles if ui == u.index]
        assert [(a, b) for a, b, _ in enc] == tiles and [j for _, _, j in enc] == list(range(u.n_ps))
        assert u.n_enc == u.n_ps
    # owners round-robin inside a group, over the group's PS tiles in unit order
    for g in range(pl.n_groups):
        by_order = []
        for ui in pl.group_units[g]:
            u = pl.units[ui]
            e = u.ps_rows if u.kind == P.KIND_ENTRY else P.DENSE_TILE_ELEMS
            by_order.extend((ui, a) for a in range(0, u.numel, e))
        owner_of = {(ui, a): o for (ui, a, b, o) in pl.ps_tiles}
        assert sorted(by_order) == sorted((ui, a) for (ui, a, b, o) in pl.ps_tiles if pl.units[ui].group == g)
        assert [owner_of[k] for k in by_order] == [j % owners for j in range(len(by_order))]
    # slots: disjoint, 16-byte aligned headers and entries, inside the arena
    spans = []
    for u in entry_units:
        assert u.slot_off % 4 == 0
        last = u.numel - (u.n_ps - 1) * P.ENTRY_TILE_ELEMS
        for j in range(u.n_ps):
            assert P.entry_words_off(u.n_ps, j) % 4 == 0
            assert P.entry_words_off(u.n_ps, j) >= P.entry_hdr_off(u.n_ps)      # entries after every header
        end = u.slot_off + P.entry_words_off(u.n_ps, u.n_ps - 1) + last
        spans.append((u.slot_off, end))
    spans.sort()
    assert all(a1 >= b0 for (a0, b0), (a1, b1) in zip(spans, spans[1:]))
    assert spans[-1][1] <= pl.arena_floats
    # byte accounting: 4 bytes per expected atom, 16 per tile header
    want = sum(4 * coder.atoms_for(p.numel) for p in pl.params if p.is_w) + \
        16 * sum(-(-p.numel // P.ENTRY_TILE_ELEMS) for p in pl.params if p.is_w)
    assert pl.entry_bytes() == pytest.approx(want, rel=1e-12)
    assert pl.expected_factor_bytes() == pytest.approx(want, rel=1e-12)
    assert pl.qsgd_bytes() == 0 and pl.factor_bytes_per_worker() == 0
    assert pl.dense_bytes() == 4 * sum(p.numel for p in pl.params if not p.is_w)


def test_plan2_other_codes_ignore_the_entry_budget():
    for code in ("svd", "qsvd", "sgd", "qsgd", "terngrad"):
        a = P.build_plan2(NET_SHAPES, code, 3, n_owners=2, n_groups=3)
        for b in (0.01, 0.25, 1000.0, -1.0):
            c = P.build_plan2(NET_SHAPES, code, 3, n_owners=2, n_groups=3, entry_budget=b)
            assert a.units_bytes() == c.units_bytes() and a.ps_tiles == c.ps_tiles and a.enc_tiles == c.enc_tiles
            assert a.enc_range == c.enc_range and a.ps_range == c.ps_range
            assert a.arena_floats == c.arena_floats and a.n_coded == c.n_coded and c.entry_bytes() == 0


def test_plan2_entry_refuses_non_positive_budget():
    for b in (0.0, -0.05, float("nan")):
        with pytest.raises(ValueError):
            P.build_plan2(NET_SHAPES, "entrywise", entry_budget=b)


@pytest.mark.parametrize("kw", [{"prob_rule": "waterfill"}, {"sampling": "systematic"}, {"entry_budget": 0.0},
                                {"entry_budget": -2.0}])
def test_shadow_engine_entrywise_refuses_unsupported_settings(kw):
    """Checked before any CUDA work, so a bad flag fails the same way on every machine."""
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    with pytest.raises(ValueError):
        ShadowEngine(None, 0, 1, code="entrywise", **kw)


# ---------------------------------------------------------------------------------------------------- GPU harness
def _ext():
    from atomo_b200.ops._ext import load
    return load()


class HE:
    """Loopback harness: one rank that is worker 0..W-1 (virtual) and the only owner."""

    def __init__(self, shapes, budget=0.05, W=1, lr=0.1, momentum=0.0, wd=0.0, nesterov=False, opt=0, seed=7,
                 num_aggregate=0):
        self.C = _ext()
        dev = self.dev = torch.device("cuda", 0)
        self.W, self.budget = W, budget
        self.plan = pl = P.build_plan2(shapes, "entrywise", n_owners=1, n_groups=1, entry_budget=budget)
        u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)
        self.t_units = u8(pl.units_bytes())
        self.t_enc = u8(P.Plan2.tiles_bytes(pl.enc_tiles))
        self.t_ps = u8(P.Plan2.tiles_bytes(pl.ps_tiles))
        nc = max(pl.n_coded, 1)
        z = lambda n, dt=torch.float32: torch.zeros(n, dtype=dt, device=dev)
        self.l1 = z(nc, torch.float64)
        self.partials = z(len(pl.enc_tiles), torch.float64)
        self.counters = z(nc + 32, torch.int32)
        self.arena = z(pl.arena_floats * W)
        self.signals = z(1024, torch.int32)
        self.signals[256] = 1
        self.ctrl = u8(P.pack_ctrl2(step=1, lr=lr, momentum=momentum, weight_decay=wd, nesterov=nesterov, seed=seed,
                                    opt=opt, num_aggregate=num_aggregate))
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.master = torch.randn(pl.w_total, device=dev, generator=g)
        self.wshadow = self.master.to(torch.bfloat16)
        self.vparams = torch.randn(pl.v_total, device=dev, generator=g)
        self.mom, self.vmom = z(pl.w_total), z(pl.v_total)
        self.sq, self.vsq, self.sqmax, self.vsqmax = z(pl.w_total), z(pl.v_total), z(pl.w_total), z(pl.v_total)
        self.vgrads = [z(pl.v_total) for _ in range(W)]
        self.wgrads = [None] * W
        i64 = lambda xs: torch.tensor(list(xs), dtype=torch.int64, device=dev)
        self.t_arena_peer = i64([self.arena.data_ptr()])
        self.t_sig_peer = i64([self.signals.data_ptr()])
        self.t_wshadow_peer = i64([self.wshadow.data_ptr()])
        self.t_vparams_peer = i64([self.vparams.data_ptr()])
        self.t_vgrads_peer = i64([t.data_ptr() for t in self.vgrads])
        self.tstats = z(32, torch.int64)

    def set_step(self, step):
        self.ctrl.view(torch.int32)[0] = step

    def fill(self, w, seed, zero=(), spike=()):
        """Random bf16 gradients of virtual worker w (params in `zero` all zero, params in `spike` with a few large
        entries); returns {param index: fp32 physical-order flat tensor}."""
        pl, dev = self.plan, self.dev
        g = torch.Generator(device="cuda").manual_seed(seed)
        grads, phys = [], {}
        for q in pl.params:
            if q.is_w:
                x = torch.randn(q.shape, device=dev, generator=g)
                if q.index in zero:
                    x.zero_()
                if q.index in spike:
                    x.view(-1)[::997] = 300.0
                x = x.to(torch.bfloat16)
                t = x.contiguous(memory_format=torch.channels_last) if x.dim() == 4 else x.contiguous()
                grads.append(t)
                phys[q.index] = (t.permute(0, 2, 3, 1) if t.dim() == 4 else t).reshape(-1).float()
            else:
                v = torch.randn(q.numel, device=dev, generator=g)
                self.vgrads[w][q.off:q.off + q.numel] = v
                phys[q.index] = v
        self.wgrads[w] = grads
        return phys

    def encode(self, w, uniforms=None):
        C, pl = self.C, self.plan
        gptr = torch.tensor([t.data_ptr() for t in self.wgrads[w]], dtype=torch.int64, device=self.dev)
        self._gptr = gptr
        t0, nt = pl.enc_range[0]
        C.v2_entry_stats(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr.data_ptr(),
                         self.partials.data_ptr(), self.counters.data_ptr(), self.l1.data_ptr(), 0, 0)
        C.v2_entry_encode(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr.data_ptr(), self.l1.data_ptr(),
                          self.t_arena_peer.data_ptr(), self.t_sig_peer.data_ptr(), 1, pl.arena_floats, w, 0,
                          self.ctrl.data_ptr(), self.counters.data_ptr() + 4 * (pl.n_coded + 8),
                          uniforms.data_ptr() if uniforms is not None else 0, 0, False)
        torch.cuda.synchronize()

    def ps(self, grid=64):
        C, pl = self.C, self.plan
        t0, nt = pl.ps_range[0][0]
        C.v2_ps_entry(self.t_units.data_ptr(), self.t_ps.data_ptr(), t0, nt, self.W, 1, 0, True, 0,
                      self.master.data_ptr(), self.mom.data_ptr(), self.sq.data_ptr(), self.sqmax.data_ptr(),
                      self.vmom.data_ptr(), self.vsq.data_ptr(), self.vsqmax.data_ptr(), 0,
                      self.t_wshadow_peer.data_ptr(), self.vparams.data_ptr(), 0, self.t_vparams_peer.data_ptr(), 0,
                      self.t_vgrads_peer.data_ptr(), self.arena.data_ptr(), pl.arena_floats, self.signals.data_ptr(),
                      self.t_sig_peer.data_ptr(), self.ctrl.data_ptr(), self.counters.data_ptr() + 4 * (pl.n_coded + 16),
                      int(5e9), self.tstats.data_ptr(), 1.0 / self.W, grid)
        torch.cuda.synchronize()

    def tiles(self, u, w):
        """Per PS tile of unit u in worker w's slot: (stamp, count, scale, int32 words of the 16-byte groups)."""
        base = self.arena[w * self.plan.arena_floats + u.slot_off:]
        out = []
        for j in range(u.n_ps):
            h = base[P.entry_hdr_off(j):P.entry_hdr_off(j) + 4]
            stamp, count = (int(v) for v in h.view(torch.int32)[:2].tolist())
            wo = P.entry_words_off(u.n_ps, j)
            words = base[wo:wo + (count + 3) // 4 * 4].view(torch.int32).clone()
            out.append((stamp, count, float(h[2]), words))
        return out

    def decode(self, u, w):
        """(element indices inside the unit, fp32 values, exact-flag) of the entries worker w pushed for unit u."""
        idx, val, flag = [], [], []
        for j, (_, count, scale, words) in enumerate(self.tiles(u, w)):
            e = words[:count]
            g = (e & -65536).view(torch.float32)
            f = (e & 0x1000) != 0
            idx.append(j * P.ENTRY_TILE_ELEMS + (e & 0xFFF).long())
            val.append(torch.where(f, g, torch.copysign(torch.full_like(g, scale), g)))
            flag.append(f)
        return torch.cat(idx), torch.cat(val), torch.cat(flag)


def _bf16_bits(x):
    return (x.to(torch.bfloat16).view(torch.int16).to(torch.int32) & 0xFFFF)


# ---------------------------------------------------------------------------------------------------- GPU: encode
@pytest.mark.gpu
@pytest.mark.parametrize("budget", [0.01, 0.05, 0.25, 200.0])
def test_v2_entry_encode_matches_oracle(budget):
    h = HE(ORACLE_SHAPES, budget)
    pl = h.plan
    step = 3
    h.set_step(step)
    phys = h.fill(0, 11, zero=(ZERO_PARAM,), spike=(SPIKE_PARAM,))
    uni = torch.rand(pl.w_total + 64, device=h.dev, generator=torch.Generator(device="cuda").manual_seed(5))
    h.encode(0, uni)
    coder = _entry_budget_of(budget)
    saw_exact = False
    for u in pl.units:
        if u.kind != P.KIND_ENTRY:
            continue
        flat = phys[u.param]
        n = u.numel
        tiles = h.tiles(u, 0)
        for j, (stamp, count, scale, words) in enumerate(tiles):
            tlen = min(P.ENTRY_TILE_ELEMS, n - j * P.ENTRY_TILE_ELEMS)
            assert stamp == step and 0 <= count <= tlen
            offs = (words[:count] & 0xFFF).long()
            assert bool((offs[1:] > offs[:-1]).all()) and (count == 0 or int(offs[-1]) < tlen)   # sorted, unique
            assert bool((words[count:] == 0).all())                  # the padding of the last 16-byte store
        idx, val, flag = h.decode(u, 0)
        s = coder.atoms_for(n)
        l1 = float(flat.double().abs().sum())
        if l1 == 0:
            assert idx.numel() == 0 and all(t[1] == 0 for t in tiles), u.param
            continue
        # every entry carries its gradient's bf16 bits; flagged entries decode to them, the others to +-scale
        gbits = _bf16_bits(flat)
        words = torch.cat([t[3][:t[1]] for t in tiles])
        assert torch.equal((words >> 16) & 0xFFFF, gbits[idx])
        assert torch.equal(val[flag], flat[idx][flag])
        for (_, count, scale, _) in tiles:
            assert abs(scale - l1 / s) <= 1e-6 * (l1 / s)
        assert torch.equal(val[~flag].abs(), torch.full_like(val[~flag], tiles[0][2]))
        saw_exact = saw_exact or bool(flag.any())
        # the kept set is the oracle's except where the uniform lies within rounding of p
        ref = coder.encode(flat.cpu(), uniforms=uni[u.w_off:u.w_off + n].cpu())
        mine = torch.zeros(n, dtype=torch.bool)
        mine[idx.cpu()] = True
        want = torch.zeros(n, dtype=torch.bool)
        want[ref["idx"].long()] = True
        p = (s * flat.double().abs() / l1).cpu()
        uu = uni[u.w_off:u.w_off + n].double().cpu()
        diff = mine != want
        assert bool(((uu - p.clamp(max=1.0)).abs()[diff] <= 1e-5 * p[diff]).all()), u.param
        assert int(diff.sum()) <= 2 + n // 1000, (u.param, int(diff.sum()))
        # flags: p_i == 1 up to rounding of s / L1
        pf = torch.zeros(n, dtype=torch.bool)
        pf[idx.cpu()[flag.cpu()]] = True
        fdiff = (pf != (p >= 1.0)) & mine
        assert bool(((p - 1.0).abs()[fdiff] <= 1e-5).all()), u.param
        # values: the oracle's g / p wherever both keep the element
        both = mine & want
        ref_val = torch.zeros(n)
        ref_val[ref["idx"].long()] = ref["val"]
        my_val = torch.zeros(n)
        my_val[idx.cpu()] = val.cpu()
        assert torch.allclose(my_val[both], ref_val[both], rtol=1e-5, atol=0), u.param
    assert saw_exact                                            # the spiky tensor has entries with p_i clamped to 1
    assert int(h.signals[0]) == step


@pytest.mark.gpu
def test_v2_entry_encode_is_repeatable():
    h = HE(ORACLE_SHAPES, 0.05)
    h.set_step(4)
    h.fill(0, 3, spike=(SPIKE_PARAM,))
    h.encode(0)
    first = h.arena.clone()
    h.arena.zero_()
    h.encode(0)
    assert torch.equal(h.arena.view(torch.int32), first.view(torch.int32))
    assert int((first != 0).sum()) > 0
    h.set_step(5)                                               # another step draws other uniforms
    h.encode(0)
    assert not torch.equal(h.arena.view(torch.int32), first.view(torch.int32))


@pytest.mark.gpu
def test_v2_entry_philox_sampling_is_unbiased():
    shapes = [(32, 16, 3, 3), (40, 30)]
    h = HE(shapes, 0.25)
    phys = h.fill(0, 5)
    units = [u for u in h.plan.units if u.kind == P.KIND_ENTRY]
    acc = {u.index: torch.zeros(u.numel, device=h.dev) for u in units}
    cnt = {u.index: 0 for u in units}
    T = 1000
    for t in range(T):
        h.set_step(t + 1)
        h.encode(0)
        for u in units:
            idx, val, _ = h.decode(u, 0)
            acc[u.index][idx] += val
            cnt[u.index] += idx.numel()
    for u in units:
        flat = phys[u.param]
        p = (u.budget * flat.double().abs() / flat.double().abs().sum()).clamp(max=1.0)
        mean = acc[u.index] / T
        var = torch.where(p > 0, flat.double() ** 2 * (1 - p) / p.clamp(min=1e-30), torch.zeros_like(p))
        bound = 4 * (var / T).sqrt() + 1e-6 * float(flat.abs().max())
        frac_out = float(((mean.double() - flat.double()).abs() > bound).float().mean())
        assert frac_out < 1e-3, (u.param, frac_out)
        assert float((mean - flat).norm() / flat.norm()) < 0.2
        sp = float(p.sum())
        sd = float((p * (1 - p)).sum()) ** 0.5
        assert abs(cnt[u.index] / T - sp) <= 4 * sd / T ** 0.5 + 1e-3 * sp, (u.param, cnt[u.index] / T, sp)


# ---------------------------------------------------------------------------------------------------- GPU: PS
def _opt_ref(p, g, m, s2, s2m, step, lr, momentum, nesterov, wd, opt):
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


def _decoded_sum(h, workers):
    """sum over `workers` (in worker order, fp32) of the entries actually in the arena, physical order."""
    est = torch.zeros(h.plan.w_total, device=h.dev)
    for w in workers:
        for u in h.plan.units:
            if u.kind == P.KIND_ENTRY:
                idx, val, _ = h.decode(u, w)
                est[u.w_off + idx] += val          # one worker's indices are distinct: one rounding per element
    return est


def _used(pl, dev):
    used = torch.zeros(pl.w_total, dtype=torch.bool, device=dev)
    vused = torch.zeros(pl.v_total, dtype=torch.bool, device=dev)
    for q in pl.params:
        (used if q.is_w else vused)[q.off:q.off + q.numel] = True
    return used, vused


@pytest.mark.gpu
def test_v2_ps_entry_mean_is_bitwise_the_decodes():
    """With lr = 1, no momentum / weight decay and a zero master, the PS writes master = -g exactly, so the kernel's
    averaged gradient can be compared bit for bit with the entries summed in worker order, times 1/W."""
    W = 3
    h = HE(NET_SHAPES, 0.25, W=W, lr=1.0)
    for w in range(W):
        h.fill(w, 70 + w, spike=(3,))
        h.encode(w)
    want = _decoded_sum(h, range(W)) * torch.tensor(1.0 / W, dtype=torch.float32)
    h.master.zero_()
    h.ps()
    assert int(h.ctrl.view(torch.int32)[1]) == 0
    used, _ = _used(h.plan, h.dev)
    assert torch.equal(-h.master[used], want[used])
    assert int((want[used] != 0).sum()) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("momentum,nesterov,wd,opt", [(0.0, False, 0.0, 0), (0.9, True, 1e-3, 0), (0.9, False, 0.0, 0),
                                                      (0.0, False, 0.0, 1), (0.0, False, 1e-3, 2)])
def test_v2_ps_entry_matches_reference(momentum, nesterov, wd, opt):
    W, lr = 3, 0.05
    h = HE(NET_SHAPES, 0.05, W=W, lr=lr, momentum=momentum, wd=wd, nesterov=nesterov, opt=opt)
    pl = h.plan
    used, vused = _used(pl, h.dev)
    for step in (1, 2):
        h.set_step(step)
        for w in range(W):
            h.fill(w, 10 * step + w)
            h.encode(w)
        gw = _decoded_sum(h, range(W)) / W
        gv = sum(h.vgrads) / W
        rp, rm = _opt_ref(h.master.clone(), gw, h.mom.clone(), h.sq.clone(), h.sqmax.clone(), step, lr, momentum,
                          nesterov, wd, opt)
        rv, _ = _opt_ref(h.vparams.clone(), gv, h.vmom.clone(), h.vsq.clone(), h.vsqmax.clone(), step, lr, momentum,
                         nesterov, wd, opt)
        h.ps()
        assert int(h.ctrl.view(torch.int32)[1]) == 0
        assert int(h.signals[256]) == step + 1
        tol = dict(rtol=3e-4, atol=3e-5) if opt == 0 else dict(rtol=2e-3, atol=2e-4)
        assert torch.allclose(h.master[used], rp[used], **tol), float((h.master - rp)[used].abs().max())
        assert torch.allclose(h.vparams[vused], rv[vused], **tol)
        assert torch.equal(h.wshadow[used], h.master.to(torch.bfloat16)[used])


@pytest.mark.gpu
def test_v2_ps_entry_num_aggregate_and_stale_slots():
    """num_aggregate = 2 of 3 workers, worker 1 never pushes: only {0, 2} are averaged.  Then a slot whose stamp is
    of another step is skipped and flagged with ERR2_SLOT_STEP."""
    lr = 0.1
    h = HE(NET_SHAPES, 0.05, W=3, lr=lr, num_aggregate=2)
    pl = h.plan
    for w in (0, 2):
        h.fill(w, 40 + w)
        h.encode(w)
    h.vgrads[1].fill_(1e6)                         # garbage a skipped worker may hold
    assert int(h.signals[0]) == 1 and int(h.signals[1]) == 0 and int(h.signals[2]) == 1
    est = _decoded_sum(h, (0, 2))
    p0, v0 = h.master.clone(), h.vparams.clone()
    h.ps()
    assert int(h.ctrl.view(torch.int32)[1]) == 0 and int(h.signals[256]) == 2
    assert int(h.signals[320]) == 0b101 and int(h.signals[321]) == 1
    used, vused = _used(pl, h.dev)
    assert torch.allclose(h.master[used], (p0 - lr * est / 2)[used], rtol=3e-4, atol=3e-5)
    assert torch.allclose(h.vparams[vused], (v0 - lr * (h.vgrads[0] + h.vgrads[2]) / 2)[vused], rtol=3e-4, atol=3e-5)

    # stale stamp: worker 1's slot still holds step 0 (never written) while its flag claims step 1
    hs = HE(NET_SHAPES, 0.05, W=2, lr=lr)
    hs.fill(0, 1)
    hs.encode(0)
    hs.signals[1] = 1
    hs.ps()
    assert int(hs.ctrl.view(torch.int32)[1]) & 4          # ERR2_SLOT_STEP


# ---------------------------------------------------------------------------------------------------- GPU: engine
def _batch(net, n=32, seed=0):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import input_shape
    x, y = SyntheticImageDataset(input_shape(net), 10, 4096, seed=seed).materialize(n)
    return x.pin_memory(), y.pin_memory()


def _engine(net, graph, overlap, budget, seed=3):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    return ShadowEngine(build_model(net, 10), 0, 1, code="entrywise", entry_budget=budget, lr=0.05, momentum=0.9,
                        use_graph=graph, overlap=overlap, seed=seed)


@pytest.mark.gpu
@pytest.mark.parametrize("net", ["ResNet18", "VGG11"])
@pytest.mark.parametrize("graph,overlap", [(True, True), (False, False)])
def test_shadow_engine_entrywise_trains_single_gpu(net, graph, overlap, tmp_path, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)      # bitwise-reproducible backward
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    budget = 0.25
    x, y = _batch(net, 64)
    masters = []
    for rep in range(2):
        eng = _engine(net, graph, overlap, budget)
        assert eng.vprev is None                        # no spectral warm-start state
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
            assert side["entry_budget"] == budget and side["code"] == "entrywise"
            want = m.clone()
            eng.close()
            b = _engine(net, graph, overlap, budget)
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
@pytest.mark.parametrize("ps_mode", ["sharded", "colocated"])
def test_shadow_engine_entrywise_multi_gpu_replicas_identical(ps_mode):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    from test_gpu_v2 import _run_mp
    world = 2 if n < 8 else (8 if os.environ.get("ATOMO_TEST_WORLD8") else 2)
    port = 29760 + 7 * ["sharded", "colocated"].index(ps_mode)
    res = _run_mp(world, {"code": "entrywise", "ps_mode": ps_mode, "net": "VGG11"}, port)
    for rank, err, same, l0, l1, mode, mc, _ in res:
        assert err == 0 and same, res
    assert all(r[4] < r[3] for r in res), res


@pytest.mark.gpu
@pytest.mark.multigpu
def test_shadow_engine_entrywise_protocol_survives_random_delays():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    from test_gpu_v2 import _run_mp
    world = 2 if n < 8 else (8 if os.environ.get("ATOMO_TEST_WORLD8") else 2)
    res = _run_mp(world, {"code": "entrywise", "ps_mode": "sharded", "graph": False, "steps": 8, "warmup": 0,
                          "jitter_us": 300.0}, 29780)
    for r in res:
        assert r[1] == 0 and r[2], res

"""Helpers shared by the test files: loopback harnesses of the bf16 engine's kernels, the error-feedback loopback
engine, the single-GPU and multi-GPU training helpers and the launcher argv.  Not a test file itself: pytest puts this
directory on ``sys.path``, and the tests import from here."""
import argparse
import math
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn as nn

from atomo_b200.codings import signum as S
from atomo_b200.ops import plan2 as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ext():
    from atomo_b200.ops._ext import load
    return load()


def physical(t):
    """A weight tensor in the engine's storage order: channels-last if 4-d."""
    return t.contiguous(memory_format=torch.channels_last) if t.dim() == 4 else t.contiguous()


def flat(t):
    """Physical-order flat view of a tensor in storage order."""
    return (t.permute(0, 2, 3, 1) if t.dim() == 4 else t).view(-1)


# ---------------------------------------------------------------------------------------------------- bf16 engine
class LoopbackPS:
    """Loopback harness of the bf16 engine: one GPU that is virtual worker 0..W-1 and virtual owner 0..n_owners-1.

    Subclasses name the code's PS binding (``PS``), launch the code's encode, decode its slots, and may change a drawn
    gradient tensor in ``tensor``.  ``counters`` (int32; every kernel resets the words it used) is laid out as
    ``[0, nc)`` per coded unit (stats / selection kernels, by ``ts_index``), ``nc + g`` the encode of group g and
    ``nc + 8 (1 + o) + g`` the PS launch of owner o for group g, so up to 8 groups never share a word."""

    PS = None

    def __init__(self, shapes, code, W=1, lr=0.1, momentum=0.0, wd=0.0, nesterov=False, opt=0, seed=7,
                 num_aggregate=0, n_groups=1, n_owners=1, stage=False, **plan_kw):
        assert n_groups <= 8
        self.C = ext()
        dev = self.dev = torch.device("cuda", 0)
        self.W, self.seed, self.n_owners, self.step = W, seed, n_owners, 1
        self.plan = pl = P.build_plan2(shapes, code, n_owners=n_owners, n_groups=n_groups, **plan_kw)
        u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)
        self.t_units = u8(pl.units_bytes())
        self.t_enc = u8(P.Plan2.tiles_bytes(pl.enc_tiles))
        self.t_ps = u8(P.Plan2.tiles_bytes(pl.ps_tiles))
        nc = self.nc = max(pl.n_coded, 1)
        z = self.zeros = lambda n, dt=torch.float32: torch.zeros(n, dtype=dt, device=dev)
        self.counters = z(nc + 8 * (1 + n_owners), torch.int32)
        # one arena and one signal region per owner
        self.arenas = [z(pl.arena_floats * W) for _ in range(n_owners)]
        self.sigs = [z(1024, torch.int32) for _ in range(n_owners)]
        for s in self.sigs:
            s[256:256 + n_owners] = 1
        self.arena, self.signals = self.arenas[0], self.sigs[0]
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
        self.stage = [z(pl.stage_total, torch.bfloat16) for _ in range(W)] if stage else None
        i64 = lambda xs: torch.tensor(list(xs), dtype=torch.int64, device=dev)
        self.t_arena_peer = i64(t.data_ptr() for t in self.arenas)
        self.t_sig_peer = i64(t.data_ptr() for t in self.sigs)
        self.t_sig_own = [i64([t.data_ptr()]) for t in self.sigs]      # an owner's PS reads its own region only
        self.t_wshadow_peer = i64([self.wshadow.data_ptr()])
        self.t_vparams_peer = i64([self.vparams.data_ptr()])
        self.t_vgrads_peer = i64(t.data_ptr() for t in self.vgrads)
        self.t_stage_peer = i64(t.data_ptr() for t in self.stage) if stage else None
        self.ps_tail = ()                # the code's last PS arguments
        self.tstats = z(32, torch.int64)

    def counter(self, g=0, owner=None):
        """Address of the counter of group g's encode, or of owner's PS launch for group g."""
        return self.counters.data_ptr() + 4 * (self.nc + g if owner is None else self.nc + 8 * (1 + owner) + g)

    def set_step(self, step):
        self.step = step
        self.ctrl.view(torch.int32)[0] = step

    def tensor(self, q, x, g, **kw):
        """The fp32 gradient of weight q before its bf16 rounding, given the normal draw x (logical layout) and the
        generator g for further draws.  To set entries in physical order, return ``physical(x)`` changed through
        ``flat``."""
        return x

    def fill(self, w, seed, **kw):
        """Random bf16 gradients of virtual worker w (``tensor`` may change each); returns {param index: fp32
        physical-order flat tensor}."""
        pl, dev = self.plan, self.dev
        g = torch.Generator(device="cuda").manual_seed(seed)
        grads, phys = [], {}
        for q in pl.params:
            if q.is_w:
                x = self.tensor(q, torch.randn(q.shape, device=dev, generator=g), g, **kw)
                t = physical(x.to(torch.bfloat16))
                grads.append(t)
                phys[q.index] = flat(t).float()
            else:
                v = torch.randn(q.numel, device=dev, generator=g)
                self.vgrads[w][q.off:q.off + q.numel] = v
                phys[q.index] = v
        self.wgrads[w] = grads
        return phys

    def gptr(self, w):
        """Device table of worker w's gradient pointers (kept alive until the next call)."""
        self._gptr = torch.tensor([t.data_ptr() for t in self.wgrads[w]] or [0], dtype=torch.int64, device=self.dev)
        return self._gptr.data_ptr()

    def ps(self, grid=64):
        """The PS launch of every owner for every group, ``final`` on the last group."""
        pl = self.plan
        stage = [self.t_stage_peer.data_ptr()] if self.stage is not None else []
        for g in range(pl.n_groups):
            for o in range(self.n_owners):
                t0, nt = pl.ps_range[g][o]
                getattr(self.C, self.PS)(
                    self.t_units.data_ptr(), self.t_ps.data_ptr(), t0, nt, self.W, 1, g, g == pl.n_groups - 1, o,
                    self.master.data_ptr(), self.mom.data_ptr(), self.sq.data_ptr(), self.sqmax.data_ptr(),
                    self.vmom.data_ptr(), self.vsq.data_ptr(), self.vsqmax.data_ptr(), 0,
                    self.t_wshadow_peer.data_ptr(), self.vparams.data_ptr(), 0, self.t_vparams_peer.data_ptr(), 0,
                    self.t_vgrads_peer.data_ptr(), *stage, self.arenas[o].data_ptr(), pl.arena_floats,
                    self.sigs[o].data_ptr(), self.t_sig_own[o].data_ptr(), self.ctrl.data_ptr(), self.counter(g, o),
                    int(5e9), self.tstats.data_ptr(), 1.0 / self.W, grid, *self.ps_tail)
        torch.cuda.synchronize()

    def used(self):
        mw = torch.zeros(self.plan.w_total, dtype=torch.bool, device=self.dev)
        mv = torch.zeros(self.plan.v_total, dtype=torch.bool, device=self.dev)
        for q in self.plan.params:
            (mw if q.is_w else mv)[q.off:q.off + q.numel] = True
        return mw, mv


class H2(LoopbackPS):
    """Spectral ATOMO (svd / qsvd) and the dense code: fills return fp32 gradients in the logical layout."""

    PS = "v2_ps"

    def __init__(self, shapes, code="svd", rank=3, W=1, lr=0.1, momentum=0.0, wd=0.0, nesterov=False, opt=0, seed=7,
                 systematic=False, groups=1, warm=False, max_sweeps=0):
        super().__init__(shapes, code, W, lr, momentum, wd, nesterov, opt, seed, n_groups=groups, stage=True,
                         rank=rank, systematic=systematic)
        self.P = P
        pl, dev, z = self.plan, self.dev, self.zeros
        nc = self.nc
        self.gpart, self.vsel, self.sigma = z(pl.gpart_floats), z(nc * 64 * 32), z(nc * 64)
        self.selcount = z(nc, torch.int32)
        self.max_sweeps = max_sweeps
        self.vprev = None
        if warm:
            self.vprev = z(nc * 64 * 64)
            for u in pl.units:
                if u.coded:
                    self.vprev[u.ts_index * 4096:u.ts_index * 4096 + u.cols * u.cols] = torch.eye(u.cols, device=dev).reshape(-1)

    def tensor(self, q, x, g, lowrank=True):
        if lowrank and len(q.shape) >= 2:
            dev = self.dev
            m = x.reshape(q.shape[0], -1)
            k = min(m.shape)
            a = torch.randn(m.shape[0], k, device=dev, generator=g) * torch.logspace(0, -1.5, k, device=dev)
            x = (a @ torch.linalg.qr(torch.randn(m.shape[1], k, device=dev, generator=g)).Q.T).reshape(q.shape)
        return x

    def fill(self, w, seed, lowrank=True):
        """Random gradients for virtual worker w; returns {param index: fp32 tensor in the logical layout}."""
        logical = super().fill(w, seed, lowrank=lowrank)
        for q in self.plan.params:
            if q.is_w:
                logical[q.index] = self.wgrads[w][q.widx].float()
        return logical

    def encode(self, w, random_sample=True, waterfill=False, systematic=False, uniforms=None, resample_empty=False):
        C, pl = self.C, self.plan
        gptr = self.gptr(w)
        for g in range(pl.n_groups):
            t0, nt = pl.enc_range[g]
            C.v2_encode(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr, self.gpart.data_ptr(),
                        self.counters.data_ptr(), self.vsel.data_ptr(), self.selcount.data_ptr(), self.sigma.data_ptr(),
                        self.t_arena_peer.data_ptr(), 1, pl.arena_floats, self.stage[w].data_ptr(), self.ctrl.data_ptr(),
                        uniforms.data_ptr() if uniforms is not None else 0,
                        self.vprev.data_ptr() if self.vprev is not None else 0, self.max_sweeps, random_sample,
                        waterfill, systematic, w, resample_empty, 0, 0, g)
            C.v2_project(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr, self.vsel.data_ptr(),
                         self.selcount.data_ptr(), self.t_arena_peer.data_ptr(), self.t_sig_peer.data_ptr(), 1,
                         pl.arena_floats, w, g, self.ctrl.data_ptr(), self.counter(g), 0, 0, False, False)
        torch.cuda.synchronize()

    # ---- references ---------------------------------------------------------------------------------------
    def unit_matrix(self, u, logical):
        """fp32 tall matrix of a coded unit, in the kernel's row/column convention."""
        q = self.plan.params[u.param]
        t = logical[q.index]
        if u.kind == P.KIND_SLAB:
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
        uo = P.slot_u_off(u.rcap, u.cols)
        if u.ubits == 8:      # QSVD: int8 U with one fp32 scale per row
            q = base[uo:uo + u.rows * u.rcap // 4].view(torch.int8).view(u.rows, u.rcap)[:, :count].float()
            so = P.slot_scale_off(u.rows, u.cols, u.rcap)
            U = q * (base[so:so + u.rows] / 127.0).unsqueeze(1)
        else:
            U = base[uo:uo + u.rows * u.rcap].view(u.rows, u.rcap)[:, :count]
        return count, s, V, U, int(hdr[1])

    def write_unit(self, u, flat, mat):
        """Scatter a tall unit matrix into a flat fp32 array indexed like wshadow (physical order)."""
        q = self.plan.params[u.param]
        if u.kind == P.KIND_SLAB:
            o, i, kh, kw = q.shape
            logical = mat.reshape(o, i, kh, kw)
            flat[q.off:q.off + q.numel] = logical.permute(0, 2, 3, 1).reshape(-1)
        else:
            torch.as_strided(flat, (u.rows, u.cols), (u.rs, u.cs), u.w_off).copy_(mat)


class HE(LoopbackPS):
    """Entry-wise ATOMO; ``fill`` zeroes the params in ``zero`` and puts a few large entries into those in ``spike``."""

    PS = "v2_ps_entry"
    CODE = "entrywise"

    def __init__(self, shapes, budget=0.05, W=1, lr=0.1, momentum=0.0, wd=0.0, nesterov=False, opt=0, seed=7,
                 num_aggregate=0):
        super().__init__(shapes, self.CODE, W, lr, momentum, wd, nesterov, opt, seed, num_aggregate,
                         entry_budget=budget)
        self.budget = budget
        self.l1 = self.zeros(self.nc, torch.float64)
        self.partials = self.zeros(len(self.plan.enc_tiles), torch.float64)

    def tensor(self, q, x, g, zero=(), spike=()):
        if q.index in zero:
            x.zero_()
        if q.index in spike:
            x.view(-1)[::997] = 300.0
        return x

    def encode(self, w, uniforms=None):
        C, pl = self.C, self.plan
        gptr = self.gptr(w)
        t0, nt = pl.enc_range[0]
        C.v2_entry_stats(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr, self.partials.data_ptr(),
                         self.counters.data_ptr(), self.l1.data_ptr(), 0, 0)
        C.v2_entry_encode(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr, self.l1.data_ptr(),
                          self.t_arena_peer.data_ptr(), self.t_sig_peer.data_ptr(), 1, pl.arena_floats, w, 0,
                          self.ctrl.data_ptr(), self.counter(), uniforms.data_ptr() if uniforms is not None else 0, 0,
                          False)
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


# -------------------------------------------------------------------------------------------- Signum / Distributed Lion
# the 1728-element stem, 3x3 convs (one a multiple of the 4096-element tile, one with a half tile), fc layers, tensors
# whose size is not a multiple of 64 (or of 16), vectors, an all-zero tensor (ZERO), one with +0 / -0 / bf16 subnormals
# (SIGNED_ZERO) and one that gets a NaN (NAN)
SIGNUM_SHAPES = [(64, 3, 3, 3), (64,), (64, 32, 3, 3), (128, 64, 3, 3), (128,), (96, 64, 3, 3), (10, 512), (7, 20),
                 (5, 3), (10,), (32, 16, 3, 3), (40, 30), (48, 16, 3, 3)]
ZERO, SIGNED_ZERO, NAN = 10, 11, 12


class HSG(LoopbackPS):
    """Signum: per virtual worker a momentum buffer (beta > 0) and the coin's external uniforms."""

    PS = "v2_ps_signum"

    def __init__(self, shapes, W=1, beta=0.0, lr=0.0625, seed=7, num_aggregate=0, n_groups=1, n_owners=1):
        super().__init__(shapes, "signum", W, lr, 0.0, 0.0, False, 0, seed, num_aggregate, n_groups, n_owners)
        pl, z = self.plan, self.zeros
        self.beta = beta
        self.wmom = [z(pl.w_total) for _ in range(W)] if beta > 0 else None
        self.vmom_w = [z(pl.v_total) for _ in range(W)] if beta > 0 else None
        chunks, self.vec_range = P.vec_chunks(pl)
        self.t_vchunks = torch.frombuffer(bytearray(chunks or b"\0" * 24), dtype=torch.uint8).to(self.dev)
        g = torch.Generator(device="cuda").manual_seed(seed + 1)
        self.unif = [torch.rand(pl.w_total, device=self.dev, generator=g) for _ in range(W)]
        self.vext = torch.rand(W * pl.v_total, device=self.dev, generator=g)
        self.ps_tail = (self.vext.data_ptr(), pl.v_total)

    def tensor(self, q, x, g, special=False, who=0, negate=None):
        if special and q.index == ZERO:
            x.zero_()
        elif special and q.index == SIGNED_ZERO:
            r = torch.rand(q.shape, device=self.dev, generator=g)
            z = torch.zeros_like(x)
            x = torch.where(r < 0.3, z, torch.where(r < 0.6, -z, torch.where(r < 0.7, x.sign() * 1e-39, x)))
        if special and q.index == NAN and who == 0:
            x = physical(x)
            flat(x)[100] = float("nan")
        return x

    def encode(self, w, coin=False):
        C, pl = self.C, self.plan
        gptr = self.gptr(w)
        for g in range(pl.n_groups):
            t0, nt = pl.enc_range[g]
            v0, nv = self.vec_range[g]
            if self.beta == 0:
                nv = 0
            C.v2_signum_encode(self.t_units.data_ptr(), self.t_enc.data_ptr(), t0, nt, gptr,
                               self.t_vchunks.data_ptr() + 24 * v0, nv, self.vgrads[w].data_ptr(),
                               self.wmom[w].data_ptr() if self.wmom else 0,
                               self.vmom_w[w].data_ptr() if self.vmom_w else 0, self.beta,
                               self.t_arena_peer.data_ptr(), self.t_sig_peer.data_ptr(), self.n_owners,
                               pl.arena_floats, w, g, self.ctrl.data_ptr(), self.counter(g), 0,
                               g == pl.n_groups - 1, 0 if coin else self.unif[w].data_ptr())
        torch.cuda.synchronize()


class SignumOracle:
    """The fp32 numpy oracle of a HSG run: the workers' momenta, the pushed bits per tile, the owners' state."""

    def __init__(self, h):
        pl = self.plan = h.plan
        self.h = h
        self.u = [np.zeros(pl.w_total, np.float32) for _ in range(h.W)]
        self.uv = [np.zeros(pl.v_total, np.float32) for _ in range(h.W)]
        self.x, self.xv = [None] * h.W, [None] * h.W
        self.master = h.master.cpu().numpy().copy()
        self.vparams = h.vparams.cpu().numpy().copy()
        self.unif = [t.cpu().numpy() for t in h.unif]
        self.vext = h.vext.cpu().numpy().reshape(h.W, pl.v_total)

    def push(self, w, phys, coin=False):
        pl, beta = self.plan, self.h.beta
        x, xv = np.zeros(pl.w_total, np.float32), np.zeros(pl.v_total, np.float32)
        for q in pl.params:
            g = phys[q.index].cpu().numpy().astype(np.float32)
            sl = slice(q.off, q.off + q.numel)
            st, dst = (self.u[w], x) if q.is_w else (self.uv[w], xv)
            if beta > 0:
                st[sl] = S.momentum_step(st[sl], g, beta)
                dst[sl] = st[sl]
            else:
                dst[sl] = g
        self.x[w], self.xv[w] = x, xv
        if coin:
            self.unif[w] = np.zeros(pl.w_total, np.float32)
            for u in pl.units:
                if u.kind == P.KIND_SIGNUM:
                    self.unif[w][u.w_off:u.w_off + u.numel] = S.coin_uniforms(self.h.seed, u.index,
                                                                               np.arange(u.numel), self.h.step, w)

    def tile_bits(self, w, u, a, b):
        sl = slice(u.w_off + a, u.w_off + a + b)
        return S.bits(self.x[w][sl], self.unif[w][sl]), S.nonfinite(self.x[w][sl])

    def vec_bits(self, w, u, a, b, coin=False):
        sl = slice(u.w_off + a, u.w_off + a + b)
        un = S.coin_uniforms(self.h.seed, u.index, np.arange(a, a + b), self.h.step, w) if coin else self.vext[w][sl]
        return S.bits(self.xv[w][sl], un), S.nonfinite(self.xv[w][sl])

    def ps(self, counted, coin=False):
        pl, lr = self.plan, np.float32(self.h_lr())
        for (ui, a, b, o) in pl.ps_tiles:
            u = pl.units[ui]
            rows, bad = [], []
            for w in counted:
                r, nf = self.vec_bits(w, u, a, b, coin) if u.kind == P.KIND_VEC else self.tile_bits(w, u, a, b)
                rows.append(r)
                bad.append(nf)
            v = S.vote(rows, b, bad)
            dst = self.vparams if u.kind == P.KIND_VEC else self.master
            dst[u.w_off + a:u.w_off + a + b] = S.step(dst[u.w_off + a:u.w_off + a + b], v, lr)

    def h_lr(self):
        return float(self.h.ctrl.view(torch.float32)[2])


def signum_check_push(h, o, w):
    """Worker w's words, status words and stamps in the owners' arenas, and its momenta, against the oracle."""
    pl = h.plan
    arenas = [t.cpu().numpy() for t in h.arenas]
    for u in pl.units:
        if u.kind != P.KIND_SIGNUM:
            continue
        for j in range(u.n_ps):
            a, b = 4096 * j, min(4096, u.numel - 4096 * j)
            ar = arenas[(u.own0 + j) % h.n_owners]
            base = w * pl.arena_floats + u.slot_off
            bits, nf = o.tile_bits(w, u, a, b)
            wo = base + P.qsgd_words_off(u.n_ps, u.rows) + 2 * j * u.cols
            nw = -(-b // 64)
            got = ar[wo:wo + 2 * nw].view(np.uint64)
            assert np.array_equal(got, S.pack(bits)), (u.index, j, w)
            status = ar[base + P.qsgd_norms_off(u.n_ps) + j]
            assert (math.isnan(status) if nf else status == 0.0), (u.index, j, w, status)
            assert int(ar[base:base + u.n_ps].view(np.int32)[j]) == h.step
    if h.beta > 0:
        used = np.zeros(pl.w_total, bool)
        for q in pl.params:
            if q.is_w:
                used[q.off:q.off + q.numel] = True
        got = h.wmom[w].cpu().numpy()
        assert np.array_equal(got[used], o.u[w][used], equal_nan=True)
        assert np.array_equal(h.vmom_w[w].cpu().numpy(), o.uv[w], equal_nan=True)
    assert np.array_equal(h.vgrads[w].cpu().numpy(), o.xv[w], equal_nan=True)


def signum_check_ps(h, o):
    assert int(h.ctrl.view(torch.int32)[1]) == 0
    assert np.array_equal(h.master.cpu().numpy(), o.master, equal_nan=True)
    assert np.array_equal(h.vparams.cpu().numpy(), o.vparams, equal_nan=True)
    a, b = h.wshadow.float(), torch.from_numpy(o.master).cuda().bfloat16().float()
    assert torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num())


def opt_ref(p, g, m, s2, s2m, step, lr, momentum, nesterov, wd, opt):
    """One PS optimizer step in fp32 PyTorch: (new params, new momentum) for SGD (opt 0), Adam (1), AMSGrad (2)."""
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


# ---------------------------------------------------------------------------------------------------- fp32-flat engine
class Harness:
    """One rank that is both worker 0 and the PS (world == 1): peer pointers are local."""

    def __init__(self, shapes, code="svd", rank=3, systematic=False, lr=0.1, momentum=0.0, wd=0.0, nesterov=False,
                 seed=7):
        from atomo_b200.ops import plan as P
        from atomo_b200.runtime.flat import FlatLayout
        self.C, self.P = ext(), P
        dev = torch.device("cuda", 0)
        self.dev = dev
        self.layout = FlatLayout(shapes)
        self.plan = P.build_plan(shapes, code, rank, systematic, offsets=self.layout.offsets)
        pl = self.plan
        total = pl.total_elems
        u8 = lambda b: torch.frombuffer(bytearray(b if len(b) else b"\0" * 16), dtype=torch.uint8).to(dev)
        self.t_layers = u8(pl.layers_bytes())
        self.t_enc = u8(P.Plan.tiles_bytes(pl.enc_tiles))
        self.t_ps = u8(P.Plan.tiles_bytes(pl.ps_tiles))
        self.t_dense = u8(P.Plan.tiles_bytes(pl.dense_tiles))
        self.t_ts = torch.tensor(pl.ts_layers or [0], dtype=torch.int32, device=dev)
        n_ts = max(len(pl.ts_layers), 1)
        self.gpart = torch.zeros(pl.gpart_floats, device=dev)
        self.vsel = torch.zeros(n_ts * P.TS_MAX_COLS * P.RCAP_MAX, device=dev)
        self.selcount = torch.zeros(n_ts, dtype=torch.int32, device=dev)
        self.sigma = torch.zeros(n_ts * P.TS_MAX_COLS, device=dev)
        self.arena = torch.zeros(pl.arena_floats, device=dev)
        self.flags = torch.zeros(1024, dtype=torch.int32, device=dev)
        self.params = torch.randn(total, device=dev)
        self.grads = torch.zeros(total, device=dev)
        self.mom = torch.zeros(total, device=dev)
        self.ctrl = u8(P.pack_ctrl(step=1, lr=lr, momentum=momentum, weight_decay=wd, nesterov=nesterov, seed=seed))
        self.t_params_peer = torch.tensor([self.params.data_ptr()], dtype=torch.int64, device=dev)
        self.t_grads_peer = torch.tensor([self.grads.data_ptr()], dtype=torch.int64, device=dev)
        self.t_flag_peer = torch.tensor([self.flags.data_ptr() + 4 * 64], dtype=torch.int64, device=dev)
        self.rank_budget = rank
        self.systematic = systematic

    def set_step(self, step):
        self.ctrl.view(torch.int32)[0] = step

    def grad_views(self):
        return self.layout.views(self.grads)

    def encode(self, random_sample=True, waterfill=False, uniforms=None, rank=None):
        C, pl = self.C, self.plan
        C.gram(self.grads, self.t_layers, self.t_enc, len(pl.enc_tiles), self.gpart)
        C.eig_sample(self.t_layers, self.t_ts, self.gpart, self.vsel, self.selcount, self.sigma,
                     self.arena.data_ptr(), pl.arena_floats, self.ctrl, uniforms,
                     self.rank_budget if rank is None else rank, random_sample, waterfill, self.systematic, 0, 1024)
        C.project_push(self.grads, self.t_layers, self.t_enc, len(pl.enc_tiles), self.vsel, self.selcount,
                       self.arena.data_ptr(), pl.arena_floats, self.flags.data_ptr(), self.ctrl, 0, True)

    def ps_update(self):
        C, pl = self.C, self.plan
        C.ps_update(self.t_layers, self.t_ps, len(pl.ps_tiles), 1, 1, 1, self.params, self.mom, self.t_params_peer,
                    0, self.t_grads_peer, 0, self.arena.data_ptr(), pl.arena_floats, self.flags.data_ptr(),
                    self.t_flag_peer, self.ctrl, int(5e9), 1.0, min(len(pl.ps_tiles), 296))

    def slot(self, layer):
        P = self.P
        base = self.arena[layer.slot_off:]
        hdr = base[:4].view(torch.int32)
        count = int(hdr[0])
        rc, n = layer.rcap, layer.cols
        s = base[4:4 + rc][:count]
        V = base[4 + rc:4 + rc + rc * n].view(rc, n)[:count]
        uo = P.slot_u_off(rc, n)
        U = base[uo:uo + layer.rows * rc].view(layer.rows, rc)[:, :count]
        return count, s, V, U

    def tall(self, layer, flat):
        """tall (rows x cols) view of a layer inside a flat buffer"""
        t = flat[layer.off:layer.off + layer.numel]
        return torch.as_strided(t, (layer.rows, layer.cols), (layer.row_stride, layer.col_stride))


# ---------------------------------------------------------------------------------------------------- error feedback
# stem (MAT units), 3x3 convs (SLAB units; one a multiple of 4096 elements, one not), fc layers (MAT blocks), a tensor
# smaller than an absolute budget, a vector
SHAPES = [(64, 3, 3, 3), (64, 32, 3, 3), (128, 64, 3, 3), (10, 512), (300, 200), (7, 20), (32, 16, 3, 3), (64,)]


def ef_grads(seed=0):
    """bf16-representable gradients of SHAPES, scaled up tensor by tensor."""
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(s, generator=g) * (0.01 * (1 + i))).bfloat16().float().cuda() for i, s in enumerate(SHAPES)]


class Linear(nn.Module):
    """loss = sum_p <p, G_p>: the gradient of every parameter is G_p whatever the weights are."""

    def __init__(self, grads):
        super().__init__()
        self.ps = nn.ParameterList([nn.Parameter(torch.zeros(g.shape)) for g in grads])
        self.gs = grads

    def forward(self, x):
        s = sum((p.float() * g).sum() for p, g in zip(self.ps, self.gs))
        return s.reshape(1, 1).expand(x.shape[0], 2)


class Loopback:
    """One rank that is the only worker and the only owner, fed a fixed gradient.  With lr = 1, no momentum and the
    fp32 master zeroed before every step, the master after the step is minus what the owner reconstructed from this
    worker's slot: g_hat."""

    def __init__(self, code, grads, ef=True, **kw):
        from atomo_b200.runtime.shadow_engine import ShadowEngine
        torch.cuda.set_device(0)
        self.eng = ShadowEngine(Linear(grads), 0, 1, code=code, lr=1.0, momentum=0.0, use_graph=False, overlap=False,
                                warm_start=False, criterion=lambda lg, y: lg[0, 0], error_feedback=ef, seed=5, **kw)
        self.x, self.y = torch.zeros(4, 2), torch.zeros(4, dtype=torch.long)
        self.eng.prepare(self.x, self.y, warmup=0)
        self.eng.heap.tensor("arena").zero_()      # slot words no push writes compare equal across engines
        pl = self.eng.plan
        self.w = [q for q in pl.params if q.is_w]
        g = torch.zeros(pl.w_total, dtype=torch.float64, device="cuda")
        for q in self.w:
            t = grads[q.index].double()
            g[q.off:q.off + q.numel] = (t.permute(0, 2, 3, 1) if t.dim() == 4 else t).reshape(-1)
        self.g = g
        self.mask = torch.zeros(pl.w_total, dtype=torch.bool, device="cuda")
        for q in self.w:
            self.mask[q.off:q.off + q.numel] = True

    def residual(self):
        r = self.eng.residual
        return r.double().clone() if r is not None else torch.zeros_like(self.g)

    def step(self):
        """(g_hat, residual after the step), fp64, physical order (zero outside the weight tensors)."""
        self.eng.master.zero_()
        self.eng.train_step(self.x, self.y)
        torch.cuda.synchronize()
        assert self.eng.error_code() == 0
        return (-self.eng.master.double()) * self.mask, self.residual() * self.mask

    def close(self):
        self.eng.close()


# ---------------------------------------------------------------------------------------------------- engine
@pytest.fixture
def deterministic_cudnn(monkeypatch):
    """cuDNN with deterministic, heuristically chosen algorithms (as bench.py runs it) for one test."""
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)


_BATCHES = {}


def engine_batch(net, step, n=32, seed=0, period=4):
    """The device batch of training step `step`: n synthetic samples of `net`'s input shape drawn with seed
    ``seed + step % period``, the same tensors on every call.  Test files share the cache, so its key holds the seed."""
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import input_shape
    k = (net, seed, step % period, n)
    if k not in _BATCHES:
        x, y = SyntheticImageDataset(input_shape(net), 10, 4096, seed=seed + k[2]).materialize(n)
        _BATCHES[k] = (x.cuda(), y.cuda())
    return _BATCHES[k]


def make_engine(net="ResNet18", rank=0, world=1, seed=7, prepare_n=None, data_seed=0, **kw):
    """ShadowEngine(**kw) on device `rank` for ``build_model(net)`` drawn from torch seed 0.  With `prepare_n` it is
    prepared without warm-up on the step-0 `engine_batch` of prepare_n samples drawn from `data_seed`."""
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    torch.cuda.set_device(rank)
    eng = ShadowEngine(build_model(net, 10), rank, world, seed=seed, **kw)
    if prepare_n is not None:
        x, y = engine_batch(net, 0, prepare_n, data_seed)
        eng.prepare(x, y, warmup=0)
    return eng


def step(eng, batch, check=True):
    """One synchronized training step on `batch` (x, y); the loss.  With `check` the device error must be clear."""
    loss = eng.train_step(*batch)
    torch.cuda.synchronize()
    if check:
        assert eng.error_code() == 0
    return float(loss[0])


def state(eng, keys):
    """Copies of the engine tensors named in `keys`, skipping those the engine does not allocate."""
    return {k: getattr(eng, k).clone() for k in keys if getattr(eng, k, None) is not None}


def differs(a, b, keys=None):
    """The names among `keys` (default: all of a's, which must be b's) whose tensors are not bitwise equal."""
    if keys is None:
        assert a.keys() == b.keys()
        keys = a.keys()
    return [k for k in keys if not torch.equal(a[k], b[k])]


def batch(net, n=32, seed=0):
    """n synthetic samples of the input shape of `net`, in pinned memory."""
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import input_shape
    x, y = SyntheticImageDataset(input_shape(net), 10, 4096, seed=seed).materialize(n)
    return x.pin_memory(), y.pin_memory()


def train(net, graph, ef, steps=6, lr=0.05, seed=3, **code):
    """`steps` steps of the single-GPU engine on one fixed batch, graph replay and overlap both `graph`, error feedback
    `ef`: (fp32 master, losses, error-feedback norms).  `code` holds the code and its settings."""
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model, input_shape
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    x, y = SyntheticImageDataset(input_shape(net), 10, 4096, seed=0).materialize(32)
    eng = ShadowEngine(build_model(net, 10), 0, 1, lr=lr, momentum=0.9, use_graph=graph, overlap=graph, seed=seed,
                       error_feedback=ef, **code)
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


def model_shapes(net, dataset=""):
    from atomo_b200.models import build_model
    return [tuple(p.shape) for p in build_model(net, 10, dataset).parameters()]


MODELS = {"ResNet18": ("ResNet18", ""), "VGG11": ("VGG11", ""), "ResNet50-ImageNet": ("ResNet50", "ImageNet")}


# ---------------------------------------------------------------------------------------------------- multi GPU
def nccl_init(rank, world, port):
    """Join the NCCL process group of `world` local ranks on 127.0.0.1:`port` as `rank`, on device `rank`."""
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))


def spawn(world, target, *args, timeout=600):
    """Run ``target(rank, world, *args, out)`` in `world` spawned processes; each puts one result tuple that starts
    with its rank on the queue `out`.  The results are taken before the processes are joined (a full queue would
    keep a process from exiting) and returned sorted by rank; every process must exit with code 0."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    procs = [ctx.Process(target=target, args=(r, world, *args, out)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted((out.get(timeout=timeout) for _ in range(world)), key=lambda r: r[0])
    for p in procs:
        p.join(timeout)
        assert p.exitcode == 0
    return res


def mp_worker(rank, world, port, cfg, out):
    import torch.distributed as dist
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    nccl_init(rank, world, port)
    torch.manual_seed(0)
    net = cfg.get("net", "ResNet18")
    eng = ShadowEngine(build_model(net, 10), rank, world, code=cfg["code"], svd_rank=3, lr=0.05, momentum=0.9,
                       use_graph=cfg.get("graph", True), seed=5, ps_mode=cfg["ps_mode"], timeout_s=20.0,
                       debug_jitter_us=cfg.get("jitter_us", 0.0))
    x, y = batch(net, 32, seed=rank)
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


def run_mp(world, cfg, port):
    """`world` spawned ranks of ``mp_worker``; their result tuples sorted by rank."""
    return spawn(world, mp_worker, port, cfg, timeout=300)


# ---------------------------------------------------------------------------------------------------- launcher
SVD3 = ("--code", "svd", "--svd-rank", "3")     # launcher flags of spectral ATOMO at rank 3


def fit_args(tmp_path, *extra):
    """Launcher flags of a short synthetic LeNet / MNIST run writing to tmp_path, then `extra`."""
    from atomo_b200.utils.flags import add_fit_args
    return add_fit_args(argparse.ArgumentParser(), [
        "--network", "LeNet", "--dataset", "MNIST", "--synthetic", "1", "--train-len", "512", "--test-len", "128",
        "--batch-size", "32", "--test-batch-size", "64", "--lr", "0.05", "--log-interval", "1", "--eval-freq", "100",
        "--train-dir", str(tmp_path) + "/", *extra])



class StandInEngine:
    """Plain SGD on the CPU behind the engine interface the launcher uses.  Every instance is appended to `instances`,
    which a test clears before it runs the launcher; subclasses record what their test reads."""
    first_worker, W, is_worker, is_ps, is_owner = 0, 1, True, True, True
    instances = []

    def __init__(self, model, args):
        self.model, self.lr, self.step, self.args = model, args.lr, 1, args
        self.opt = torch.optim.SGD(model.parameters(), lr=args.lr)
        self.plan = types.SimpleNamespace(factor_bytes_per_worker=lambda: 1 << 20, dense_bytes=lambda: 1 << 18,
                                          expected_factor_bytes=lambda: 1 << 20)
        StandInEngine.instances.append(self)

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
        hit = out.argmax(1).eq(y).float().mean() * 100
        return torch.stack([loss.detach(), hit, hit])

    def phase_stats(self, reset=True):
        return {"param_wait_us": 10.0, "encode_us": 300.0, "to_push_us": 1500.0}

    def error_code(self):
        return 0

    def save_checkpoint(self, train_dir, step):
        pass

    def load_checkpoint(self, train_dir, step):
        pass

    def close(self):
        pass


def role_master(tmp_path, **kw):
    """The gloo role path's master (``SyncReplicasMaster_NN``) of a 2-process LeNet / MNIST run writing to tmp_path,
    with the settings `kw`, its model built from torch seed 0."""
    from atomo_b200.runtime import master as M
    m = M.SyncReplicasMaster_NN(types.SimpleNamespace(world_size=2), network="LeNet", dataset="MNIST",
                                train_dir=str(tmp_path) + "/", **kw)
    torch.manual_seed(0)
    return m.build_model(10)


def role_run(d, port, max_steps, *flags):
    """A 2-process gloo role-path run (``distributed_nn``) of synthetic LeNet / MNIST with the dense code, writing to
    d and evaluating every step, then `flags`; its stdout.  It must exit with code 0."""
    cmd = [sys.executable, "-m", "atomo_b200.distributed_nn", "--synthetic", "1", "--train-len", "512",
           "--test-len", "128", "--batch-size", "32", "--lr", "0.01", "--test-batch-size", "64", "--nproc", "2",
           "--network", "LeNet", "--dataset", "MNIST", "--code", "sgd", "--max-steps", str(max_steps), "--eval-freq",
           "1", "--train-dir", d, "--master-port", str(port), *flags]
    env = dict(os.environ, ATOMO_HANG_DUMP_S="400", PYTHONPATH=ROOT, OMP_NUM_THREADS="2", MKL_NUM_THREADS="2")
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=420)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout

def forbid_cuda(monkeypatch):
    """Make ShadowEngine fail on its first CUDA work, so a refusal is shown to come before any."""
    from atomo_b200.runtime import shadow_engine as S

    def no_cuda(*a, **k):
        raise AssertionError("refused only after CUDA work started")
    monkeypatch.setattr(S, "load_ext", no_cuda)

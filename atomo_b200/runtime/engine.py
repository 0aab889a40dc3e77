"""Fused H100 engine: the whole PS training step on NVLink peer memory.

Where the reference runs (SURVEY.md 3.2/3.3) ``Bcast(float64) x P -> fwd/bwd ->
host SVD x P -> pickle -> isend x P -> waitany -> np.dot decode -> SGD`` with
every tensor staged through host numpy, this engine keeps everything on the
GPUs and issues, per step and per rank, a fixed sequence of kernels that can be
captured in ONE CUDA graph:

  wait_params (spin on the step flag the PS wrote into our HBM)        [K9]
  -> forward / backward (PyTorch, parameters and gradients are views into
     flat buffers that live in the symmetric heap)
  -> encode + push: gram / eig_sample / project_push  (or qsgd / entry-wise);
     factors are stored straight into rank 0's arena through NVLink     [K1/K3/K5]
  -> rank 0 only: ps_update — wait for W push flags, low-rank reconstruct or
     NVLS in-switch dense reduce, momentum-SGD, multicast the new
     parameters to every rank, raise the step flags                     [K2/K7/K8]
  -> advance the device-side step counter.

Cross-GPU ordering is carried entirely by step-stamped flags in peer memory, so
no host synchronisation, NCCL call or MPI-style handshake sits on the path.
Rank 0 hosts the PS and (``ps_mode='colocated'``, default) also trains; with
``ps_mode='dedicated'`` it only serves, like the reference's rank 0.
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F

from ..ops import plan as P
from ..ops._ext import load as load_ext
from ..parallel.symm import SymmetricHeap
from .flat import bind_gradients, bind_parameters, FlatLayout

SIGNAL_INTS = 1024
PARAM_FLAG_SLOT = 64  # index of the param flag inside the signal region


def _dev_bytes(b: bytes, device) -> torch.Tensor:
    t = torch.frombuffer(bytearray(b if len(b) else b"\0" * 16), dtype=torch.uint8)
    return t.to(device)


class FusedEngine:
    def __init__(self, model: nn.Module, rank: int = 0, world: int = 1, code: str = "svd", svd_rank: int = 3,
                 lr: float = 0.01, momentum: float = 0.0, weight_decay: float = 0.0, nesterov: bool = False,
                 dampening: float = 0.0, ps_mode: str = "colocated", sampling: str = "bernoulli",
                 prob_rule: str = "reference", random_sample: bool = True, seed: int = 1,
                 quantization_level: int = 4, bucket_size: int = 512, entry_budget: float = 0.05,
                 dtype: str = "fp32", channels_last: bool = False, use_graph: bool = True, group=None,
                 multicast: bool = True, heap_mode: str = "auto", timeout_s: float = 30.0,
                 criterion: Optional[nn.Module] = None, device: Optional[torch.device] = None,
                 subspace="auto", power_iters: int = 0, gemm_impl: str = "auto", fused_bn="auto"):
        self.C = load_ext()
        self.rank, self.world, self.group = rank, world, group
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        self.code = code.lower()
        if self.code in ("dense", "lossless"):
            self.code = "sgd"
        self.svd_rank = int(svd_rank)
        self.ps_mode = ps_mode if world > 1 else "colocated"
        self.first_worker = 0 if self.ps_mode == "colocated" else 1
        self.W = world - self.first_worker
        self.is_ps = rank == 0
        self.is_worker = rank >= self.first_worker
        self.worker_index = rank - self.first_worker
        self.systematic = sampling == "systematic"
        self.waterfill = prob_rule == "waterfill"
        self.random_sample = random_sample
        self.q, self.bucket = int(quantization_level), int(bucket_size)
        self.entry_budget = float(entry_budget)
        self.autocast = dtype == "bf16"
        self.channels_last = channels_last
        self.use_graph = use_graph
        self.criterion = criterion or nn.CrossEntropyLoss()
        self.timeout_ticks = int(timeout_s * 1.5e9)
        self.step = 1
        self.lr = lr
        self.model = model.to(self.device)
        self.launches_per_step = 0
        self.nvtx = bool(os.environ.get("ATOMO_NVTX"))   # NVTX ranges around the phases (eager mode)

        # ---- plan + symmetric heap -----------------------------------------------------------
        self.layout = FlatLayout.from_module(self.model)
        shapes = self.layout.shapes
        plan_code = self.code if self.code == "svd" else "sgd"
        self.plan = P.build_plan(shapes, plan_code, self.svd_rank, self.systematic, offsets=self.layout.offsets,
                                 subspace=bool(subspace))
        if subspace == "auto" and self.plan.ext is not None:
            # the range-finder pipeline is ~10 small dependent launches: only worth it when the square-ish
            # layers hold a real share of the model (ResNet-50 1x1 convs, fc-heavy nets), not ResNet-18's 1.5%
            ext_elems = sum(l.numel for l in self.plan.ext.layers)
            if ext_elems < 0.05 * self.layout.total:
                self.plan = P.build_plan(shapes, plan_code, self.svd_rank, self.systematic,
                                         offsets=self.layout.offsets, subspace=False)
        self.power_iters = int(power_iters)
        self.gemm_impl = gemm_impl
        assert self.plan.total_elems == self.layout.total
        total = self.plan.total_elems
        nb = (total + self.bucket - 1) // self.bucket
        E = 64 // (2 + self.q)
        self.q_words = (self.bucket + E - 1) // E
        exp_atoms = self._entry_expected(total)
        self.ew_capacity = int(exp_atoms * 1.25) + 4096
        need = 4 * SIGNAL_INTS + 2 * 4 * total + 4096
        if self.code == "svd":
            need += 4 * self.plan.arena_floats * self.W
        elif self.code in ("qsgd", "terngrad"):
            need += self.W * (8 * nb * self.q_words + 4 * nb + 512)
        elif self.code == "entrywise":
            need += self.W * (8 * self.ew_capacity + 1024)
        self.heap = SymmetricHeap(need + (1 << 20), rank, world, self.device.index, group=group,
                                  multicast=multicast, mode=heap_mode)
        h = self.heap
        h.alloc("signals", 4 * SIGNAL_INTS)
        h.alloc("params", 4 * total)
        h.alloc("grads", 4 * total)
        if self.code == "svd":
            h.alloc("arena", 4 * self.plan.arena_floats * self.W)
        elif self.code in ("qsgd", "terngrad"):
            h.alloc("qwords", 8 * nb * self.q_words * self.W)
            h.alloc("qnorms", 4 * nb * self.W)
        elif self.code == "entrywise":
            h.alloc("ew_idx", 4 * self.ew_capacity * self.W)
            h.alloc("ew_val", 4 * self.ew_capacity * self.W)
            h.alloc("ew_cnt", 256 * self.W)
        self.nbuckets = nb

        self.flat_params = h.tensor("params")
        self.flat_grads = h.tensor("grads")
        self.signals = h.tensor("signals", torch.int32)
        bind_parameters(self.model, self.flat_params, self.layout)
        self.grad_views = bind_gradients(self.model, self.flat_grads, self.layout)
        if fused_bn == "auto":
            fused_bn = self.autocast and channels_last
        if fused_bn:
            from ..ops.fused_bn import enable_fused_bn
            self.fused_bn_layers, self.bn_arena = enable_fused_bn(self.model, True, arena_device=self.device)
        else:
            self.fused_bn_layers, self.bn_arena = 0, None
        if channels_last:
            self.model = self.model.to(memory_format=torch.channels_last)  # activations only; weights stay flat views
            bind_parameters(self.model, self.flat_params, self.layout)
        if self.fused_bn_layers:
            # the fused BN backward writes dgamma / dbeta straight into the flat gradient buffer (the views that
            # are these parameters' .grad): no AccumulateGrad add kernels for the 2 x #BN vectors
            from ..ops.fused_bn import BNAct
            for m in self.model.modules():
                if isinstance(m, BNAct) and m.fused and m.weight is not None:
                    m._grad_sink = (m.weight.grad, m.bias.grad)

        # ---- device tables --------------------------------------------------------------------
        dev = self.device
        self.t_layers = _dev_bytes(self.plan.layers_bytes(), dev)
        self.t_enc_tiles = _dev_bytes(P.Plan.tiles_bytes(self.plan.enc_tiles), dev)
        self.t_ps_tiles = _dev_bytes(P.Plan.tiles_bytes(self.plan.ps_tiles), dev)
        self.t_dense_tiles = _dev_bytes(P.Plan.tiles_bytes(self.plan.dense_tiles), dev)
        self.t_ts_layers = torch.tensor(self.plan.ts_layers or [0], dtype=torch.int32, device=dev)
        n_ts = max(len(self.plan.ts_layers), 1)
        self.gpart = torch.zeros(self.plan.gpart_floats, dtype=torch.float32, device=dev)
        self.vsel = torch.zeros(n_ts * P.TS_MAX_COLS * P.RCAP_MAX, dtype=torch.float32, device=dev)
        self.selcount = torch.zeros(n_ts, dtype=torch.int32, device=dev)
        self.sigma = torch.zeros(n_ts * P.TS_MAX_COLS, dtype=torch.float32, device=dev)
        self.ctrl = _dev_bytes(P.pack_ctrl(step=1, lr=lr, momentum=momentum, dampening=dampening,
                                           weight_decay=weight_decay, nesterov=nesterov, first_step=1, seed=seed), dev)
        self.ctrl_i32 = self.ctrl.view(torch.int32)
        self.ctrl_f32 = self.ctrl.view(torch.float32)
        ranks = list(range(world))
        workers = list(range(self.first_worker, world))
        self.t_params_peer = torch.tensor([h.region_ptr("params", r) for r in ranks], dtype=torch.int64, device=dev)
        self.t_grads_peer = torch.tensor([h.region_ptr("grads", r) for r in workers], dtype=torch.int64, device=dev)
        self.t_flag_peer = torch.tensor([h.region_ptr("signals", r) + 4 * PARAM_FLAG_SLOT for r in ranks],
                                        dtype=torch.int64, device=dev)
        self.params_mc = h.region_mc_ptr("params")
        self.grads_mc = h.region_mc_ptr("grads")
        self.ps_push_flags = h.region_ptr("signals", 0)           # on the PS
        self.local_param_flag = h.region_ptr("signals") + 4 * PARAM_FLAG_SLOT
        if self.is_ps:
            self.momentum_buf = torch.zeros(total, dtype=torch.float32, device=dev)
        if self.code in ("qsgd", "terngrad", "entrywise"):
            self.dense_plan = P.dense_only_plan(shapes, offsets=self.layout.offsets)
            self.t_dense_layers = _dev_bytes(self.dense_plan.layers_bytes(), dev)
            self.t_dense_ps_tiles = _dev_bytes(P.Plan.tiles_bytes(self.dense_plan.ps_tiles), dev)
            if self.is_ps:
                self.out_sum = torch.zeros(total, dtype=torch.float32, device=dev)
                self.t_out_sum_ptr = torch.tensor([self.out_sum.data_ptr()], dtype=torch.int64, device=dev)
        if self.code in ("qsgd", "terngrad") and self.is_ps:
            wb, nbs = h.region_ptr("qwords", 0), h.region_ptr("qnorms", 0)
            self.t_qwords = torch.tensor([wb + 8 * nb * self.q_words * w for w in range(self.W)], dtype=torch.int64, device=dev)
            self.t_qnorms = torch.tensor([nbs + 4 * nb * w for w in range(self.W)], dtype=torch.int64, device=dev)
        if self.code == "terngrad":
            self.clip = torch.zeros(1, dtype=torch.float32, device=dev)
        if self.code == "entrywise":
            self.l1 = torch.zeros(len(shapes), dtype=torch.float32, device=dev)
            self.ew_local_count = torch.zeros(1, dtype=torch.int32, device=dev)
            if self.is_ps:
                ib, vb, cb = (h.region_ptr(n, 0) for n in ("ew_idx", "ew_val", "ew_cnt"))
                self.t_ew_idx = torch.tensor([ib + 4 * self.ew_capacity * w for w in range(self.W)], dtype=torch.int64, device=dev)
                self.t_ew_val = torch.tensor([vb + 4 * self.ew_capacity * w for w in range(self.W)], dtype=torch.int64, device=dev)
                self.t_ew_cnt = torch.tensor([cb + 256 * w for w in range(self.W)], dtype=torch.int64, device=dev)
        if self.plan.ext is not None:
            self._setup_ext()
        sm = torch.cuda.get_device_properties(dev).multi_processor_count
        self.ps_grid = min(len(self.plan.ps_tiles), sm * 3)
        max_cols = max([l.cols for l in self.plan.layers if l.route == P.ROUTE_SVD_TS] or [0])
        self.eig_threads = 1024 if max_cols > 32 else 256

        # ---- metrics + static batch ----------------------------------------------------------
        self.loss_buf = torch.zeros(3, dtype=torch.float32, device=dev)  # loss, prec1, prec5
        # device-side phase accounting (globaltimer ns): [0] PS wait-for-pushes, [1] PS work, [2] PS steps,
        # [3] wait-for-params, [4] steps
        self.tstats = torch.zeros(8, dtype=torch.int64, device=dev)
        self.static_x = None
        self.static_y = None
        self.graph = None

        self._initial_sync()

    # ------------------------------------------------------------------------------------------
    def _aux_tables(self, aux):
        dev = self.device
        n_ts = max(len(aux.ts_layers), 1)
        return {
            "plan": aux, "layers": _dev_bytes(aux.layers_bytes(), dev),
            "tiles": _dev_bytes(P.Plan.tiles_bytes(aux.enc_tiles), dev),
            "ts": torch.tensor(aux.ts_layers or [0], dtype=torch.int32, device=dev),
            "gpart": torch.zeros(aux.gpart_floats, dtype=torch.float32, device=dev),
            "vsel": torch.zeros(n_ts * P.TS_MAX_COLS * P.RCAP_MAX, dtype=torch.float32, device=dev),
            "selcount": torch.zeros(n_ts, dtype=torch.int32, device=dev),
            "arena": torch.zeros(aux.arena_floats, dtype=torch.float32, device=dev),
        }

    def _setup_ext(self):
        """Scratch + auxiliary tables of the subspace-iteration route (square-ish layers)."""
        ext, dev = self.plan.ext, self.device
        self.ext_scratch = torch.zeros(ext.scratch_floats, dtype=torch.float32, device=dev)
        self.aux_y = self._aux_tables(ext.aux_y)
        self.aux_b = self._aux_tables(ext.aux_b)
        self.t_ext_descs = _dev_bytes(ext.descs_bytes(), dev)
        self.t_fin_tiles = _dev_bytes(P.Plan.tiles_bytes(ext.fin_tiles), dev)
        assert self.C.ext_desc_bytes() == P.EXT_BYTES
        self.ext_views = []
        for l, d, ly in zip(ext.layers, ext.descs, ext.aux_y.layers):
            a_off, xt_off, y_off, b_off, qslot_off = d[0], d[1], d[2], d[3], d[4]
            sk = l.sketch
            A = torch.as_strided(self.flat_grads, (l.rows, l.cols), (l.row_stride, l.col_stride), a_off)
            Xt = self.ext_scratch[xt_off:xt_off + sk * l.cols].view(sk, l.cols)
            Y = self.ext_scratch[y_off:y_off + l.rows * sk].view(l.rows, sk)
            B = self.ext_scratch[b_off:b_off + l.cols * sk].view(l.cols, sk)
            qo = qslot_off + P.slot_u_off(sk, sk)
            Q = self.aux_y["arena"][qo:qo + l.rows * sk].view(l.rows, sk)
            self.ext_views.append((A, Xt, Y, B, Q))
        if self.gemm_impl == "auto":
            self.gemm_impl = "wgmma"
        if self.gemm_impl == "wgmma":
            self._setup_gemm_tiles()

    def _setup_gemm_tiles(self):
        """Tile tables of the grouped wgmma skinny GEMMs (csrc/gemm_kernels.cu: struct GemmTile)."""
        import struct
        assert self.C.gemm_tile_bytes() == 72
        gp = self.flat_grads.data_ptr()
        sm = torch.cuda.get_device_properties(self.device).multi_processor_count

        def vec_mode(base_elems, sa_i, sa_k):
            if sa_k == 1 and sa_i % 4 == 0 and base_elems % 4 == 0:
                return 1
            if sa_i == 1 and sa_k % 4 == 0 and base_elems % 4 == 0:
                return 2
            return 0

        def tile(A_ptr, B_ptr, C_ptr, sa_i, sa_k, sb_j, sb_k, ldc, M, N, K, av, kb=0, klen=0, atomic=0):
            return struct.pack("<3Q12i", A_ptr, B_ptr, C_ptr, sa_i, sa_k, sb_j, sb_k, ldc, M, N, K, av, kb, klen,
                               atomic)

        def ksplits(ntiles, K):
            """split the reduction so that a handful of output tiles still fills every SM (two CTAs each)"""
            want = -(-2 * sm // max(ntiles, 1))
            return max(1, min(want, K // 128))

        layers = self.plan.ext.layers
        n_f = sum(-(-l.rows // 128) for l in layers)
        n_b = sum(-(-l.cols // 128) for l in layers)
        fwd_x, fwd_b, bwd = [], [], []
        self.gemm_fwd_atomic = self.gemm_bwd_atomic = False
        for l, (A, Xt, Y, B, Q) in zip(layers, self.ext_views):
            sk, m, n, rs, cs = l.sketch, l.rows, l.cols, l.row_stride, l.col_stride
            sf, sb = ksplits(n_f, n), ksplits(n_b, m)
            klen_f = -(-(-(-n // sf)) // 32) * 32
            klen_b = -(-(-(-m // sb)) // 32) * 32
            for r0 in range(0, m, 128):      # Y[r0:r0+128] = A[r0:r0+128, :] @ X
                base = l.off + r0 * rs
                av = vec_mode(base, rs, cs)
                for kb in range(0, n, klen_f):
                    at = int(sf > 1)
                    self.gemm_fwd_atomic |= bool(at)
                    fwd_x.append(tile(gp + 4 * base, Xt.data_ptr(), Y.data_ptr() + 4 * r0 * sk, rs, cs, n, 1, sk,
                                      min(128, m - r0), sk, n, av, kb, klen_f, at))
                    # power iteration: X is the (n x l) buffer B
                    fwd_b.append(tile(gp + 4 * base, B.data_ptr(), Y.data_ptr() + 4 * r0 * sk, rs, cs, 1, sk, sk,
                                      min(128, m - r0), sk, n, av, kb, klen_f, at))
            for c0 in range(0, n, 128):      # B[c0:c0+128] = A[:, c0:c0+128]^T @ Q
                base = l.off + c0 * cs
                for kb in range(0, m, klen_b):
                    at = int(sb > 1)
                    self.gemm_bwd_atomic |= bool(at)
                    bwd.append(tile(gp + 4 * base, Q.data_ptr(), B.data_ptr() + 4 * c0 * sk, cs, rs, 1, sk, sk,
                                    min(128, n - c0), sk, m, vec_mode(base, cs, rs), kb, klen_b, at))
        self.n_fwd_tiles, self.n_bwd_tiles = len(fwd_x), len(bwd)
        self.t_gemm_fwd_x = _dev_bytes(b"".join(fwd_x), self.device)
        self.t_gemm_fwd_b = _dev_bytes(b"".join(fwd_b), self.device)
        self.t_gemm_bwd = _dev_bytes(b"".join(bwd), self.device)
        self.gemm_grid = torch.cuda.get_device_properties(self.device).multi_processor_count * 2
        ext = self.plan.ext
        self.ext_y_all = self.ext_scratch[ext.y_range[0]:ext.y_range[1]]
        self.ext_b_all = self.ext_scratch[ext.b_range[0]:ext.b_range[1]]

    def _gemm_fwd(self, from_b: bool = False):
        if self.gemm_impl == "wgmma":
            if self.gemm_fwd_atomic:
                self.ext_y_all.zero_()   # split-K partial sums are accumulated with atomics
            self.C.skinny_gemm(self.t_gemm_fwd_b if from_b else self.t_gemm_fwd_x, self.n_fwd_tiles, self.ctrl,
                               self.gemm_grid)
            return 1
        for A, Xt, Y, B, Q in self.ext_views:
            torch.mm(A, B if from_b else Xt.t(), out=Y)
        return 0

    def _gemm_bwd(self):
        if self.gemm_impl == "wgmma":
            if self.gemm_bwd_atomic:
                self.ext_b_all.zero_()
            self.C.skinny_gemm(self.t_gemm_bwd, self.n_bwd_tiles, self.ctrl, self.gemm_grid)
            return 1
        for A, Xt, Y, B, Q in self.ext_views:
            torch.mm(A.t(), Q, out=B)
        return 0

    def _aux_factorize(self, aux, rank, random_sample, signal_worker):
        """gram -> eig_sample -> project on an auxiliary tall-skinny plan (local arena)."""
        C, pl = self.C, aux["plan"]
        C.gram(self.ext_scratch, aux["layers"], aux["tiles"], len(pl.enc_tiles), aux["gpart"])
        C.eig_sample(aux["layers"], aux["ts"], aux["gpart"], aux["vsel"], aux["selcount"], None,
                     aux["arena"].data_ptr(), 0, self.ctrl, None, rank, random_sample, self.waterfill,
                     self.systematic, signal_worker, 256)
        C.project_push(self.ext_scratch, aux["layers"], aux["tiles"], len(pl.enc_tiles), aux["vsel"],
                       aux["selcount"], aux["arena"].data_ptr(), 0, self.ps_push_flags, self.ctrl, 0, False)
        return 3

    def _encode_ext(self):
        """Randomized range finder + ATOMO sampling for the square-ish layers; factors land in the PS slot."""
        ext = self.plan.ext
        n = 0
        xr = ext.xt_range
        self.ext_scratch[xr[0]:xr[1]].normal_()          # fresh Gaussian test matrices X for every layer
        n += self._gemm_fwd()                            # Y = A X            (wgmma skinny GEMM)
        sk = ext.layers[0].sketch
        n += self._aux_factorize(self.aux_y, sk, False, 0)       # Q = orth(Y)
        for _ in range(self.power_iters):                # optional power iterations: Y = A (A^T Q)
            n += self._gemm_bwd()
            n += self._gemm_fwd(from_b=True)
            n += self._aux_factorize(self.aux_y, sk, False, 0)
        n += self._gemm_bwd()                            # B = A^T Q          (wgmma skinny GEMM)
        n += self._aux_factorize(self.aux_b, self.svd_rank, self.random_sample, self.worker_index)
        self.C.ext_finalize(self.t_ext_descs, self.t_fin_tiles, len(ext.fin_tiles), self.aux_y["arena"],
                            self.aux_b["arena"], self.heap.region_ptr("arena", 0), self.plan.arena_floats,
                            self.ctrl, self.worker_index)
        return n + 1

    def _entry_expected(self, total: int) -> float:
        b = self.entry_budget
        return b * total if b < 1.0 else b * len(self.layout.shapes)

    def _barrier(self):
        torch.cuda.synchronize(self.device)
        if self.world > 1:
            dist.barrier(group=self.group)

    def _initial_sync(self):
        """K8: every rank starts from rank 0's parameters; flags say 'step 1 ready'."""
        self._barrier()
        if self.is_ps and self.world > 1:
            self.C.param_bcast(self.flat_params, self.t_params_peer, self.params_mc, self.world, self.rank,
                               self.plan.total_elems)
        self._barrier()
        self.signals.zero_()
        self.signals[PARAM_FLAG_SLOT] = 1
        self._barrier()

    def set_lr(self, lr: float):
        self.lr = lr
        self.ctrl_f32[2] = lr  # Ctrl::lr (device write ordered on the stream)

    def phase_stats(self, reset: bool = True) -> dict:
        """Average device-side microseconds per step since the last reset."""
        t = self.tstats.tolist()
        out = {"param_wait_us": t[3] / max(t[4], 1) / 1e3}
        if self.is_ps:
            out["ps_wait_push_us"] = t[0] / max(t[2], 1) / 1e3
            out["ps_work_us"] = t[1] / max(t[2], 1) / 1e3
        if reset:
            self.tstats.zero_()
        return out

    def error_code(self) -> int:
        return int(self.ctrl_i32[1].item())

    def device_step(self) -> int:
        return int(self.ctrl_i32[0].item())

    # ------------------------------------------------------------------------------------------
    def _forward_backward(self):
        x, y = self.static_x, self.static_y
        if self.autocast:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                logits = self.model(x)
                loss = self.criterion(logits.float(), y)
        else:
            logits = self.model(x)
            loss = self.criterion(logits, y)
        loss.backward()
        with torch.no_grad():
            lg = logits.detach().float()
            k = min(5, lg.size(1))
            top = lg.topk(k, 1).indices
            hit = top.eq(y.view(-1, 1))
            self.loss_buf[0] = loss.detach()
            self.loss_buf[1] = hit[:, :1].float().sum() * (100.0 / y.numel())
            self.loss_buf[2] = hit.float().sum() * (100.0 / y.numel())

    def _encode_push(self):
        C, pl = self.C, self.plan
        n = 0
        if self.code == "svd":
            arena0 = self.heap.region_ptr("arena", 0)
            if pl.ext is not None:
                n += self._encode_ext()
            if pl.enc_tiles:
                C.gram(self.flat_grads, self.t_layers, self.t_enc_tiles, len(pl.enc_tiles), self.gpart)
                C.eig_sample(self.t_layers, self.t_ts_layers, self.gpart, self.vsel, self.selcount, self.sigma,
                             arena0, pl.arena_floats, self.ctrl, None, self.svd_rank, self.random_sample,
                             self.waterfill, self.systematic, self.worker_index, self.eig_threads)
                n += 2
            C.project_push(self.flat_grads, self.t_layers, self.t_enc_tiles, len(pl.enc_tiles), self.vsel,
                           self.selcount, arena0, pl.arena_floats, self.ps_push_flags, self.ctrl,
                           self.worker_index, True)
            n += 1
        elif self.code == "sgd":
            C.signal_push(self.ps_push_flags, self.ctrl, self.worker_index)
            n += 1
        elif self.code in ("qsgd", "terngrad"):
            total, nb = pl.total_elems, self.nbuckets
            tern = self.code == "terngrad"
            clip = None
            if tern:
                self.clip.copy_((2.5 * self.flat_grads.std(unbiased=False)).reshape(1))
                clip = self.clip
            wout = self.heap.region_ptr("qwords", 0) + 8 * nb * self.q_words * self.worker_index
            nout = self.heap.region_ptr("qnorms", 0) + 4 * nb * self.worker_index
            C.qsgd_encode(self.flat_grads, total, self.bucket, self.q, tern, clip, wout, nout, self.ctrl,
                          self.worker_index, None)
            C.signal_push(self.ps_push_flags, self.ctrl, self.worker_index)
            n += 2
        elif self.code == "entrywise":
            w = self.worker_index
            C.entrywise_encode(self.flat_grads, self.t_layers, self.t_dense_tiles, len(pl.dense_tiles), self.l1,
                               self.entry_budget, self.heap.region_ptr("ew_idx", 0) + 4 * self.ew_capacity * w,
                               self.heap.region_ptr("ew_val", 0) + 4 * self.ew_capacity * w,
                               self.heap.region_ptr("ew_cnt", 0) + 256 * w, self.ew_capacity, self.ew_local_count,
                               self.ps_push_flags, self.ctrl, w, None, True)
            n += 2
        else:
            raise ValueError("unsupported --code for the fused engine: %s" % self.code)
        return n

    def _ps_update(self):
        C, pl = self.C, self.plan
        n = 0
        if self.code in ("svd", "sgd"):
            arenas = self.heap.region_ptr("arena", 0) if self.code == "svd" else 0
            C.ps_update(self.t_layers, self.t_ps_tiles, len(pl.ps_tiles), self.W, self.W, self.world,
                        self.flat_params, self.momentum_buf, self.t_params_peer, self.params_mc, self.t_grads_peer,
                        self.grads_mc, arenas, pl.arena_floats, self.ps_push_flags, self.t_flag_peer, self.ctrl,
                        self.timeout_ticks, 1.0 / self.W, self.ps_grid, self.tstats.data_ptr())
            return 1
        if self.code in ("qsgd", "terngrad"):
            C.qsgd_decode_sum(self.t_qwords, self.t_qnorms, self.W, pl.total_elems, self.bucket, self.q,
                              self.code == "terngrad", self.out_sum, self.ps_push_flags, self.ctrl,
                              self.timeout_ticks)
            n += 1
        elif self.code == "entrywise":
            C.entrywise_scatter(self.t_ew_idx, self.t_ew_val, self.t_ew_cnt, self.W, self.ew_capacity, self.out_sum,
                                pl.total_elems, self.ps_push_flags, self.ctrl, self.timeout_ticks)
            n += 1
        dp = self.dense_plan
        C.ps_update(self.t_dense_layers, self.t_dense_ps_tiles, len(dp.ps_tiles), 1, 0, self.world,
                    self.flat_params, self.momentum_buf, self.t_params_peer, self.params_mc, self.t_out_sum_ptr, 0,
                    0, dp.arena_floats, self.ps_push_flags, self.t_flag_peer, self.ctrl, self.timeout_ticks,
                    1.0 / self.W, min(len(dp.ps_tiles), self.ps_grid), self.tstats.data_ptr())
        return n + 1

    def _step_body(self):
        """One full step on the current stream (capturable)."""
        C = self.C
        n = 0
        nvtx = self.nvtx and not torch.cuda.is_current_stream_capturing()
        C.wait_params(self.local_param_flag, self.ctrl, self.timeout_ticks, self.tstats.data_ptr()); n += 1
        if self.is_worker:
            self.flat_grads.zero_()
            if self.bn_arena is not None:
                self.bn_arena.zero_()          # per-channel accumulators of every fused BN layer
            if nvtx:
                torch.cuda.nvtx.range_push("fwd_bwd")
            self._forward_backward()
            n += 4 * self.fused_bn_layers      # stats + apply, backward reduce + apply (csrc/bn_kernels.cu)
            if nvtx:
                torch.cuda.nvtx.range_pop()
                torch.cuda.nvtx.range_push("encode_push")
            n += self._encode_push()
            if nvtx:
                torch.cuda.nvtx.range_pop()
        if self.is_ps:
            if nvtx:
                torch.cuda.nvtx.range_push("ps_update")
            n += self._ps_update()
            if nvtx:
                torch.cuda.nvtx.range_pop()
        C.advance_step(self.ctrl); n += 1
        self.launches_per_step = n

    # ------------------------------------------------------------------------------------------
    def prepare(self, x_example: torch.Tensor, y_example: torch.Tensor, warmup: int = 3):
        """Allocate static inputs, warm up eagerly, then capture the step in a CUDA graph."""
        self.static_x = torch.empty_like(x_example, device=self.device)
        if self.channels_last and self.static_x.dim() == 4:
            self.static_x = self.static_x.contiguous(memory_format=torch.channels_last)
        self.static_y = torch.empty_like(y_example, device=self.device)
        self.static_x.copy_(x_example)
        self.static_y.copy_(y_example)
        self.model.train()
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            for _ in range(warmup):
                self._step_body()
                self.step += 1
        torch.cuda.current_stream(self.device).wait_stream(s)
        torch.cuda.synchronize(self.device)
        if self.use_graph:
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._step_body()
            # capture does not execute: the device step counter is unchanged
        return self

    def train_step(self, x: Optional[torch.Tensor] = None, y: Optional[torch.Tensor] = None):
        """Run one step.  ``x``/``y`` may live in pinned host memory (async H2D)."""
        if x is not None and self.is_worker:
            self.static_x.copy_(x, non_blocking=True)
            self.static_y.copy_(y, non_blocking=True)
        if self.graph is not None:
            self.graph.replay()
        else:
            self._step_body()
        self.step += 1
        return self.loss_buf

    # ------------------------------------------------------------------------------------------
    # checkpoint / resume (SURVEY 5.4: same `model_step_<N>` file for the evaluator + an `_optim` sidecar)
    def save_checkpoint(self, train_dir: str, step: Optional[int] = None) -> Optional[str]:
        """Call on every rank.  The FIRST TRAINING rank writes the model file the polling evaluator consumes: its
        parameters are the PS's (multicast every step) and its BatchNorm running statistics are real — a PS that
        never runs a forward pass (``ps_mode='dedicated'``) would save untrained BN buffers, which is why the
        reference kept PS checkpointing off for ResNet (sync_replicas_master_nn.py:228-230).  The PS rank writes the
        ``_optim`` sidecar (momentum, step, LR, RNG seed) so a later run can resume exactly."""
        from ..utils import checkpoint as ckpt
        step = (self.step - 1) if step is None else step
        torch.cuda.synchronize(self.device)
        path = None
        if self.rank == self.first_worker:
            path = ckpt.save_model(train_dir, step, self.model)
        if self.is_ps:
            side_path = ckpt.model_path(train_dir, step) + "_optim"
            os.makedirs(os.path.dirname(side_path) or ".", exist_ok=True)
            side = {"step": step, "lr": self.lr, "momentum_buffer": self.momentum_buf.detach().cpu(),
                    "ctrl": bytes(self.ctrl.cpu().numpy().tobytes()), "code": self.code, "svd_rank": self.svd_rank}
            torch.save(side, side_path + ".tmp")
            os.replace(side_path + ".tmp", side_path)
        return path

    def load_checkpoint(self, train_dir: str, step: int) -> None:
        """Collective: every rank calls this with the same ``step``.  Rank 0 restores model + momentum from
        disk, the parameters are re-broadcast over the heap and every rank's device step / flags jump to
        ``step + 1``."""
        from ..utils import checkpoint as ckpt
        self._barrier()
        if self.is_ps:
            ckpt.load_model(train_dir, step, self.model, map_location=self.device)   # in place: params are heap views
            side_path = ckpt.model_path(train_dir, step) + "_optim"
            if os.path.exists(side_path):
                side = torch.load(side_path, map_location="cpu", weights_only=False)
                self.momentum_buf.copy_(side["momentum_buffer"].to(self.device))
                if side.get("lr") is not None:
                    self.set_lr(float(side["lr"]))
        self._barrier()
        if self.is_ps and self.world > 1:
            self.C.param_bcast(self.flat_params, self.t_params_peer, self.params_mc, self.world, self.rank,
                               self.plan.total_elems)
        self._barrier()
        self.step = step + 1
        self.ctrl_i32[0] = self.step          # Ctrl::step; first_step stays 1 so momentum is not re-initialised
        self.signals[PARAM_FLAG_SLOT] = self.step
        self._barrier()

    def close(self):
        torch.cuda.synchronize(self.device)
        if self.world > 1:
            dist.barrier(group=self.group)
        self.graph = None
        self.heap.close()


# ----------------------------------------------------------------------------------------------
def run_p2p_training(args):
    """``--backend p2p`` entry of the launcher (kept here for the old import path)."""
    from .p2p_launcher import run_p2p_training as _run
    return _run(args)

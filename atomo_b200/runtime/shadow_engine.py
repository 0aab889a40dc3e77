"""Overlapped, sharded bf16 engine — the H100 headline path (``--backend p2p`` with ``--dtype bf16``).

Differences against ``runtime/engine.py`` (round 1: fp32 flat parameters, encode after the whole backward,
one central PS kernel at the end of the step):

* **bf16 working weights, fp32 master on the PS.**  Every conv / linear weight the model trains with is a
  bf16 *leaf* tensor in cuDNN's layout (``channels_last``) living in the symmetric heap (``wshadow``).  No
  autocast weight casts, no NHWC weight copies, no fp32 gradient casts, no AccumulateGrad adds: autograd
  hands over the bf16 ``wgrad`` tensor cuDNN wrote and the coding kernels read it in place (pointer table).
  The fp32 master copy and the optimizer state live only on the PS owner of each tile; the PS epilogue
  rounds to bf16 and multicasts 2 bytes per weight instead of 4.
* **Push during backward** (the reference's only overlap design, ``src/model_ops/resnet_split.py:259-360``):
  parameters are split into backward groups; a post-accumulate-grad hook fires when the last gradient of a
  group exists, forks a side stream *inside the captured CUDA graph* and runs gram+eig / project+push of that
  group there while cuDNN continues with the earlier layers.
* **Sharded parameter server.**  Every GPU owns ``1/n_owners`` of each group's tiles (``ps_mode='sharded'``):
  workers store the U rows of a tile straight into its owner's arena, the owner reconstructs, steps the
  optimizer and multicasts its shard; nobody is the serial tail.  ``'colocated'`` (rank 0 owns everything,
  all ranks train) and ``'dedicated'`` (rank 0 only serves, like the reference's rank 0) keep the centralized
  topology of ``src/sync_replicas_master_nn.py``.
* Optimizers fused in the PS epilogue: momentum-SGD (``src/optim/sgd.py:57-90``), Adam / AMSGrad
  (``src/optim/adam.py:37-94``).

Per step and rank: ``wait_params`` -> forward -> backward [group hooks -> encode, project+push on stream E;
PS launch of the group on stream P] -> join -> ``advance_step``.  All cross-GPU ordering is carried by
step-stamped flags in peer memory (``csrc/v2_common.cuh``); no NCCL call on the path.
"""
from __future__ import annotations

import os
from typing import List, Optional

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn

from ..ops import plan2 as P2
from ..ops._ext import load as load_ext
from ..parallel.symm import SymmetricHeap

SIGNAL_INTS = 1024


def _dev_bytes(b: bytes, device) -> torch.Tensor:
    return torch.frombuffer(bytearray(b if len(b) else b"\0" * 16), dtype=torch.uint8).to(device)


class ShadowEngine:
    def __init__(self, model: nn.Module, rank: int = 0, world: int = 1, code: str = "svd", svd_rank: int = 3,
                 lr: float = 0.01, momentum: float = 0.0, weight_decay: float = 0.0, nesterov: bool = False,
                 dampening: float = 0.0, optimizer: str = "sgd", betas=(0.9, 0.999), eps: float = 1e-8,
                 amsgrad: bool = False, ps_mode: str = "sharded", groups: int = 5, sampling: str = "bernoulli",
                 prob_rule: str = "reference", random_sample: bool = True, seed: int = 1, use_graph: bool = True,
                 group=None, multicast: bool = True, heap_mode: str = "auto", timeout_s: float = 30.0,
                 criterion: Optional[nn.Module] = None, device: Optional[torch.device] = None,
                 ps_grid: int = 0, overlap: bool = True, fused_bn: bool = True, num_aggregate: int = 0,
                 warm_start: bool = True, max_sweeps: int = 1, main_priority: int = 0, debug_jitter_us: float = 0.0,
                 side_priority: int = -1, resample_empty: bool = False):
        self.C = load_ext()
        C = self.C
        assert C.v2_unit_bytes() == P2.UNIT_BYTES and C.v2_ctrl_bytes() == P2.CTRL2_BYTES
        self.rank, self.world, self.group = rank, world, group
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        dev = self.device
        self.code = {"dense": "sgd", "lossless": "sgd"}.get(code.lower(), code.lower())
        if self.code not in ("svd", "sgd", "qsvd"):
            raise ValueError("ShadowEngine codes: svd | qsvd | sgd (qsgd / terngrad / entrywise run on FusedEngine)")
        self.svd_rank = int(svd_rank)
        if world == 1:
            ps_mode = "colocated"
        self.ps_mode = ps_mode
        if ps_mode == "sharded":
            self.owner_ranks, self.worker_ranks = list(range(world)), list(range(world))
        elif ps_mode == "colocated":
            self.owner_ranks, self.worker_ranks = [0], list(range(world))
        elif ps_mode == "dedicated":
            self.owner_ranks, self.worker_ranks = [0], list(range(1, world))
        else:
            raise ValueError("ps_mode: sharded | colocated | dedicated")
        self.n_owners, self.W = len(self.owner_ranks), len(self.worker_ranks)
        assert self.W <= P2.MAX_WORKERS
        self.is_owner = rank in self.owner_ranks
        self.is_worker = rank in self.worker_ranks
        self.is_ps = rank == 0
        self.owner_index = self.owner_ranks.index(rank) if self.is_owner else -1
        self.worker_index = self.worker_ranks.index(rank) if self.is_worker else 0
        self.first_worker = self.worker_ranks[0]
        self.systematic = sampling == "systematic"
        self.waterfill = prob_rule == "waterfill"
        self.random_sample = random_sample
        self.resample_empty = resample_empty
        self.kflags = 1 if os.environ.get("ATOMO_NO_TMA") else 0     # bit 0: plain loads instead of TMA bulk copies
        # protocol fuzzing (tests): random device-side delays before every push / PS launch, different on every rank
        self._jitter_us = float(debug_jitter_us)
        self._jitter_rng = np.random.default_rng(1234 + rank)
        self.use_graph, self.overlap = use_graph, overlap
        self.criterion = criterion or nn.CrossEntropyLoss()
        self.timeout_ticks = int(timeout_s * 1.5e9)
        self.step, self.lr = 1, lr
        self.opt = {"sgd": P2.OPT_SGD, "adam": P2.OPT_AMSGRAD if amsgrad else P2.OPT_ADAM}[optimizer.lower()]
        self.launches_per_step = 0

        # ---- model: NHWC activations, fused BN ------------------------------------------------------------
        self.model = model.to(dev).to(memory_format=torch.channels_last)
        self.fused_bn_layers, self.bn_arena = 0, None
        if fused_bn:
            from ..ops.fused_bn import enable_fused_bn
            self.fused_bn_layers, self.bn_arena = enable_fused_bn(self.model, True, arena_device=dev)
        self.params = list(self.model.parameters())
        shapes = [tuple(p.shape) for p in self.params]
        self.plan = P2.build_plan2(shapes, self.code, self.svd_rank, self.systematic, n_owners=self.n_owners,
                                   n_groups=groups if overlap else 1)
        pl = self.plan
        self.G = pl.n_groups

        # ---- symmetric heap ---------------------------------------------------------------------------------
        need = 4 * SIGNAL_INTS + 2 * pl.w_total + 8 * pl.v_total + 2 * pl.stage_total + \
            4 * pl.arena_floats * self.W + (1 << 16)
        self.heap = h = SymmetricHeap(need + (1 << 20), rank, world, dev.index, group=group, multicast=multicast,
                                      mode=heap_mode)
        h.alloc("signals", 4 * SIGNAL_INTS)
        h.alloc("wshadow", 2 * pl.w_total)
        h.alloc("vparams", 4 * pl.v_total)
        h.alloc("vgrads", 4 * pl.v_total)
        h.alloc("wstage", 2 * pl.stage_total)
        h.alloc("arena", 4 * pl.arena_floats * self.W)
        self.signals = h.tensor("signals", torch.int32)
        self.wshadow = h.tensor("wshadow", torch.bfloat16)
        self.vparams = h.tensor("vparams")
        self.vgrads = h.tensor("vgrads")
        self.wstage = h.tensor("wstage", torch.bfloat16)
        self.signals.zero_(); self.wshadow.zero_(); self.vparams.zero_(); self.vgrads.zero_(); self.wstage.zero_()

        # ---- bind parameters --------------------------------------------------------------------------------
        # master (fp32, physical order) is built from the fp32 initial values BEFORE they are rounded to bf16
        self.master = torch.zeros(pl.w_total, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for p, q in zip(self.params, pl.params):
                src = p.data.to(dev, torch.float32)
                if q.is_w:
                    phys = src.permute(0, 2, 3, 1).contiguous().reshape(-1) if src.dim() == 4 else src.reshape(-1)
                    self.master[q.off:q.off + q.numel].copy_(phys)
                else:
                    self.vparams[q.off:q.off + q.numel].copy_(src.reshape(-1))
        if world > 1:   # everyone starts from rank 0's initial values
            dist.broadcast(self.master, src=0, group=group)
            vtmp = self.vparams.clone()
            dist.broadcast(vtmp, src=0, group=group)
            self.vparams.copy_(vtmp)
        self.wshadow.copy_(self.master.to(torch.bfloat16))
        self.w_params, self.v_params = [], []
        for p, q in zip(self.params, pl.params):
            if q.is_w:
                p.data = torch.as_strided(self.wshadow, q.shape, q.phys_strides(), q.off)
                p.grad = None
                self.w_params.append(p)
            else:
                p.data = self.vparams[q.off:q.off + q.numel].view(q.shape)
                p.grad = self.vgrads[q.off:q.off + q.numel].view(q.shape)
                self.v_params.append(p)
        sinked = set()
        if self.fused_bn_layers:
            from ..ops.fused_bn import BNAct
            for m in self.model.modules():
                if isinstance(m, BNAct) and m.fused and m.weight is not None and m.num_features % 8 == 0 \
                        and m.num_features <= 2048:
                    m._grad_sink = (m.weight.grad, m.bias.grad)
                    sinked.add(id(m.weight)); sinked.add(id(m.bias))
        # group bookkeeping: a group fires when every hooked parameter of it has its gradient
        self.group_of = [q.group for q in pl.params]
        self.group_size = [0] * self.G
        self._hooks = []
        if self.is_worker:
            for i, (p, q) in enumerate(zip(self.params, pl.params)):
                if id(p) in sinked:
                    continue
                self.group_size[q.group] += 1
                self._hooks.append(p.register_post_accumulate_grad_hook(self._make_hook(i)))
        self.w_range = []   # per group: range of gradient-pointer-table entries
        for g in range(self.G):
            idx = [q.widx for q in pl.params if q.is_w and q.group == g]
            self.w_range.append((min(idx), max(idx) + 1) if idx else (0, 0))

        # ---- owner state ----------------------------------------------------------------------------------
        z = lambda n: torch.zeros(n, dtype=torch.float32, device=dev)
        adam = self.opt != P2.OPT_SGD
        if self.is_owner:
            self.mom, self.vmom = z(pl.w_total), z(pl.v_total)
            self.sq, self.vsq = (z(pl.w_total), z(pl.v_total)) if adam else (None, None)
            self.sqmax, self.vsqmax = (z(pl.w_total), z(pl.v_total)) if self.opt == P2.OPT_AMSGRAD else (None, None)
        else:
            self.master = None

        # ---- device tables ---------------------------------------------------------------------------------
        self.t_units = _dev_bytes(pl.units_bytes(), dev)
        self.t_enc_tiles = _dev_bytes(P2.Plan2.tiles_bytes(pl.enc_tiles), dev)
        self.t_ps_tiles = _dev_bytes(P2.Plan2.tiles_bytes(pl.ps_tiles), dev)
        nc = max(pl.n_coded, 1)
        self.gpart = z(pl.gpart_floats)
        self.vsel = z(nc * P2.MAX_COLS * P2.RCAP_MAX)
        self.selcount = torch.zeros(nc, dtype=torch.int32, device=dev)
        self.sigma = z(nc * P2.MAX_COLS)
        # eigenbasis of the previous step per coded unit (Jacobi warm start); identity to begin with
        self.max_sweeps = int(max_sweeps) if warm_start else 0
        self.vprev = None
        if warm_start:
            self.vprev = z(nc * P2.MAX_COLS * P2.MAX_COLS)
            for u in pl.units:
                if u.coded:
                    o = u.ts_index * P2.MAX_COLS * P2.MAX_COLS
                    self.vprev[o:o + u.cols * u.cols].copy_(torch.eye(u.cols, device=dev).reshape(-1))
        self.counters = torch.zeros(nc + 2 * P2.MAX_GROUPS + 8, dtype=torch.int32, device=dev)
        self.cnt_enc_group = self.counters.data_ptr() + 4 * nc
        self.cnt_ps_group = self.cnt_enc_group + 4 * P2.MAX_GROUPS
        self.ctrl = _dev_bytes(P2.pack_ctrl2(step=1, lr=lr, momentum=momentum, dampening=dampening,
                                             weight_decay=weight_decay, nesterov=nesterov, first_step=1, seed=seed,
                                             beta1=betas[0], beta2=betas[1], eps=eps, opt=self.opt,
                                             num_aggregate=num_aggregate), dev)
        self.ctrl_i32, self.ctrl_f32 = self.ctrl.view(torch.int32), self.ctrl.view(torch.float32)
        n_w = max(len(self.w_params), 1)
        self.t_gptr = torch.zeros(n_w, dtype=torch.int64, device=dev)
        self.host_gptr = np.zeros(n_w, dtype=np.int64)
        i64 = lambda xs: torch.tensor(list(xs) or [0], dtype=torch.int64, device=dev)
        self.t_arena_peer = i64(h.region_ptr("arena", r) for r in self.owner_ranks)
        self.t_sig_owner = i64(h.region_ptr("signals", r) for r in self.owner_ranks)
        self.t_sig_all = i64(h.region_ptr("signals", r) for r in range(world))
        self.t_wshadow_peer = i64(h.region_ptr("wshadow", r) for r in range(world))
        self.t_vparams_peer = i64(h.region_ptr("vparams", r) for r in range(world))
        self.t_vgrads_peer = i64(h.region_ptr("vgrads", r) for r in self.worker_ranks)
        self.t_stage_peer = i64(h.region_ptr("wstage", r) for r in self.worker_ranks)
        self.wshadow_mc, self.vparams_mc = h.region_mc_ptr("wshadow"), h.region_mc_ptr("vparams")
        self.vgrads_mc = h.region_mc_ptr("vgrads")
        sm = torch.cuda.get_device_properties(dev).multi_processor_count
        self.ps_grid = ps_grid or 3 * sm
        self.tstats = torch.zeros(32, dtype=torch.int64, device=dev)
        self.loss_buf = torch.zeros(3, dtype=torch.float32, device=dev)
        self.static_x = self.static_y = self.graph = None

        # ---- streams / events --------------------------------------------------------------------------------
        self.s_enc = torch.cuda.Stream(device=dev, priority=side_priority)
        self.s_ps = torch.cuda.Stream(device=dev, priority=side_priority)
        self.s_main = torch.cuda.Stream(device=dev, priority=main_priority)   # warm-up + capture stream
        self.ev_ready = [torch.cuda.Event() for _ in range(self.G)]
        self.ev_push = [torch.cuda.Event() for _ in range(self.G)]
        self.ev_enc_done, self.ev_ps_done = torch.cuda.Event(), torch.cuda.Event()
        self._pending, self._fired, self._nlaunch = list(self.group_size), 0, 0
        self._capturing = False
        self._initial_sync()

    # ------------------------------------------------------------------------------------------------------
    def _barrier(self):
        torch.cuda.synchronize(self.device)
        if self.world > 1:
            dist.barrier(group=self.group)

    def _initial_sync(self):
        self._barrier()
        self.signals.zero_()
        self.signals[256:256 + self.n_owners] = 1      # SIG_PARAM: parameters of step 1 are in place
        self._barrier()

    def set_lr(self, lr: float):
        self.lr = lr
        self.ctrl_f32[2] = lr

    def error_code(self) -> int:
        return int(self.ctrl_i32[1].item())

    def device_step(self) -> int:
        return int(self.ctrl_i32[0].item())

    def phase_stats(self, reset: bool = True) -> dict:
        """Average device-side microseconds per step since the last reset (globaltimer stamps taken inside the
        kernels, so they are valid under CUDA-graph replay):

        * ``param_wait_us``  blocked at the start of a step until every owner published the parameters,
        * ``encode_us``      encode + project kernels of all groups (first CTA in -> last CTA out; they overlap with
                             backward except for the final group),
        * ``to_push_us``     step start -> this worker's last push flag (forward + backward + its encode tail),
        * ``to_params_us``   step start -> this owner's parameters published (owners only),
        * ``ps_wait_push_us`` / ``ps_work_us``  per step, summed over the groups this owner serves."""
        t = self.tstats.tolist()
        steps = max(t[4], 1)
        out = {"param_wait_us": t[3] / steps / 1e3, "encode_us": t[5] / steps / 1e3, "to_push_us": t[8] / steps / 1e3}
        if self.is_owner:
            out["ps_wait_push_us"] = t[0] / steps / 1e3
            out["ps_work_us"] = t[1] / steps / 1e3
            out["to_params_us"] = t[7] / steps / 1e3
        if reset:
            self.tstats[:9].zero_()
        return out

    # ------------------------------------------------------------------------------------------------------
    def _make_hook(self, i: int):
        q = self.plan.params[i]

        def hook(p):
            if q.is_w:
                self.host_gptr[q.widx] = p.grad.data_ptr()
            g = q.group
            self._pending[g] -= 1
            if self._pending[g] == 0:
                self._launch_group(g)
        return hook

    def _launch_encode(self, g: int):
        C, pl = self.C, self.plan
        t0, nt = pl.enc_range[g]
        if not self._capturing:
            lo, hi = self.w_range[g]
            if hi > lo:   # pageable source: staged synchronously, safe against the host table changing next step
                self.t_gptr[lo:hi].copy_(torch.from_numpy(self.host_gptr[lo:hi].copy()))
        if nt > 0 and self.code in ("svd", "qsvd"):
            C.v2_encode(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                        self.gpart.data_ptr(), self.counters.data_ptr(), self.vsel.data_ptr(),
                        self.selcount.data_ptr(), self.sigma.data_ptr(), self.t_arena_peer.data_ptr(), self.n_owners,
                        pl.arena_floats, self.wstage.data_ptr(), self.ctrl.data_ptr(), 0,
                        self.vprev.data_ptr() if self.vprev is not None else 0, self.max_sweeps, self.random_sample,
                        self.waterfill, self.systematic, self.worker_index, self.resample_empty, self.kflags,
                        self.tstats.data_ptr(), g)
            self._nlaunch += 1
        elif nt > 0:
            # dense code: only the staging copies of the bf16 gradients
            C.v2_encode(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                        self.gpart.data_ptr(), self.counters.data_ptr(), self.vsel.data_ptr(),
                        self.selcount.data_ptr(), 0, self.t_arena_peer.data_ptr(), self.n_owners, pl.arena_floats,
                        self.wstage.data_ptr(), self.ctrl.data_ptr(), 0, 0, 0, False, False, False, self.worker_index, False, self.kflags,
                        self.tstats.data_ptr(), g)
            self._nlaunch += 1
        C.v2_project(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                     self.vsel.data_ptr(), self.selcount.data_ptr(), self.t_arena_peer.data_ptr(),
                     self.t_sig_owner.data_ptr(), self.n_owners, pl.arena_floats, self.worker_index, g,
                     self.ctrl.data_ptr(), self.cnt_enc_group + 4 * g, self.kflags, self.tstats.data_ptr(),
                     self._fired == self.G, nt > 0)
        self._nlaunch += 1

    def _launch_ps(self, g: int, final: bool):
        C, pl = self.C, self.plan
        t0, nt = pl.ps_range[g][self.owner_index]
        p = lambda t: t.data_ptr() if t is not None else 0
        C.v2_ps(self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), t0, nt, self.W, self.world, g, final,
                self.owner_index, p(self.master), p(self.mom), p(self.sq), p(self.sqmax), p(self.vmom), p(self.vsq),
                p(self.vsqmax), self.wshadow_mc, self.t_wshadow_peer.data_ptr(), self.vparams.data_ptr(),
                self.vparams_mc, self.t_vparams_peer.data_ptr(), self.vgrads_mc, self.t_vgrads_peer.data_ptr(),
                self.t_stage_peer.data_ptr(), self.heap.region_ptr("arena"), pl.arena_floats,
                self.signals.data_ptr(), self.t_sig_all.data_ptr(), self.ctrl.data_ptr(), self.cnt_ps_group + 4 * g,
                self.timeout_ticks, self.tstats.data_ptr(), 1.0 / self.W, max(1, min(self.ps_grid, max(nt, 1))))
        self._nlaunch += 1

    def _launch_group(self, g: int):
        """Called from the autograd thread when the last gradient of group ``g`` exists: fork the encode stream
        (and, on an owner, the PS stream) off the stream backward is running on."""
        final = self._fired == self.G - 1
        self._fired += 1
        if not self.overlap:
            self._launch_encode(g)
            if self.is_owner:
                self._launch_ps(g, final)
            return
        cur = torch.cuda.current_stream(self.device)
        self.ev_ready[g].record(cur)
        self.s_enc.wait_event(self.ev_ready[g])
        with torch.cuda.stream(self.s_enc):
            if self._jitter_us:
                torch.cuda._sleep(int(self._jitter_rng.uniform(0, self._jitter_us) * 1900))
            self._launch_encode(g)
            self.ev_push[g].record(self.s_enc)
            if final:
                self.ev_enc_done.record(self.s_enc)
        if self.is_owner:
            self.s_ps.wait_event(self.ev_push[g])
            with torch.cuda.stream(self.s_ps):
                if self._jitter_us:
                    torch.cuda._sleep(int(self._jitter_rng.uniform(0, self._jitter_us) * 1900))
                self._launch_ps(g, final)
                if final:
                    self.ev_ps_done.record(self.s_ps)

    def _forward_backward(self):
        x, y = self.static_x, self.static_y
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits = self.model(x)
            loss = self.criterion(logits.float(), y)
        loss.backward()
        with torch.no_grad():
            lg = logits.detach().float()
            k = min(5, lg.size(1))
            hit = lg.topk(k, 1).indices.eq(y.view(-1, 1))
            self.loss_buf[0] = loss.detach()
            self.loss_buf[1] = hit[:, :1].float().sum() * (100.0 / y.numel())
            self.loss_buf[2] = hit.float().sum() * (100.0 / y.numel())

    def _step_body(self):
        C = self.C
        self._nlaunch = 0
        C.v2_wait_params(self.signals.data_ptr(), self.n_owners, self.ctrl.data_ptr(), self.timeout_ticks,
                         self.tstats.data_ptr())
        self._nlaunch += 1
        if self.is_worker:
            self.vgrads.zero_()
            if self.bn_arena is not None:
                self.bn_arena.zero_()
            for p in self.w_params:
                p.grad = None
            self._pending, self._fired = list(self.group_size), 0
            self._forward_backward()
            self._nlaunch += 4 * self.fused_bn_layers
            assert self._fired == self.G, "a backward group never fired (%d of %d)" % (self._fired, self.G)
            if self.overlap:
                cur = torch.cuda.current_stream(self.device)
                cur.wait_event(self.ev_enc_done)
                if self.is_owner:
                    cur.wait_event(self.ev_ps_done)
        elif self.is_owner:      # dedicated PS: serve the groups in order on the main stream
            for g in range(self.G):
                self._launch_ps(g, g == self.G - 1)
        C.v2_advance_step(self.ctrl.data_ptr())
        self._nlaunch += 1
        self.launches_per_step = self._nlaunch

    # ------------------------------------------------------------------------------------------------------
    def prepare(self, x_example: torch.Tensor, y_example: torch.Tensor, warmup: int = 3):
        self.static_x = torch.empty_like(x_example, device=self.device)
        if self.static_x.dim() == 4:
            self.static_x = self.static_x.contiguous(memory_format=torch.channels_last)
        self.static_y = torch.empty_like(y_example, device=self.device)
        self.static_x.copy_(x_example)
        self.static_y.copy_(y_example)
        # double-buffered input staging: the host->device copy of batch t runs on its own stream while step t-1 is
        # still executing; the step itself starts with a 1.5 MB device-to-device copy instead of a PCIe transfer
        self.s_copy = torch.cuda.Stream(device=self.device)
        self.stage_x = [torch.empty_like(self.static_x) for _ in range(2)]
        self.stage_y = [torch.empty_like(self.static_y) for _ in range(2)]
        self._stage_ready = [torch.cuda.Event() for _ in range(2)]
        self._stage_free = [torch.cuda.Event() for _ in range(2)]
        self._stage_i = 0
        self.model.train()
        s = self.s_main
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            for _ in range(warmup):
                self._step_body()
                self.step += 1
        torch.cuda.current_stream(self.device).wait_stream(s)
        torch.cuda.synchronize(self.device)
        if self.use_graph:
            self.graph = torch.cuda.CUDAGraph()
            self._capturing = True
            try:
                with torch.cuda.graph(self.graph, stream=self.s_main):
                    self._step_body()
            finally:
                self._capturing = False
            # the gradient tensors allocated during capture live at fixed addresses of the graph's pool
            self.t_gptr.copy_(torch.from_numpy(self.host_gptr.copy()))
            torch.cuda.synchronize(self.device)
        return self

    def train_step(self, x: Optional[torch.Tensor] = None, y: Optional[torch.Tensor] = None):
        if x is not None and self.is_worker:
            if x.is_cuda:
                self.static_x.copy_(x, non_blocking=True)
                self.static_y.copy_(y, non_blocking=True)
            else:
                k = self._stage_i
                self._stage_i ^= 1
                cur = torch.cuda.current_stream(self.device)
                with torch.cuda.stream(self.s_copy):
                    self.s_copy.wait_event(self._stage_free[k])      # the step that consumed this buffer has read it
                    self.stage_x[k].copy_(x, non_blocking=True)
                    self.stage_y[k].copy_(y, non_blocking=True)
                    self._stage_ready[k].record(self.s_copy)
                cur.wait_event(self._stage_ready[k])
                self.static_x.copy_(self.stage_x[k], non_blocking=True)
                self.static_y.copy_(self.stage_y[k], non_blocking=True)
                self._stage_free[k].record(cur)
        if self.graph is not None:
            self.graph.replay()
        else:
            self._step_body()
        self.step += 1
        return self.loss_buf

    # ------------------------------------------------------------------------------------------------------
    # fp32 views of the sharded state (checkpointing, tests)
    def _owned_mask(self):
        """1.0 where this owner holds the authoritative fp32 value (per weight element / per vector element)."""
        pl = self.plan
        mw = torch.zeros(pl.w_total, dtype=torch.float32, device=self.device)
        mv = torch.zeros(pl.v_total, dtype=torch.float32, device=self.device)
        if not self.is_owner:
            return mw, mv
        for (ui, a, b, o) in pl.ps_tiles:
            if o != self.owner_index:
                continue
            u = pl.units[ui]
            if u.kind == P2.KIND_VEC:
                mv[u.w_off + a:u.w_off + a + b] = 1
            elif u.kind == P2.KIND_DENSE16:
                mw[u.w_off + a:u.w_off + a + b] = 1
            elif u.kind == P2.KIND_SLAB:
                half = u.I // 2
                e0 = u.w_off + (a // half) * u.K * u.I
                mw[e0:e0 + (b // half) * u.K * u.I] = 1
            else:
                torch.as_strided(mw, (b, u.cols), (u.rs, u.cs), u.w_off + a * u.rs).fill_(1)
        return mw, mv

    def gather_fp32(self, what: str = "master") -> torch.Tensor:
        """Full fp32 array (weight indexing) assembled from the owners' shards: 'master' | 'mom' | 'sq' | 'sqmax'."""
        src = {"master": self.master, "mom": getattr(self, "mom", None), "sq": getattr(self, "sq", None),
               "sqmax": getattr(self, "sqmax", None)}[what]
        torch.cuda.synchronize(self.device)
        mw, _ = self._owned_mask()
        out = (src * mw) if (self.is_owner and src is not None) else torch.zeros_like(mw)
        if self.world > 1:
            dist.all_reduce(out, group=self.group)
        return out

    def fp32_state_dict(self) -> dict:
        """state_dict in the standard (OIHW, fp32) layout — the evaluator's ``model_step_<N>`` contract.  Weights
        come from the fp32 master copies on the owners; BN running statistics from THIS rank's model (call it on
        a rank that trains: the reference's PS checkpoints carried untrained BN statistics, SURVEY 2.9)."""
        full = self.gather_fp32("master")
        sd = {}
        byid = {id(p): q for p, q in zip(self.params, self.plan.params)}
        for name, t in self.model.state_dict().items():
            sd[name] = t.detach().float().clone() if t.is_floating_point() else t.detach().clone()
        for name, p in self.model.named_parameters():
            q = byid[id(p)]
            if q.is_w:
                flat = full[q.off:q.off + q.numel]
                if len(q.shape) == 4:
                    o, i, kh, kw = q.shape
                    sd[name] = flat.view(o, kh, kw, i).permute(0, 3, 1, 2).contiguous()
                else:
                    sd[name] = flat.view(q.shape).clone()
        return sd

    def save_checkpoint(self, train_dir: str, step: Optional[int] = None) -> Optional[str]:
        """Collective.  The first training rank writes ``model_step_<N>`` (fp32, trained BN statistics) and the
        ``_optim`` sidecar (momentum — for Adam / AMSGrad also the second moments —, step, LR) so a later run can
        resume."""
        from ..utils import checkpoint as ckpt
        step = (self.step - 1) if step is None else step
        sd = self.fp32_state_dict()
        mom = self.gather_fp32("mom")
        vmom = self.vmom if self.is_owner else torch.zeros_like(self.vparams)
        _, mv = self._owned_mask()
        vm = vmom * mv
        if self.world > 1:
            dist.all_reduce(vm, group=self.group)
        adam_state = {}
        if self.opt != P2.OPT_SGD:      # Adam / AMSGrad: second moments too (collective gathers, every rank takes part)
            names = [("sq", "vsq")] + ([("sqmax", "vsqmax")] if self.opt == P2.OPT_AMSGRAD else [])
            for wname, vname in names:
                vt = (getattr(self, vname) if self.is_owner else torch.zeros_like(self.vparams)) * mv
                if self.world > 1:
                    dist.all_reduce(vt, group=self.group)
                adam_state[wname + "_w"] = self.gather_fp32(wname).cpu()
                adam_state[wname + "_v"] = vt.cpu()
        if self.rank != self.first_worker:
            return None
        path = ckpt.model_path(train_dir, step)
        os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
        tmp = path + ".tmp"
        torch.save({k: v.cpu() for k, v in sd.items()}, tmp)
        os.replace(tmp, path)
        side = {"step": step, "lr": self.lr, "mom_w": mom.cpu(), "mom_v": vm.cpu(), "code": self.code,
                "svd_rank": self.svd_rank, "engine": "shadow"}
        side.update(adam_state)
        torch.save(side, path + "_optim.tmp")
        os.replace(path + "_optim.tmp", path + "_optim")
        return path

    def load_checkpoint(self, train_dir: str, step: int) -> None:
        """Collective: every rank reads the same files (shared directory) and jumps to ``step + 1``."""
        from ..utils import checkpoint as ckpt
        self._barrier()
        path = ckpt.model_path(train_dir, step)
        sd = torch.load(path, map_location="cpu", weights_only=False)
        byname = dict(self.model.named_parameters())
        byid = {id(p): q for p, q in zip(self.params, self.plan.params)}
        with torch.no_grad():
            for name, t in sd.items():
                if name in byname:
                    q = byid[id(byname[name])]
                    src = t.to(self.device, torch.float32)
                    if q.is_w:
                        phys = src.permute(0, 2, 3, 1).contiguous().reshape(-1) if src.dim() == 4 else src.reshape(-1)
                        if self.is_owner:
                            self.master[q.off:q.off + q.numel].copy_(phys)
                        self.wshadow[q.off:q.off + q.numel].copy_(phys.to(torch.bfloat16))
                    else:
                        self.vparams[q.off:q.off + q.numel].copy_(src.reshape(-1))
                else:
                    buf = dict(self.model.named_buffers()).get(name)
                    if buf is not None:
                        buf.copy_(t.to(buf.device, buf.dtype))
            if os.path.exists(path + "_optim") and self.is_owner:
                side = torch.load(path + "_optim", map_location="cpu", weights_only=False)
                if "mom_w" in side:
                    self.mom.copy_(side["mom_w"].to(self.device))
                    self.vmom.copy_(side["mom_v"].to(self.device))
                for wname, vname in (("sq", "vsq"), ("sqmax", "vsqmax")):      # Adam / AMSGrad second moments
                    if wname + "_w" in side and getattr(self, wname, None) is not None:
                        getattr(self, wname).copy_(side[wname + "_w"].to(self.device))
                        getattr(self, vname).copy_(side[vname[1:] + "_v"].to(self.device))
                if side.get("lr") is not None:
                    self.set_lr(float(side["lr"]))
        self.step = step + 1
        self.ctrl_i32[0] = self.step
        self._barrier()
        self.signals[256:256 + self.n_owners] = self.step
        self._barrier()

    def close(self):
        torch.cuda.synchronize(self.device)
        if self.world > 1:
            dist.barrier(group=self.group)
        for hk in self._hooks:
            hk.remove()
        self.graph = None
        self.heap.close()

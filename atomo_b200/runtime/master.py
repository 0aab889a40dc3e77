"""Parameter-server role.

Parity: ``SyncReplicasMaster_NN`` (``/root/reference/src/sync_replicas_master_nn.py:94-359``):
``__init__(comm, **kwargs)`` with the same kwargs, ``build_model(num_classes)``,
``train()``; per step: send step -> broadcast weights -> gather coded gradients
-> decode -> aggregate (sum / num_workers) -> optimizer step -> LR schedule ->
checkpoint.  Log line: ``master:221``.

Fixes (SURVEY.md 2.9): the aggregate buffer is fully zeroed each step; the LR
decay reaches the optimizer; ``--num-aggregate`` really implements
backup-worker aggregation (proceed after N arrivals, drop stale stragglers);
checkpointing every ``eval_freq`` steps is enabled; every ``--code`` builds.
"""
from __future__ import annotations

import os
import time
from typing import Optional

import numpy as np
import torch

from .. import codings
from ..models import build_model
from ..optim import LAMB, LARS, SGD, Adam, AdamW, Lion
from ..parallel.transport import Transport, STOP_STEP
from ..utils import checkpoint as ckpt
from ..utils.flags import check_clip_grad_norm, check_ema_decay
from ..utils.logging import MetricsWriter, master_line
from .flat import FlatLayout, bind_parameters
from .nn_ops import NN_Trainer

STEP_START_ = 1


def build_coder(kwargs: dict, worker_side: bool):
    """Coder selection shared by PS and workers (master:134-144, worker:127-137)."""
    code = kwargs.get("code", "sgd")
    if code in ("sgd", "dense", "lossless"):
        return codings.build("sgd", compress=bool(kwargs.get("compress", False)))
    if code == "svd":
        return codings.build("svd", rank=kwargs.get("svd_rank", 0), random_sample=worker_side, compress=True,
                             prob_rule=kwargs.get("prob_rule", "reference"),
                             scheme=kwargs.get("sampling", "bernoulli"))
    if code in ("qsgd", "terngrad"):
        return codings.build(code, bucket_size=kwargs.get("bucket_size", 512),
                             quantization_level=kwargs.get("quantization_level", 4))
    if code == "entrywise":
        return codings.build("entrywise", budget=kwargs.get("entry_budget", 0.05),
                             prob_rule=kwargs.get("prob_rule", "reference"))
    if code == "fp8":
        raise ValueError("--code fp8 runs on the --backend p2p bf16 engine (--dtype bf16) only; the gloo / nccl "
                         "backends have no fp8 coder")
    if code == "hadamard":
        raise ValueError("--code hadamard runs on the --backend p2p bf16 engine (--dtype bf16) only; the gloo / nccl "
                         "backends have no randomized-Hadamard coder")
    if code == "powersgd":
        raise ValueError("--code powersgd runs on the --backend p2p bf16 engine (--dtype bf16), which keeps each "
                         "worker's warm state and error-feedback residual; the gloo / nccl coders keep neither")
    if code == "sign":
        raise ValueError("--code sign runs on the --backend p2p bf16 engine (--dtype bf16), which keeps the "
                         "error-feedback residual; scaled sign without it is biased, and the gloo / nccl coders keep "
                         "none")
    if code == "signum":
        raise ValueError("--code signum runs on the --backend p2p bf16 engine (--dtype bf16), which keeps each "
                         "worker's momentum and takes the owners' majority vote; the gloo / nccl coders keep neither")
    if code == "dlion":
        raise ValueError("--code dlion runs on the --backend p2p bf16 engine (--dtype bf16), which keeps each "
                         "worker's Lion momentum and aggregates the signs on the owners; the gloo / nccl coders keep "
                         "neither")
    if code == "topk":
        raise ValueError("--code topk runs on the --backend p2p bf16 engine (--dtype bf16), which keeps the "
                         "error-feedback residual; top-k without it is biased, and the gloo / nccl coders keep none")
    if code == "bsvd":
        return codings.build("bsvd", rank=kwargs.get("svd_rank", 0) or 3, random_sample=worker_side,
                             prob_rule=kwargs.get("prob_rule", "reference"),
                             scheme=kwargs.get("sampling", "bernoulli"))
    if code == "qsvd":
        return codings.build("qsvd", rank=kwargs.get("svd_rank", 0), random_sample=worker_side,
                             quantization_level=kwargs.get("quantization_level", 4),
                             bucket_size=kwargs.get("bucket_size", 512))
    raise ValueError("args.code not recognized")


class GradientAccumulator:
    """Per-parameter aggregate buffers + arrival counters
    (parity: ``GradientAccumulator``, master:57-91 — without the pickled
    bytearray receive slots: the transport delivers tensors)."""

    def __init__(self, layout: FlatLayout, device, dtype=torch.float64):
        self.layout = layout
        self.flat = torch.zeros(layout.total, dtype=dtype, device=device)
        self.gradient_aggregator = layout.views(self.flat)
        self.gradient_aggregate_counter = [0] * len(layout)

    def add(self, layer_idx: int, grad: torch.Tensor):
        self.gradient_aggregator[layer_idx].add_(grad.to(self.flat.device, self.flat.dtype))
        self.gradient_aggregate_counter[layer_idx] += 1

    def meset_everything(self):
        self.flat.zero_()
        self.gradient_aggregate_counter = [0] * len(self.layout)


def clip_grad_norm(grads, max_norm: float):
    """``torch.nn.utils.clip_grad_norm_`` on a list of gradients: scaled by ``min(1, max_norm / (||g|| + 1e-6))``, the
    norm taken over all of them, in their own precision.  Returns the scaled gradients and ``(total, coef)``."""
    total = torch.nn.utils.get_total_norm(grads)
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    return [g * coef.to(g.device) for g in grads], (float(total), float(coef))


class SyncReplicasMaster_NN(NN_Trainer):
    ema = None      # --ema-decay: the fp32 average of flat_params (build_model), None when off

    def __init__(self, comm: Transport, **kwargs):
        self.comm = comm
        self.world_size = comm.world_size
        self.cur_step = STEP_START_
        self.lr = kwargs["learning_rate"]
        self._lr_shrinkage = kwargs.get("lr_shrinkage", 0.95)
        self._base_lr = kwargs["learning_rate"]
        self.shrinkage_freq = kwargs.get("shrinkage_freq", 50)
        self.shrink_counter = 0
        self.momentum = kwargs.get("momentum", 0.5)
        self.network_config = kwargs["network"]
        self.dataset = kwargs.get("dataset", "")
        self.comm_type = kwargs.get("comm_method", "Bcast")
        self._num_workers = self.world_size - 1
        self._eval_freq = kwargs.get("eval_freq", 50)
        self._train_dir = kwargs.get("train_dir", "output/models/")
        self._max_steps = kwargs.get("max_steps", 10000)
        self._compress = kwargs.get("compress", False)
        self._enable_gpu = bool(kwargs.get("enable_gpu", False)) and torch.cuda.is_available()
        na = kwargs.get("num_aggregate", None)
        self._num_aggregate = self._num_workers if not na else max(1, min(int(na), self._num_workers))
        self._svd_rank = kwargs.get("svd_rank", 0)
        self._quantization_level = kwargs.get("quantization_level", 4)
        self._bucket_size = kwargs.get("bucket_size", 512)
        self._optimizer_name = kwargs.get("optimizer", "sgd")
        self._clip_grad_norm = check_clip_grad_norm(kwargs.get("clip_grad_norm", 0.0))
        self.last_grad_norm = None      # (total, coef) of the last update with clipping on
        # --ema-decay: an fp32 average of flat_params after every optimizer step, e <- e + w (p - e), w = fp32(1 - d)
        self._ema_decay = check_ema_decay(kwargs.get("ema_decay", 0.0))
        self._ema_w = float(np.float32(1.0 - self._ema_decay))
        self._save_checkpoints = kwargs.get("save_checkpoints", True)
        self._resume = kwargs.get("resume", False)
        self._verbose = kwargs.get("verbose", True)
        self.device = torch.device("cuda", torch.cuda.current_device()) if self._enable_gpu else torch.device("cpu")
        self._coder = build_coder(kwargs, worker_side=False)
        self._kwargs = kwargs
        self._metrics = MetricsWriter(kwargs.get("metrics_file", ""), 0, "ps")

    def build_model(self, num_classes: int = 10):
        self.network = build_model(self.network_config, num_classes, self.dataset).to(self.device)
        self.layout = FlatLayout.from_module(self.network)
        self.flat_params = torch.zeros(self.layout.total, dtype=torch.float32, device=self.device)
        bind_parameters(self.network, self.flat_params, self.layout)
        if self._optimizer_name == "adam":
            self.optimizer = Adam(self.network.parameters(), lr=self.lr)
        elif self._optimizer_name == "lars":
            self.optimizer = LARS(self.network.parameters(), lr=self.lr, momentum=self.momentum,
                                  weight_decay=self._kwargs.get("weight_decay", 0.0),
                                  trust_coefficient=self._kwargs.get("trust_coefficient", 0.001),
                                  nesterov=self._kwargs.get("nesterov", False))
        elif self._optimizer_name == "adamw":
            self.optimizer = AdamW(self.network.parameters(), lr=self.lr,
                                   weight_decay=self._kwargs.get("weight_decay", 0.0))
        elif self._optimizer_name == "lion":
            self.optimizer = Lion(self.network.parameters(), lr=self.lr,
                                  betas=tuple(self._kwargs.get("lion_betas", (0.9, 0.99))),
                                  weight_decay=self._kwargs.get("weight_decay", 0.0))
        elif self._optimizer_name == "lamb":
            self.optimizer = LAMB(self.network.parameters(), lr=self.lr,
                                  weight_decay=self._kwargs.get("weight_decay", 0.0))
        else:
            self.optimizer = SGD(self.network.parameters(), lr=self.lr, momentum=self.momentum,
                                 weight_decay=self._kwargs.get("weight_decay", 0.0),
                                 nesterov=self._kwargs.get("nesterov", False))
        agg_dtype = torch.float64 if self.device.type == "cpu" else torch.float32
        self.grad_accumulator = GradientAccumulator(self.layout, self.device, agg_dtype)
        self._model_shapes = [tuple(p.shape) for p in self.network.parameters()]
        last = ckpt.latest_step(self._train_dir) if self._resume else None
        if last is not None:
            ckpt.load_model(self._train_dir, last, self.network, map_location=self.device)
            side = ckpt.load_sidecar(self._train_dir, last, self.optimizer, map_location=self.device)
            self.cur_step = last + 1
            if side and side.get("lr") is not None:
                self.lr = side["lr"]
                self.optimizer.set_lr(self.lr)
                self.shrink_counter = side.get("shrink_counter", 0)
        if self._ema_decay:
            self.ema = self.flat_params.clone()     # the initial (or loaded) weights
            if last is not None:
                self._load_ema(ckpt.model_path(self._train_dir, last) + "_ema")
        return self

    def _ema_views(self) -> dict:
        """Parameter name -> its view of ``ema``."""
        return {n: v for (n, _), v in zip(self.network.named_parameters(), self.layout.views(self.ema))}

    def _load_ema(self, path: str):
        if not os.path.exists(path):
            print("%s missing: the weight average starts at the loaded weights" % path, flush=True)
            return
        sd = torch.load(path, map_location=self.device, weights_only=False)
        with torch.no_grad():
            for name, v in self._ema_views().items():
                v.copy_(sd[name])

    def _update_ema(self):
        """e <- e + w (p - e) over flat_params, each operation rounded to fp32 (the bf16 engine's csrc/v2_ema.cu)."""
        w = torch.tensor(self._ema_w, dtype=torch.float32, device=self.device)
        d = torch.sub(self.flat_params, self.ema)
        d.mul_(w)
        self.ema.add_(d)

    # ------------------------------------------------------------------
    def train(self):
        first = self.cur_step
        for i in range(first, self._max_steps + 1):
            self.network.train()
            if self._verbose:
                print("Master node is entering step: {}".format(i))
            if self.comm.backup_rounds:
                # backup workers: point-to-point announcement to the workers that owe nothing (transport.py)
                self.comm.send_round(self.cur_step, self.flat_params, self._num_aggregate)
            else:
                self.async_bcast_step()
                self.async_bcast_layer_weights_bcast()

            gather_start = time.time()
            coded_msgs = self.comm.gather(self.cur_step, need=self._num_aggregate)
            gather_duration = time.time() - gather_start
            if self._num_aggregate < self._num_workers:
                # backup-worker mode: the update uses the first N arrivals.  With --straggler-kill the others are
                # told to abandon the step (tag 77, lenet.py:173-180).  Nobody is waited for: late messages are
                # step-stamped and dropped when they surface; on NCCL (no any-source receive) gather() already
                # waited for everyone.
                if self._kwargs.get("kill_stragglers", False):
                    for w in self.comm.asked_workers():
                        if w not in coded_msgs:
                            self.comm.send_kill(w, self.cur_step)
                if not self.comm.backup_rounds:
                    self.comm.drain()

            self._take_aux_buffers(coded_msgs)
            decode_start = time.time()
            n_used = self._decode(coded_msgs)
            decode_dur = time.time() - decode_start
            print(master_line(self.cur_step, decode_dur, self.lr, gather_duration))
            self._metrics.write(step=self.cur_step, gather=gather_duration, decode=decode_dur, lr=self.lr,
                                used_workers=sorted(coded_msgs), stale_dropped=getattr(self.comm, "_stale_dropped", 0),
                                lost_workers=self.comm.lost_workers())
            self._model_update(n_used)
            self.grad_accumulator.meset_everything()

            if self._save_checkpoints and self.cur_step % self._eval_freq == 0:
                self._save_model(self._generate_model_path())
            self.cur_step += 1
            if self.cur_step % self.shrinkage_freq == 0:
                self.shrink_counter += 1
                self.lr = self._base_lr * self._lr_shrinkage ** self.shrink_counter
                self.optimizer.set_lr(self.lr)  # the reference never did this (master:232-234)
        self.comm.finish()      # collect what stragglers still owe, then STOP every worker

    def async_bcast_step(self):
        self.comm.send_step(self.cur_step)

    def async_bcast_layer_weights_bcast(self):
        self.comm.bcast_params(self.flat_params)

    def _take_aux_buffers(self, coded_msgs: dict):
        """Strip the auxiliary entries workers append to their code lists; BatchNorm running statistics sent by the
        first worker on checkpoint steps are copied into the PS's network before it is saved."""
        for w, codes in coded_msgs.items():
            if codes and isinstance(codes[-1], dict) and codes[-1].get("__aux__") == "buffers":
                aux = codes.pop()
                with torch.no_grad():
                    for b, t in zip(self.network.buffers(), aux["tensors"]):
                        b.copy_(t.to(b.device, b.dtype))

    def _decode(self, coded_msgs: dict) -> int:
        for _, codes in coded_msgs.items():
            for layer_idx, code in enumerate(codes):
                grad = self._coder.decode(code)
                if tuple(grad.shape) != self._model_shapes[layer_idx]:
                    grad = grad.reshape(self._model_shapes[layer_idx])
                self.aggregate_gradient(grad, layer_idx)
        return max(len(coded_msgs), 1)

    def aggregate_gradient(self, gradient: torch.Tensor, layer_idx: int):
        self.grad_accumulator.add(layer_idx, gradient)

    def _model_update(self, n_used: Optional[int] = None):
        n = float(n_used or self._num_workers)
        grads = [g / n for g in self.grad_accumulator.gradient_aggregator]
        if self._clip_grad_norm:
            grads, self.last_grad_norm = clip_grad_norm(grads, self._clip_grad_norm)
        self.optimizer.step(grads=grads, cuda=self._enable_gpu)
        if self.ema is not None:
            self._update_ema()

    def _generate_model_path(self):
        return ckpt.model_path(self._train_dir, self.cur_step)

    def _save_model(self, file_path=None):
        ckpt.save_model(self._train_dir, self.cur_step, self.network)
        if self.ema is not None:
            # the averaged weights with the live BN running statistics (from the first worker, _take_aux_buffers)
            sd = self.network.state_dict()
            sd.update({n: v.clone() for n, v in self._ema_views().items()})
            path = ckpt.model_path(self._train_dir, self.cur_step) + "_ema"
            torch.save(sd, path + ".tmp")
            os.replace(path + ".tmp", path)
        ckpt.save_sidecar(self._train_dir, self.cur_step, self.optimizer, lr=self.lr,
                          extra={"shrink_counter": self.shrink_counter})

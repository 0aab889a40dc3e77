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
* **Quantizing codes** (``code="qsgd" | "terngrad"``): every weight tensor is one QSGD unit of the plan; its
  buckets are quantized and bit-packed by the workers during backward straight into the owners' arenas
  (``csrc/v2_qsgd.cu``, TernGrad adds a per-tensor clip launch), and the owners decode, sum and step the
  optimizer in one launch per group.  BN and bias vectors stay fp32 (``multimem.ld_reduce``).
* **Entry-wise ATOMO** (``code="entrywise"``, ``entry_budget``): every weight tensor is one entry unit; a stats
  launch takes its fp64 L1 norm, the encode launch samples entries with ``p_i = min(1, s |g_i| / ||g||_1)`` and
  pushes them as 4-byte words (``csrc/v2_entrywise.cu``), and the owners scatter-add them in worker order and step
  the optimizer.  BN and bias vectors stay fp32, as above.
* **Top-k** (``code="topk"``, ``entry_budget``): the entry units, slots and PS of entry-wise ATOMO with ``k =
  floor(s)`` entries per tensor.  Two selection launches find each tensor's threshold magnitude from histograms of the
  bf16 bits, and the encode pushes the ``k`` largest entries exactly (``csrc/v2_topk.cu``).  Deterministic and
  biased on its own: it is the contractive code for ``error_feedback=True``.
* **Scaled sign** (``code="sign"``, ``bucket_size``): every weight's buckets are pushed as one bit per element and one
  fp32 scale ``||b||_1 / |b|`` in the slots and tiles of QSGD (``csrc/v2_sign.cu``, one encode launch per group); the
  owners decode ``+-scale``, sum in worker order and step the optimizer.  Deterministic, dense and biased on its own:
  the contractive code of EF-SignSGD for ``error_feedback=True``.
* **Signum with majority vote** (``code="signum"``, ``momentum`` = beta in ``[0, 1)``; SGD only): each worker keeps an
  fp32 momentum ``u <- beta u + g`` per weight and vector element (no buffer with ``beta == 0``: ``u = g``) and pushes
  ``sign(u)``, one bit per element and no scale, in the slots of sign with one 4096-element bucket per tile
  (``csrc/v2_signum.cu``, one encode launch per group that also forms the vectors' momentum in ``vgrads``).  A zero
  takes a fair Philox coin.  The owners count the 1 bits of the counted workers per element and step
  ``p <- p - lr * vote``, ``vote`` in {-1, 0, +1} (NaN when a counted worker's tile is not finite); vectors are voted on
  the sign of each worker's ``vgrads``.  Weight decay is decoupled and owner-side, the pass of AdamW before the PS
  launch.  The momentum lives in momentum correction's buffers and checkpoint keys.
* **Distributed Lion** (``code="dlion"``, ``betas`` = (b1, b2) default ``(0.9, 0.99)``, ``dlion_aggregate`` = ``"vote"``
  or ``"mean"``; SGD only): Signum's plan, push, buffers and decay with Lion's worker rule.  Each worker pushes the sign
  of ``c = b1 m + (1 - b1) g``, then ``m <- b2 m + (1 - b2) g`` (``v2_dlion_encode``; no buffer with ``b1 == 0``:
  ``c = g``).  The owners step ``p <- p - lr * v`` with ``v`` the vote (Signum's PS kernel) or the mean
  ``(pos - neg) / counted`` of the counted signs (``v2_ps_signum(mean=True)``).  ``momentum`` is ignored.
* **PowerSGD** (``code="powersgd"``, ``svd_rank`` = r in ``[1, 4]``): every weight matrix (``[O][C]`` in its physical
  layout) is pushed as a rank-``r`` pair from one power step warm-started by the previous step's right factor
  (``csrc/v2_powersgd.cu``, two encode launches per group); the owners reconstruct ``P_hat Q'^T`` in worker order and
  step the optimizer.  Deterministic, low-rank and biased on its own: a contractive code for ``error_feedback=True``.
  The warm state is per worker and is checkpointed with the residuals (``save_checkpoint``).
* **FP8** (``code="fp8"``, ``bucket_size``): every weight's buckets are pushed as one e4m3 byte per element and one
  power-of-two fp32 scale in the slots and tiles of sign (``csrc/v2_fp8.cu``, one encode launch per group); each
  scaled magnitude is rounded to one of its two e4m3 neighbours with Philox draws, so the code is unbiased.  The
  owners decode with the hardware conversion, sum in worker order and step the optimizer.
* **Randomized Hadamard** (``code="hadamard"``, ``quantization_level`` = bits in {2, 4, 8}, ``bucket_size`` a power
  of two): every weight's buckets are rotated by ``H D`` (Philox signs shared by all workers in a step) and pushed as
  ``bits``-bit codes between the bucket's min and max, stochastically rounded, with an fp32 ``(lo, step)`` per bucket
  (``csrc/v2_hadamard.cu``, one encode launch per group).  Unbiased.  The owners sum the workers' decodes in the
  rotated domain, apply one inverse transform per bucket and step the optimizer.
* **Error feedback** (``error_feedback=True``; svd, entrywise, topk, qsgd, sign, powersgd, fp8, hadamard): each worker keeps an fp32 residual ``e`` per
  weight element and codes ``A = g + e``.  An apply launch per group (``csrc/v2_feedback.cu``) writes ``bf16(A)`` into
  autograd's gradient buffer in place and keeps ``A - bf16(A)``; the encoders' epilogues add ``bf16(A) - g_hat``, the
  part of ``A`` this push did not carry.  Nothing is discarded, only delayed.  Each worker checkpoints its residual
  and warm-start state in ``model_step_<N>_worker<R>`` (``save_checkpoint``), so a resume continues bit for bit.
* **Gradient accumulation** (``accumulate_steps=N``): a step runs ``N`` micro-batches of ``B / N`` samples and pushes
  once.  For every micro-batch but the last, each group's hook adds the bf16 gradients into an fp32 accumulator on the
  encode stream (``csrc/v2_accum.cu``) and releases autograd's buffers, so no bf16 add ever happens; the vectors'
  ``vgrads`` are added and zeroed the same way.  Before the last micro-batch's encode a fold launch writes
  ``bf16((sum g_j) / N (+ e))`` into its gradient buffers in place (with error feedback it takes the place of the apply
  launch), so every code, ``code_stats`` and the residual work unchanged.  BN statistics take one update per
  micro-batch.  ``N = 1`` launches exactly what it launched before.
* **Momentum correction** (``momentum_correction=True``; top-k with error feedback and SGD only): Deep Gradient
  Compression's momentum on the workers, before the gradient is sparsified.  Each worker keeps an fp32 momentum ``u``
  per weight and vector element; per group, an apply launch (``csrc/v2_momentum.cu``, in place of the error-feedback
  apply) forms ``u = m u + g + wd w`` (``w`` the worker's bf16 weight) and codes ``A = u + e`` (Nesterov: ``d + m u +
  e``), and the top-k encode zeroes ``u`` at every entry it sent (momentum-factor masking).  Vectors travel exactly:
  ``vgrads`` becomes their momentum direction, unmasked.  The PS runs plain SGD on what it receives.  Unlike
  ``torch.optim.SGD``, weight decay uses the bf16 weight the worker trained with, not the owner's fp32 master.
* Optimizers fused in the PS epilogue: momentum-SGD (``src/optim/sgd.py:57-90``), Adam / AMSGrad
  (``src/optim/adam.py:37-94``).  LARS and LAMB (``optimizer="lars" | "lamb"``, ``trust_coefficient``) need whole-tensor
  norms first: the code's PS kernel runs its layer-wise instantiation (moments, direction, per-tile partials; vectors
  finished), then ``csrc/v2_layerwise.cu`` takes the norms across tiles and owners, the trust ratios and the step of
  the weights, and broadcasts them (``optim/lars.py`` / ``optim/lamb.py`` are the oracles).
* Gradient-norm clipping (``clip_grad_norm=MAX``, ``torch.nn.utils.clip_grad_norm_`` semantics): the code's PS kernel
  runs its gather instantiation per group (mean gradient and sum g^2 per tile, nothing stepped), then one launch per
  owner after the final group (``csrc/v2_clip.cu``) takes the whole-model norm across tiles and owners and steps every
  tile of the owner on ``coef * g`` (LARS / LAMB: their phase 2 follows per group).  ``grad_norm()`` reports it.
* Exponential moving average of the weights (``ema_decay=d``, ``0 < d < 1``): every owner keeps an fp32 average of
  every value it holds, ``ema`` indexed like ``master`` and ``vema`` like ``vparams``, starting at the initial
  weights.  Per group, one launch on the PS stream right after the launch that writes the group's final master values
  (``csrc/v2_ema.cu``; with clipping that is the end of the step) forms ``e <- e + w (p - e)`` with ``w = fp32(1 - d)``,
  each operation rounded to fp32.  ``ema_state_dict()`` gathers the averaged model; BN running statistics are not
  averaged: it carries the live ones.  Checkpoints add ``model_step_<N>_ema``.
* AdamW (``optimizer="adamw"``, ``torch.optim.AdamW`` with two parameter groups): per group, one launch on the PS
  stream right before the launch that steps the group's tiles (the PS launch; with clipping, the clip launch) scales
  the owner's weight elements of ``master`` by ``f = fp32(1 - lr * wd)`` (``csrc/v2_ema.cu``), read from
  ``Ctrl2.decay_factor``, which ``set_lr`` rewrites.  The PS kernels then run Adam (AMSGrad with ``amsgrad=True``)
  with weight decay 0.  1-D parameters (BN, biases) take no decay.  With ``weight_decay=0`` it is ``adam``, bit for
  bit, and launches nothing new.
* Lion (``optimizer="lion"``, ``betas`` default ``(0.9, 0.99)``; ``optim/lion.py`` is the oracle): the code's PS
  kernel runs its Lion instantiation (``v2_ps_lion``): ``p -= lr sign(b1 m + (1 - b1) g)``, ``m = b2 m + (1 - b2) g``
  on ``master`` / ``mom`` and ``vparams`` / ``vmom``, no second moments allocated.  Weight decay is AdamW's decay
  launch before it.  Clipping, Nesterov, AMSGrad, ``code="signum" | "dlion"`` and momentum correction are refused.

Per step and rank: ``wait_params`` -> forward -> backward [group hooks -> encode, project+push on stream E;
PS launch of the group on stream P] -> join -> ``advance_step``.  All cross-GPU ordering is carried by
step-stamped flags in peer memory (``csrc/v2_common.cuh``); no NCCL call on the path.
"""
from __future__ import annotations

import math
import numbers
import os
import struct
from typing import List, Optional

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn

from ..ops import plan2 as P2
from ..ops._ext import load as load_ext
from ..parallel.symm import SymmetricHeap
from ..utils.flags import check_clip_grad_norm, check_ema_decay

SIGNAL_INTS = 1024


def _dev_bytes(b: bytes, device) -> torch.Tensor:
    return torch.frombuffer(bytearray(b if len(b) else b"\0" * 16), dtype=torch.uint8).to(device)


class ShadowEngine:
    def __init__(self, model: nn.Module, rank: int = 0, world: int = 1, code: str = "svd", svd_rank: int = 3,
                 lr: float = 0.01, momentum: float = 0.0, weight_decay: float = 0.0, nesterov: bool = False,
                 dampening: float = 0.0, optimizer: str = "sgd", betas=None, eps: float = 1e-8,
                 amsgrad: bool = False, ps_mode: str = "sharded", groups: int = 5, sampling: str = "bernoulli",
                 prob_rule: str = "reference", random_sample: bool = True, seed: int = 1, use_graph: bool = True,
                 group=None, multicast: bool = True, heap_mode: str = "auto", timeout_s: float = 30.0,
                 criterion: Optional[nn.Module] = None, device: Optional[torch.device] = None,
                 ps_grid: int = 0, overlap: bool = True, fused_bn: bool = True, num_aggregate: int = 0,
                 warm_start: bool = True, max_sweeps: int = 1, main_priority: int = 0, debug_jitter_us: float = 0.0,
                 side_priority: int = -1, resample_empty: bool = False, quantization_level: int = 4,
                 bucket_size: int = 512, entry_budget: float = 0.05, code_stats: bool = False,
                 error_feedback: bool = False, accumulate_steps: int = 1, trust_coefficient: float = 0.001,
                 clip_grad_norm: float = 0.0, momentum_correction: bool = False, ema_decay: float = 0.0,
                 dlion_aggregate: str = "vote"):
        self.optimizer = optimizer.lower()
        if self.optimizer not in ("sgd", "adam", "adamw", "lars", "lamb", "lion"):      # checked before any CUDA work
            raise ValueError("ShadowEngine optimizers: sgd | adam | adamw | lars | lamb | lion (got %r)" % (optimizer,))
        self.code = {"dense": "sgd", "lossless": "sgd"}.get(code.lower(), code.lower())
        # Signum and Distributed Lion: the workers push the 1-bit sign of their own momentum and the owners step by the
        # aggregate; dlion differs only in the worker rule (two betas) and may average instead of voting
        self.dlion = self.code == "dlion"
        self.signum = self.code in ("signum", "dlion")
        self.lion = self.optimizer == "lion"
        if betas is None:
            betas = (0.9, 0.99) if self.lion or self.dlion else (0.9, 0.999)
        if self.lion or self.dlion:       # checked before any CUDA work
            if len(betas) != 2 or not all(not isinstance(b, bool) and isinstance(b, numbers.Real) and 0 <= b < 1
                                          for b in betas):
                raise ValueError("%s: betas must be two finite numbers in [0, 1) (got %r)"
                                 % ("lion" if self.lion else "dlion", betas))
        if self.lion:       # checked before any CUDA work
            if nesterov:
                raise ValueError("lion takes no Nesterov momentum: nesterov=False")
            if amsgrad:
                raise ValueError("lion keeps no second moment: amsgrad=False")
            if self.dlion:
                raise ValueError("lion cannot be combined with code='dlion': the owners step by the aggregate of the "
                                 "workers' Lion signs (code='dlion' alone runs Lion on the workers)")
            if self.signum:
                raise ValueError("lion cannot be combined with code='signum': the owners step by the vote")
            if momentum_correction:
                raise ValueError("lion cannot be combined with momentum_correction: the parameter server must run "
                                 "plain SGD")
            if check_clip_grad_norm(clip_grad_norm) > 0:
                raise ValueError("lion cannot be combined with clip_grad_norm yet: the clip launch steps Adam and "
                                 "momentum-SGD only")
        self.betas = (float(betas[0]), float(betas[1]))
        # AdamW, Lion and Signum: the PS kernels run with weight_decay 0; the decoupled decay of the weights is its own
        # pass
        self.adamw_wd = 0.0
        if self.optimizer in ("adamw", "lion") or self.signum:      # checked before any CUDA work
            if isinstance(weight_decay, bool) or not isinstance(weight_decay, numbers.Real) \
                    or not 0 <= weight_decay < math.inf:
                raise ValueError("%s: weight_decay must be finite and >= 0 (got %r)"
                                 % (self.code if self.signum else self.optimizer, weight_decay))
            self.adamw_wd, weight_decay = float(weight_decay), 0.0
        self.decay_on = self.adamw_wd > 0     # with weight_decay 0 AdamW is Adam: nothing new is launched
        self.layerwise = self.optimizer in ("lars", "lamb")
        if self.optimizer == "lars" and (nesterov or dampening != 0):
            raise ValueError("lars takes plain momentum: nesterov=False and dampening=0")
        if self.optimizer == "lars" and not trust_coefficient > 0:
            raise ValueError("lars: trust_coefficient must be positive (got %r)" % (trust_coefficient,))
        if self.optimizer == "lamb" and amsgrad:
            raise ValueError("lamb has no AMSGrad variant (amsgrad=False)")
        self.trust_coefficient = float(trust_coefficient)
        if isinstance(accumulate_steps, bool) or not isinstance(accumulate_steps, numbers.Integral) \
                or accumulate_steps < 1:        # checked before any CUDA work
            raise ValueError("accumulate_steps must be an integer >= 1 (got %r)" % (accumulate_steps,))
        self.clip_grad_norm = check_clip_grad_norm(clip_grad_norm)      # checked before any CUDA work
        self.clip_on = self.clip_grad_norm > 0
        self.ema_decay = check_ema_decay(ema_decay)      # checked before any CUDA work
        self.ema_w = float(np.float32(1.0 - self.ema_decay))    # the average's step weight, rounded once
        if self.code not in ("svd", "sgd", "qsvd", "qsgd", "terngrad", "entrywise", "topk", "sign", "signum", "dlion",
                             "powersgd", "fp8", "hadamard"):
            raise ValueError("ShadowEngine codes: svd | qsvd | sgd | qsgd | terngrad | entrywise | topk | sign | signum "
                             "| dlion | powersgd | fp8 | hadamard")
        self.dlion_aggregate = dlion_aggregate
        if self.dlion:      # checked before any CUDA work; momentum is ignored, as Lion ignores it
            if self.optimizer != "sgd":
                raise ValueError("dlion runs Lion on the workers and steps the owners by the aggregate of their signs: "
                                 "optimizer='sgd' only (got %r)" % (optimizer,))
            if nesterov:
                raise ValueError("dlion takes Lion's momentum on the workers: nesterov=False")
            if dampening != 0:
                raise ValueError("dlion takes dampening=0 (got %r)" % (dampening,))
            if error_feedback:
                raise ValueError("dlion sends the sign of the Lion direction without a residual: error_feedback=False")
            if code_stats:
                raise ValueError("code_stats has no estimator model for an aggregate of signs (dlion)")
            if check_clip_grad_norm(clip_grad_norm) > 0:
                raise ValueError("dlion cannot be combined with clip_grad_norm: the aggregate of signs has no gradient "
                                 "norm to clip")
            if momentum_correction:
                raise ValueError("dlion keeps its own worker momentum: momentum_correction=False")
            if dlion_aggregate not in ("vote", "mean"):
                raise ValueError("dlion_aggregate: vote | mean (got %r)" % (dlion_aggregate,))
        elif self.signum:     # checked before any CUDA work
            if self.optimizer != "sgd":
                raise ValueError("signum steps the owners by the vote of the workers' momentum signs: optimizer='sgd' "
                                 "only (got %r)" % (optimizer,))
            if nesterov:
                raise ValueError("signum takes heavy-ball momentum on the workers: nesterov=False")
            if dampening != 0:
                raise ValueError("signum takes dampening=0 (got %r)" % (dampening,))
            if isinstance(momentum, bool) or not isinstance(momentum, numbers.Real) or not 0 <= momentum < 1:
                raise ValueError("signum: momentum (the workers' beta) must be in [0, 1) (got %r)" % (momentum,))
            if error_feedback:
                raise ValueError("signum sends sign(momentum) without a residual: error_feedback=False (use "
                                 "code='sign' for EF-SignSGD)")
            if code_stats:
                raise ValueError("code_stats has no estimator model for a majority vote (signum)")
            if check_clip_grad_norm(clip_grad_norm) > 0:
                raise ValueError("signum cannot be combined with clip_grad_norm: every step has length lr per element")
            if momentum_correction:
                raise ValueError("signum keeps its own worker momentum: momentum_correction=False")
        self.power = self.code == "powersgd"
        if self.power and not 1 <= int(svd_rank) <= P2.POWER_MAX_RANK:      # checked before any CUDA work
            raise ValueError("powersgd: svd_rank must be in [1, %d] (got %r)" % (P2.POWER_MAX_RANK, svd_rank))
        self.error_feedback = bool(error_feedback)
        if self.error_feedback:     # checked before any CUDA work
            if self.code == "qsvd":
                raise ValueError("error_feedback: QSVD rounds its int8 left factors after the residual would be "
                                 "formed (use code='svd')")
            if self.code == "terngrad":
                raise ValueError("error_feedback: TernGrad's owners rescale every worker by a shared max norm, so a "
                                 "worker cannot know what it contributed")
            if self.code == "sgd":
                raise ValueError("error_feedback: the dense code sends the gradient exactly; there is nothing to "
                                 "feed back")
            n_workers = world - 1 if (ps_mode == "dedicated" and world > 1) else world
            if 0 < num_aggregate < n_workers:
                raise ValueError("error_feedback needs every push counted (num_aggregate=0 or >= workers): a "
                                 "dropped push would lose its residual credit")
        if code_stats:      # checked before any CUDA work: the closed forms of code_stats() do not hold for these
            if self.code == "qsvd":
                raise ValueError("code_stats does not model the int8 quantization of QSVD's left factors")
            if resample_empty:
                raise ValueError("code_stats needs resample_empty=False: redrawing empty selections biases the "
                                 "estimator, and the closed-form error no longer holds")
        self.entry = self.code in ("entrywise", "topk")
        self.topk = self.code == "topk"
        self.entry_budget = float(entry_budget)
        if self.entry:      # checked before any CUDA work
            if prob_rule != "reference" or sampling != "bernoulli":
                raise ValueError("%s on ShadowEngine runs with prob_rule='reference' and sampling='bernoulli' only "
                                 "(got %r / %r)" % (self.code, prob_rule, sampling))
            if not self.entry_budget > 0:
                raise ValueError("entry_budget must be positive (a fraction of numel below 1, else an atom count)")
        self.sign = self.code == "sign"
        self.fp8 = self.code == "fp8"
        if self.sign or self.fp8:       # checked before any CUDA work
            if not (P2.SIGN_MIN_BUCKET <= int(bucket_size) <= P2.SIGN_MAX_BUCKET and int(bucket_size) % 64 == 0):
                raise ValueError("%s: bucket_size must be a multiple of 64 in [%d, %d] (got %r)"
                                 % (self.code, P2.SIGN_MIN_BUCKET, P2.SIGN_MAX_BUCKET, bucket_size))
        self.hadamard = self.code == "hadamard"
        if self.hadamard:       # checked before any CUDA work
            if int(quantization_level) not in P2.HADAMARD_BITS:
                raise ValueError("hadamard: quantization_level (bits) must be 2, 4 or 8 (got %r)" % (quantization_level,))
            hb = int(bucket_size)
            if not (P2.HADAMARD_MIN_BUCKET <= hb <= P2.HADAMARD_MAX_BUCKET and hb & (hb - 1) == 0):
                raise ValueError("hadamard: bucket_size must be a power of two in [%d, %d] (got %r)"
                                 % (P2.HADAMARD_MIN_BUCKET, P2.HADAMARD_MAX_BUCKET, bucket_size))
        self.momentum_correction = bool(momentum_correction)
        if self.momentum_correction:        # checked before any CUDA work
            if self.code != "topk" or not self.error_feedback:
                raise ValueError("momentum_correction needs code='topk' with error_feedback=True: masking the momentum "
                                 "of the entries sent has no meaning for the other codes (got code=%r, "
                                 "error_feedback=%r)" % (self.code, self.error_feedback))
            if self.optimizer != "sgd":
                raise ValueError("momentum_correction moves momentum-SGD to the workers: optimizer='sgd' only "
                                 "(got %r)" % (optimizer,))
            if dampening != 0:
                raise ValueError("momentum_correction takes dampening=0 (got %r)" % (dampening,))
            if isinstance(momentum, bool) or not isinstance(momentum, numbers.Real) or not 0 <= momentum < math.inf:
                raise ValueError("momentum_correction needs a finite momentum >= 0 (got %r)" % (momentum,))
            if self.clip_on:
                raise ValueError("momentum_correction cannot be combined with clip_grad_norm: the workers' momentum "
                                 "would run on the unclipped gradient")
            if accumulate_steps != 1:
                raise ValueError("momentum_correction cannot be combined with accumulate_steps > 1")
        self.C = load_ext()
        C = self.C
        assert C.v2_unit_bytes() == P2.UNIT_BYTES and C.v2_ctrl_bytes() == P2.CTRL2_BYTES
        self.rank, self.world, self.group = rank, world, group
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        dev = self.device
        self.svd_rank = int(svd_rank)
        self.quant = self.code in ("qsgd", "terngrad")
        self.quantization_level, self.bucket_size = int(quantization_level), int(bucket_size)
        if self.quant:
            if not 1 <= self.quantization_level <= P2.QSGD_MAX_LEVEL:
                raise ValueError("quantization_level must be in [1, %d]" % P2.QSGD_MAX_LEVEL)
            if not (32 <= self.bucket_size <= P2.QSGD_MAX_BUCKET and self.bucket_size % 8 == 0):
                raise ValueError("bucket_size must be a multiple of 8 in [32, %d]" % P2.QSGD_MAX_BUCKET)
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
        # micro-batches per step; a dedicated PS rank runs no backward and ignores the setting
        self.accum = int(accumulate_steps) if self.is_worker else 1
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
        adam_opt = P2.OPT_AMSGRAD if amsgrad else P2.OPT_ADAM
        self.opt = {"sgd": P2.OPT_SGD, "adam": adam_opt, "adamw": adam_opt, "lars": P2.OPT_LARS,
                    "lamb": P2.OPT_LAMB, "lion": P2.OPT_LION}[self.optimizer]
        self.launches_per_step = 0

        # ---- model: NHWC activations, fused BN ------------------------------------------------------------
        self.model = model.to(dev).to(memory_format=torch.channels_last)
        self.fused_bn_layers, self.bn_arena = 0, None
        if fused_bn:
            from ..ops.fused_bn import enable_fused_bn
            self.fused_bn_layers, self.bn_arena = enable_fused_bn(self.model, True, arena_device=dev)
        self.params = list(self.model.parameters())
        shapes = [tuple(p.shape) for p in self.params]
        self.plan = P2.build_plan2(shapes, "signum" if self.dlion else self.code, self.svd_rank, self.systematic, n_owners=self.n_owners,
                                   n_groups=groups if overlap else 1, quantization_level=self.quantization_level,
                                   bucket_size=self.bucket_size, entry_budget=self.entry_budget)
        pl = self.plan
        self.G = pl.n_groups

        # ---- symmetric heap ---------------------------------------------------------------------------------
        # LARS / LAMB: per group, the per-tensor norms every owner exchanges ([2 step parities][owner][tensor][2] fp64)
        self.lw_tile_layer, self.lw_layers = P2.layerwise_tables(pl) if self.layerwise else ([], [])
        self.lw_xch_off = [2 * 2 * self.n_owners * sum(self.lw_layers[:g]) for g in range(self.G)]
        xch_doubles = 2 * 2 * self.n_owners * sum(self.lw_layers)
        # gradient-norm clipping: every owner's sum of g^2 ([2 step parities][owner] fp64)
        clip_doubles = 2 * self.n_owners if self.clip_on else 0
        need = 4 * SIGNAL_INTS + 2 * pl.w_total + 8 * pl.v_total + 2 * pl.stage_total + \
            4 * pl.arena_floats * self.W + 8 * xch_doubles + 8 * clip_doubles + (1 << 16)
        self.heap = h = SymmetricHeap(need + (1 << 20), rank, world, dev.index, group=group, multicast=multicast,
                                      mode=heap_mode)
        h.alloc("signals", 4 * SIGNAL_INTS)
        h.alloc("wshadow", 2 * pl.w_total)
        h.alloc("vparams", 4 * pl.v_total)
        h.alloc("vgrads", 4 * pl.v_total)
        h.alloc("wstage", 2 * pl.stage_total)
        h.alloc("arena", 4 * pl.arena_floats * self.W)
        if self.layerwise:
            h.alloc("lwx", 8 * max(xch_doubles, 2))
        if self.clip_on:
            h.alloc("clipx", 8 * clip_doubles)
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
        adam = self.opt in (P2.OPT_ADAM, P2.OPT_AMSGRAD, P2.OPT_LAMB)
        if self.is_owner:
            self.mom, self.vmom = z(pl.w_total), z(pl.v_total)
            self.sq, self.vsq = (z(pl.w_total), z(pl.v_total)) if adam else (None, None)
            self.sqmax, self.vsqmax = (z(pl.w_total), z(pl.v_total)) if self.opt == P2.OPT_AMSGRAD else (None, None)
        else:
            self.master = None
        # exponential moving average of the weights (csrc/v2_ema.cu): the owner's fp32 average of master and vparams,
        # starting at the initial weights every rank now holds
        self.ema = self.vema = None
        if self.ema_decay and self.is_owner:
            self.ema, self.vema = self.master.clone(), self.vparams.clone()

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
        self.warm_start = bool(warm_start)
        self.max_sweeps = int(max_sweeps) if warm_start else 0
        self.vprev = None
        if warm_start and not self.quant and not self.entry and not self.sign and not self.power and not self.fp8 \
                and not self.hadamard and not self.signum:
            self.vprev = z(nc * P2.MAX_COLS * P2.MAX_COLS)      # set by _fresh_worker_state()
        # QSGD: largest level / bucket of the plan (checked by the bindings), TernGrad clip per unit + its partials
        qunits = [u for u in pl.units if u.kind == P2.KIND_QSGD]
        self.q_max_level = max((u.I for u in qunits), default=0)
        self.q_max_bucket = max((u.K for u in qunits), default=0)
        self.clip = self.clip_partials = None
        if self.code == "terngrad":
            self.clip = z(nc)
            self.clip_partials = torch.zeros(2 * max(len(pl.enc_tiles), 1), dtype=torch.float64, device=dev)
        # entry-wise: fp64 L1 norm per unit and its per-tile partials
        self.l1 = self.l1_partials = None
        # top-k: selection state and histogram per unit (the histogram is zero between launches), tie counts per tile
        self.topk_sel = self.topk_hist = self.topk_tiles = None
        if self.topk:
            n_state, n_hi, n_lo = C.v2_topk_sizes()
            assert (n_state, n_hi, n_lo) == (P2.TOPK_STATE_INTS, P2.TOPK_HI_BINS, P2.TOPK_LO_BINS)
            i32 = lambda n: torch.zeros(n, dtype=torch.int32, device=dev)
            self.topk_sel, self.topk_hist = i32(nc * n_state), i32(nc * n_hi)
            self.topk_tiles = i32(max(len(pl.enc_tiles), 1) * n_lo)
        elif self.entry:
            self.l1 = torch.zeros(nc, dtype=torch.float64, device=dev)
            self.l1_partials = torch.zeros(max(len(pl.enc_tiles), 1), dtype=torch.float64, device=dev)
        # PowerSGD: pass-B tiles, fp64 Gram partials per pass-A tile, per-unit state (R^{-1}, mask, draw counter, unit
        # counters); the factors and the warm Q_w live in ``gpart`` (ops/plan2.py pw_scratch_floats)
        self.pw_state = self.pw_gram = self.t_pw_tiles = None
        if self.power:
            self.t_pw_tiles = _dev_bytes(P2.Plan2.tiles_bytes(pl.pw_tiles), dev)
            self.pw_gram = torch.zeros(P2.PW_GRAM * max(len(pl.enc_tiles), 1), dtype=torch.float64, device=dev)
            self.pw_state = torch.zeros(nc * C.v2_powersgd_state_bytes(), dtype=torch.uint8, device=dev)
        self.counters = torch.zeros(nc + 2 * P2.MAX_GROUPS + 8, dtype=torch.int32, device=dev)
        self.cnt_enc_group = self.counters.data_ptr() + 4 * nc
        self.cnt_ps_group = self.cnt_enc_group + 4 * P2.MAX_GROUPS
        # momentum correction: momentum, weight decay and Nesterov act on the workers (v2_mc_apply), the PS runs plain SGD
        self.mc_momentum, self.mc_weight_decay, self.mc_nesterov = float(momentum), float(weight_decay), bool(nesterov)
        if self.momentum_correction or self.signum or self.lion:     # lion: --momentum is ignored, as for Adam
            momentum, dampening, weight_decay, nesterov = 0.0, 0.0, 0.0, False
        self.ctrl = _dev_bytes(P2.pack_ctrl2(step=1, lr=lr, momentum=momentum, dampening=dampening,
                                             weight_decay=weight_decay, nesterov=nesterov, first_step=1, seed=seed,
                                             beta1=self.betas[0], beta2=self.betas[1], eps=eps, opt=self.opt,
                                             num_aggregate=num_aggregate,
                                             trust_coefficient=self.trust_coefficient if self.layerwise else 0.0,
                                             clip_grad_norm=self.clip_grad_norm,
                                             decay_factor=self.decay_factor(lr) if self.decay_on else 0.0), dev)
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
        # LARS / LAMB (csrc/v2_layerwise.cu): the owner's direction per weight element (indexed like master), the
        # (sum w^2, sum x^2) of every PS tile, the tensor of every PS tile, the exchange slots and the trust ratios
        self.lw_dir = self.lw_part = self.t_lw_tile_layer = self.lw_ratio = self.lw_counter = None
        self.t_lw_xch_peer = []
        if self.layerwise:
            if max(self.lw_layers, default=0) > C.v2_layerwise_max_layers():
                raise ValueError("lars / lamb: at most %d weight tensors per backward group (use more groups)"
                                 % C.v2_layerwise_max_layers())
            self.lw_ratio = z(max(sum(self.lw_layers), 1))
            self.lw_counter = torch.zeros(P2.MAX_GROUPS, dtype=torch.int32, device=dev)
            if self.is_owner:
                self.lw_dir = z(pl.w_total)
                self.lw_part = z(2 * max(len(pl.ps_tiles), 1))
                self.t_lw_tile_layer = torch.tensor(self.lw_tile_layer or [0], dtype=torch.int32, device=dev)
            self.t_lw_xch_peer = [i64(h.region_ptr("lwx", r) + 8 * self.lw_xch_off[g] for r in range(world))
                                  for g in range(self.G)]
        # gradient-norm clipping (csrc/v2_clip.cu): the owner's mean gradient per element (LARS / LAMB: in lw_dir, which
        # phase 2 overwrites with the direction) and per vector element, sum g^2 of every PS tile, the owner's PS tiles
        # of every group, a completion counter, the exchange slots and the last (total, coef)
        self.clip_grad = self.clip_vgrad = self.clip_part = self.t_clip_tiles = self.clip_counter = None
        self.clip_norm, self.clip_tiles, self.t_clip_xch_peer = None, [], None
        if self.clip_on:
            self.clip_norm = z(2)
            if self.is_owner:
                self.clip_grad = self.lw_dir if self.layerwise else z(pl.w_total)
                self.clip_vgrad = z(pl.v_total)
                self.clip_part = z(2 * max(len(pl.ps_tiles), 1))
                self.clip_tiles = P2.owner_ps_tiles(pl, self.owner_index)
                self.t_clip_tiles = torch.tensor(self.clip_tiles or [0], dtype=torch.int32, device=dev)
                self.clip_counter = torch.zeros(1, dtype=torch.int32, device=dev)
            self.t_clip_xch_peer = i64(h.region_ptr("clipx", r) for r in range(world))
        self.tstats = torch.zeros(32, dtype=torch.int64, device=dev)
        # --code-stats: per coded unit fp64 sums over steps (v2_stats.cu), the per-tile partials and unit counters
        self.code_stats_on = bool(code_stats)
        self.stats_acc = self.stats_partials = self.stats_counters = None
        if self.code_stats_on and self.code != "sgd":
            self.stats_acc = torch.zeros(nc * C.v2_stats_fields(), dtype=torch.float64, device=dev)
            self.stats_partials = torch.zeros(max(len(pl.enc_tiles), 1) * C.v2_stats_partials(), dtype=torch.float64,
                                              device=dev)
            self.stats_counters = torch.zeros(nc, dtype=torch.int32, device=dev)
        # error feedback: fp32 residual per weight element (wshadow's physical order) and the apply chunks per group
        self.residual = self.t_ef_chunks = None
        self.ef_range = []
        if (self.error_feedback or self.accum > 1) and self.is_worker:
            assert C.v2_ef_chunk_bytes() == struct.calcsize(P2.EF_CHUNK_FMT)
            if self.error_feedback:
                self.residual = z(pl.w_total)
            chunks, self.ef_range = P2.ef_chunks(pl)
            self.t_ef_chunks = _dev_bytes(chunks, dev)
        # gradient accumulation (accumulate_steps > 1, csrc/v2_accum.cu): fp32 sums of the micro-batches' weight and
        # vector gradients (zero at every step boundary), the vector chunks per group, and one gradient-pointer table
        # per micro-batch before the last (each micro-batch's gradients live at their own addresses; the last one
        # uses t_gptr, which the encoders read)
        self.acc = self.vacc = self.t_vec_chunks = self.t_aptr = self.host_aptr = None
        self.vec_range = []
        if self.accum > 1 or ((self.momentum_correction or self.signum) and self.is_worker):
            vchunks, self.vec_range = P2.vec_chunks(pl)
            self.t_vec_chunks = _dev_bytes(vchunks, dev)
        if self.accum > 1:
            self.acc, self.vacc = z(pl.w_total), z(pl.v_total)
            self.t_aptr = torch.zeros((self.accum - 1, n_w), dtype=torch.int64, device=dev)
            self.host_aptr = np.zeros((self.accum - 1, n_w), dtype=np.int64)
        self.inv_n = float(np.float32(1.0 / self.accum))
        # momentum correction (csrc/v2_momentum.cu), Signum with beta > 0 and Distributed Lion with b1 > 0
        # (csrc/v2_signum.cu): the worker's fp32 momentum per weight element (wshadow's physical order, the residual's
        # offsets) and per vector element (vgrads' order)
        self.mc_mom = self.mc_vmom = None
        worker_beta = self.betas[0] if self.dlion else self.mc_momentum
        if (self.momentum_correction or (self.signum and worker_beta > 0)) and self.is_worker:
            self.mc_mom, self.mc_vmom = z(pl.w_total), z(pl.v_total)
        self.pw_warm = P2.pw_warm_ranges(pl) if self.power else []     # Q_w inside gpart (checkpointed)
        self._fresh_worker_state()
        self.loss_buf = torch.zeros(3, dtype=torch.float32, device=dev)
        self.static_x = self.static_y = self.graph = None

        # ---- streams / events --------------------------------------------------------------------------------
        self.s_enc = torch.cuda.Stream(device=dev, priority=side_priority)
        self.s_ps = torch.cuda.Stream(device=dev, priority=side_priority)
        self.s_main = torch.cuda.Stream(device=dev, priority=main_priority)   # warm-up + capture stream
        # with the fused BN, the convolutions' weight gradients run on a stream of their own, beside the backward
        # chain (ops/split_conv.py); the encode of a group waits for it.  Same priority as the backward: the main
        # stream is at the lowest priority by default, and the wgrad is as urgent as the rest of the backward.
        self.s_wgrad, self.ev_wgrad, self.split_wgrad_layers = None, [], 0
        self.group_w_params = [[p for p, q in zip(self.params, pl.params) if q.is_w and q.group == g]
                               for g in range(self.G)]
        if self.fused_bn_layers and self.is_worker:
            from ..ops.split_conv import enable_split_wgrad
            self.s_wgrad = torch.cuda.Stream(device=dev, priority=main_priority)
            self.split_wgrad_layers = enable_split_wgrad(self.model, self.s_wgrad)
            if self.split_wgrad_layers:
                self.ev_wgrad = [torch.cuda.Event() for _ in range(self.G)]
            else:
                self.s_wgrad = None
        self.ev_ready = [torch.cuda.Event() for _ in range(self.G)]
        self.ev_push = [torch.cuda.Event() for _ in range(self.G)]
        self.ev_enc_done, self.ev_ps_done = torch.cuda.Event(), torch.cuda.Event()
        self.ev_acc_done = torch.cuda.Event()      # the adds of a micro-batch have read (and zeroed) vgrads
        self._pending, self._fired, self._nlaunch, self._micro = list(self.group_size), 0, 0, 0
        self._capturing = False
        self._initial_sync()

    # ------------------------------------------------------------------------------------------------------
    def _fresh_worker_state(self):
        """Per-worker state as a new run starts it: residual ``e = 0``, the identity as the Jacobi warm start, and
        PowerSGD's first draw of ``Q_w`` (Philox keyed by seed, unit, column) with a cleared unit state."""
        if self.residual is not None:
            self.residual.zero_()
        if self.mc_mom is not None:
            self.mc_mom.zero_()
            self.mc_vmom.zero_()
        if self.vprev is not None:
            self.vprev.zero_()
            for u in self.plan.units:
                if u.coded:
                    o = u.ts_index * P2.MAX_COLS * P2.MAX_COLS
                    self.vprev[o:o + u.cols * u.cols].copy_(torch.eye(u.cols, device=self.device).reshape(-1))
        if self.power and self.is_worker:
            self.pw_state.zero_()
            self.C.v2_powersgd_init(self.t_units.data_ptr(), len(self.plan.units), self.gpart.data_ptr(),
                                    self.ctrl.data_ptr())

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
        if self.decay_on:
            self.ctrl_f32[17] = self.decay_factor(lr)      # Ctrl2::decay_factor, read by every decay launch

    def decay_factor(self, lr: float) -> float:
        """AdamW, Lion and Signum: the factor of the decoupled weight decay at learning rate ``lr``, ``1 - lr * wd`` in double
        (as torch.optim.AdamW computes it in Python) rounded to fp32 once."""
        return float(np.float32(1.0 - float(lr) * self.adamw_wd))

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

    def code_stats(self, reset: bool = True) -> dict:
        """Estimator statistics of this worker's code since the last reset (``code_stats=True``), as means per step:
        per parameter tensor (the block units of a tensor summed) and for the whole model,

        * ``gsq``       ``||g||^2`` of the bf16 gradient the encoder read (coded tensors; None for tensors that travel
                        exactly: 1-D vectors in fp32, dense bf16 weights).  With ``error_feedback=True`` the encoder
                        reads the coded input ``bf16(g + e)``, so every statistic describes that input, not ``g``,
        * ``mse``       the expected ``||g_hat - g||^2`` given that gradient, in closed form (exact, not sampled);
                        ``rel_var`` = ``mse / gsq``,
        * ``bias_sq``   TernGrad's clip bias ``||clip(g) - g||^2`` (0 for the other codes; not part of ``mse``),
        * ``exp_atoms`` / ``atoms``  expected and realized atoms (QSGD / TernGrad / sign / fp8 / hadamard: every element; PowerSGD: the
                        non-degenerate columns of ``P_hat``), exact tensors their element count,
        * ``bytes``     realized push bytes: the spectral slot layout, ``entry_bytes()`` / ``qsgd_bytes()`` applied to
                        the realized counts, dense bytes for exact tensors.

        The whole-model ``rel_var`` is the summed ``mse`` over the summed ``gsq`` of the coded tensors.  Reading it
        synchronises the device; ``reset`` zeroes the sums."""
        if not self.code_stats_on:
            raise RuntimeError("code_stats() needs ShadowEngine(..., code_stats=True)")
        pl, nf = self.plan, self.C.v2_stats_fields()
        acc = self.stats_acc.view(-1, nf).tolist() if self.stats_acc is not None else []
        names = {id(p): n for n, p in self.model.named_parameters()}
        per = {}
        for u in pl.units:
            q = pl.params[u.param]
            name = names.get(id(self.params[u.param]), str(u.param))
            t = per.setdefault(name, {"numel": q.numel, "gsq": None, "mse": 0.0, "bias_sq": 0.0, "exp_atoms": 0.0,
                                      "atoms": 0.0, "bytes": 0.0})
            if u.kind in (P2.KIND_SLAB, P2.KIND_MAT, P2.KIND_ENTRY, P2.KIND_QSGD, P2.KIND_SIGN, P2.KIND_POWER,
                          P2.KIND_FP8, P2.KIND_HADAMARD) and acc:
                gsq, mse, ex, bias, real, real4, n = acc[u.ts_index]
                n = max(n, 1.0)
                t["gsq"] = (t["gsq"] or 0.0) + gsq / n
                t["mse"] += mse / n
                t["bias_sq"] += bias / n
                t["exp_atoms"] += ex / n
                t["atoms"] += real / n
                if u.kind in (P2.KIND_QSGD, P2.KIND_SIGN, P2.KIND_FP8):
                    t["bytes"] += 8.0 * u.rows * u.cols + 4.0 * u.rows
                elif u.kind == P2.KIND_HADAMARD:
                    t["bytes"] += 8.0 * u.rows * u.cols + 8.0 * u.rows
                elif u.kind == P2.KIND_POWER:
                    t["bytes"] += 4.0 * u.rcap * (u.rows + u.cols)
                elif u.kind == P2.KIND_ENTRY:
                    t["bytes"] += 4.0 * real / n + 16.0 * u.n_ps
                else:
                    t["bytes"] += 4.0 * (4 + u.rcap + u.rcap * u.cols) + 4.0 * u.rows * real4 / n
            else:       # travels exactly: fp32 vector, or a dense bf16 weight
                t["exp_atoms"] += u.numel
                t["atoms"] += u.numel
                t["bytes"] += (2.0 if u.kind == P2.KIND_DENSE16 else 4.0) * u.numel
        for t in per.values():
            t["rel_var"] = t["mse"] / t["gsq"] if t["gsq"] else (0.0 if t["gsq"] is None else None)
        coded = [t for t in per.values() if t["gsq"] is not None]
        tot = {k: sum(t[k] for t in per.values()) for k in ("mse", "bias_sq", "exp_atoms", "atoms", "bytes")}
        tot["gsq"] = sum(t["gsq"] for t in coded)
        tot["rel_var"] = tot["mse"] / tot["gsq"] if tot["gsq"] > 0 else 0.0
        steps = int(acc[0][-1]) if acc else 0
        if reset and self.stats_acc is not None:
            self.stats_acc.zero_()
        return {"code": self.code, "steps": steps, "model": tot, "tensors": per}

    def error_feedback_norm(self) -> dict:
        """``||e||`` of this worker's error-feedback residual: per weight tensor and for the whole model
        (``error_feedback=True``).  Reading it synchronises the device."""
        if self.residual is None:
            raise RuntimeError("error_feedback_norm() needs ShadowEngine(..., error_feedback=True) on a worker")
        names = {id(p): n for n, p in self.model.named_parameters()}
        ws = [(names.get(id(p), str(q.index)), q) for p, q in zip(self.params, self.plan.params) if q.is_w]
        sq = torch.stack([self.residual[q.off:q.off + q.numel].double().square().sum() for _, q in ws]).tolist()
        return {"model": float(sum(sq)) ** 0.5, "tensors": {n: v ** 0.5 for (n, _), v in zip(ws, sq)}}

    def momentum_correction_norm(self) -> dict:
        """``||u||`` of this worker's momentum (``momentum_correction=True``, ``code="signum"`` with
        ``momentum > 0``, or ``code="dlion"`` with ``b1 > 0``): per parameter tensor (weights and vectors) and for the
        whole model.  Reading it synchronises the device."""
        if self.mc_mom is None:
            raise RuntimeError("momentum_correction_norm() needs ShadowEngine(..., momentum_correction=True), "
                               "code='signum' with momentum > 0 or code='dlion' with b1 > 0, on a worker")
        names = {id(p): n for n, p in self.model.named_parameters()}
        ts = [(names.get(id(p), str(q.index)), (self.mc_mom if q.is_w else self.mc_vmom)[q.off:q.off + q.numel])
              for p, q in zip(self.params, self.plan.params)]
        sq = torch.stack([t.double().square().sum() for _, t in ts]).tolist()
        return {"model": float(sum(sq)) ** 0.5, "tensors": {n: v ** 0.5 for (n, _), v in zip(ts, sq)}}

    def _launch_code_stats(self, g: int):
        """Estimator statistics of group ``g``: after its push on the same stream (the gradient, this step's sigma /
        selcount / L1 / clip and this worker's slot headers and norms are live until the next encode)."""
        t0, nt = self.plan.enc_range[g]
        if self.stats_acc is None or nt == 0:
            return
        p = lambda t: t.data_ptr() if t is not None else 0
        if self.power:
            self.C.v2_powersgd_code_stats(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt,
                                          self.t_gptr.data_ptr(), self.gpart.data_ptr(), self.pw_state.data_ptr(),
                                          self.stats_partials.data_ptr(), self.stats_counters.data_ptr(),
                                          self.stats_acc.data_ptr())
            self._nlaunch += 1
            return
        if self.hadamard:
            self.C.v2_hadamard_code_stats(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt,
                                          self.t_gptr.data_ptr(), self.t_arena_peer.data_ptr(), self.n_owners,
                                          self.plan.arena_floats, self.worker_index, self.ctrl.data_ptr(),
                                          self.stats_partials.data_ptr(), self.stats_counters.data_ptr(),
                                          self.stats_acc.data_ptr())
            self._nlaunch += 1
            return
        if self.sign or self.fp8:
            stats = self.C.v2_sign_code_stats if self.sign else self.C.v2_fp8_code_stats
            stats(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                  self.t_arena_peer.data_ptr(), self.n_owners, self.plan.arena_floats, self.worker_index,
                  self.stats_partials.data_ptr(), self.stats_counters.data_ptr(), self.stats_acc.data_ptr())
            self._nlaunch += 1
            return
        if self.topk:
            self.C.v2_topk_code_stats(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt,
                                      self.t_gptr.data_ptr(), self.topk_sel.data_ptr(), self.topk_tiles.data_ptr(),
                                      self.t_arena_peer.data_ptr(), self.n_owners, self.plan.arena_floats,
                                      self.worker_index, self.stats_partials.data_ptr(),
                                      self.stats_counters.data_ptr(), self.stats_acc.data_ptr())
            self._nlaunch += 1
            return
        spectral = self.code == "svd"
        self.C.v2_code_stats(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                             self.sigma.data_ptr() if spectral else 0, self.selcount.data_ptr(), p(self.l1),
                             p(self.clip), self.t_arena_peer.data_ptr(), self.n_owners, self.plan.arena_floats,
                             self.worker_index, self.random_sample, self.waterfill, self.stats_partials.data_ptr(),
                             self.stats_counters.data_ptr(), self.stats_acc.data_ptr())
        self._nlaunch += 1

    # ------------------------------------------------------------------------------------------------------
    def _make_hook(self, i: int):
        q = self.plan.params[i]

        def hook(p):
            if q.is_w:
                j = self._micro
                (self.host_gptr if j == self.accum - 1 else self.host_aptr[j])[q.widx] = p.grad.data_ptr()
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
        res = self.residual.data_ptr() if self.residual is not None else 0
        if self.acc is not None:
            # the last micro-batch: A = (sum of the micro-batches) / N (+ e) into its gradient buffers (bf16), the
            # rounding remainder into the residual, the vectors' mean into vgrads; the accumulators back to zero
            (c0, nw), (v0, nv), cb = self.ef_range[g], self.vec_range[g], struct.calcsize(P2.EF_CHUNK_FMT)
            C.v2_accum_fold(self.t_ef_chunks.data_ptr() + cb * c0, nw, self.t_vec_chunks.data_ptr() + cb * v0, nv,
                            self.t_gptr.data_ptr(), self.acc.data_ptr(), self.vacc.data_ptr(), self.vgrads.data_ptr(),
                            self.inv_n, res)
            self._nlaunch += 1
        elif self.momentum_correction:
            # momentum correction: u = m u + g (+ wd w), A = u (Nesterov: d + m u) + e into the gradient buffers
            # (bf16) and the residual; the vectors' direction into vgrads
            (c0, nw), (v0, nv), cb = self.ef_range[g], self.vec_range[g], struct.calcsize(P2.EF_CHUNK_FMT)
            C.v2_mc_apply(self.t_ef_chunks.data_ptr() + cb * c0, nw, self.t_vec_chunks.data_ptr() + cb * v0, nv,
                          self.t_gptr.data_ptr(), self.wshadow.data_ptr(), self.mc_mom.data_ptr(), res,
                          self.vgrads.data_ptr(), self.vparams.data_ptr(), self.mc_vmom.data_ptr(), self.mc_momentum,
                          self.mc_weight_decay, self.mc_nesterov)
            self._nlaunch += 1
        elif res:     # A = g + e into the gradient buffers (bf16) and the residual (its rounding remainder)
            c0, ncs = self.ef_range[g]
            C.v2_ef_apply(self.t_ef_chunks.data_ptr(), c0, ncs, self.t_gptr.data_ptr(), res)
            self._nlaunch += 1
        if nt > 0 and self.quant:
            # quantize + push straight into the owners' arenas; the encode launch raises the group's push flag
            if self.clip is not None:
                C.v2_qsgd_stats(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                                self.clip_partials.data_ptr(), self.counters.data_ptr(), self.clip.data_ptr(),
                                self.tstats.data_ptr(), g)
                self._nlaunch += 1
            C.v2_qsgd_encode(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                             self.clip.data_ptr() if self.clip is not None else 0, self.t_arena_peer.data_ptr(),
                             self.t_sig_owner.data_ptr(), self.n_owners, pl.arena_floats, self.worker_index, g,
                             self.ctrl.data_ptr(), self.cnt_enc_group + 4 * g, 0, self.tstats.data_ptr(),
                             self._fired == self.G, self.clip is None, self.q_max_level, self.q_max_bucket,
                             self.code == "terngrad", res)
            self._nlaunch += 1
            return
        if self.signum and (nt > 0 or self.mc_vmom is not None):
            # worker momentum of the weights and (beta > 0) of the vectors, sign bits pushed into the owners' arenas; the
            # encode raises the push flag
            (v0, nv), cb = self.vec_range[g], struct.calcsize(P2.EF_CHUNK_FMT)
            if self.mc_vmom is None:
                nv = 0
            p = lambda t: t.data_ptr() if t is not None else 0
            if self.dlion:      # Lion's worker rule: the sign of b1 m + (1 - b1) g, then m = b2 m + (1 - b2) g
                C.v2_dlion_encode(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                                  self.t_vec_chunks.data_ptr() + cb * v0, nv, self.vgrads.data_ptr(), p(self.mc_mom),
                                  p(self.mc_vmom), self.betas[0], self.betas[1], self.t_arena_peer.data_ptr(),
                                  self.t_sig_owner.data_ptr(), self.n_owners, pl.arena_floats, self.worker_index, g,
                                  self.ctrl.data_ptr(), self.cnt_enc_group + 4 * g, self.tstats.data_ptr(),
                                  self._fired == self.G)
            else:
                C.v2_signum_encode(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                                   self.t_vec_chunks.data_ptr() + cb * v0, nv, self.vgrads.data_ptr(), p(self.mc_mom),
                                   p(self.mc_vmom), self.mc_momentum, self.t_arena_peer.data_ptr(),
                                   self.t_sig_owner.data_ptr(), self.n_owners, pl.arena_floats, self.worker_index, g,
                                   self.ctrl.data_ptr(), self.cnt_enc_group + 4 * g, self.tstats.data_ptr(),
                                   self._fired == self.G)
            self._nlaunch += 1
            return
        if self.power:
            # pass A (P = M Q_w, Gram, R^{-1}), pass B (Q' = M^T P_hat, pushes, warm state, push flag), EF pass
            p0, npw = pl.pw_range[g]
            C.v2_powersgd_encode(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt,
                                 self.t_pw_tiles.data_ptr(), p0, npw, self.t_gptr.data_ptr(), self.gpart.data_ptr(),
                                 self.pw_gram.data_ptr(), self.pw_state.data_ptr(), self.wstage.data_ptr(),
                                 self.t_arena_peer.data_ptr(), self.t_sig_owner.data_ptr(), self.n_owners,
                                 pl.arena_floats, self.worker_index, g, self.ctrl.data_ptr(), self.cnt_enc_group + 4 * g,
                                 self.tstats.data_ptr(), self._fired == self.G, res)
            self._nlaunch += (1 if nt > 0 else 0) + 1 + (1 if res and nt > 0 else 0)
            return
        if nt > 0 and (self.sign or self.fp8 or self.hadamard):
            # scales + sign bits / e4m3 bytes / (lo, step) + rotated codes pushed straight into the owners' arenas; the
            # encode raises the push flag
            encode = C.v2_sign_encode if self.sign else C.v2_fp8_encode if self.fp8 else C.v2_hadamard_encode
            encode(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                   self.t_arena_peer.data_ptr(), self.t_sig_owner.data_ptr(), self.n_owners, pl.arena_floats,
                   self.worker_index, g, self.ctrl.data_ptr(), self.cnt_enc_group + 4 * g, self.tstats.data_ptr(),
                   self._fired == self.G, res)
            self._nlaunch += 1
            return
        if nt > 0 and self.topk:
            # per-tensor threshold magnitude (two histogram launches), then the k largest entries pushed exactly
            C.v2_topk_select(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                             self.topk_hist.data_ptr(), self.topk_tiles.data_ptr(), self.counters.data_ptr(),
                             self.topk_sel.data_ptr(), self.tstats.data_ptr(), g)
            C.v2_topk_encode(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                             self.topk_sel.data_ptr(), self.topk_tiles.data_ptr(), self.t_arena_peer.data_ptr(),
                             self.t_sig_owner.data_ptr(), self.n_owners, pl.arena_floats, self.worker_index, g,
                             self.ctrl.data_ptr(), self.cnt_enc_group + 4 * g, self.tstats.data_ptr(),
                             self._fired == self.G, res, self.mc_mom.data_ptr() if self.mc_mom is not None else 0)
            self._nlaunch += 3
            return
        if nt > 0 and self.entry:
            # per-tensor L1 norms, then sample + compact + push into the owners' arenas (raises the push flag)
            C.v2_entry_stats(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                             self.l1_partials.data_ptr(), self.counters.data_ptr(), self.l1.data_ptr(),
                             self.tstats.data_ptr(), g)
            C.v2_entry_encode(self.t_units.data_ptr(), self.t_enc_tiles.data_ptr(), t0, nt, self.t_gptr.data_ptr(),
                              self.l1.data_ptr(), self.t_arena_peer.data_ptr(), self.t_sig_owner.data_ptr(),
                              self.n_owners, pl.arena_floats, self.worker_index, g, self.ctrl.data_ptr(),
                              self.cnt_enc_group + 4 * g, 0, self.tstats.data_ptr(), self._fired == self.G, res)
            self._nlaunch += 2
            return
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
                     self._fired == self.G, nt > 0, res, max(self.owner_index, 0))
        self._nlaunch += 1

    def _launch_ps(self, g: int, final: bool):
        t0, nt = self.plan.ps_range[g][self.owner_index]
        if self.clip_on:
            self._launch_ps_clip(g, final, t0, nt)
        elif self.layerwise:
            self._launch_ps_layerwise(g, final, t0, nt)
        else:
            self._launch_decay(g)
            if self.lion:
                self._launch_ps_lion(g, final, t0, nt)
            else:
                self._launch_ps_code(g, final, t0, nt)
            self._launch_ema(g)

    def _launch_ps_code(self, g: int, final: bool, t0: int, nt: int):
        """The code's PS kernel for group ``g``: decode, optimizer step, broadcast of the new parameters."""
        C, pl = self.C, self.plan
        p = lambda t: t.data_ptr() if t is not None else 0
        if self.quant:
            C.v2_ps_qsgd(self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), t0, nt, self.W, self.world, g, final,
                         self.owner_index, p(self.master), p(self.mom), p(self.sq), p(self.sqmax), p(self.vmom),
                         p(self.vsq), p(self.vsqmax), self.wshadow_mc, self.t_wshadow_peer.data_ptr(),
                         self.vparams.data_ptr(), self.vparams_mc, self.t_vparams_peer.data_ptr(), self.vgrads_mc,
                         self.t_vgrads_peer.data_ptr(), self.heap.region_ptr("arena"), pl.arena_floats,
                         self.signals.data_ptr(), self.t_sig_all.data_ptr(), self.ctrl.data_ptr(),
                         self.cnt_ps_group + 4 * g, self.timeout_ticks, self.tstats.data_ptr(), 1.0 / self.W,
                         max(1, min(self.ps_grid, max(nt, 1))), self.q_max_level, self.q_max_bucket)
            self._nlaunch += 1
            return
        if self.power:
            C.v2_ps_powersgd(self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), t0, nt, self.W, self.world, g, final,
                             self.owner_index, p(self.master), p(self.mom), p(self.sq), p(self.sqmax), p(self.vmom),
                             p(self.vsq), p(self.vsqmax), self.wshadow_mc, self.t_wshadow_peer.data_ptr(),
                             self.vparams.data_ptr(), self.vparams_mc, self.t_vparams_peer.data_ptr(), self.vgrads_mc,
                             self.t_vgrads_peer.data_ptr(), self.t_stage_peer.data_ptr(), self.heap.region_ptr("arena"),
                             pl.arena_floats, self.signals.data_ptr(), self.t_sig_all.data_ptr(), self.ctrl.data_ptr(),
                             self.cnt_ps_group + 4 * g, self.timeout_ticks, self.tstats.data_ptr(), 1.0 / self.W,
                             max(1, min(self.ps_grid, max(nt, 1))))
            self._nlaunch += 1
            return
        if self.sign or self.fp8 or self.hadamard:
            ps = C.v2_ps_sign if self.sign else C.v2_ps_fp8 if self.fp8 else C.v2_ps_hadamard
            ps(self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), t0, nt, self.W, self.world, g, final,
               self.owner_index, p(self.master), p(self.mom), p(self.sq), p(self.sqmax), p(self.vmom), p(self.vsq),
               p(self.vsqmax), self.wshadow_mc, self.t_wshadow_peer.data_ptr(), self.vparams.data_ptr(),
               self.vparams_mc, self.t_vparams_peer.data_ptr(), self.vgrads_mc, self.t_vgrads_peer.data_ptr(),
               self.heap.region_ptr("arena"), pl.arena_floats, self.signals.data_ptr(), self.t_sig_all.data_ptr(),
               self.ctrl.data_ptr(), self.cnt_ps_group + 4 * g, self.timeout_ticks, self.tstats.data_ptr(),
               1.0 / self.W, max(1, min(self.ps_grid, max(nt, 1))))
            self._nlaunch += 1
            return
        if self.signum:
            C.v2_ps_signum(self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), t0, nt, self.W, self.world, g, final,
                           self.owner_index, p(self.master), p(self.mom), p(self.sq), p(self.sqmax), p(self.vmom),
                           p(self.vsq), p(self.vsqmax), self.wshadow_mc, self.t_wshadow_peer.data_ptr(),
                           self.vparams.data_ptr(), self.vparams_mc, self.t_vparams_peer.data_ptr(), self.vgrads_mc,
                           self.t_vgrads_peer.data_ptr(), self.heap.region_ptr("arena"), pl.arena_floats,
                           self.signals.data_ptr(), self.t_sig_all.data_ptr(), self.ctrl.data_ptr(),
                           self.cnt_ps_group + 4 * g, self.timeout_ticks, self.tstats.data_ptr(), 1.0 / self.W,
                           max(1, min(self.ps_grid, max(nt, 1))), mean=self.dlion and self.dlion_aggregate == "mean")
            self._nlaunch += 1
            return
        if self.entry:
            C.v2_ps_entry(self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), t0, nt, self.W, self.world, g, final,
                          self.owner_index, p(self.master), p(self.mom), p(self.sq), p(self.sqmax), p(self.vmom),
                          p(self.vsq), p(self.vsqmax), self.wshadow_mc, self.t_wshadow_peer.data_ptr(),
                          self.vparams.data_ptr(), self.vparams_mc, self.t_vparams_peer.data_ptr(), self.vgrads_mc,
                          self.t_vgrads_peer.data_ptr(), self.heap.region_ptr("arena"), pl.arena_floats,
                          self.signals.data_ptr(), self.t_sig_all.data_ptr(), self.ctrl.data_ptr(),
                          self.cnt_ps_group + 4 * g, self.timeout_ticks, self.tstats.data_ptr(), 1.0 / self.W,
                          max(1, min(self.ps_grid, max(nt, 1))))
            self._nlaunch += 1
            return
        C.v2_ps(self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), t0, nt, self.W, self.world, g, final,
                self.owner_index, p(self.master), p(self.mom), p(self.sq), p(self.sqmax), p(self.vmom), p(self.vsq),
                p(self.vsqmax), self.wshadow_mc, self.t_wshadow_peer.data_ptr(), self.vparams.data_ptr(),
                self.vparams_mc, self.t_vparams_peer.data_ptr(), self.vgrads_mc, self.t_vgrads_peer.data_ptr(),
                self.t_stage_peer.data_ptr(), self.heap.region_ptr("arena"), pl.arena_floats,
                self.signals.data_ptr(), self.t_sig_all.data_ptr(), self.ctrl.data_ptr(), self.cnt_ps_group + 4 * g,
                self.timeout_ticks, self.tstats.data_ptr(), 1.0 / self.W, max(1, min(self.ps_grid, max(nt, 1))))
        self._nlaunch += 1

    def _launch_ps_lion(self, g: int, final: bool, t0: int, nt: int):
        """Lion: the code's PS kernel with the Lion epilogue (decode and sum as the plain launch; ``master`` / ``mom``
        and ``vparams`` / ``vmom`` stepped, the new parameters broadcast; the last group publishes them)."""
        C, pl = self.C, self.plan
        C.v2_ps_lion(self._ps_kind(), self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), t0, nt, self.W, self.world,
                     g, final, self.owner_index, self.master.data_ptr(), self.mom.data_ptr(), self.vmom.data_ptr(),
                     self.wshadow_mc, self.t_wshadow_peer.data_ptr(), self.vparams.data_ptr(), self.vparams_mc,
                     self.t_vparams_peer.data_ptr(), self.vgrads_mc, self.t_vgrads_peer.data_ptr(),
                     self.t_stage_peer.data_ptr(), self.heap.region_ptr("arena"), pl.arena_floats,
                     self.signals.data_ptr(), self.t_sig_all.data_ptr(), self.ctrl.data_ptr(),
                     self.cnt_ps_group + 4 * g, self.timeout_ticks, self.tstats.data_ptr(), 1.0 / self.W,
                     max(1, min(self.ps_grid, max(nt, 1))), self.q_max_level, self.q_max_bucket)
        self._nlaunch += 1

    def _launch_ps_layerwise(self, g: int, final: bool, t0: int, nt: int):
        """LARS / LAMB: phase 1 (the code's PS kernel with the layer-wise epilogue: moments, direction, tile
        partials, vectors finished), then phase 2 (norms across tiles and owners, trust ratios, the step of the
        weights and their bf16 broadcast; the last group publishes the parameters)."""
        C, pl = self.C, self.plan
        p = lambda t: t.data_ptr() if t is not None else 0
        grid = max(1, min(self.ps_grid, max(nt, 1)))
        part = self.lw_part.data_ptr() + 8 * t0
        C.v2_ps_layerwise(self._ps_kind(), self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), t0, nt, self.W, self.world, g,
                          self.owner_index, p(self.master), p(self.mom), p(self.sq), p(self.vmom), p(self.vsq),
                          self.vparams.data_ptr(), self.vparams_mc, self.t_vparams_peer.data_ptr(), self.vgrads_mc,
                          self.t_vgrads_peer.data_ptr(), self.t_stage_peer.data_ptr(), self.heap.region_ptr("arena"),
                          pl.arena_floats, self.signals.data_ptr(), self.t_sig_all.data_ptr(), self.ctrl.data_ptr(),
                          self.cnt_ps_group + 4 * g, self.timeout_ticks, self.tstats.data_ptr(), 1.0 / self.W,
                          self.lw_dir.data_ptr(), part, grid, self.q_max_level, self.q_max_bucket)
        self._nlaunch += 1
        self._launch_layerwise(g, final)

    def _launch_layerwise(self, g: int, final: bool):
        """LARS / LAMB phase 2 of group ``g`` (csrc/v2_layerwise.cu), on the direction and tile partials phase 1 (or
        the clip launch) left."""
        C = self.C
        p = lambda t: t.data_ptr() if t is not None else 0
        t0, nt = self.plan.ps_range[g][self.owner_index]
        part = self.lw_part.data_ptr() + 8 * t0
        C.v2_layerwise(self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), t0, nt,
                       self.t_lw_tile_layer.data_ptr() + 4 * t0, self.lw_layers[g], part, self.lw_dir.data_ptr(),
                       self.world, g, final, self.owner_index, self.n_owners, p(self.master), p(self.mom),
                       self.wshadow_mc, self.t_wshadow_peer.data_ptr(),
                       self.heap.region_ptr("lwx") + 8 * self.lw_xch_off[g], self.t_lw_xch_peer[g].data_ptr(),
                       self.signals.data_ptr(), self.t_sig_all.data_ptr(), self.ctrl.data_ptr(),
                       self.lw_counter.data_ptr() + 4 * g, self.timeout_ticks, self.tstats.data_ptr(),
                       self.lw_ratio.data_ptr() + 4 * sum(self.lw_layers[:g]), max(1, min(self.ps_grid, max(nt, 1))))
        self._nlaunch += 1
        self._launch_ema(g)

    def _launch_decay(self, g: int):
        """AdamW's decoupled weight decay of group ``g`` (csrc/v2_ema.cu): ``p <- p * f`` over the weight elements of
        this owner's PS tiles of the group, ``f`` from ``Ctrl2.decay_factor``, on the stream of the launch that steps
        those tiles, right before it."""
        t0, nt = self.plan.ps_range[g][self.owner_index]
        if not self.decay_on or nt == 0:
            return
        self.C.v2_decay(self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), t0, nt, self.master.data_ptr(),
                        self.ctrl.data_ptr(), max(1, min(self.ps_grid, nt)))
        self._nlaunch += 1

    def _launch_ema(self, g: int):
        """The average of group ``g`` (``ema_decay``, csrc/v2_ema.cu): ``e <- e + w (p - e)`` over this owner's PS tiles
        of the group, on the stream of the launch that wrote their final master values, right after it."""
        t0, nt = self.plan.ps_range[g][self.owner_index]
        if self.ema is None or nt == 0:
            return
        self.C.v2_ema(self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), t0, nt, self.master.data_ptr(),
                      self.vparams.data_ptr(), self.ema.data_ptr(), self.vema.data_ptr(), self.ema_w,
                      max(1, min(self.ps_grid, nt)))
        self._nlaunch += 1

    def _ps_kind(self) -> int:
        """The PS kernel of the code, as the phase-1 launches (v2_ps_layerwise, v2_ps_gather) select it."""
        return 1 if self.quant else 2 if self.entry else 3 if self.sign else 4 if self.fp8 else 5 if self.hadamard \
            else 6 if self.power else 0

    def _launch_ps_clip(self, g: int, final: bool, t0: int, nt: int):
        """Gradient-norm clipping: phase 1 of every group (the code's PS kernel with the gather epilogue: mean gradient
        and sum g^2 per tile, nothing stepped); after the final group, phase 2 (the whole-model norm across tiles and
        owners, the coefficient, and the step of every tile of this owner on coef * g), and for LARS / LAMB their
        phase 2 per group, unchanged (the last one publishes the parameters)."""
        C, pl = self.C, self.plan
        p = lambda t: t.data_ptr() if t is not None else 0
        C.v2_ps_gather(self._ps_kind(), self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), t0, nt, self.W,
                       self.world, g, self.owner_index, self.vgrads_mc, self.t_vgrads_peer.data_ptr(),
                       self.t_stage_peer.data_ptr(), self.heap.region_ptr("arena"), pl.arena_floats,
                       self.signals.data_ptr(), self.t_sig_all.data_ptr(), self.ctrl.data_ptr(),
                       self.cnt_ps_group + 4 * g, self.timeout_ticks, self.tstats.data_ptr(), 1.0 / self.W,
                       self.clip_grad.data_ptr(), self.clip_vgrad.data_ptr(), self.clip_part.data_ptr() + 8 * t0,
                       max(1, min(self.ps_grid, max(nt, 1))), self.q_max_level, self.q_max_bucket)
        self._nlaunch += 1
        if not final:
            return
        for gg in range(self.G):        # AdamW: every group's decay before the clip launch steps its tiles
            self._launch_decay(gg)
        n = len(self.clip_tiles)
        C.v2_clip(self.layerwise, self.t_units.data_ptr(), self.t_ps_tiles.data_ptr(), self.t_clip_tiles.data_ptr(), n,
                  self.clip_part.data_ptr(), self.clip_grad.data_ptr(), self.clip_vgrad.data_ptr(), self.world,
                  self.owner_index, self.n_owners, p(self.master), p(self.mom), p(self.sq), p(self.sqmax),
                  p(self.vmom), p(self.vsq), p(self.vsqmax), self.wshadow_mc, self.t_wshadow_peer.data_ptr(),
                  self.vparams.data_ptr(), self.vparams_mc, self.t_vparams_peer.data_ptr(), p(self.lw_dir),
                  p(self.lw_part), self.heap.region_ptr("clipx"), self.t_clip_xch_peer.data_ptr(),
                  self.signals.data_ptr(), self.t_sig_all.data_ptr(), self.ctrl.data_ptr(),
                  self.clip_counter.data_ptr(), self.timeout_ticks, self.tstats.data_ptr(), self.clip_norm.data_ptr(),
                  max(1, min(self.ps_grid, max(n, 1))))
        self._nlaunch += 1
        for gg in range(self.G):
            if self.layerwise:
                self._launch_layerwise(gg, gg == self.G - 1)
            else:
                self._launch_ema(gg)

    def grad_norm(self) -> tuple:
        """Gradient-norm clipping: ``(total, coef)`` of the last step, the whole-model norm of the mean gradient the
        owners received and the factor they stepped with, as this owner's clip launch computed them (zeros on a rank
        that owns no PS tiles).  Reading it synchronises the device."""
        if not self.clip_on:
            raise RuntimeError("grad_norm() needs ShadowEngine(..., clip_grad_norm=MAX) with MAX > 0")
        total, coef = self.clip_norm.tolist()
        return total, coef

    def trust_ratios(self) -> dict:
        """LARS / LAMB: the trust ratio of every weight tensor in the last step (parameter name -> ratio), as this
        owner's phase 2 computed it.  Reading it synchronises the device."""
        if not self.layerwise:
            raise RuntimeError("trust_ratios() needs ShadowEngine(..., optimizer='lars' | 'lamb')")
        names = {id(p): n for n, p in self.model.named_parameters()}
        r = self.lw_ratio.tolist()
        base = [sum(self.lw_layers[:g]) for g in range(self.G)]
        out, seen = {}, [0] * self.G
        for p, q in zip(self.params, self.plan.params):
            if q.is_w:
                out[names.get(id(p), str(q.index))] = r[base[q.group] + seen[q.group]]
                seen[q.group] += 1
        return out

    def _launch_group(self, g: int):
        """Called from the autograd thread when the last gradient of group ``g`` exists: fork the encode stream
        (and, on an owner, the PS stream) off the stream backward is running on."""
        final = self._fired == self.G - 1
        self._fired += 1
        cur = torch.cuda.current_stream(self.device)
        if self.s_wgrad is not None:
            # the wgrad stream runs in launch order: this event covers the weight gradients of the group
            self.ev_wgrad[g].record(self.s_wgrad)
            reader = cur if not self.overlap else self.s_enc
            reader.wait_event(self.ev_wgrad[g])
            for p in self.group_w_params[g]:
                p.grad.record_stream(reader)
        if self._micro < self.accum - 1:
            self._launch_accum(g, cur)
            return
        if not self.overlap:
            self._launch_encode(g)
            self._launch_code_stats(g)
            if self.is_owner:
                self._launch_ps(g, final)
            return
        self.ev_ready[g].record(cur)
        self.s_enc.wait_event(self.ev_ready[g])
        with torch.cuda.stream(self.s_enc):
            if self._jitter_us:
                torch.cuda._sleep(int(self._jitter_rng.uniform(0, self._jitter_us) * 1900))
            self._launch_encode(g)
            self.ev_push[g].record(self.s_enc)
            self._launch_code_stats(g)
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

    def _launch_accum(self, g: int, cur):
        """Group ``g`` of a micro-batch before the last: add its gradients into the accumulators (on the encode
        stream, or on ``cur`` without overlap), then release the gradient buffers, so that the next backward hands
        over fresh ones instead of adding into them in bf16."""
        j = self._micro
        reader = self.s_enc if self.overlap else cur
        if self.overlap:
            self.ev_ready[g].record(cur)
            self.s_enc.wait_event(self.ev_ready[g])
        with torch.cuda.stream(reader):
            lo, hi = self.w_range[g]
            if not self._capturing and hi > lo:     # as in _launch_encode; after a capture prepare() fills the table
                self.t_aptr[j, lo:hi].copy_(torch.from_numpy(self.host_aptr[j, lo:hi].copy()))
            (c0, nw), (v0, nv), cb = self.ef_range[g], self.vec_range[g], struct.calcsize(P2.EF_CHUNK_FMT)
            self.C.v2_accum_add(self.t_ef_chunks.data_ptr() + cb * c0, nw, self.t_vec_chunks.data_ptr() + cb * v0, nv,
                                self.t_aptr[j].data_ptr(), self.acc.data_ptr(), self.vacc.data_ptr(),
                                self.vgrads.data_ptr(), j == 0)
            self._nlaunch += 1
            if self._fired == self.G:
                self.ev_acc_done.record(reader)
        for p in self.group_w_params[g]:
            p.grad.record_stream(reader)        # not reused before the add has read it
            p.grad = None

    def _forward_backward(self, j: int = 0):
        """Forward and backward of micro-batch ``j`` (the whole static batch when ``accumulate_steps`` is 1); the
        loss and precisions in ``loss_buf`` are means over the whole batch."""
        n = self.accum
        x, y = self.static_x, self.static_y
        if n > 1:
            b = x.size(0) // n
            x, y = x[j * b:(j + 1) * b], y[j * b:(j + 1) * b]
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits = self.model(x)
            loss = self.criterion(logits.float(), y)
        if j > 0 and self.overlap:      # the previous micro-batch's adds read vgrads, which this backward rewrites
            torch.cuda.current_stream(self.device).wait_event(self.ev_acc_done)
        loss.backward()
        with torch.no_grad():
            lg = logits.detach().float()
            k = min(5, lg.size(1))
            hit = lg.topk(k, 1).indices.eq(y.view(-1, 1))
            vals = (loss.detach() if n == 1 else loss.detach() / n, hit[:, :1].float().sum() * (100.0 / (y.numel() * n)),
                    hit.float().sum() * (100.0 / (y.numel() * n)))
            for i, v in enumerate(vals):
                if j == 0:
                    self.loss_buf[i] = v
                else:
                    self.loss_buf[i] += v

    def _step_body(self):
        C = self.C
        self._nlaunch = 0
        C.v2_wait_params(self.signals.data_ptr(), self.n_owners, self.ctrl.data_ptr(), self.timeout_ticks,
                         self.tstats.data_ptr())
        self._nlaunch += 1
        if self.is_worker:
            self.vgrads.zero_()
            for p in self.w_params:
                p.grad = None
            if self.s_wgrad is not None:
                # fork the wgrad stream here, so that it is part of a graph capture before any group records on it;
                # the encode's waits on the last group's event join it again
                self.s_wgrad.wait_stream(torch.cuda.current_stream(self.device))
            for j in range(self.accum):     # only the last micro-batch codes, pushes and steps the PS
                self._micro = j
                self._pending, self._fired = list(self.group_size), 0
                self._forward_backward(j)
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
        if x_example.size(0) % self.accum:
            raise ValueError("accumulate_steps=%d needs a batch divisible by it (got %d samples)"
                             % (self.accum, x_example.size(0)))
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
            if self.t_aptr is not None:
                self.t_aptr.copy_(torch.from_numpy(self.host_aptr.copy()))
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
            elif u.kind in (P2.KIND_DENSE16, P2.KIND_QSGD, P2.KIND_ENTRY, P2.KIND_SIGN, P2.KIND_FP8,
                            P2.KIND_HADAMARD, P2.KIND_SIGNUM):                                           # (first, count)
                mw[u.w_off + a:u.w_off + a + b] = 1
            elif u.kind == P2.KIND_POWER:                                                # (first row, rows)
                mw[u.w_off + a * u.cols:u.w_off + (a + b) * u.cols] = 1
            elif u.kind == P2.KIND_SLAB:
                half = u.I // 2
                e0 = u.w_off + (a // half) * u.K * u.I
                mw[e0:e0 + (b // half) * u.K * u.I] = 1
            else:
                torch.as_strided(mw, (b, u.cols), (u.rs, u.cs), u.w_off + a * u.rs).fill_(1)
        return mw, mv

    def gather_fp32(self, what: str = "master") -> torch.Tensor:
        """Full fp32 array assembled from the owners' shards: 'master' | 'mom' | 'sq' | 'sqmax' | 'ema' (weight
        indexing) or 'vema' (vector indexing, ``vparams``')."""
        src = {"master": self.master, "mom": getattr(self, "mom", None), "sq": getattr(self, "sq", None),
               "sqmax": getattr(self, "sqmax", None), "ema": self.ema, "vema": self.vema}[what]
        torch.cuda.synchronize(self.device)
        mw, mv = self._owned_mask()
        m = mv if what == "vema" else mw
        out = (src * m) if (self.is_owner and src is not None) else torch.zeros_like(m)
        if self.world > 1:
            dist.all_reduce(out, group=self.group)
        return out

    def fp32_state_dict(self) -> dict:
        """state_dict in the standard (OIHW, fp32) layout — the evaluator's ``model_step_<N>`` contract.  Weights
        come from the fp32 master copies on the owners; BN running statistics from THIS rank's model (call it on
        a rank that trains: the reference's PS checkpoints carried untrained BN statistics, SURVEY 2.9)."""
        return self._state_dict(self.gather_fp32("master"))

    def ema_state_dict(self) -> dict:
        """Collective.  The averaged model (``ema_decay``) in the layout of :meth:`fp32_state_dict`: weights and BN /
        bias vectors from the owners' fp32 averages, BN running statistics from THIS rank's live model (they are not
        averaged, as ``torch.optim.swa_utils.AveragedModel(use_buffers=False)``)."""
        if not self.ema_decay:
            raise RuntimeError("ema_state_dict() needs ShadowEngine(..., ema_decay=d) with 0 < d < 1")
        return self._state_dict(self.gather_fp32("ema"), self.gather_fp32("vema"))

    def _state_dict(self, full: torch.Tensor, vfull: Optional[torch.Tensor] = None) -> dict:
        """This rank's model state_dict (fp32) with the weights taken from ``full`` (weight indexing, physical order)
        and, when given, the vectors from ``vfull`` (``vparams``' indexing)."""
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
            elif vfull is not None:
                sd[name] = vfull[q.off:q.off + q.numel].view(q.shape).clone()
        return sd

    def save_checkpoint(self, train_dir: str, step: Optional[int] = None) -> Optional[str]:
        """Collective.  Every training rank ``R`` writes ``model_step_<N>_worker<R>`` (its own state, below); after a
        barrier the first training rank writes ``model_step_<N>`` (fp32, trained BN statistics), the ``_optim``
        sidecar and, with ``ema_decay``, ``model_step_<N>_ema`` (:meth:`ema_state_dict`, the evaluator's layout).  So
        when the model file exists, its worker files exist too.  After ``load_checkpoint`` on the same
        configuration, training continues bit for bit as if it had never stopped.

        Every device buffer the engine keeps across steps is in one of these classes:

        (a) owner state and BN buffers, in ``model_step_<N>`` / ``_optim``: ``master`` (``wshadow`` is rebuilt from
            it as ``bf16(master)``, what the PS epilogue publishes), ``vparams``, ``mom`` / ``vmom``, for Adam
            ``sq`` / ``vsq`` and for AMSGrad ``sqmax`` / ``vsqmax``, the BN running statistics, and the step and LR
            of ``ctrl``; with ``ema_decay`` the averages ``ema`` / ``vema``, in ``model_step_<N>_ema``.
        (b) per-worker state, in ``model_step_<N>_worker<R>`` (:meth:`_worker_tensors`, physical order):
            ``residual`` (``error_feedback``, fp32 per weight element); ``mom`` / ``vmom_w``
            (``momentum_correction``, the worker's fp32 momentum per weight / vector element); ``vprev`` (svd / qsvd with ``warm_start``,
            the previous step's Jacobi basis per coded unit); PowerSGD's warm ``Q_w`` (only those ranges of
            ``gpart``, ``ops/plan2.py`` ``pw_warm_ranges``) and ``pw_state`` (160 bytes per unit: the draw counter
            carries over; ``R^{-1}``, the mask and the non-finite flag are rewritten by pass A before pass B reads
            them; its unit counters are zero between launches); the device's default CUDA generator (seed and
            offset), from which the model's dropout layers draw their masks (VGG's classifier).
        (c) scratch, rewritten every step before it is read: LARS / LAMB's direction ``lw_dir``, tile partials
            ``lw_part``, exchange slots and trust ratios; gradient-norm clipping's ``clip_grad``, ``clip_vgrad``,
            ``clip_part``, exchange slots and ``clip_norm``; the rest of ``gpart`` (Gram partials, ``P``,
            ``P_hat``, ``Q'``), ``vsel``, ``selcount``, ``sigma``, ``clip`` / ``clip_partials``, ``l1`` /
            ``l1_partials``, ``topk_sel``, ``topk_tiles``, ``pw_gram``, ``stats_partials``, ``vgrads``, ``wstage``,
            the gradient-accumulation sums ``acc`` / ``vacc`` (zero at every step boundary) and pointer tables,
            the arena slots (step-stamped), the fused-BN statistics arena, ``loss_buf`` and the input staging; zero
            between launches by design: ``counters``, ``stats_counters``, ``topk_hist``; ``signals`` carries step
            stamps, and ``load_checkpoint`` raises the parameter flags to the resumed step.
        (d) diagnostics that never feed the step, not saved: ``tstats`` (phase timings) and ``stats_acc``
            (``code_stats`` sums); a resumed run starts them afresh."""
        from ..utils import checkpoint as ckpt
        step = (self.step - 1) if step is None else step
        sd = self.fp32_state_dict()
        ema_sd = self.ema_state_dict() if self.ema_decay else None
        mom = self.gather_fp32("mom")
        vmom = self.vmom if self.is_owner else torch.zeros_like(self.vparams)
        _, mv = self._owned_mask()
        vm = vmom * mv
        if self.world > 1:
            dist.all_reduce(vm, group=self.group)
        adam_state = {}
        if self.opt in (P2.OPT_ADAM, P2.OPT_AMSGRAD, P2.OPT_LAMB):      # Adam / AMSGrad / LAMB: second moments too
            # (collective gathers, every rank takes part)
            names = [("sq", "vsq")] + ([("sqmax", "vsqmax")] if self.opt == P2.OPT_AMSGRAD else [])
            for wname, vname in names:
                vt = (getattr(self, vname) if self.is_owner else torch.zeros_like(self.vparams)) * mv
                if self.world > 1:
                    dist.all_reduce(vt, group=self.group)
                adam_state[wname + "_w"] = self.gather_fp32(wname).cpu()
                adam_state[wname + "_v"] = vt.cpu()
        path = ckpt.model_path(train_dir, step)
        os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
        if self.is_worker:
            ckpt.save_worker_state(train_dir, step, self.rank, self._worker_config(), self._worker_tensors())
        self._barrier()         # every worker file is in place before the model file names this step
        if self.rank != self.first_worker:
            return None
        tmp = path + ".tmp"
        torch.save({k: v.cpu() for k, v in sd.items()}, tmp)
        os.replace(tmp, path)
        if ema_sd is not None:
            torch.save({k: v.cpu() for k, v in ema_sd.items()}, path + "_ema.tmp")
            os.replace(path + "_ema.tmp", path + "_ema")
        side = {"step": step, "lr": self.lr, "mom_w": mom.cpu(), "mom_v": vm.cpu(), "code": self.code,
                "svd_rank": self.svd_rank, "engine": "shadow", "optimizer": self.optimizer}
        if self.quant or self.hadamard:
            side.update(quantization_level=self.quantization_level, bucket_size=self.bucket_size)
        if self.sign or self.fp8:
            side.update(bucket_size=self.bucket_size)
        if self.entry:
            side.update(entry_budget=self.entry_budget)
        if self.momentum_correction:
            side.update(momentum_correction=True)
        if self.dlion:
            side.update(dlion_betas=self.betas, dlion_aggregate=self.dlion_aggregate, weight_decay=self.adamw_wd)
        elif self.signum:
            side.update(signum_momentum=self.mc_momentum, weight_decay=self.adamw_wd)
        if self.lion:       # Lion's one state is mom_w / mom_v above
            side.update(lion_betas=self.betas, weight_decay=self.adamw_wd)
        side.update(adam_state)
        torch.save(side, path + "_optim.tmp")
        os.replace(path + "_optim.tmp", path + "_optim")
        return path

    def _worker_config(self) -> dict:
        """What this worker's state depends on: a worker file is applied only where every field matches."""
        cfg = {"code": self.code, "plan": P2.plan_digest(self.plan), "error_feedback": self.error_feedback,
               "warm_start": self.warm_start, "world": self.world, "ps_mode": self.ps_mode, "worker": self.worker_index}
        if self.momentum_correction:
            cfg["momentum_correction"] = True
        if self.dlion:
            cfg["dlion_betas"] = self.betas
        elif self.signum:
            cfg["signum_momentum"] = self.mc_momentum
        return cfg

    def _worker_tensors(self) -> dict:
        """Class (b) of :meth:`save_checkpoint`: this worker's tensors that carry over between steps.  ``pw_qw`` is a
        gathered copy of the ``Q_w`` ranges of ``gpart`` and ``cuda_rng`` the state of the device's default generator;
        the others are the engine's own tensors."""
        out = {}
        if self.residual is not None:
            out["residual"] = self.residual
        if self.mc_mom is not None:
            out["mom"], out["vmom_w"] = self.mc_mom, self.mc_vmom
        if self.vprev is not None:
            out["vprev"] = self.vprev
        if self.power:
            out["pw_qw"] = torch.cat([self.gpart[o:o + n] for o, n in self.pw_warm]) if self.pw_warm else self.gpart[:0]
            out["pw_state"] = self.pw_state
        out["cuda_rng"] = torch.cuda.get_rng_state(self.device)     # dropout masks draw from it (VGG's classifier)
        return out

    def _load_worker_state(self, train_dir: str, step: int) -> bool:
        """Copy this worker's saved state into the existing tensors (no new allocation: a captured graph keeps its
        addresses).  A missing or non-matching file leaves the state fresh (:meth:`_fresh_worker_state`), whatever
        warm-up steps wrote into it, and the CUDA generator where it is; it prints one line."""
        from ..utils import checkpoint as ckpt
        state = ckpt.load_worker_state(train_dir, step, self.rank)
        mine = self._worker_tensors()
        bad = ["file missing"] if state is None else \
            ckpt.worker_state_mismatch(state, step, self._worker_config(), mine)
        if bad:
            self._fresh_worker_state()
            print("rank %d: per-worker state of step %d not restored (%s): residuals and warm-start state start fresh"
                  % (self.rank, step, ", ".join(bad)), flush=True)
            return False
        saved = state["tensors"]
        for name, t in mine.items():
            if name not in ("pw_qw", "cuda_rng"):
                t.copy_(saved[name])
        torch.cuda.set_rng_state(saved["cuda_rng"], self.device)    # a captured graph reads seed and offset at replay
        i = 0
        for o, n in self.pw_warm:
            self.gpart[o:o + n].copy_(saved["pw_qw"][i:i + n])
            i += n
        return True

    def load_checkpoint(self, train_dir: str, step: int) -> None:
        """Collective: every rank reads the same files (shared directory) and jumps to ``step + 1``.  Each training
        rank also restores its own worker file (:meth:`_load_worker_state`).  With ``ema_decay`` the owners restore
        the average from ``model_step_<N>_ema``; without that file it starts at the loaded weights (one line says
        so).  Without ``ema_decay`` the file is ignored."""
        from ..utils import checkpoint as ckpt
        self._barrier()
        path = ckpt.model_path(train_dir, step)
        if os.path.exists(path + "_optim"):     # refused before any state changes
            side = torch.load(path + "_optim", map_location="cpu", weights_only=False)
            saved = side.get("optimizer", "sgd or adam")
            own_state = ("lars", "lamb", "lion")       # optimizers whose state no other optimizer can continue
            if (self.optimizer in own_state or saved in own_state) and saved != self.optimizer:
                raise ValueError("checkpoint %s was written by optimizer %s; this engine runs %s" % (path, saved,
                                                                                                  self.optimizer))
            if bool(side.get("momentum_correction", False)) != self.momentum_correction:
                raise ValueError("checkpoint %s was written with momentum_correction=%s; this engine runs %s"
                                 % (path, bool(side.get("momentum_correction", False)), self.momentum_correction))
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
            if self.ema_decay:
                self._load_ema(path + "_ema", byname, byid)
            if self.is_worker:
                self._load_worker_state(train_dir, step)
        self.step = step + 1
        self.ctrl_i32[0] = self.step
        self._barrier()
        self.signals[256:256 + self.n_owners] = self.step
        self._barrier()

    def _load_ema(self, path: str, byname: dict, byid: dict) -> None:
        """The owners' averages from ``path`` (weights permuted to the physical order, as ``master``), or from the
        loaded master and vectors when the file is missing."""
        if not os.path.exists(path):
            if self.is_owner:
                self.ema.copy_(self.master)
                self.vema.copy_(self.vparams)
            if self.rank == self.first_worker:
                print("%s missing: the weight average starts at the loaded weights" % path, flush=True)
            return
        if not self.is_owner:
            return
        for name, t in torch.load(path, map_location="cpu", weights_only=False).items():
            if name in byname:
                q = byid[id(byname[name])]
                src = t.to(self.device, torch.float32)
                if q.is_w:
                    phys = src.permute(0, 2, 3, 1).contiguous().reshape(-1) if src.dim() == 4 else src.reshape(-1)
                    self.ema[q.off:q.off + q.numel].copy_(phys)
                else:
                    self.vema[q.off:q.off + q.numel].copy_(src.reshape(-1))

    def close(self):
        torch.cuda.synchronize(self.device)
        if self.world > 1:
            dist.barrier(group=self.group)
        for hk in self._hooks:
            hk.remove()
        self.graph = None
        self.heap.close()

"""Checkpoint layout (parity: SURVEY.md 5.4).

Model file: ``<train_dir> + "model_step_" + str(step)`` — plain string
concatenation exactly like ``sync_replicas_master_nn.py:331-336`` /
``distributed_worker.py:337-342`` (``torch.save(network.state_dict(), f)``), so
the polling evaluator's contract (``distributed_evaluator.py:76-88``) holds.
New: a sidecar ``..._optim`` with optimizer state, step, LR and RNG state for
true resume (the reference cannot resume), and on the bf16 engine one
``..._worker<R>`` per training rank ``R`` with that worker's own state
(error-feedback residual, warm-start state) and the configuration it belongs to.
"""
from __future__ import annotations

import os
from typing import List, Optional

import torch


def model_path(train_dir: str, step: int) -> str:
    return train_dir + "model_step_" + str(step)


def save_model(train_dir: str, step: int, network: torch.nn.Module) -> str:
    path = model_path(train_dir, step)
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        torch.save(network.state_dict(), f)
    os.replace(tmp, path)  # atomic: the evaluator never sees a partial file
    return path


def save_sidecar(train_dir: str, step: int, optimizer=None, lr: Optional[float] = None, extra: Optional[dict] = None) -> str:
    path = model_path(train_dir, step) + "_optim"
    state = {"step": step, "lr": lr, "rng": torch.get_rng_state(),
             "optimizer": optimizer.state_dict() if optimizer is not None else None}
    if extra:
        state.update(extra)
    tmp = path + ".tmp"
    torch.save(state, tmp)
    os.replace(tmp, path)
    return path


def latest_step(train_dir: str) -> Optional[int]:
    d = os.path.dirname(train_dir + "x") or "."
    prefix = os.path.basename(train_dir + "model_step_")
    best = None
    if not os.path.isdir(d):
        return None
    for name in os.listdir(d):
        if name.startswith(prefix) and not name.endswith(("_optim", ".tmp")):
            try:
                s = int(name[len(prefix):])
            except ValueError:
                continue
            best = s if best is None else max(best, s)
    return best


WORKER_STATE_FORMAT = 1


def worker_path(train_dir: str, step: int, rank: int) -> str:
    return model_path(train_dir, step) + "_worker%d" % rank


def save_worker_state(train_dir: str, step: int, rank: int, config: dict, tensors: dict) -> str:
    """``model_step_<N>_worker<R>``: format version, step, the configuration the tensors depend on, and the tensors
    (host copies).  Written atomically, like the model file."""
    path = worker_path(train_dir, step, rank)
    state = {"format": WORKER_STATE_FORMAT, "step": step, "config": dict(config),
             "tensors": {k: v.detach().cpu() for k, v in tensors.items()}}
    tmp = path + ".tmp"
    torch.save(state, tmp)
    os.replace(tmp, path)
    return path


def load_worker_state(train_dir: str, step: int, rank: int) -> Optional[dict]:
    path = worker_path(train_dir, step, rank)
    if not os.path.exists(path):
        return None
    return torch.load(path, map_location="cpu", weights_only=True)


def worker_state_mismatch(state: dict, step: int, config: dict, tensors: dict) -> List[str]:
    """What keeps a worker sidecar from applying to this worker: the names of the fields that differ (``format``,
    ``step``, configuration keys, ``tensors`` when a tensor is missing, extra or of another shape or dtype).  Empty
    when it applies."""
    if state.get("format") != WORKER_STATE_FORMAT:
        return ["format"]
    bad = [] if state.get("step") == step else ["step"]
    saved = state.get("config") or {}
    bad += sorted(k for k in set(config) | set(saved) if saved.get(k) != config.get(k))
    st = state.get("tensors") or {}
    if set(st) != set(tensors) or any(tuple(st[k].shape) != tuple(t.shape) or st[k].dtype != t.dtype
                                      for k, t in tensors.items()):
        bad.append("tensors")
    return bad


def load_model(train_dir: str, step: int, network: torch.nn.Module, map_location="cpu") -> None:
    with open(model_path(train_dir, step), "rb") as f:
        network.load_state_dict(torch.load(f, map_location=map_location))


def load_sidecar(train_dir: str, step: int, optimizer=None, map_location="cpu") -> Optional[dict]:
    path = model_path(train_dir, step) + "_optim"
    if not os.path.exists(path):
        return None
    state = torch.load(path, map_location=map_location, weights_only=False)
    if optimizer is not None and state.get("optimizer") is not None:
        optimizer.load_state_dict(state["optimizer"])
    return state

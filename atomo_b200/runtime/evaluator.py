"""Checkpoint-polling evaluator (separate process, coupled only through files).

Parity: ``DistributedEvaluator`` (``/root/reference/src/distributed_evaluator.py:58-134``):
poll ``<model_dir>model_step_<N>``; when it exists rebuild the net,
``load_state_dict(torch.load)``, report NLL + top-1/top-5 on the test set,
``N += eval_freq``; else sleep.  Works for every ``--network`` (the reference's
only works for LeNet, SURVEY.md 2.9) and can stop (``max_evals`` / ``timeout``)
instead of looping forever.  ``ema=True`` polls ``model_step_<N>_ema`` instead, the averaged weights that
``--ema-decay`` writes beside each model file.
"""
from __future__ import annotations

import os
import time
from typing import Optional

import torch
import torch.nn.functional as F

from ..models import build_model
from ..utils import checkpoint as ckpt
from .nn_ops import NN_Trainer, accuracy


class DistributedEvaluator(NN_Trainer):
    def __init__(self, **kwargs):
        self._cur_step = 0
        self._model_dir = kwargs.get("model_dir", "output/models/")
        self._eval_freq = int(kwargs.get("eval_freq", 50))
        self._eval_batch_size = kwargs.get("eval_batch_size", 10000)
        self.network_config = kwargs.get("network", "LeNet")
        self.dataset = kwargs.get("dataset", "MNIST")
        self.num_classes = kwargs.get("num_classes", 10)
        self.device = torch.device(kwargs.get("device", "cpu"))
        self._poll_s = float(kwargs.get("poll_seconds", 10.0))
        self._suffix = "_ema" if kwargs.get("ema", False) else ""
        self._next_step_to_fetch = self._eval_freq
        self.results = []

    def evaluate(self, validation_loader, max_evals: Optional[int] = None, timeout: Optional[float] = None):
        t0 = time.time()
        while True:
            path = ckpt.model_path(self._model_dir, self._next_step_to_fetch) + self._suffix
            if os.path.isfile(path):
                self._load_model(path)
                print("Evaluator evaluating results on step {}".format(self._next_step_to_fetch))
                self.results.append(self._evaluate_model(validation_loader))
                self._next_step_to_fetch += self._eval_freq
                if max_evals is not None and len(self.results) >= max_evals:
                    return self.results
            else:
                if timeout is not None and time.time() - t0 > timeout:
                    return self.results
                time.sleep(self._poll_s)

    def _load_model(self, file_path: str):
        self.network = build_model(self.network_config, self.num_classes, self.dataset).to(self.device)
        with open(file_path, "rb") as f:
            self.network.load_state_dict(torch.load(f, map_location=self.device))

    @torch.no_grad()
    def _evaluate_model(self, test_loader):
        self.network.eval()
        test_loss, p1, p5, nb, n = 0.0, 0.0, 0.0, 0, 0
        for data, target in test_loader:
            data, target = data.to(self.device), target.to(self.device)
            output = self.network(data)
            test_loss += F.nll_loss(F.log_softmax(output, dim=1), target, reduction="sum").item()
            a1, a5 = accuracy(output, target, topk=(1, 5))
            p1 += a1.item(); p5 += a5.item(); nb += 1; n += len(target)
        nb = max(nb, 1)
        res = {"step": self._next_step_to_fetch, "loss": test_loss / max(n, 1), "prec1": p1 / nb, "prec5": p5 / nb}
        print("Test set: Average loss: {:.4f}, Prec@1: {} Prec@5: {}".format(res["loss"], res["prec1"], res["prec5"]))
        return res

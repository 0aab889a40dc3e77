"""GPU-resident training input (``--gpu-data``).

``GpuLoader`` uploads a rank's shard of the training (or test) set to the device once and builds every batch there
with one ``augment_gather`` kernel launch (``csrc/data_kernels.cu``): gather in the epoch's sample order, then
pad -> random crop -> random horizontal flip -> ToTensor -> Normalize.  It yields the same samples in the same order
as ``data.loader.DataLoader`` (``shuffle=True, drop_last=True``) with the same seed, and its normalisation is bit
for bit torchvision's.  Only the crop offsets and flips differ: they come from Philox keyed by
(seed, epoch, position in the epoch) instead of torch's CPU generator.

Sources: torchvision ``CIFAR10`` / ``CIFAR100`` / ``MNIST``, ``data.datasets.SVHN``, :class:`UInt8ImageDataset`
(uint8 images) and ``SyntheticImageDataset`` (fp32, gathered without augmentation, as on the CPU path), each
optionally wrapped in the ``Subset`` of ``shard_dataset``.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Tuple

import numpy as np
import torch
from torch.utils.data import Dataset, Subset

from .datasets import SVHN, _CIFAR_MEAN, _CIFAR_STD, _MNIST_MEAN, _MNIST_STD, _SVHN_MEAN, _SVHN_STD
from .synthetic import SyntheticImageDataset


class UInt8ImageDataset(Dataset):
    """An in-memory image set laid out like torchvision's ``CIFAR10``: ``.data`` is uint8 ``[N, H, W, C]``,
    ``.targets`` a list of ints, and ``__getitem__`` applies a PIL ``transform``."""

    def __init__(self, data, targets, transform=None):
        self.data = np.ascontiguousarray(np.asarray(data, dtype=np.uint8))
        if self.data.ndim != 4:
            raise ValueError("UInt8ImageDataset: data must be [N, H, W, C], got shape %s" % (self.data.shape,))
        self.targets = [int(t) for t in targets]
        if len(self.targets) != len(self.data):
            raise ValueError("UInt8ImageDataset: %d images but %d targets" % (len(self.data), len(self.targets)))
        self.transform = transform

    def __len__(self):
        return len(self.data)

    def __getitem__(self, index):
        from PIL import Image

        img = self.data[index]
        img = Image.fromarray(img[:, :, 0], mode="L") if img.shape[2] == 1 else Image.fromarray(img)
        if self.transform is not None:
            img = self.transform(img)
        return img, self.targets[index]


@dataclass(frozen=True)
class TransformSpec:
    """What ``datasets.real_transforms`` does to a uint8 image, in the kernel's terms."""
    mean: Tuple[float, ...]
    std: Tuple[float, ...]
    pad: int          # RandomCrop padding (0: no crop)
    reflect: bool     # reflect padding, else zeros
    augment: bool     # draw a crop offset and a flip per sample


def transform_spec(dataset: str, train: bool) -> TransformSpec:
    """The device pipeline equal to ``datasets.real_transforms(dataset)[0 if train else 1]``."""
    k = dataset.lower()
    if k == "imagenet":
        raise ValueError("--gpu-data cannot reproduce --dataset ImageNet: its pipeline resizes to 227x227 "
                         "(Resize is not implemented on the device); run it without --gpu-data")
    if k == "mnist":
        return TransformSpec(tuple(_MNIST_MEAN), tuple(_MNIST_STD), 0, False, False)
    if k in ("cifar10", "cifar100"):
        mean, std, reflect = _CIFAR_MEAN, _CIFAR_STD, True
    elif k == "svhn":
        mean, std, reflect = _SVHN_MEAN, _SVHN_STD, False
    else:
        raise ValueError("--gpu-data: unknown dataset %r" % dataset)
    if not train:
        return TransformSpec(tuple(mean), tuple(std), 0, False, False)
    return TransformSpec(tuple(mean), tuple(std), 4, reflect, True)


class ShuffleOrder:
    """Per-epoch sample order of ``data.loader.DataLoader(shuffle=True, seed=seed)``, from the same generator draws:
    each epoch's iterator takes one int64 base seed, ``RandomSampler`` one ``randperm(n)`` for the epoch and one more
    when the exhausted sampler is asked for the (empty) remainder."""

    def __init__(self, n: int, seed: int):
        self.n = int(n)
        self._gen = torch.Generator().manual_seed(seed)

    def next_epoch(self) -> torch.Tensor:
        torch.empty((), dtype=torch.int64).random_(generator=self._gen)
        perm = torch.randperm(self.n, generator=self._gen)
        torch.randperm(self.n, generator=self._gen)
        return perm


def _unwrap(ds: Dataset):
    if isinstance(ds, Subset):
        return ds.dataset, torch.as_tensor(list(ds.indices), dtype=torch.int64)
    return ds, None


def _max_device_bytes(device) -> int:
    free, _ = torch.cuda.mem_get_info(device)
    return free // 2       # leave the other half to the engine


def _upload_source(ds: Dataset, device):
    """(images [n, H, W, C] uint8 or fp32, labels [n] int64) of ``ds`` on ``device``, in ``ds``'s index order."""
    base, idx = _unwrap(ds)
    n = len(ds)
    if isinstance(base, SyntheticImageDataset):
        c, h, w = base.shape
        need = n * c * h * w * 4
        if need > _max_device_bytes(device):
            raise ValueError("--gpu-data: the synthetic set needs %.1f GB on the device, more than half of the free "
                             "memory; use --train-len / --test-len or run without --gpu-data" % (need / 1e9))
        ids = range(n) if idx is None else idx.tolist()
        items = [base[i] for i in ids]
        x = torch.stack([t for t, _ in items]).permute(0, 2, 3, 1).contiguous()
        y = torch.tensor([l for _, l in items], dtype=torch.int64)
        return x.to(device), y.to(device)
    if not hasattr(base, "data"):
        raise ValueError("--gpu-data: cannot upload a %s (expected a torchvision CIFAR10/CIFAR100/MNIST, SVHN, "
                         "UInt8ImageDataset or SyntheticImageDataset)" % type(base).__name__)
    data = torch.as_tensor(np.asarray(base.data))
    labels = base.labels if isinstance(base, SVHN) else base.targets
    labels = torch.as_tensor(np.asarray(labels), dtype=torch.int64)
    if isinstance(base, SVHN):
        data = data.permute(0, 2, 3, 1)            # stored NCHW
    elif data.dim() == 3:
        data = data.unsqueeze(-1)                  # MNIST: [N, 28, 28]
    if data.dtype != torch.uint8 or data.dim() != 4:
        raise ValueError("--gpu-data: %s.data must be uint8 images" % type(base).__name__)
    if idx is not None:
        data, labels = data[idx], labels[idx]
    return data.contiguous().to(device), labels.contiguous().to(device)


class GpuLoader:
    """``DataLoader``-like training input built on the device.

    ``train=True``: shuffled per epoch exactly like ``DataLoader(shuffle=True, drop_last=True, seed=seed)``, with the
    dataset's augmentation.  ``train=False``: in order, the last partial batch kept, no augmentation.
    ``next_batch()`` returns ``(x, y)`` on the device, ``x`` fp32 ``[B, C, H, W]`` (channels_last when asked: the
    layout of ``ShadowEngine``'s static input), ``y`` int64.
    """

    def __init__(self, dataset: Dataset, batch_size: int, dataset_key: str, train: bool = True, seed: int = 0,
                 device=None, channels_last: bool = False):
        from ..ops._ext import load

        self._C = load(required=True)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if self.device.type != "cuda":
            raise ValueError("GpuLoader builds batches on a CUDA device, got %s" % self.device)
        spec = transform_spec(dataset_key, train)
        self.batch_size, self.train, self.seed = int(batch_size), bool(train), int(seed)
        self.channels_last = channels_last
        self.n = len(dataset)
        if len(self) == 0:
            raise ValueError("GpuLoader: %d samples give no batch of %d (a worker's shard is smaller than "
                             "--batch-size?)" % (self.n, self.batch_size))
        self.src, self.labels = _upload_source(dataset, self.device)
        if self.src.dtype == torch.uint8:
            self.spec = spec
        else:      # synthetic: the CPU path applies no transform
            self.spec = TransformSpec((0.0,) * self.src.shape[3], (1.0,) * self.src.shape[3], 0, False, False)
        if len(self.spec.mean) != self.src.shape[3]:
            raise ValueError("GpuLoader: %s has %d channels, its transform normalises %d"
                             % (dataset_key, self.src.shape[3], len(self.spec.mean)))
        self.mean_std = torch.tensor([self.spec.mean, self.spec.std], dtype=torch.float32, device=self.device)
        self._shuffle = ShuffleOrder(self.n, seed) if self.train else None
        self.epochs_completed = 0
        self._pos = 0
        self._order = self._next_order()

    def __len__(self):
        return self.n // self.batch_size if self.train else -(-self.n // self.batch_size)

    def _next_order(self) -> torch.Tensor:
        order = self._shuffle.next_epoch() if self.train else torch.arange(self.n)
        return order.to(torch.int32).pin_memory().to(self.device, non_blocking=True)

    def _batch(self, pos0: int):
        b = min(self.batch_size, self.n - pos0)
        _, h, w, c = self.src.shape
        x = torch.empty((b, c, h, w), dtype=torch.float32, device=self.device,
                        memory_format=torch.channels_last if self.channels_last else torch.contiguous_format)
        y = torch.empty(b, dtype=torch.int64, device=self.device)
        s = self.spec
        self._C.augment_gather(self.src, self.labels, self._order, pos0, self.mean_std, s.pad, s.reflect, s.augment,
                               self.seed & 0xFFFFFFFFFFFFFFFF, self.epochs_completed, None, x, y)
        return x, y

    def next_batch(self):
        """The next (images, labels) batch on the device, wrapping across epochs."""
        if self._pos + (self.batch_size if self.train else 1) > self.n:
            self.epochs_completed += 1
            self._order = self._next_order()
            self._pos = 0
        x, y = self._batch(self._pos)
        self._pos += len(y)
        return x, y

    def __iter__(self):
        """One pass over the current epoch's batches (the evaluation loop), leaving ``next_batch()``'s place."""
        for i in range(len(self)):
            yield self._batch(i * self.batch_size)

    def close(self):
        self.src = self.labels = self._order = self.mean_std = None

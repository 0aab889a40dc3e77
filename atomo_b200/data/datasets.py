"""Dataset registry for the ``--dataset`` flag.

Parity: dataset/transform construction in
``/root/reference/src/distributed_nn.py:93-207`` (MNIST, Cifar10, SVHN,
Cifar100, "ImageNet" = CIFAR-10 upscaled to 227) and ``src/datasets.py``
(``SVHN`` 113-228, the ``next_batch``-style wrappers 11-57).

Real data is used when it already exists under ``root`` (no downloads are
attempted: there is no network); otherwise — or with ``synthetic=True`` — the
synthetic dataset of the same shape is returned.  Unlike the reference, the
training set handed to worker ``k`` of ``W`` is *sharded and seeded*
(:func:`shard_indices`), fixing "every worker shuffles the full set with no
seed" (SURVEY.md 2.9).
"""
from __future__ import annotations

import os
from typing import Optional, Tuple

import numpy as np
import torch
from torch.utils.data import Dataset, Subset

from .synthetic import SHAPES, synthetic_pair

_CIFAR_MEAN = [x / 255.0 for x in [125.3, 123.0, 113.9]]
_CIFAR_STD = [x / 255.0 for x in [63.0, 62.1, 66.7]]
_SVHN_MEAN, _SVHN_STD = (0.4914, 0.4822, 0.4465), (0.2023, 0.1994, 0.2010)
_MNIST_MEAN, _MNIST_STD = (0.1307,), (0.3081,)


def num_classes_of(name: str) -> int:
    return SHAPES[_key(name)][1]


def _key(name: str) -> str:
    k = name.lower()
    if k == "imagenet":
        return "imagenet"
    return k


class SVHN(Dataset):
    """SVHN from the ``*_32x32.mat`` files (parity: ``src/datasets.py:113-228``).

    Label 10 is remapped to 0 like torchvision/the reference.  No download.
    """

    filenames = {"train": "train_32x32.mat", "test": "test_32x32.mat", "extra": "extra_32x32.mat"}

    def __init__(self, root, split="train", transform=None, target_transform=None, download=False):
        import scipy.io as sio

        self.root = os.path.expanduser(root)
        self.transform, self.target_transform, self.split = transform, target_transform, split
        if split not in self.filenames:
            raise ValueError('Wrong split entered! Please use split="train" or "extra" or "test"')
        path = os.path.join(self.root, self.filenames[split])
        if not os.path.exists(path):
            raise RuntimeError("Dataset not found at %s (downloads are disabled offline)" % path)
        mat = sio.loadmat(path)
        self.data = np.transpose(mat["X"], (3, 2, 0, 1))
        self.labels = mat["y"].astype(np.int64).squeeze()
        np.place(self.labels, self.labels == 10, 0)

    def __getitem__(self, index):
        from PIL import Image

        img, target = self.data[index], int(self.labels[index])
        img = Image.fromarray(np.transpose(img, (1, 2, 0)))
        if self.transform is not None:
            img = self.transform(img)
        if self.target_transform is not None:
            target = self.target_transform(target)
        return img, target

    def __len__(self):
        return len(self.data)


class BatchDataset:
    """``.images/.labels/.next_batch`` wrapper (parity: ``MNISTDataset`` /
    ``Cifar10Dataset``, ``src/datasets.py:11-57``) over in-memory tensors."""

    def __init__(self, images: torch.Tensor, labels: torch.Tensor, seed: int = 0):
        self.images, self.labels = images, labels
        self.epochs_completed = 0
        self._pos = 0
        self._gen = torch.Generator().manual_seed(seed)
        self._perm = torch.randperm(len(images), generator=self._gen)

    def __len__(self):
        return len(self.images)

    def next_batch(self, batch_size: int):
        if self._pos + batch_size > len(self.images):
            self.epochs_completed += 1
            self._perm = torch.randperm(len(self.images), generator=self._gen)
            self._pos = 0
        idx = self._perm[self._pos:self._pos + batch_size]
        self._pos += batch_size
        return self.images[idx], self.labels[idx]


MNISTDataset = BatchDataset
Cifar10Dataset = BatchDataset


def real_transforms(name: str):
    """(train, test) torchvision transforms of the real ``--dataset name`` (mnist, cifar10, cifar100, svhn,
    imagenet).  ``data.gpu_loader`` reproduces the same pipeline on the device."""
    from torchvision import transforms as T

    k = name.lower()
    if k == "mnist":
        tf = T.Compose([T.ToTensor(), T.Normalize(_MNIST_MEAN, _MNIST_STD)])
        return tf, tf
    if k in ("cifar10", "cifar100", "imagenet"):
        norm = T.Normalize(_CIFAR_MEAN, _CIFAR_STD)
        size = 227 if k == "imagenet" else 32
        pre = [T.Resize((227, 227))] if k == "imagenet" else []
        train_tf = T.Compose(pre + [T.RandomCrop(size, padding=4, padding_mode="reflect"),
                                    T.RandomHorizontalFlip(), T.ToTensor(), norm])
        return train_tf, T.Compose(pre + [T.ToTensor(), norm])
    if k == "svhn":
        norm = T.Normalize(_SVHN_MEAN, _SVHN_STD)
        train_tf = T.Compose([T.RandomCrop(32, padding=4), T.RandomHorizontalFlip(), T.ToTensor(), norm])
        return train_tf, T.Compose([T.ToTensor(), norm])
    raise ValueError("no real-data transforms for dataset %r" % name)


def _real_pair(name: str, root: str):
    """Try to build (train, test) from files already on disk; None if absent."""
    try:
        from torchvision import datasets as tvd
    except Exception:
        return None
    k = name.lower()
    try:
        if k == "mnist":
            train_tf, test_tf = real_transforms(k)
            return (tvd.MNIST(os.path.join(root, "mnist_data"), train=True, download=False, transform=train_tf),
                    tvd.MNIST(os.path.join(root, "mnist_data"), train=False, download=False, transform=test_tf))
        if k in ("cifar10", "cifar100", "imagenet"):
            train_tf, test_tf = real_transforms(k)
            cls = tvd.CIFAR100 if k == "cifar100" else tvd.CIFAR10
            sub = "cifar100_data" if k == "cifar100" else "cifar10_data"
            return (cls(os.path.join(root, sub), train=True, download=False, transform=train_tf),
                    cls(os.path.join(root, sub), train=False, download=False, transform=test_tf))
        if k == "svhn":
            train_tf, test_tf = real_transforms(k)
            return (SVHN(os.path.join(root, "svhn_data"), "train", train_tf),
                    SVHN(os.path.join(root, "svhn_data"), "test", test_tf))
    except Exception:
        return None
    return None


def build_datasets(name: str, root: str = ".", synthetic: Optional[bool] = None, seed: int = 0,
                   train_len: Optional[int] = None, test_len: Optional[int] = None):
    """(train, test, num_classes) for ``--dataset name``."""
    key = name.lower()
    if key == "imagenet":
        # the reference's ImageNet branch: CIFAR-10 classes at 227x227
        syn_key, classes = "imagenet-ref", 10
    else:
        syn_key, classes = key, SHAPES[key][1]
    if synthetic is not True:
        pair = _real_pair(name, root)
        if pair is not None:
            return pair[0], pair[1], classes
        if synthetic is False:
            raise RuntimeError("dataset %s not found under %s and synthetic=False" % (name, root))
    train, test = synthetic_pair(syn_key, seed=seed, train_len=train_len, test_len=test_len)
    return train, test, classes


def shard_indices(n: int, worker: int, num_workers: int, seed: int = 0, epoch: int = 0) -> torch.Tensor:
    """Disjoint, seeded, per-epoch shard of ``range(n)`` for ``worker``."""
    g = torch.Generator().manual_seed(seed * 7919 + epoch)
    perm = torch.randperm(n, generator=g)
    per = n // num_workers
    return perm[worker * per:(worker + 1) * per]


def shard_dataset(ds: Dataset, worker: int, num_workers: int, seed: int = 0) -> Dataset:
    if num_workers <= 1:
        return ds
    return Subset(ds, shard_indices(len(ds), worker, num_workers, seed).tolist())

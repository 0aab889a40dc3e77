"""GPU-resident training input (``--gpu-data``): transform specs, epoch order and launcher flag (CPU); the
``augment_gather`` kernel against torchvision bit for bit, its Philox draws, and training through ``GpuLoader`` on
both engines' paths (GPU)."""
import argparse

import numpy as np
import pytest
import torch

from atomo_b200.data import DataLoader, SyntheticImageDataset, UInt8ImageDataset, real_transforms, shard_dataset
from atomo_b200.data.gpu_loader import GpuLoader, ShuffleOrder, transform_spec
from atomo_b200.utils.flags import add_fit_args


def _u8_set(n, hw=32, c=3, key="cifar10", train=True, seed=0, classes=10):
    """Learnable uint8 images: a per-class colour plus noise, labels i % classes."""
    rng = np.random.default_rng(seed)
    y = np.arange(n) % classes
    base = rng.integers(0, 256, size=(classes, 1, 1, c))
    img = np.clip(base[y] + rng.integers(-60, 61, size=(n, hw, hw, c)), 0, 255).astype(np.uint8)
    tf = real_transforms(key)[0 if train else 1]
    return UInt8ImageDataset(img, y.tolist(), tf)


# ---------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("key", ["MNIST", "Cifar10", "cifar100", "svhn"])
@pytest.mark.parametrize("train", [True, False])
def test_transform_spec_matches_the_torchvision_pipeline(key, train):
    from torchvision import transforms as T
    spec = transform_spec(key, train)
    tf = real_transforms(key)[0 if train else 1].transforms
    norm = [t for t in tf if isinstance(t, T.Normalize)][0]
    assert spec.mean == tuple(norm.mean) and spec.std == tuple(norm.std)
    crop = [t for t in tf if isinstance(t, T.RandomCrop)]
    flips = [t for t in tf if isinstance(t, T.RandomHorizontalFlip)]
    assert spec.augment == bool(crop) == bool(flips)
    assert all(isinstance(t, (T.RandomCrop, T.RandomHorizontalFlip, T.ToTensor, T.Normalize)) for t in tf)
    if crop:
        assert spec.pad == crop[0].padding == 4 and crop[0].fill == 0 and crop[0].size == (32, 32)
        assert spec.reflect == (crop[0].padding_mode == "reflect")
        assert flips[0].p == 0.5
    else:
        assert spec.pad == 0


def test_imagenet_is_refused():
    with pytest.raises(ValueError, match="ImageNet"):
        transform_spec("ImageNet", True)
    with pytest.raises(ValueError, match="unknown dataset"):
        transform_spec("stl10", True)


def test_gpu_data_flag_parses():
    assert add_fit_args(argparse.ArgumentParser(), []).gpu_data is False
    assert add_fit_args(argparse.ArgumentParser(), ["--gpu-data", "1"]).gpu_data is True
    assert add_fit_args(argparse.ArgumentParser(), ["--gpu-data", "0"]).gpu_data is False


def test_gloo_backend_refuses_gpu_data(monkeypatch):
    from atomo_b200 import distributed_nn
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    args = add_fit_args(argparse.ArgumentParser(), ["--backend", "gloo", "--gpu-data", "1", "--synthetic", "1"])
    with pytest.raises(SystemExit, match="--gpu-data"):
        distributed_nn.run_rank(args)


def _cpu_labels(ds, batch, seed, nbatches):
    loader = DataLoader(ds, batch_size=batch, shuffle=True, seed=seed, drop_last=True, pin_memory=True, prefetch=2)
    try:
        return torch.cat([loader.next_batch()[1] for _ in range(nbatches)])
    finally:
        loader.close()


@pytest.mark.parametrize("shard", [False, True])
def test_epoch_order_equals_the_cpu_loader(shard):
    n, batch, seed = 300, 32, 11
    full = UInt8ImageDataset(np.zeros((n, 4, 4, 3), np.uint8), list(range(1000, 1000 + n)),
                             real_transforms("cifar10")[1])
    ds = shard_dataset(full, 1, 3, seed=5) if shard else full
    per_epoch = len(ds) // batch
    want = _cpu_labels(ds, batch, seed, 2 * per_epoch + 1)       # two epochs and the first batch of the third
    targets = torch.tensor([ds[i][1] for i in range(len(ds))])
    order = ShuffleOrder(len(ds), seed)
    got = torch.cat([targets[order.next_epoch()[:per_epoch * batch]] for _ in range(3)])
    assert torch.equal(got[:len(want)], want)


# ---------------------------------------------------------------------------------------------------- GPU: kernel
def _C():
    from atomo_b200.ops._ext import load
    return load(required=True)


ALL_DRAWS = [(t, l, f) for t in range(9) for l in range(9) for f in (0, 1)]      # 81 crop offsets x both flips


def _reference(ds_images, order, draws, mean, std, pad, mode):
    """torchvision's pad -> crop -> hflip -> to_tensor -> normalize on PIL images."""
    from PIL import Image
    from torchvision.transforms import functional as TF
    out = []
    for s, (top, left, flip) in zip(order, draws):
        a = ds_images[s]
        img = Image.fromarray(a[:, :, 0], mode="L") if a.shape[2] == 1 else Image.fromarray(a)
        h, w = img.height, img.width
        if pad:
            img = TF.pad(img, pad, fill=0, padding_mode=mode)
            img = TF.crop(img, top, left, h, w)
        if flip:
            img = TF.hflip(img)
        out.append(TF.normalize(TF.to_tensor(img), list(mean), list(std)))
    return torch.stack(out)


def _gather(src, labels, order, pos0, b, mean, std, pad, reflect, augment, seed=0, epoch=0, draws=None,
            channels_last=False):
    dev = src.device
    _, h, w, c = src.shape
    x = torch.empty((b, c, h, w), device=dev,
                    memory_format=torch.channels_last if channels_last else torch.contiguous_format)
    y = torch.empty(b, dtype=torch.int64, device=dev)
    ms = torch.tensor([list(mean), list(std)], dtype=torch.float32, device=dev)
    ext = None if draws is None else torch.tensor(draws, dtype=torch.int32, device=dev)
    _C().augment_gather(src, labels, order, pos0, ms, pad, reflect, augment, seed, epoch, ext, x, y)
    return x, y


@pytest.mark.gpu
@pytest.mark.parametrize("hw,c,key,reflect", [(32, 3, "cifar10", True), (32, 3, "svhn", False),
                                              (28, 1, "mnist", True), (28, 1, "mnist", False)])
@pytest.mark.parametrize("channels_last", [False, True])
def test_augment_gather_is_bitwise_torchvision(hw, c, key, reflect, channels_last):
    """Every crop offset and flip, fed through the external-draws hook.  28x28 images make the flat
    (sample, pixel) grid end in a partial CTA; the batch is the 162 combinations plus 3 more samples."""
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(hw + c + reflect)
    n = 200
    imgs = rng.integers(0, 256, size=(n, hw, hw, c), dtype=np.uint8)
    labels = rng.integers(0, 100, size=n)
    mean, std = (transform_spec(key, True).mean, transform_spec(key, True).std) if c == 3 else ((0.1307,), (0.3081,))
    draws = ALL_DRAWS + [(0, 8, 1), (8, 0, 0), (4, 4, 1)]
    b = len(draws)
    order = rng.permutation(n)[:b + 7].astype(np.int32)
    pos0 = 7
    src = torch.from_numpy(imgs).to(dev)
    x, y = _gather(src, torch.from_numpy(labels).to(dev), torch.from_numpy(order).to(dev), pos0, b, mean, std, 4,
                   reflect, True, draws=draws, channels_last=channels_last)
    want = _reference(imgs, order[pos0:], draws, mean, std, 4, "reflect" if reflect else "constant")
    assert x.is_contiguous(memory_format=torch.channels_last if channels_last else torch.contiguous_format)
    assert torch.equal(x.cpu(), want)
    assert torch.equal(y.cpu(), torch.from_numpy(labels[order[pos0:]]))


@pytest.mark.gpu
@pytest.mark.parametrize("key,hw,c", [("cifar10", 32, 3), ("svhn", 32, 3), ("mnist", 28, 1)])
def test_test_loader_is_in_order_unaugmented_and_keeps_the_partial_batch(key, hw, c):
    ds = _u8_set(300, hw=hw, c=c, key=key, train=False)
    gl = GpuLoader(ds, 128, key, train=False, device="cuda:0")
    cpu = list(torch.utils.data.DataLoader(ds, batch_size=128, shuffle=False))
    got = list(gl)
    assert len(gl) == len(got) == len(cpu) == 3 and len(got[-1][1]) == 300 - 256
    for (gx, gy), (cx, cy) in zip(got, cpu):
        assert torch.equal(gx.cpu(), cx) and torch.equal(gy.cpu(), cy)
    for (gx, _), (nx, _) in zip(got, [gl.next_batch() for _ in range(3)]):
        assert torch.equal(gx, nx)
    assert gl.epochs_completed == 0
    gl.next_batch()
    assert gl.epochs_completed == 1


@pytest.mark.gpu
def test_mnist_train_loader_normalises_only():
    ds = _u8_set(200, hw=28, c=1, key="mnist")
    gl = GpuLoader(ds, 64, "MNIST", train=True, seed=3, device="cuda:0")
    perm = ShuffleOrder(200, 3).next_epoch()
    x, y = gl.next_batch()
    want = torch.stack([ds[int(i)][0] for i in perm[:64]])
    assert torch.equal(x.cpu(), want) and torch.equal(y.cpu(), torch.tensor([ds.targets[int(i)] for i in perm[:64]]))


@pytest.mark.gpu
@pytest.mark.parametrize("shard", [False, True])
def test_synthetic_source_is_bitwise_the_dataset(shard):
    full = SyntheticImageDataset((3, 32, 32), 10, 500, seed=4)
    ds = shard_dataset(full, 0, 2, seed=1) if shard else full
    gl = GpuLoader(ds, 96, "Cifar10", train=True, seed=9, device="cuda:0", channels_last=True)
    perm = ShuffleOrder(len(ds), 9).next_epoch()
    for k in range(2):
        x, y = gl.next_batch()
        ids = perm[k * 96:(k + 1) * 96].tolist()
        assert x.is_contiguous(memory_format=torch.channels_last)
        assert torch.equal(x.cpu(), torch.stack([ds[i][0] for i in ids]))
        assert y.tolist() == [ds[i][1] for i in ids]


@pytest.mark.gpu
@pytest.mark.parametrize("shard", [False, True])
def test_gpu_loader_labels_follow_the_cpu_loader(shard):
    full = _u8_set(420)
    ds = shard_dataset(full, 2, 3, seed=2) if shard else full
    per_epoch = len(ds) // 32
    want = _cpu_labels(ds, 32, 6, 2 * per_epoch)
    gl = GpuLoader(ds, 32, "cifar10", train=True, seed=6, device="cuda:0")
    got = torch.cat([gl.next_batch()[1].cpu() for _ in range(2 * per_epoch)])
    assert torch.equal(got, want) and gl.epochs_completed == 1


def _coordinate_source(dev):
    """One 32x32 image whose channel 0 holds the row and channel 1 the column: the draws can be read back."""
    r, c = np.meshgrid(np.arange(32), np.arange(32), indexing="ij")
    img = np.stack([r, c, np.zeros_like(r)], -1).astype(np.uint8)[None]
    return torch.from_numpy(img).to(dev), torch.zeros(1, dtype=torch.int64, device=dev)


def _decode_draws(x):
    """(top, left, flip) per sample from the coordinate image with zero padding, mean 0 and std 1."""
    u = torch.round(x[:, :2, 16, 16:18] * 255).to(torch.int64)          # [B, 2 channels, 2 columns]
    flip = (u[:, 1, 1] < u[:, 1, 0]).to(torch.int64)
    top = u[:, 0, 0] - 12
    left = u[:, 1, 0] - 12 + flip
    return torch.stack([top, left, flip], 1)


def _philox_draws(src, labels, n, seed, epoch, chunk=20000):
    order = torch.zeros(n, dtype=torch.int32, device=src.device)
    out = []
    for p in range(0, n, chunk):
        x, _ = _gather(src, labels, order, p, min(chunk, n - p), (0.0,) * 3, (1.0,) * 3, 4, False, True, seed=seed,
                       epoch=epoch)
        out.append(_decode_draws(x))
    return torch.cat(out).cpu()


@pytest.mark.gpu
def test_philox_draws_repeat_differ_across_epochs_and_are_uniform():
    from scipy.stats import chisquare
    src, labels = _coordinate_source(torch.device("cuda", 0))
    n = 100000
    d = _philox_draws(src, labels, n, seed=123, epoch=0)
    assert ((d[:, :2] >= 0) & (d[:, :2] <= 8)).all()
    assert torch.equal(_philox_draws(src, labels, 5000, seed=123, epoch=0), d[:5000])
    other = _philox_draws(src, labels, 5000, seed=123, epoch=1)
    assert (other != d[:5000]).any(1).float().mean() > 0.95
    cells = torch.bincount(d[:, 0] * 9 + d[:, 1], minlength=81).numpy()
    assert chisquare(cells).pvalue > 1e-3, cells
    flips = torch.bincount(d[:, 2], minlength=2).numpy()
    assert chisquare(flips).pvalue > 1e-3, flips


@pytest.mark.gpu
def test_gpu_loader_philox_batches_are_bitwise_torchvision():
    """A loader over the coordinate image reveals the draws the kernel takes at each position; a loader with the
    same seed over real-format images must equal torchvision fed those draws."""
    dev = torch.device("cuda", 0)
    n, batch = 256, 100
    ds = _u8_set(n)
    gl = GpuLoader(ds, batch, "cifar10", train=True, seed=21, device=dev, channels_last=True)
    coord, clab = _coordinate_source(dev)
    perm = ShuffleOrder(n, 21).next_epoch()
    spec = transform_spec("cifar10", True)
    for k in range(n // batch):
        x, y = gl.next_batch()
        xc, _ = _gather(coord, clab, torch.zeros(n, dtype=torch.int32, device=dev), k * batch, batch, (0.0,) * 3,
                        (1.0,) * 3, 4, False, True, seed=21, epoch=0)
        draws = _decode_draws(xc).tolist()
        ids = perm[k * batch:(k + 1) * batch].numpy()
        assert torch.equal(x.cpu(), _reference(ds.data, ids, draws, spec.mean, spec.std, 4, "reflect"))
        assert torch.equal(y.cpu(), torch.tensor(ds.targets)[ids])


# ---------------------------------------------------------------------------------------------------- GPU: end to end
def _train_shadow(ds, steps=20):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    eng = ShadowEngine(build_model("ResNet18", 10), 0, 1, code="sgd", lr=0.05, momentum=0.9, seed=3)
    gl = GpuLoader(ds, 64, "cifar10", train=True, seed=1, device="cuda:0", channels_last=True)
    x0, y0 = gl.next_batch()
    eng.prepare(x0, y0, warmup=2)
    losses = [float(eng.train_step(*gl.next_batch())[0]) for _ in range(steps)]
    torch.cuda.synchronize()
    assert eng.error_code() == 0
    master = eng.gather_fp32("master").clone()
    eng.close()
    gl.close()
    return losses, master


@pytest.mark.gpu
def test_shadow_engine_trains_from_the_gpu_loader(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)      # bitwise-reproducible backward
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    ds = _u8_set(512)
    losses, m1 = _train_shadow(ds)
    assert all(np.isfinite(losses))
    assert np.mean(losses[-4:]) < np.mean(losses[:4]), losses
    _, m2 = _train_shadow(ds)
    assert torch.equal(m1.view(torch.int32), m2.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["synthetic", "uint8"])
def test_launcher_trains_and_evaluates_with_gpu_data(source, tmp_path, monkeypatch, capsys):
    import atomo_b200.data as data
    from atomo_b200.runtime import p2p_launcher as L
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    if source == "uint8":
        monkeypatch.setattr(data, "build_datasets", lambda *a, **k: (_u8_set(1024), _u8_set(300, train=False), 10))
    args = add_fit_args(argparse.ArgumentParser(), [
        "--network", "ResNet18", "--dataset", "Cifar10", "--synthetic", "1", "--train-len", "1024", "--test-len",
        "300", "--batch-size", "64", "--test-batch-size", "128", "--gpu-data", "1", "--engine", "shadow", "--dtype",
        "bf16", "--code", "svd", "--svd-rank", "3", "--lr", "0.05", "--momentum", "0.9", "--max-steps", "8",
        "--eval-freq", "4", "--log-interval", "1", "--train-dir", str(tmp_path) + "/"])
    L.run_p2p_training(args)
    out = capsys.readouterr().out
    assert "Test set: Step: 4," in out and "Test set: Step: 8," in out, out
    assert "Worker: 0, Step: 8," in out and "device error" not in out

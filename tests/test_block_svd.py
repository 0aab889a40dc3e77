"""Block-spectral coder (codings/block_svd.py): the estimator of the sm_90a bf16 engine as a PyTorch oracle."""
import pytest
import torch

from atomo_b200 import codings
from atomo_b200.codings.block_svd import unit_table


def test_unit_table_is_the_gpu_planners():
    assert unit_table((64, 64, 3, 3), 3) == (("slab", 2048, 18, 0, 3.0),)
    assert unit_table((128, 64, 1, 1), 3) == (("block", 128, 32, 0, 2.0), ("block", 128, 32, 32, 2.0))
    assert unit_table((10, 512), 3) == (("block", 512, 10, 0, 3.0),)        # wide fc layer: coded transposed
    assert unit_table((64, 3, 3, 3), 3)[0][0] == "dense"                    # 3-channel stem
    assert unit_table((512,), 3)[0][0] == "dense"
    t = unit_table((1000, 2048), 8)                                          # ResNet-50 fc: 2048 x 1000 tall
    assert len(t) == 32 and all(k == "block" and r == 2048 for k, r, _, _, _ in t)
    assert sum(c for _, _, c, _, _ in t) == 1000 and all(b == 1.0 for *_, b in t)


@pytest.mark.parametrize("shape", [(64, 64, 3, 3), (128, 64, 1, 1), (10, 512), (40, 24)])
def test_full_budget_without_sampling_is_exact(shape):
    g = torch.randn(shape, generator=torch.Generator().manual_seed(1))
    c = codings.build("bsvd", rank=64, random_sample=False)
    code = c.encode(g)
    assert torch.allclose(c.decode(code), g, atol=2e-5)


def test_slab_units_use_the_reference_matricization_and_probabilities():
    """A 3x3 convolution is one unit over the reference's (O*I/2, 2*kh*kw) matricization: the Gram route finds the
    same singular values as torch.linalg.svd, hence the same inclusion probabilities as --code svd."""
    from atomo_b200.codings.sampling import atom_probabilities
    from atomo_b200.codings.svd import resize_to_2d
    g = torch.randn(32, 16, 3, 3, generator=torch.Generator().manual_seed(2))
    a = resize_to_2d(g)
    s = torch.linalg.svdvals(a)
    lam = torch.linalg.eigvalsh(a.t() @ a).flip(0).clamp_min(0).sqrt()
    assert torch.allclose(lam, s, rtol=1e-4, atol=1e-4)
    assert torch.allclose(atom_probabilities(lam, 3), atom_probabilities(s, 3), atol=1e-5)


@pytest.mark.parametrize("shape,rank", [((48, 32, 3, 3), 3), ((96, 80), 4), ((128, 64, 1, 1), 2)])
def test_estimator_is_unbiased(shape, rank):
    """Mean of n decodes -> g at the 1/sqrt(n) rate the estimator's own variance predicts (a biased estimator — the
    reference's redraw-until-non-empty, round 1's truncated subspace — plateaus instead)."""
    gen = torch.Generator().manual_seed(3)
    m = torch.randn(shape, generator=gen)
    flat = m.reshape(shape[0], -1)
    u, s, vT = torch.linalg.svd(flat, full_matrices=False)
    g = ((u * (s * torch.logspace(0, -2, len(s)))) @ vT).reshape(shape)      # decaying spectrum, like real gradients
    c = codings.build("bsvd", rank=rank, generator=gen)
    n = 600
    acc, var = torch.zeros_like(g), 0.0
    for _ in range(n):
        d = c.decode(c.encode(g))
        acc += d
        var += float((d - g).pow(2).sum())
    err2 = float((acc / n - g).pow(2).sum())
    predicted = var / n / n                     # E||mean - g||^2 = Var / n for an unbiased estimator
    assert 0.5 * predicted < err2 < 2.0 * predicted, (err2, predicted)
    assert err2 ** 0.5 / float(g.norm()) < 0.25


def test_code_is_smaller_than_the_tensor_and_survives_the_wire():
    from atomo_b200.parallel import wire
    gen = torch.Generator().manual_seed(11)
    g = torch.randn(256, 128, 3, 3, generator=gen)
    c = codings.build("bsvd", rank=3, generator=gen)
    sizes = []
    for _ in range(20):
        code = c.encode(g)
        n = len(code["units"][0]["s"])
        assert codings.Coding.wire_bytes(code) == 4 * n * (16384 + 1 + 18)      # U column + s + V row per atom
        sizes.append(n)
    assert 2.0 < sum(sizes) / len(sizes) < 4.0                                  # the budget is the EXPECTED count
    assert 4 * 3 * (16384 + 19) < 0.2 * g.numel() * 4                           # ~6x fewer bytes than the tensor
    back = wire.unpack(wire.pack({"codes": [code]}))["codes"][0]
    assert torch.equal(c.decode(back), c.decode(code))

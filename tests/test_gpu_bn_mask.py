"""The ReLU mask the fused BatchNorm forward writes for its backward: bit i of byte e is (y > 0) for channel i of the
e-th 8-channel vector of the bf16 output y."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("with_res", [False, True])
def test_bn_relu_mask_bits_are_bf16_output_positive(with_res):
    from atomo_b200.ops._ext import load
    C = load()
    dev = torch.device("cuda", 0)
    n, ch, hw = 16, 64, 8
    x = (torch.randn(n, ch, hw, hw, device=dev) * 2 + 0.3).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    gamma = torch.empty(ch, device=dev).uniform_(0.5, 1.5)
    beta = torch.empty(ch, device=dev).uniform_(-0.5, 0.5)
    # gamma = 0 makes a channel's output the constant beta: positive fp32 values below half of bf16's smallest
    # subnormal (2^-133) round to bf16 zero and must give a 0 bit; the bf16 subnormals and smallest normals around them
    tiny = [2.0 ** -149, 2.0 ** -140, 2.0 ** -135, 2.0 ** -134, 2.0 ** -133, 2.0 ** -130, 2.0 ** -127, 2.0 ** -126,
            2.0 ** -120, -2.0 ** -130, 0.0, 1e-3, -1e-3]
    k = len(tiny)
    gamma[:k] = 0.0
    beta[:k] = torch.tensor(tiny, device=dev)
    res = None
    if with_res:
        r = torch.randn(n, ch, hw, hw, device=dev)
        r[:, :k] = 0.0
        res = r.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.empty_like(x)
    mask = torch.empty(x.numel() // 8, dtype=torch.uint8, device=dev)
    acc = torch.empty(2 * ch, device=dev)
    mean, invstd = torch.empty(ch, device=dev), torch.empty(ch, device=dev)
    C.bn_forward(x, res, y, mask, acc, gamma, beta, mean, invstd, None, None, 1e-5, 0.1)
    torch.cuda.synchronize()
    rows = y.permute(0, 2, 3, 1).reshape(-1, ch).float()          # [N*H*W][C], the kernel's row order
    bits = (mask.view(-1, ch // 8, 1).int() >> torch.arange(8, device=dev, dtype=torch.int32)) & 1
    assert torch.equal(bits.reshape(-1, ch).bool(), rows > 0)
    assert bool((rows > 0).any()) and bool((rows == 0).any())

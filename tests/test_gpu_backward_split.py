"""The bf16 engine's convolutions compute their weight gradients on a stream of their own, beside the backward chain.
Every value must stay bit for bit what the stock autograd node computes."""
import pytest
import torch

from shadow_harness import deterministic_cudnn  # noqa: F401

pytestmark = pytest.mark.gpu

CL = torch.channels_last


def _bf16(shape):
    return torch.randn(*shape, device="cuda").to(torch.bfloat16).contiguous(memory_format=CL)


@pytest.mark.parametrize("k,stride", [(3, 1), (3, 2), (1, 2), (1, 1)])
@pytest.mark.parametrize("graph", [False, True])
def test_split_conv_backward_equals_convolution_backward(deterministic_cudnn, k, stride, graph):
    from atomo_b200.ops.split_conv import Conv2d
    cin, cout = 64, 128
    conv = Conv2d(cin, cout, k, stride, k // 2, bias=False).cuda().to(torch.bfloat16).to(memory_format=CL)
    side = torch.cuda.Stream()
    conv.wgrad_stream = side
    x = _bf16((32, cin, 16, 16)).requires_grad_(True)
    ho = (16 + 2 * (k // 2) - k) // stride + 1
    dy = _bf16((32, cout, ho, ho))
    want = torch.ops.aten.convolution_backward(dy, x.detach(), conv.weight.detach(), None, conv.stride, conv.padding,
                                               conv.dilation, False, (0, 0), 1, (True, True, False))

    def step():
        x.grad = conv.weight.grad = None
        y = conv(x)
        y.backward(dy)
        torch.cuda.current_stream().wait_stream(side)      # join the wgrad stream

    if graph:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        x.grad.zero_(), conv.weight.grad.zero_()
        g.replay()
    else:
        step()
    torch.cuda.synchronize()
    assert torch.equal(x.grad, want[0])
    assert torch.equal(conv.weight.grad, want[1])


@pytest.mark.parametrize("use_graph,overlap", [(True, True), (False, False)])
def test_shadow_engine_steps_equal_the_stock_backward(deterministic_cudnn, use_graph, overlap):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model
    from atomo_b200.ops.split_conv import enable_split_wgrad
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    x, y = SyntheticImageDataset((3, 32, 32), 10, 512).materialize(64)
    runs = []
    for new in (True, False):
        torch.manual_seed(0)
        eng = ShadowEngine(build_model("ResNet18", 10), 0, 1, code="svd", svd_rank=3, lr=0.01, momentum=0.9,
                           use_graph=use_graph, overlap=overlap, groups=5, seed=1)
        assert eng.split_wgrad_layers == 20
        if not new:
            enable_split_wgrad(eng.model, None)
        eng.prepare(x.pin_memory(), y.pin_memory(), warmup=2)
        losses = [eng.train_step().clone() for _ in range(10)]
        torch.cuda.synchronize()
        assert eng.error_code() == 0
        runs.append((torch.stack(losses), eng.gather_fp32("master").clone()))
        eng.close()
    assert torch.equal(runs[0][0], runs[1][0])
    assert torch.equal(runs[0][1], runs[1][1])


def test_trace_has_wgrad_on_a_second_stream(deterministic_cudnn):
    from torch.profiler import ProfilerActivity, profile
    from atomo_b200.models import build_model
    from atomo_b200.ops.fused_bn import enable_fused_bn
    from atomo_b200.ops.split_conv import Conv2d, enable_split_wgrad
    model = build_model("ResNet18", 10).cuda().to(memory_format=CL)
    for m in model.modules():
        if isinstance(m, Conv2d):
            m.weight.data = m.weight.data.to(torch.bfloat16)
    enable_fused_bn(model, True)
    side = torch.cuda.Stream()
    assert enable_split_wgrad(model, side) == 20
    x = torch.randn(32, 3, 32, 32, device="cuda").contiguous(memory_format=CL)
    y = torch.randint(0, 10, (32,), device="cuda")

    def step():
        model.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(model(x).float(), y)
        loss.backward()
        torch.cuda.current_stream().wait_stream(side)
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
            and "Memcpy" not in e.name and "Memset" not in e.name]
    main = {e.device_resource_id for e in kern if "bn_bwd_reduce" in e.name}
    assert len(main) == 1
    main = main.pop()
    wgrad = [e for e in kern if "wgrad" in e.name]
    assert wgrad and all(e.device_resource_id != main for e in wgrad)
    side_kernels = [e.name for e in kern if e.device_resource_id != main]
    assert len(side_kernels) >= 20, side_kernels                          # at least one wgrad kernel per conv

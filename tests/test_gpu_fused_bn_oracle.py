"""The fused BatchNorm kernels (csrc/bn_kernels.cu) against float64 oracles on the same bf16 inputs.

Two oracles, both float64 PyTorch:
- full: F.batch_norm (+ residual) (+ ReLU) with autograd, and the usual running update from the unbiased variance;
- element: the kernels' own elementwise formulas evaluated on the kernel's statistics (save_mean, save_invstd, the
  backward's sums and the ReLU mask), so a wrong reduction and a wrong elementwise pass fail different checks.

With integer inputs in [-8, 8] and R <= 2^18 rows every partial sum of x, x^2 and dy is an integer below 2^24, exact
in fp32 in any order: the sums must then come out exact, which catches a row dropped or counted twice at any R.
"""
import copy
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from shadow_harness import ext

pytestmark = pytest.mark.gpu

# The statistics bound: every kernel sum is a chain of at most ~300 dependent fp32 adds for the shapes here (worst
# C = 8: a thread's few rows, RL = 256 rows in the shared-memory sum, then the per-CTA partials), so it is within
# 300 eps * sum|x| < 2^-14 / 3 * sum|x|.  One 2^-14 covers sum(x^2), the division and the mean^2 of E[x^2] - mean^2.
STAT = 2.0 ** -14
CTAS = 296  # the reduction grid cap (ATOMO_BN_REDUCE_CTAS at its default)


def _rl(c):
    """rows per reduction CTA: 256 threads / (C / 8) channel groups"""
    return 256 // (c // 8)


# R = a * RL + b: the boundaries of the stats kernel's 4-row and the backward reduction's 2-row loops, their
# remainder loops and the grid cap.  For C >= 1032 RL is 1, so RL - 1 is the empty batch (its own test below), RL + 1
# is 2, and 2^16 + 3 rows would exceed 64 MB.
_R = {"2": (0, 2), "7": (0, 7), "RL-1": (1, -1), "RL+1": (1, 1), "cap-1": (CTAS, -1), "cap+1": (CTAS, 1),
      "4cap-1": (4 * CTAS, -1), "4cap+1": (4 * CTAS, 1), "2^16+3": (0, 2 ** 16 + 3)}

# (C, R, residual, relu, momentum, eps)
GEOMETRY = [
    (8, "2", False, False, 0.1, 1e-5), (24, "7", True, True, 0.01, 1e-3),
    (8, "RL-1", False, True, 0.1, 1e-5), (24, "RL-1", True, True, 0.1, 1e-3),
    (96, "RL+1", False, False, 0.1, 1e-5), (120, "RL+1", True, False, 0.01, 1e-5),
    (8, "cap-1", True, False, 0.1, 1e-3), (96, "cap+1", False, True, 0.01, 1e-5),
    (120, "cap-1", True, True, 0.1, 1e-5), (24, "cap+1", False, False, 0.1, 1e-5),
    (8, "4cap-1", True, True, 0.1, 1e-5), (24, "4cap+1", False, False, 0.01, 1e-3),
    (96, "4cap-1", True, False, 0.01, 1e-3), (120, "4cap+1", False, True, 0.1, 1e-5),
    (8, "2^16+3", False, True, 0.01, 1e-5), (120, "2^16+3", True, False, 0.1, 1e-3),
    (512, "RL-1", True, True, 0.1, 1e-5), (512, "cap+1", False, False, 0.01, 1e-5),
    (512, "4cap-1", True, False, 0.1, 1e-3), (1032, "2", True, True, 0.1, 1e-5),
    (2040, "7", False, False, 0.01, 1e-3), (2048, "RL+1", False, True, 0.1, 1e-3),
    (1032, "cap-1", False, True, 0.01, 1e-5), (2040, "cap+1", True, False, 0.1, 1e-5),
    (2048, "cap-1", True, True, 0.01, 1e-3), (1032, "4cap+1", True, False, 0.1, 1e-3),
    (2040, "4cap-1", False, True, 0.1, 1e-5), (2048, "4cap+1", False, False, 0.01, 1e-5),
    (1032, "7", False, False, 0.01, 1e-5),
]


def _rows(t):
    """a channels_last NCHW tensor as the kernels see it: [R = N*H*W][C]"""
    return t.permute(0, 2, 3, 1).reshape(-1, t.size(1))


def _nchw(rows, n, h, w):
    return rows.view(n, h, w, rows.size(1)).permute(0, 3, 1, 2)


def _bits(mask, R, C):
    """the ReLU mask as bool [R][C]: bit i of byte e is channel i of the e-th 8-channel vector"""
    sh = torch.arange(8, device=mask.device, dtype=torch.int32)
    return ((mask.view(R, C // 8, 1).int() >> sh) & 1).reshape(R, C).bool()


def _ulp(v, mant, tiny):
    """one ulp, in a format with `mant` stored mantissa bits, of the float64 values v (at least `tiny`)"""
    return torch.exp2(torch.floor(torch.log2(v.abs())) - mant).clamp_min(tiny)


def _le(got, want, bound, what):
    err = (got.double() - want).abs()
    bad = ~(err <= bound)  # a NaN fails too
    assert not bool(bad.any()), "%s: %d of %d beyond the bound, worst %.3g vs bound %.3g" % (
        what, int(bad.sum()), bad.numel(), float((err - bound)[bad].max()), float(bound[bad].max()))


def _same_bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    ints = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.uint8: torch.uint8}
    return torch.equal(a.view(ints[a.dtype]), b.view(ints[b.dtype]))


def _inputs(R, C, res, exact, gen):
    """[R][C] bf16 rows.  exact: integers in [-8, 8] and gamma = 1; else normal channels with std in [0.5, 2] and
    mean/std in [-1, 1], 10 or 100 (the offset channels pin the E[x^2] - mean^2 contract), gamma of either sign"""
    dev = torch.device("cuda", 0)
    if exact:
        def draw():
            return torch.randint(-8, 9, (R, C), generator=gen, device=dev).to(torch.bfloat16)
        x, r, dy = draw(), draw(), draw()
        gamma = torch.ones(C, device=dev)
    else:
        std = torch.rand(C, generator=gen, device=dev) * 1.5 + 0.5
        k = torch.rand(C, generator=gen, device=dev) * 2 - 1
        k[3::8], k[5::8] = 10.0, 100.0
        x = (torch.randn(R, C, generator=gen, device=dev) * std + k * std).to(torch.bfloat16)
        r = torch.randn(R, C, generator=gen, device=dev).to(torch.bfloat16)
        dy = torch.randn(R, C, generator=gen, device=dev).to(torch.bfloat16)
        sign = torch.where(torch.rand(C, generator=gen, device=dev) < 0.2, -1.0, 1.0)
        gamma = (torch.rand(C, generator=gen, device=dev) + 0.5) * sign
    beta = torch.rand(C, generator=gen, device=dev) - 0.5
    return dict(x=x, res=r if res else None, dy=dy, gamma=gamma, beta=beta)


def _run_binding(inp, relu, rm, rv, eps, momentum):
    """both kernel chains through the binding on [R][C] rows viewed as (1, C, R, 1); rm / rv are updated in place"""
    K = ext()
    x = _nchw(inp["x"], 1, inp["x"].size(0), 1)
    res = None if inp["res"] is None else _nchw(inp["res"], 1, x.size(2), 1)
    dy = _nchw(inp["dy"], 1, x.size(2), 1)
    R, C = inp["x"].shape
    f32 = lambda n: torch.empty(n, device=x.device)
    k = dict(y=torch.empty_like(x), acc_f=f32(2 * C), mean=f32(C), invstd=f32(C), dx=torch.empty_like(x),
             dres=torch.empty_like(x) if res is not None else None, acc_b=f32(2 * C), dgamma=f32(C), dbeta=f32(C),
             mask=torch.empty(R * C // 8, dtype=torch.uint8, device=x.device) if relu else None)
    K.bn_forward(x, res, k["y"], k["mask"], k["acc_f"], inp["gamma"], inp["beta"], k["mean"], k["invstd"], rm, rv, eps,
                 momentum)
    K.bn_backward(dy, x, k["mask"], k["dx"], k["dres"], k["mean"], k["invstd"], inp["gamma"], k["acc_b"], k["dgamma"],
                  k["dbeta"])
    for n in ("y", "dx", "dres"):
        if k[n] is not None:
            k[n] = _rows(k[n])
    return k


def _oracle(inp, relu, eps, momentum, rm, rv, k=None):
    """float64 on the kernels' bf16 inputs, [R][C].  The full oracle from the inputs and the previous running
    statistics rm / rv; with the kernel's outputs k also the element oracle on k's own statistics."""
    x, res, dy, gamma, beta = (inp[n] for n in ("x", "res", "dy", "gamma", "beta"))
    R, C = x.shape
    x64 = x.double().requires_grad_(True)
    r64 = res.double().requires_grad_(True) if res is not None else None
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    z = F.batch_norm(x64, None, None, g64, b64, training=True, eps=eps)
    if r64 is not None:
        z = z + r64
    y = torch.relu(z) if relu else z
    y.backward(dy.double())
    xd = x.double()
    mean, var = xd.mean(0), xd.var(0, unbiased=False)
    o = dict(z=z.detach(), y=y.detach(), dx=x64.grad, dres=None if r64 is None else r64.grad, dgamma=g64.grad,
             dbeta=b64.grad, mean=mean, var=var, invstd=(var + eps).rsqrt(),
             rm=(1 - momentum) * rm.double() + momentum * mean,
             rv=(1 - momentum) * rv.double() + momentum * var * R / (R - 1))
    if k is None:
        return o
    m, s = k["mean"].double(), k["invstd"].double()
    sc = gamma.double() * s
    shift = beta.double() - m * sc
    ye = xd * sc + shift + (res.double() if res is not None else 0.0)
    d = dy.double() * _bits(k["mask"], R, C) if relu else dy.double()
    xh = (xd - m) * s
    b, c = k["acc_b"][:C].double() / R, k["acc_b"][C:].double() / R
    o.update(ye=ye.clamp_min(0) if relu else ye, sc=sc, shift=shift, d=d, xh=xh, b=b, c=c,
             dxe=gamma.double() * s * (d - b - xh * c))
    return o


def _check(inp, k, relu, eps, momentum, rm_prev, rv_prev, rm, rv, exact):
    """k: what the kernels wrote ([R][C] rows); rm_prev / rv_prev the running statistics before the call, rm / rv
    after it"""
    x, res, dy, gamma, beta = (inp[n] for n in ("x", "res", "dy", "gamma", "beta"))
    R, C = x.shape
    o = _oracle(inp, relu, eps, momentum, rm_prev, rv_prev, k)
    xd = x.double()
    ax, ax2 = xd.abs().mean(0), (xd * xd).mean(0)

    # statistics vs the full oracle; var comes back from invstd = rsqrtf(var + eps), good to ~2^-21 (var + eps)
    _le(k["mean"], o["mean"], STAT * ax, "save_mean")
    _le(1 / k["invstd"].double() ** 2 - eps, o["var"], STAT * ax2 + 2.0 ** -20 * eps, "variance")
    for name, got, want, prev, stat, scale in (
            ("running_mean", rm, o["rm"], rm_prev, o["mean"], ax),
            ("running_var", rv, o["rv"], rv_prev, o["var"] * R / (R - 1), ax2 * R / (R - 1))):
        terms = (1 - momentum) * prev.double().abs() + momentum * stat.abs()
        _le(got, want, momentum * STAT * scale + 4 * _ulp(terms, 23, 2.0 ** -149), name)

    # elementwise vs the element oracle: 1 bf16 ulp for the output rounding, plus what the fp32 intermediates round
    # (forward: sc = gamma * invstd, shift = beta - mean * sc, the fma and the residual add; backward: a = gamma *
    # invstd, the two sums over R, xhat, and the three-term difference)
    ares = res.double().abs() if res is not None else 0.0
    _le(k["y"], o["ye"], _ulp(o["ye"], 7, 2.0 ** -133) +
        2.0 ** -22 * ((xd * o["sc"]).abs() + o["shift"].abs() + beta.double().abs() + ares), "y")
    _le(k["dx"], o["dxe"], _ulp(o["dxe"], 7, 2.0 ** -133) +
        2.0 ** -21 * (gamma.double() * k["invstd"].double()).abs() *
        (o["d"].abs() + o["b"].abs() + (o["xh"] * o["c"]).abs()), "dx")
    dxh = o["d"] * o["xh"]
    _le(k["dgamma"], dxh.sum(0), STAT * dxh.abs().sum(0), "dgamma")
    _le(k["dbeta"], o["d"].sum(0), STAT * o["d"].abs().sum(0), "dbeta")
    assert _same_bits(k["dbeta"], k["acc_b"][:C]) and _same_bits(k["dgamma"], k["acc_b"][C:])
    if relu:
        assert torch.equal(_bits(k["mask"], R, C), k["y"] > 0)
    if res is not None:
        want = torch.where(_bits(k["mask"], R, C), dy, torch.zeros_like(dy)) if relu else dy
        assert torch.equal(k["dres"], want)

    if exact:
        sx, sxx = xd.sum(0), (xd * xd).sum(0)
        assert torch.equal(k["acc_f"].double(), torch.cat([sx, sxx]))
        assert torch.equal(k["acc_b"][:C].double(), o["d"].sum(0))
        assert torch.equal(k["dbeta"].double(), o["d"].sum(0))
        _le(k["mean"], sx / R, 4 * _ulp(sx / R, 23, 2.0 ** -149), "save_mean (exact sums)")


@pytest.mark.parametrize("C,rname,res,relu,momentum,eps", GEOMETRY)
def test_fused_bn_kernels_match_fp64_oracle(C, rname, res, relu, momentum, eps):
    a, b = _R[rname]
    R = a * _rl(C) + b
    assert R * C * 2 <= 64 << 20
    gen = torch.Generator(device="cuda").manual_seed(1000003 * C + R)
    for exact in ([True, False] if R <= 2 ** 18 else [False]):
        rm = torch.randn(C, device="cuda", generator=gen) * 0.1
        rv = torch.rand(C, device="cuda", generator=gen) + 0.5
        for _ in range(3):  # the running statistics followed over 3 calls
            inp = _inputs(R, C, res, exact, gen)
            rm_prev, rv_prev = rm.clone(), rv.clone()
            k = _run_binding(inp, relu, rm, rv, eps, momentum)
            _check(inp, k, relu, eps, momentum, rm_prev, rv_prev, rm, rv, exact)
        # the same call again computes the same bits
        rm2, rv2 = rm_prev.clone(), rv_prev.clone()
        k2 = _run_binding(inp, relu, rm2, rv2, eps, momentum)
        for n in k:
            assert _same_bits(k[n], k2[n]), n
        assert _same_bits(rm, rm2) and _same_bits(rv, rv2)


def _model_bn_calls(name):
    """(C, H, W, residual, relu) of every BNAct call of the network at batch 2 (32 x 32 input)"""
    from atomo_b200.models import build_model
    from atomo_b200.ops.fused_bn import BNAct
    model = build_model(name, 10)
    seen = set()

    def hook(m, args, kwargs, out):
        x = args[0]
        res = kwargs.get("residual", args[1] if len(args) > 1 else None)
        relu = kwargs.get("relu", args[2] if len(args) > 2 else False)
        seen.add((x.size(1), x.size(2), x.size(3), res is not None, bool(relu)))
    for m in model.modules():
        if isinstance(m, BNAct):
            m.register_forward_hook(hook, with_kwargs=True)
    with torch.no_grad():
        model(torch.randn(2, 3, 32, 32))
    return sorted(seen)


@pytest.mark.parametrize("network", ["ResNet18", "ResNet50"])
def test_fused_bn_model_layers_match_fp64_oracle(network):
    """every BN layer shape of the network at the benchmark's per-worker batch (128), through BNAct: autograd for
    ResNet-18, the engine's gradient sink for ResNet-50"""
    from atomo_b200.ops.fused_bn import BNAct, enable_fused_bn
    dev = torch.device("cuda", 0)
    shapes = _model_bn_calls(network)
    assert len(shapes) >= 5 and {(s[3], s[4]) for s in shapes} >= {(False, True), (True, True), (False, False)}
    n = 128
    for i, (C, h, w, res, relu) in enumerate(shapes):
        R = n * h * w
        gen = torch.Generator(device="cuda").manual_seed(7919 * i + C)
        inp = _inputs(R, C, res, False, gen)
        bn = BNAct(C).to(dev)
        with torch.no_grad():
            bn.weight.copy_(inp["gamma"])
            bn.bias.copy_(inp["beta"])
        enable_fused_bn(bn, True, arena_device=dev)
        sink = None
        if network == "ResNet50":
            sink = bn._grad_sink = (torch.zeros(C, device=dev), torch.zeros(C, device=dev))
        rm_prev, rv_prev = bn.running_mean.clone(), bn.running_var.clone()
        x = _nchw(inp["x"], n, h, w).requires_grad_(True)
        r = _nchw(inp["res"], n, h, w).requires_grad_(True) if res else None
        y = bn(x, residual=r, relu=relu)
        assert y.dtype == torch.bfloat16 and y.is_contiguous(memory_format=torch.channels_last)
        _, mask, _, mean, invstd = y.grad_fn.saved_tensors
        y.backward(_nchw(inp["dy"], n, h, w))
        if sink is not None:
            assert bn.weight.grad is None and bn.bias.grad is None
        dgamma, dbeta = sink if sink is not None else (bn.weight.grad, bn.bias.grad)
        k = dict(y=_rows(y.detach()), mask=mask, acc_f=bn._acc_fwd, mean=mean, invstd=invstd, dx=_rows(x.grad),
                 dres=_rows(r.grad) if res else None, acc_b=bn._acc_bwd, dgamma=dgamma, dbeta=dbeta)
        _check(inp, k, relu, bn.eps, bn.momentum, rm_prev, rv_prev, bn.running_mean, bn.running_var, False)


@pytest.mark.parametrize("res,relu", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("where,bad", [("x", math.nan), ("x", math.inf), ("dy", math.nan), ("dy", -math.inf)])
def test_fused_bn_non_finite_values_propagate_like_stock(where, bad, res, relu):
    """One NaN or Inf in one channel: the non-finite elements of every output are the full oracle's (a diverged
    layer shows as NaN, not as a dead channel), and every other channel keeps its bits.  With ReLU the bad dy goes
    where the output is clearly positive (NaN: the gradient passes) or clearly negative (-Inf: it is masked)."""
    R, C, ch, eps, momentum = 144, 32, 5, 1e-5, 0.1
    gen = torch.Generator(device="cuda").manual_seed(11)
    inp = _inputs(R, C, res, False, gen)
    rm0 = torch.randn(C, device="cuda", generator=gen) * 0.1
    rv0 = torch.rand(C, device="cuda", generator=gen) + 0.5
    z = _oracle(inp, relu, eps, momentum, rm0, rv0)["z"][:, ch]
    row = 0
    if where == "dy" and relu:
        row = int(torch.nonzero(z > 0.5 if math.isnan(bad) else z < -0.5)[0])
    badinp = dict(inp)
    badinp[where] = inp[where].clone()
    badinp[where][row, ch] = bad

    runs = []
    for i in (inp, badinp):
        rm, rv = rm0.clone(), rv0.clone()
        k = _run_binding(i, relu, rm, rv, eps, momentum)
        k.update(rm=rm, rv=rv)
        runs.append(k)
    clean, k = runs
    o = _oracle(badinp, relu, eps, momentum, rm0, rv0)
    for n in ("y", "dx", "dres", "dgamma", "dbeta", "mean", "invstd", "rm", "rv"):
        if o[n] is not None:
            assert torch.equal(~torch.isfinite(k[n].double()), ~torch.isfinite(o[n])), n
    other = torch.arange(C, device="cuda") != ch
    for n in ("y", "dx", "dres", "mean", "invstd", "dgamma", "dbeta", "rm", "rv"):
        if k[n] is not None:
            assert _same_bits(k[n][..., other], clean[n][..., other]), n
    for n in ("acc_f", "acc_b"):
        assert _same_bits(k[n].view(2, C)[:, other], clean[n].view(2, C)[:, other]), n
    if relu:
        assert torch.equal(_bits(k["mask"], R, C)[:, other], _bits(clean["mask"], R, C)[:, other])


def _bnact_pair(C):
    from atomo_b200.ops.fused_bn import BNAct, enable_fused_bn
    dev = torch.device("cuda", 0)
    bn = BNAct(C).to(dev)
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.5, 0.5)
        bn.running_mean.uniform_(-1, 1)
        bn.running_var.uniform_(0.5, 2)
    ref = copy.deepcopy(bn)
    enable_fused_bn(bn, True)
    return bn, ref


def test_fused_bn_empty_batch_leaves_running_statistics_alone():
    bn, ref = _bnact_pair(16)
    x = torch.empty(0, 16, 4, 4, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = bn(x, relu=True)
    assert y.shape == x.shape
    assert torch.equal(bn.running_mean, ref.running_mean) and torch.equal(bn.running_var, ref.running_var)


def test_fused_bn_one_value_per_channel_raises_like_stock():
    bn, ref = _bnact_pair(16)
    x = torch.randn(1, 16, 1, 1, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    with pytest.raises(ValueError) as stock:
        nn.BatchNorm2d.forward(ref, x)
    with pytest.raises(ValueError) as fused:
        bn(x, relu=True)
    assert str(fused.value) == str(stock.value)
    assert torch.equal(bn.running_mean, ref.running_mean) and torch.equal(bn.running_var, ref.running_var)


def test_fused_bn_misaligned_view_falls_back_to_stock():
    """a channels_last view 1 element into its storage passes every layout check but cannot be read as 16-byte
    vectors: BNAct takes the stock path and the binding refuses it (the checks run before any launch)"""
    n, C, h = 4, 32, 6
    bn, ref = _bnact_pair(C)
    numel = n * C * h * h

    def view(off):
        base = torch.randn(numel + 8, device="cuda").to(torch.bfloat16)
        return base[off:off + numel].view(n, h, h, C).permute(0, 3, 1, 2)
    x, xa, r = view(1), view(0), view(1)
    assert x.is_contiguous(memory_format=torch.channels_last) and x.data_ptr() % 16 != 0
    assert bn._can_fuse(x, None) is False
    assert bn._can_fuse(xa, r) is False

    K = ext()
    f32 = lambda k: torch.empty(k, device="cuda")
    y = torch.empty_like(xa)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        K.bn_forward(x, None, y, None, f32(2 * C), bn.weight, bn.bias, f32(C), f32(C), None, None, 1e-5, 0.1)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        K.bn_forward(xa, r, y, None, f32(2 * C), bn.weight, bn.bias, f32(C), f32(C), None, None, 1e-5, 0.1)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        K.bn_backward(x, xa, None, y, None, f32(C), f32(C), bn.weight, f32(2 * C), f32(C), f32(C))
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        K.bn_backward(xa, xa, None, torch.empty_like(xa), r, f32(C), f32(C), bn.weight, f32(2 * C), f32(C), f32(C))

    for inp, res in ((x, None), (xa, r)):
        assert torch.equal(bn(inp, residual=res, relu=True), ref(inp, residual=res, relu=True))
    assert torch.equal(bn.running_mean, ref.running_mean) and torch.equal(bn.running_var, ref.running_var)

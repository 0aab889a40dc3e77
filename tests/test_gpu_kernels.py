"""sm_90a kernel numerics vs plain PyTorch fp32 references (single GPU, loopback heap)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ext():
    from atomo_b200.ops._ext import load
    return load()


class Harness:
    """One rank that is both worker 0 and the PS (world == 1): peer pointers are local."""

    def __init__(self, shapes, code="svd", rank=3, systematic=False, lr=0.1, momentum=0.0, wd=0.0, nesterov=False,
                 seed=7):
        from atomo_b200.ops import plan as P
        from atomo_b200.runtime.flat import FlatLayout
        self.C, self.P = _ext(), P
        dev = torch.device("cuda", 0)
        self.dev = dev
        self.layout = FlatLayout(shapes)
        self.plan = P.build_plan(shapes, code, rank, systematic, offsets=self.layout.offsets)
        pl = self.plan
        total = pl.total_elems
        u8 = lambda b: torch.frombuffer(bytearray(b if len(b) else b"\0" * 16), dtype=torch.uint8).to(dev)
        self.t_layers = u8(pl.layers_bytes())
        self.t_enc = u8(P.Plan.tiles_bytes(pl.enc_tiles))
        self.t_ps = u8(P.Plan.tiles_bytes(pl.ps_tiles))
        self.t_dense = u8(P.Plan.tiles_bytes(pl.dense_tiles))
        self.t_ts = torch.tensor(pl.ts_layers or [0], dtype=torch.int32, device=dev)
        n_ts = max(len(pl.ts_layers), 1)
        self.gpart = torch.zeros(pl.gpart_floats, device=dev)
        self.vsel = torch.zeros(n_ts * P.TS_MAX_COLS * P.RCAP_MAX, device=dev)
        self.selcount = torch.zeros(n_ts, dtype=torch.int32, device=dev)
        self.sigma = torch.zeros(n_ts * P.TS_MAX_COLS, device=dev)
        self.arena = torch.zeros(pl.arena_floats, device=dev)
        self.flags = torch.zeros(1024, dtype=torch.int32, device=dev)
        self.params = torch.randn(total, device=dev)
        self.grads = torch.zeros(total, device=dev)
        self.mom = torch.zeros(total, device=dev)
        self.ctrl = u8(P.pack_ctrl(step=1, lr=lr, momentum=momentum, weight_decay=wd, nesterov=nesterov, seed=seed))
        self.t_params_peer = torch.tensor([self.params.data_ptr()], dtype=torch.int64, device=dev)
        self.t_grads_peer = torch.tensor([self.grads.data_ptr()], dtype=torch.int64, device=dev)
        self.t_flag_peer = torch.tensor([self.flags.data_ptr() + 4 * 64], dtype=torch.int64, device=dev)
        self.rank_budget = rank
        self.systematic = systematic

    def set_step(self, step):
        self.ctrl.view(torch.int32)[0] = step

    def grad_views(self):
        return self.layout.views(self.grads)

    def encode(self, random_sample=True, waterfill=False, uniforms=None, rank=None):
        C, pl = self.C, self.plan
        C.gram(self.grads, self.t_layers, self.t_enc, len(pl.enc_tiles), self.gpart)
        C.eig_sample(self.t_layers, self.t_ts, self.gpart, self.vsel, self.selcount, self.sigma,
                     self.arena.data_ptr(), pl.arena_floats, self.ctrl, uniforms,
                     self.rank_budget if rank is None else rank, random_sample, waterfill, self.systematic, 0, 1024)
        C.project_push(self.grads, self.t_layers, self.t_enc, len(pl.enc_tiles), self.vsel, self.selcount,
                       self.arena.data_ptr(), pl.arena_floats, self.flags.data_ptr(), self.ctrl, 0, True)

    def ps_update(self):
        C, pl = self.C, self.plan
        C.ps_update(self.t_layers, self.t_ps, len(pl.ps_tiles), 1, 1, 1, self.params, self.mom, self.t_params_peer,
                    0, self.t_grads_peer, 0, self.arena.data_ptr(), pl.arena_floats, self.flags.data_ptr(),
                    self.t_flag_peer, self.ctrl, int(5e9), 1.0, min(len(pl.ps_tiles), 296))

    def slot(self, layer):
        P = self.P
        base = self.arena[layer.slot_off:]
        hdr = base[:4].view(torch.int32)
        count = int(hdr[0])
        rc, n = layer.rcap, layer.cols
        s = base[4:4 + rc][:count]
        V = base[4 + rc:4 + rc + rc * n].view(rc, n)[:count]
        uo = P.slot_u_off(rc, n)
        U = base[uo:uo + layer.rows * rc].view(layer.rows, rc)[:, :count]
        return count, s, V, U

    def tall(self, layer, flat):
        """tall (rows x cols) view of a layer inside a flat buffer"""
        t = flat[layer.off:layer.off + layer.numel]
        return torch.as_strided(t, (layer.rows, layer.cols), (layer.row_stride, layer.col_stride))


SHAPES = [(64, 32, 3, 3), (50, 20, 5, 5), (10, 512), (128, 64, 1, 1), (64,), (300, 200), (33, 7, 3, 3), (10,)]


def _fill_grads(h, decay=True, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    for l, v in zip(h.plan.layers, h.grad_views()):
        x = torch.randn(v.shape, device=h.dev, generator=g)
        if decay and l.route == 1:
            tall = torch.randn(l.rows, l.cols, device=h.dev, generator=g) * torch.logspace(0, -1.5, l.cols, device=h.dev)
            mix = torch.linalg.qr(torch.randn(l.cols, l.cols, device=h.dev, generator=g)).Q
            h.tall(l, h.grads).copy_(tall @ mix)
        else:
            v.copy_(x)


def test_gram_matches_torch():
    h = Harness(SHAPES)
    _fill_grads(h)
    pl = h.plan
    h.C.gram(h.grads, h.t_layers, h.t_enc, len(pl.enc_tiles), h.gpart)
    torch.cuda.synchronize()
    for l in pl.layers:
        if l.route != 1:
            continue
        A = h.tall(l, h.grads).double()
        G = h.gpart[l.gpart_off:l.gpart_off + l.ntiles * l.cols * l.cols].view(l.ntiles, l.cols, l.cols).sum(0)
        ref = (A.T @ A).float()
        assert torch.allclose(G, ref, rtol=2e-4, atol=2e-4 * float(ref.abs().max())), l.shape


def test_full_rank_topk_reconstructs_gradient_exactly():
    """random_sample=False with rank >= cols keeps every atom: U S V^T must equal A (complete basis)."""
    shapes = [(64, 32, 3, 3), (10, 512), (20, 1, 5, 5)]  # cols = 18, 10, 50 -> rcap 20, 12, 32(cap)
    h = Harness(shapes, rank=0)  # rank 0 -> slot capacity = cols (<= 32)
    _fill_grads(h)
    h.encode(random_sample=False, rank=0)
    torch.cuda.synchronize()
    for l in h.plan.layers:
        count, s, V, U = h.slot(l)
        A = h.tall(l, h.grads)
        assert count == min(l.cols, l.rcap)
        sv = torch.linalg.svdvals(A.double()).float()[:count]
        assert torch.allclose(s, sv, rtol=2e-3, atol=2e-4 * float(sv[0])), (l.shape, s, sv)
        assert torch.allclose(V @ V.T, torch.eye(count, device=h.dev), atol=2e-4)
        if count == l.cols:
            rec = (U * s) @ V
            assert float((rec - A).norm() / A.norm()) < 2e-4, l.shape


def test_sampled_atoms_are_unbiased_and_respect_budget():
    shapes = [(32, 16, 3, 3), (10, 128)]
    h = Harness(shapes, rank=3)
    _fill_grads(h, seed=3)
    acc = [torch.zeros(l.rows, l.cols, device=h.dev) for l in h.plan.layers]
    counts = [0.0 for _ in h.plan.layers]
    T = 600
    for t in range(1, T + 1):
        h.set_step(t)
        h.encode()
        for i, l in enumerate(h.plan.layers):
            c, s, V, U = h.slot(l)
            counts[i] += c
            acc[i] += (U * s) @ V
    torch.cuda.synchronize()
    for i, l in enumerate(h.plan.layers):
        A = h.tall(l, h.grads)
        rel = float((acc[i] / T - A).norm() / A.norm())
        assert rel < 0.12, (l.shape, rel)
        # E[#atoms] <= rank (single clip); resample-on-empty (svd.py:65-66) inflates it by 1/(1-P(0)) ~ 5%
        assert 0.5 <= counts[i] / T <= 3.4, counts[i] / T


def test_systematic_waterfill_sends_exactly_rank_atoms():
    h = Harness([(64, 16, 3, 3)], rank=3, systematic=True)
    _fill_grads(h)
    seen = set()
    for t in range(1, 40):
        h.set_step(t)
        h.encode(waterfill=True)
        c, s, V, U = h.slot(h.plan.layers[0])
        seen.add(c)
    assert seen <= {3}, seen


@pytest.mark.parametrize("momentum,nesterov,wd", [(0.0, False, 0.0), (0.9, False, 1e-3), (0.9, True, 0.0)])
def test_ps_update_lowrank_and_dense_matches_reference(momentum, nesterov, wd):
    h = Harness(SHAPES, rank=3, lr=0.05, momentum=momentum, wd=wd, nesterov=nesterov)
    ref_p = h.params.clone()
    ref_m = torch.zeros_like(ref_p)
    for step in (1, 2, 3):
        h.set_step(step)
        _fill_grads(h, seed=step)
        h.encode()
        torch.cuda.synchronize()
        # reference gradient estimate: decoded factors for low-rank layers, raw gradient for dense layers
        est = torch.zeros_like(ref_p)
        for l in h.plan.layers:
            if l.route == 1:
                c, s, V, U = h.slot(l)
                h.tall(l, est).copy_((U * s) @ V)
            else:
                est[l.off:l.off + l.numel] = h.grads[l.off:l.off + l.numel]
        d = est + wd * ref_p
        if momentum:
            ref_m = d.clone() if step == 1 else momentum * ref_m + d
            d = d + momentum * ref_m if nesterov else ref_m
        ref_p = ref_p - 0.05 * d
        h.ps_update()
        torch.cuda.synchronize()
        assert int(h.flags[64]) == step + 1  # param flag published
        for l in h.plan.layers:
            a, b = h.params[l.off:l.off + l.numel], ref_p[l.off:l.off + l.numel]
            assert torch.allclose(a, b, rtol=1e-4, atol=1e-5), (step, l.shape, float((a - b).abs().max()))
    assert int(h.ctrl.view(torch.int32)[1]) == 0


def test_qsgd_kernel_matches_oracle_bits():
    from atomo_b200 import codings
    C = _ext()
    dev = torch.device("cuda", 0)
    for scheme, q, bucket in (("qsgd", 4, 512), ("qsgd", 2, 256), ("terngrad", 4, 512), ("qsgd", 8, 1024)):
        torch.manual_seed(q)
        n = 5 * bucket + 37
        g = torch.randn(n, device=dev)
        u = torch.rand(((n + bucket - 1) // bucket) * bucket, device=dev)
        E = 64 // (2 + q)
        L = (bucket + E - 1) // E
        nb = (n + bucket - 1) // bucket
        words = torch.zeros(nb * L, dtype=torch.int64, device=dev)
        norms = torch.zeros(nb, device=dev)
        ctrl = torch.frombuffer(bytearray(__import__("atomo_b200.ops.plan", fromlist=["x"]).pack_ctrl()), dtype=torch.uint8).to(dev)
        clip = None
        if scheme == "terngrad":
            clip = (2.5 * g.std(unbiased=False)).reshape(1).contiguous()
        C.qsgd_encode(g, n, bucket, q, scheme == "terngrad", clip, words.data_ptr(), norms.data_ptr(), ctrl, 0, u)
        coder = codings.build(scheme, quantization_level=q, bucket_size=bucket)
        code = coder.encode(g.cpu(), uniforms=u.cpu())
        torch.cuda.synchronize()
        assert torch.allclose(norms.cpu(), code["norms"], rtol=1e-5)
        # decode both (element-level comparison tolerates 1-ulp rounding-boundary flips)
        mine = dict(code)
        mine["words"], mine["norms"] = words.cpu().view(nb, L), norms.cpu()
        a, b = coder.decode(mine), coder.decode(code)
        tol = 1e-4 * float(b.abs().max())
        mism = float(((a - b).abs() > tol).float().mean())
        assert mism < 2e-3, (scheme, q, mism)
        assert float((words.cpu().view(nb, L) != code["words"]).float().mean()) < 2e-2
        # PS-side kernel decode == oracle decode of the same words
        out = torch.zeros(n, device=dev)
        wp = torch.tensor([words.data_ptr()], dtype=torch.int64, device=dev)
        npz = torch.tensor([norms.data_ptr()], dtype=torch.int64, device=dev)
        C.qsgd_decode_sum(wp, npz, 1, n, bucket, q, scheme == "terngrad", out, 0, ctrl, 0)
        torch.cuda.synchronize()
        assert torch.allclose(out.cpu(), a, rtol=1e-5, atol=1e-6)


def test_entrywise_kernel_matches_oracle():
    from atomo_b200.ops import plan as P
    C = _ext()
    dev = torch.device("cuda", 0)
    shapes = [(64, 50), (1000,), (33, 7, 3, 3)]
    h = Harness(shapes, code="sgd")
    _fill_grads(h, decay=False)
    total = h.plan.total_elems
    cap = total
    u = torch.rand(total, device=dev)
    idx = torch.zeros(cap, dtype=torch.int32, device=dev)
    val = torch.zeros(cap, device=dev)
    cnt = torch.zeros(64, dtype=torch.int32, device=dev)
    l1 = torch.zeros(len(shapes), device=dev)
    local = torch.zeros(1, dtype=torch.int32, device=dev)
    budget = 0.1
    C.entrywise_encode(h.grads, h.t_layers, h.t_dense, len(h.plan.dense_tiles), l1, budget, idx.data_ptr(),
                       val.data_ptr(), cnt.data_ptr(), cap, local, h.flags.data_ptr(), h.ctrl, 0, u, True)
    torch.cuda.synchronize()
    n = int(cnt[0])
    dense = torch.zeros(total, device=dev)
    dense.index_add_(0, idx[:n].long(), val[:n])
    ref = torch.zeros(total, device=dev)
    for l in h.plan.layers:
        g = h.grads[l.off:l.off + l.numel]
        assert float(l1[l.index]) == pytest.approx(float(g.abs().sum()), rel=1e-4)
        p = (budget * l.numel * g.abs() / g.abs().sum()).clamp(max=1.0)
        keep = u[l.off:l.off + l.numel] < p
        ref[l.off:l.off + l.numel] = torch.where(keep, g / p, torch.zeros_like(g))
    mism = float(((dense != 0) != (ref != 0)).float().mean())
    assert mism < 1e-3
    both = (dense != 0) & (ref != 0)
    assert torch.allclose(dense[both], ref[both], rtol=1e-4)
    assert int(h.flags[0]) == 1  # push flag raised with the step
    # PS scatter
    out = torch.ones(total, device=dev)
    ip = torch.tensor([idx.data_ptr()], dtype=torch.int64, device=dev)
    vp = torch.tensor([val.data_ptr()], dtype=torch.int64, device=dev)
    cp = torch.tensor([cnt.data_ptr()], dtype=torch.int64, device=dev)
    C.entrywise_scatter(ip, vp, cp, 1, cap, out, total, 0, h.ctrl, 0)
    torch.cuda.synchronize()
    assert torch.allclose(out, dense)


def test_wgmma_skinny_gemm_matches_fp32_matmul():
    """Grouped tf32 wgmma GEMM vs torch fp32 matmul for every operand layout the subspace route uses."""
    import struct
    C = _ext()
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    ctrl = torch.frombuffer(bytearray(__import__("atomo_b200.ops.plan", fromlist=["x"]).pack_ctrl()), dtype=torch.uint8).to(dev)
    cases = []
    tiles = []

    def add(A_view, Bop, sb_j, sb_k, N, splits=1):
        """A_view: (M_total x K) strided view; Bop element (j,k) at Bop.data_ptr + (j*sb_j + k*sb_k)*4"""
        Mtot, K = A_view.shape
        sa_i, sa_k = A_view.stride()
        out = torch.zeros(Mtot, N, device=dev)
        for r0 in range(0, Mtot, 128):
            base_ptr = A_view.data_ptr() + 4 * r0 * sa_i
            if sa_k == 1 and sa_i % 4 == 0 and (base_ptr // 4) % 4 == 0:
                av = 1
            elif sa_i == 1 and sa_k % 4 == 0 and (base_ptr // 4) % 4 == 0:
                av = 2
            else:
                av = 0
            klen = -(-(-(-K // splits)) // 32) * 32
            for kb in range(0, K, klen):
                tiles.append(struct.pack("<3Q12i", base_ptr, Bop.data_ptr(), out.data_ptr() + 4 * r0 * N, sa_i, sa_k,
                                         sb_j, sb_k, N, min(128, Mtot - r0), N, K, av, kb, klen, int(splits > 1)))
        return out

    # forward: Y = A X with X^T stored (l x n); row-major A with K = 784 (not a multiple of 32), 800 rows
    A1 = torch.randn(800, 784, device=dev)
    Xt1 = torch.randn(16, 784, device=dev)
    cases.append((add(A1, Xt1, 784, 1, 16), A1 @ Xt1.t()))
    # backward: B = A^T Q (operand rows are A's columns: stride-1 along i), Q is m x l row-major
    Q1 = torch.randn(800, 16, device=dev)
    cases.append((add(A1.t(), Q1, 1, 16, 16), A1.t() @ Q1))
    cases.append((add(A1.t(), Q1, 1, 16, 16, splits=5), A1.t() @ Q1))   # split-K with atomic accumulation
    cases.append((add(A1, Xt1, 784, 1, 16, splits=3), A1 @ Xt1.t()))
    # transposed-orientation layer (tall view of a wide matrix), N = 32, odd sizes -> scalar gather path
    W = torch.randn(301, 517, device=dev)
    X2 = torch.randn(32, 301, device=dev)
    cases.append((add(W.t(), X2, 301, 1, 32), W.t() @ X2.t()))
    Q2 = torch.randn(517, 32, device=dev)
    cases.append((add(W, Q2, 1, 32, 32), W @ Q2))
    t = torch.frombuffer(bytearray(b"".join(tiles)), dtype=torch.uint8).to(dev)
    C.skinny_gemm(t, len(tiles), ctrl, 64)
    torch.cuda.synchronize()
    assert int(ctrl.view(torch.int32)[1]) == 0, "skinny GEMM rejected a tile"
    for got, ref in cases:
        err = float((got - ref).abs().max() / ref.abs().max())
        assert err < 3e-3, err  # tf32 inputs (10-bit mantissa), fp32 accumulate


@pytest.mark.parametrize("C,hw,with_res,relu,batch", [(64, 32, False, True, 16), (128, 16, True, True, 16),
                                                      (512, 4, True, True, 16), (256, 8, False, False, 16),
                                                      (96, 5, True, False, 16), (64, 32, True, True, 128),
                                                      (512, 4, False, True, 128), (2048, 2, True, True, 8)])
def test_fused_bn_matches_stock_ops(C, hw, with_res, relu, batch):
    """Fused BN(+residual)(+ReLU) NHWC bf16 kernels vs nn.BatchNorm2d + add + relu (fp32 reference)."""
    import copy
    from atomo_b200.ops.fused_bn import BNAct
    dev = torch.device("cuda", 0)
    torch.manual_seed(C + hw)
    bn = BNAct(C).to(dev)
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.5, 0.5)
    ref = copy.deepcopy(bn)
    bn.fused = True
    x32 = torch.randn(batch, C, hw, hw, device=dev) * 2 + 0.3
    r32 = torch.randn(batch, C, hw, hw, device=dev)
    x = x32.to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    r = r32.to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True) if with_res else None
    xr = x.detach().float().requires_grad_(True)          # fp32 reference on the same (bf16-rounded) values
    rr = r.detach().float().requires_grad_(True) if with_res else None
    y = bn(x, residual=r, relu=relu)
    yr = ref(xr, residual=rr, relu=relu)
    assert y.dtype == torch.bfloat16 and y.is_contiguous(memory_format=torch.channels_last)
    assert torch.allclose(y.float(), yr, rtol=2e-2, atol=2e-2)
    assert torch.allclose(bn.running_mean, ref.running_mean, rtol=1e-3, atol=1e-3)
    assert torch.allclose(bn.running_var, ref.running_var, rtol=1e-2, atol=1e-3)
    g32 = torch.randn_like(yr)
    y.backward(g32.to(torch.bfloat16).contiguous(memory_format=torch.channels_last))
    yr.backward(g32.to(torch.bfloat16).float())
    scale = float(xr.grad.abs().max())
    # a ReLU mask can flip where |y| ~ 0 (bf16 vs fp32 rounding): allow a vanishing fraction of outliers
    bad = ((x.grad.float() - xr.grad).abs() > 3e-2 * scale + 1e-3).float().mean()
    assert float(bad) < 1e-4, float(bad)
    assert torch.allclose(bn.weight.grad, ref.weight.grad, rtol=3e-2, atol=3e-2 * float(ref.weight.grad.abs().max()))
    assert torch.allclose(bn.bias.grad, ref.bias.grad, rtol=3e-2, atol=3e-2 * float(ref.bias.grad.abs().max()))
    if with_res:
        bad = ((r.grad.float() - rr.grad).abs() > 2e-2 * float(rr.grad.abs().max()) + 1e-3).float().mean()
        assert float(bad) < 1e-4, float(bad)


def test_fused_bn_graph_capture_and_grad_sinks():
    """The fused BN must replay inside a CUDA graph (the engine's step is one graph) and dgamma/dbeta must land
    in the caller's sink (no autograd gradient for weight / bias)."""
    from atomo_b200.ops.fused_bn import BNAct, enable_fused_bn
    dev = torch.device("cuda", 0)
    torch.manual_seed(3)
    bn = BNAct(128).to(dev)
    enable_fused_bn(bn, True)
    sink = (torch.zeros(128, device=dev), torch.zeros(128, device=dev))
    bn._grad_sink = sink
    x = (torch.randn(64, 128, 16, 16, device=dev)).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    x.requires_grad_(True)
    g = torch.randn(64, 128, 16, 16, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)

    def step():
        x.grad = None
        y = bn(x, relu=True)
        y.backward(g)
        return y
    for _ in range(3):
        y_eager = step().detach().clone()
    torch.cuda.synchronize()
    dx_eager, dg_eager = x.grad.clone(), sink[0].clone()
    assert bn.weight.grad is None and float(dg_eager.abs().sum()) > 0
    rm = bn.running_mean.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y_static = step()
    sink[0].zero_()
    for _ in range(5):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.allclose(y_static.float(), y_eager.float(), rtol=2e-2, atol=2e-2)   # fp32 atomics reorder
    assert torch.allclose(x.grad.float(), dx_eager.float(), rtol=1e-2, atol=1e-3)
    assert torch.allclose(sink[0], dg_eager, rtol=1e-3, atol=1e-3)
    assert not torch.equal(bn.running_mean, rm)      # the running statistics kept moving under replay


@pytest.mark.parametrize("W,rank", [(8, 3), (8, 8), (4, 16)])
def test_ps_update_many_virtual_workers_multi_chunk_K(W, rank):
    """W 'virtual workers' on one GPU (W arenas, all local): exercises the concatenated-K path of
    ps_update_kernel with K = sum_w count_w > PS_KC (several K chunks, float4 group gathers, SV reload)."""
    h = Harness(SHAPES, rank=rank, lr=0.05, momentum=0.9)
    pl = h.plan
    dev = h.dev
    arena = torch.zeros(W * pl.arena_floats, device=dev)
    grads = [torch.zeros_like(h.grads) for _ in range(W)]
    t_grads_peer = torch.tensor([g.data_ptr() for g in grads], dtype=torch.int64, device=dev)
    est = torch.zeros_like(h.params)
    for w in range(W):
        _fill_grads(h, seed=100 + w)
        grads[w].copy_(h.grads)
        C = h.C
        C.gram(h.grads, h.t_layers, h.t_enc, len(pl.enc_tiles), h.gpart)
        C.eig_sample(h.t_layers, h.t_ts, h.gpart, h.vsel, h.selcount, h.sigma, arena.data_ptr(), pl.arena_floats,
                     h.ctrl, None, rank, True, False, False, w, 1024)
        C.project_push(h.grads, h.t_layers, h.t_enc, len(pl.enc_tiles), h.vsel, h.selcount, arena.data_ptr(),
                       pl.arena_floats, h.flags.data_ptr(), h.ctrl, w, True)
        torch.cuda.synchronize()
        # reference: decode this worker's slots
        saved = h.arena
        h.arena = arena[w * pl.arena_floats:(w + 1) * pl.arena_floats]
        for l in pl.layers:
            if l.route == 1:
                c, s, V, U = h.slot(l)
                h.tall(l, est).add_((U * s) @ V)
            else:
                est[l.off:l.off + l.numel] += grads[w][l.off:l.off + l.numel]
        h.arena = saved
    assert all(int(h.flags[w]) == 1 for w in range(W))
    ref_p = h.params - 0.05 * (est / W)          # first step: momentum buffer = gradient
    h.C.ps_update(h.t_layers, h.t_ps, len(pl.ps_tiles), W, W, 1, h.params, h.mom, h.t_params_peer, 0, t_grads_peer, 0,
                  arena.data_ptr(), pl.arena_floats, h.flags.data_ptr(), h.t_flag_peer, h.ctrl, int(5e9), 1.0 / W,
                  min(len(pl.ps_tiles), 296))
    torch.cuda.synchronize()
    assert int(h.ctrl.view(torch.int32)[1]) == 0
    for l in pl.layers:
        a, b = h.params[l.off:l.off + l.numel], ref_p[l.off:l.off + l.numel]
        assert torch.allclose(a, b, rtol=2e-4, atol=2e-5), (l.shape, float((a - b).abs().max()))

"""Fused engine end-to-end on the GPU (1 GPU always; 2 GPUs when present)."""

import pytest
import torch

from shadow_harness import batch, nccl_init, spawn

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("code,net,graph", [("svd", "LeNet", False), ("svd", "ResNet18", True), ("sgd", "LeNet", True),
                                           ("qsgd", "LeNet", True), ("terngrad", "LeNet", False),
                                           ("entrywise", "LeNet", True)])
def test_single_gpu_engine_trains(code, net, graph):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.engine import FusedEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    model = build_model(net, 10)
    eng = FusedEngine(model, 0, 1, code=code, svd_rank=3, lr=0.05, momentum=0.9, use_graph=graph,
                      entry_budget=0.25, seed=3)
    x, y = batch(net, 64)
    eng.prepare(x, y, warmup=2)
    first = None
    for i in range(30):
        stats = eng.train_step(x, y)
        if first is None:
            first = float(stats[0])
    torch.cuda.synchronize()
    last = float(stats[0])
    assert eng.error_code() == 0
    assert eng.device_step() == eng.step == 33
    assert torch.isfinite(torch.tensor(last)) and last < first, (first, last)
    assert eng.launches_per_step >= 3
    eng.close()


def test_dense_engine_matches_plain_sgd():
    """--code sgd on one GPU must reproduce torch.optim.SGD exactly (same grads, fused update)."""
    import copy
    from atomo_b200.models import build_model
    from atomo_b200.runtime.engine import FusedEngine
    torch.manual_seed(1)
    torch.cuda.set_device(0)
    model = build_model("LeNet", 10)
    ref = copy.deepcopy(model).cuda()
    opt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9)
    eng = FusedEngine(model, 0, 1, code="sgd", lr=0.05, momentum=0.9, use_graph=False)
    x, y = batch("LeNet", 32)
    eng.prepare(x, y, warmup=0)
    xc, yc = x.cuda(), y.cuda()
    for _ in range(5):
        eng.train_step(x, y)
        opt.zero_grad()
        torch.nn.functional.cross_entropy(ref(xc), yc).backward()
        opt.step()
    torch.cuda.synchronize()
    for p, q in zip(eng.model.parameters(), ref.parameters()):
        assert torch.allclose(p, q, rtol=1e-4, atol=1e-5)
    eng.close()


def _two_rank_worker(rank, world, port, code, out):
    import torch.distributed as dist
    from atomo_b200.models import build_model
    from atomo_b200.runtime.engine import FusedEngine
    nccl_init(rank, world, port)
    torch.manual_seed(0)
    model = build_model("LeNet", 10)
    eng = FusedEngine(model, rank, world, code=code, svd_rank=3, lr=0.05, momentum=0.9, use_graph=True, seed=5,
                      entry_budget=0.25)
    x, y = batch("LeNet", 32, seed=rank)
    eng.prepare(x, y, warmup=2)
    losses = []
    for _ in range(20):
        losses.append(float(eng.train_step(x, y)[0]))
    torch.cuda.synchronize()
    dist.barrier()           # the PS's last launch (stores into OUR copy) has completed
    torch.cuda.synchronize()
    # every rank must hold identical parameters after the multicast / peer broadcast
    flat = eng.flat_params.clone()
    gathered = [torch.zeros_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    same = all(torch.equal(gathered[0], g) for g in gathered)
    out.put((rank, eng.error_code(), same, losses[0], losses[-1], eng.heap.mode, eng.heap.has_multicast))
    eng.close()
    dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("code", ["svd", "sgd", "qsgd", "entrywise"])
def test_two_gpu_engine_keeps_replicas_identical(code):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    port = 29620 + 3 * ["svd", "sgd", "qsgd", "entrywise"].index(code)
    res = spawn(2, _two_rank_worker, port, code, timeout=300)
    for rank, err, same, l0, l1, mode, mc in res:
        assert err == 0 and same, res
        assert l1 < l0, res
    print("heap mode:", res[0][5], "multicast:", res[0][6])


def _lowrank_plus_noise(m, n, k, dev, gen, noise=0.02):
    a = torch.randn(m, k, device=dev, generator=gen) * torch.logspace(0, -1, k, device=dev)
    b = torch.randn(k, n, device=dev, generator=gen)
    return a @ b / (k ** 0.5) + noise * torch.randn(m, n, device=dev, generator=gen)


@pytest.mark.parametrize("gemm_impl", ["torch", "wgmma"])
def test_subspace_route_matches_truncated_svd_and_ps_applies_it(gemm_impl):
    """Square-ish layers (fc) go through the randomized range finder; with top-k selection the factors in
    the PS slot must be a near-optimal rank-k approximation and ps_update must apply exactly them."""
    from atomo_b200.models import build_model
    from atomo_b200.ops import plan as P
    from atomo_b200.runtime.engine import FusedEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    eng = FusedEngine(build_model("FC", 10), 0, 1, code="svd", svd_rank=3, lr=0.1, momentum=0.0, use_graph=False,
                      random_sample=False, subspace=True, gemm_impl=gemm_impl)
    ext = eng.plan.ext
    assert ext is not None and len(ext.layers) == 2
    gen = torch.Generator(device="cuda").manual_seed(1)
    eng.flat_grads.zero_()
    truth = {}
    for l in ext.layers:
        A = _lowrank_plus_noise(l.rows, l.cols, 6, dev, gen)
        torch.as_strided(eng.flat_grads, (l.rows, l.cols), (l.row_stride, l.col_stride), l.off).copy_(A)
        truth[l.index] = A
    before = eng.flat_params.clone()
    eng._encode_push()
    torch.cuda.synchronize()
    arena = eng.heap.tensor("arena")
    for l in ext.layers:
        base = arena[l.slot_off:]
        count = int(base[:4].view(torch.int32)[0])
        assert count == 3
        s = base[4:4 + count]
        V = base[4 + l.rcap:4 + l.rcap + l.rcap * l.cols].view(l.rcap, l.cols)[:count]
        uo = P.slot_u_off(l.rcap, l.cols)
        U = base[uo:uo + l.rows * l.rcap].view(l.rows, l.rcap)[:, :count]
        A = truth[l.index]
        rec = (U * s) @ V
        sv = torch.linalg.svdvals(A)
        best = float(sv[3:].norm())
        err = float((A - rec).norm())
        assert err <= 1.25 * best + 1e-3 * float(A.norm()), (l.shape, err, best)
        assert torch.allclose(s, sv[:3], rtol=0.05), (s, sv[:3])
        truth[l.index] = rec
    eng._ps_update()
    torch.cuda.synchronize()
    assert eng.error_code() == 0
    for l in ext.layers:
        p_new = torch.as_strided(eng.flat_params, (l.rows, l.cols), (l.row_stride, l.col_stride), l.off)
        p_old = torch.as_strided(before, (l.rows, l.cols), (l.row_stride, l.col_stride), l.off)
        assert torch.allclose(p_new, p_old - 0.1 * truth[l.index], rtol=1e-4, atol=1e-5), l.shape
    eng.close()


@pytest.mark.parametrize("net", ["FC", "LeNet", "VGG11"])
def test_subspace_engine_trains(net):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.engine import FusedEngine
    torch.manual_seed(0)
    torch.cuda.set_device(0)
    eng = FusedEngine(build_model(net, 10), 0, 1, code="svd", svd_rank=3, lr=0.02, momentum=0.9, use_graph=True,
                      subspace=True)
    x, y = batch(net, 64)
    eng.prepare(x, y, warmup=2)
    first = float(eng.train_step(x, y)[0])
    for _ in range(40):
        stats = eng.train_step(x, y)
    torch.cuda.synchronize()
    assert eng.error_code() == 0 and float(stats[0]) < first
    eng.close()


def test_engine_checkpoint_resume_roundtrip(tmp_path):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model
    from atomo_b200.runtime.engine import FusedEngine
    torch.cuda.set_device(0)
    d = str(tmp_path) + "/"
    x, y = SyntheticImageDataset((1, 28, 28), 10, 512).materialize(32)
    x, y = x.pin_memory(), y.pin_memory()

    def make():
        torch.manual_seed(0)
        return FusedEngine(build_model("LeNet", 10), 0, 1, code="sgd", lr=0.05, momentum=0.9,
                           use_graph=False, seed=5)

    a = make()
    a.prepare(x, y, warmup=0)
    for _ in range(5):
        a.train_step(x, y)
    a.save_checkpoint(d)                       # step 5
    for _ in range(3):
        a.train_step(x, y)
    torch.cuda.synchronize()
    want = a.flat_params.clone()
    a.close()

    b = make()
    b.prepare(x, y, warmup=0)
    b.load_checkpoint(d, 5)
    assert b.device_step() == 6
    for _ in range(3):
        b.train_step(x, y)
    torch.cuda.synchronize()
    # dense coder: deterministic up to cuDNN's atomics.  (With a sampling coder a 1e-7 difference in a
    # probability can flip a Bernoulli draw, so resumed runs are statistically, not bitwise, identical.)
    assert torch.allclose(b.flat_params, want, rtol=1e-3, atol=1e-4)
    b.close()

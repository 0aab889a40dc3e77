#!/usr/bin/env python
"""Headline benchmark: ResNet-18 / CIFAR-10-shaped synthetic images/sec through the
fused NVLink parameter-server engine (BASELINE.json metric + config 2).

    python bench.py --gpus 1 --steps 50 --warmup 5
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \
           --master-port 29500 bench.py --gpus 8 --steps 50 --warmup 5

Rank 0 prints ONE JSON line.  ``value`` is the whole-job images/s, timed on the
device with CUDA events around exactly K steps (barrier + synchronize on both
sides, max over ranks).  ``e2e`` repeats the measurement through the public
``FusedEngine.train_step(x, y)`` API with the batch coming from pinned host
memory every step and the loss read back to the host every step.

``--dump-outputs DIR`` writes, after the timed steps, what the last step computed: ``loss.npy``
(loss, prec@1, prec@5 as returned by ``train_step``) and ``params.npy`` (rank 0's model state after the
step, every floating-point ``state_dict`` entry flattened in order, float32; a fixed seeded sample when it
exceeds 64 MB).  Inputs, initial weights and coder seeds are fixed, so two builds run with the same
arguments can be compared output for output: the step is bitwise reproducible (cuDNN runs deterministic,
heuristically chosen algorithms and the project's kernels reduce in a fixed order).  ``--cudnn-benchmark``
lets cuDNN autotune instead, which can pick different algorithms, and so different last bits (and, through
the coder's Bernoulli draws, different atoms), from run to run.

``--impl reference`` reports the reference arm (not installable here: Python-2 /
mpi4py / missing module — see DESIGN.md); ``--impl nccl-baseline`` runs the
reference *algorithm* re-hosted on torch.distributed/NCCL + torch.linalg.svd
(this repo's role classes), the bar BASELINE.md names.
"""
import argparse
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "ResNet-18 CIFAR-10 images/sec (whole box, device-timed, max over ranks)"


def metric_name(args):
    if args.network == "ResNet18" and args.dataset == "Cifar10":
        return METRIC
    return "%s %s-shaped images/sec (whole box, device-timed, max over ranks)" % (args.network, args.dataset)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=50, help="timed steps (>= 1)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", type=str, default="atomo_b200", choices=["atomo_b200", "reference", "nccl-baseline"])
    ap.add_argument("--network", type=str, default="ResNet18")
    ap.add_argument("--batch-size", type=int, default=128, help="per-worker batch (run_pytorch.sh: 128)")
    ap.add_argument("--code", type=str, default="svd")
    ap.add_argument("--svd-rank", type=int, default=3)
    ap.add_argument("--dtype", type=str, default="bf16", choices=["bf16", "fp32"])
    ap.add_argument("--ps-mode", type=str, default="sharded", choices=["sharded", "colocated", "dedicated"],
                    help="sharded: every GPU trains and owns 1/N of the PS tiles (default); colocated: rank 0 owns "
                         "the whole PS and also trains; dedicated: rank 0 only serves (the reference's topology)")
    ap.add_argument("--engine", type=str, default="auto", choices=["auto", "shadow", "fused"],
                    help="shadow = overlapped sharded bf16 engine (runtime/shadow_engine.py); fused = round-1 "
                         "fp32-flat engine (runtime/engine.py: fp32 runs, qsgd / terngrad / entrywise)")
    ap.add_argument("--groups", type=int, default=5, help="backward groups of the shadow engine")
    ap.add_argument("--no-overlap", dest="overlap", action="store_false", default=True)
    ap.add_argument("--optimizer", type=str, default="sgd", choices=["sgd", "adam"])
    ap.add_argument("--no-fp32-line", dest="fp32_line", action="store_false", default=True,
                    help="skip the nested fp32 measurement of the same config (run in a child process)")
    ap.add_argument("--fp32-line-multi", action="store_true", default=False,
                    help="also run the nested fp32 child when launched on more than one GPU (one child per rank, "
                         "rendezvous on MASTER_PORT + 53); off by default: the scaling runs stay single-purpose")
    ap.add_argument("--ps-grid", type=int, default=0)
    ap.add_argument("--main-priority", type=int, default=0)
    ap.add_argument("--side-priority", type=int, default=-1)
    ap.add_argument("--no-warm-start", dest="warm_start", action="store_false", default=True)
    ap.add_argument("--max-sweeps", type=int, default=1)
    ap.add_argument("--sampling", type=str, default="bernoulli")
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--no-channels-last", dest="channels_last", action="store_false", default=True,
                    help="activations are NHWC by default (faster convs/BN than NCHW)")
    ap.add_argument("--dataset", type=str, default="Cifar10", choices=["Cifar10", "ImageNet", "MNIST"])
    ap.add_argument("--quantization-level", type=int, default=4)
    ap.add_argument("--entry-budget", type=float, default=0.05)
    ap.add_argument("--subspace", type=str, default="auto", choices=["auto", "on", "off"])
    ap.add_argument("--fused-bn", type=str, default="auto", choices=["auto", "on", "off"])
    ap.add_argument("--cudnn-benchmark", dest="cudnn_benchmark", action="store_true", default=False,
                    help="let cuDNN autotune its algorithms: the choice (and so the outputs) can differ from run to run")
    ap.add_argument("--no-cudnn-benchmark", dest="cudnn_benchmark", action="store_false")
    ap.add_argument("--momentum", type=float, default=0.9)
    ap.add_argument("--lr", type=float, default=0.01)
    ap.add_argument("--dump-outputs", type=str, default=None, metavar="DIR",
                    help="after the timed steps, write the last step's outputs as DIR/<name>.npy")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be >= 1")
    return args


DUMP_MAX_BYTES = 64 * 2 ** 20


def dump_outputs(out_dir, stats, model):
    """What one train_step hands its caller: the returned stats and the model state it updated in place."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "loss.npy"), stats.detach().float().cpu().numpy())
    flat = torch.cat([t.detach().float().reshape(-1).cpu() for t in model.state_dict().values() if t.is_floating_point()])
    cap = (DUMP_MAX_BYTES - 4096) // 4
    if flat.numel() > cap:   # fixed seeded sample of the entries (same indices for the same model)
        g = torch.Generator().manual_seed(0)
        flat = flat[torch.randperm(flat.numel(), generator=g)[:cap].sort().values]
    np.save(os.path.join(out_dir, "params.npy"), flat.numpy())


class ClockSampler(threading.Thread):
    """Samples SM clock + throttle reasons through NVML while the timed region runs."""

    def __init__(self, index: int, period: float = 0.05):
        super().__init__(daemon=True)
        self.index, self.period = index, period
        self.samples, self.reasons, self.max_mhz = [], set(), None
        self._stop_evt = threading.Event()
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM)
        except Exception:
            self.nv = None

    def run(self):
        if self.nv is None:
            return
        nv = self.nv
        names = {
            getattr(nv, "nvmlClocksEventReasonHwSlowdown", 0x8): "hw_slowdown",
            getattr(nv, "nvmlClocksEventReasonHwThermalSlowdown", 0x40): "hw_thermal_slowdown",
            getattr(nv, "nvmlClocksEventReasonSwThermalSlowdown", 0x20): "sw_thermal_slowdown",
            getattr(nv, "nvmlClocksEventReasonSwPowerCap", 0x4): "sw_power_cap",
        }
        while not self._stop_evt.is_set():
            try:
                self.samples.append(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM))
                try:
                    mask = nv.nvmlDeviceGetCurrentClocksEventReasons(self.h)
                except Exception:
                    mask = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
                for bit, name in names.items():
                    if mask & bit:
                        self.reasons.add(name)
            except Exception:
                pass
            time.sleep(self.period)

    def stop(self):
        self._stop_evt.set()
        self.join(timeout=1.0)
        s = sorted(self.samples)
        return {"sm_mhz": s[len(s) // 2] if s else None, "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons)}


def reference_arm(args):
    if int(os.environ.get("RANK", "0")) != 0:   # launched under torchrun for N > 1: one line, from rank 0
        return
    print(json.dumps({
        "impl": "reference",
        "unavailable": "hwang595/ATOMO has no setup.py/pyproject (pip: 'not installable'), is Python-2.7 + mpi4py + "
                       "torch-0.3 and imports a module missing from its tree (codings.lossless_compress)"}))


def main():
    args = parse()
    if args.impl == "reference":
        return reference_arm(args)

    import torch
    import torch.distributed as dist

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus and world == 1 and args.gpus > 1:
        raise SystemExit("launch with torch.distributed.run --nproc-per-node %d for --gpus %d" % (args.gpus, args.gpus))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)

    if args.impl == "nccl-baseline":
        from baseline.nccl_ps import run_baseline
        return run_baseline(args, rank, world, dev)

    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model, input_shape
    from atomo_b200.runtime.engine import FusedEngine

    torch.manual_seed(0)
    torch.backends.cudnn.benchmark = args.cudnn_benchmark
    torch.backends.cudnn.deterministic = True
    ncls = 1000 if args.dataset == "ImageNet" else 10
    model = build_model(args.network, ncls, args.dataset)
    engine = args.engine
    if engine == "auto":
        engine = "shadow" if (args.dtype == "bf16" and args.code in ("svd", "qsvd", "sgd") and args.channels_last) else "fused"
    if engine == "shadow":
        from atomo_b200.runtime.shadow_engine import ShadowEngine
        eng = ShadowEngine(model, rank, world, code=args.code, svd_rank=args.svd_rank, lr=args.lr,
                           momentum=args.momentum, ps_mode=args.ps_mode, sampling=args.sampling,
                           use_graph=not args.no_graph, seed=1, timeout_s=60.0, groups=args.groups,
                           overlap=args.overlap, optimizer=args.optimizer, fused_bn=args.fused_bn != "off",
                           ps_grid=args.ps_grid, warm_start=args.warm_start, max_sweeps=args.max_sweeps,
                           main_priority=args.main_priority, side_priority=args.side_priority)
    else:
        ps_mode = "colocated" if args.ps_mode == "sharded" else args.ps_mode
        eng = FusedEngine(model, rank, world, code=args.code, svd_rank=args.svd_rank, lr=args.lr, momentum=args.momentum,
                          ps_mode=ps_mode, sampling=args.sampling, dtype=args.dtype, channels_last=args.channels_last,
                          use_graph=not args.no_graph, seed=1, timeout_s=60.0, subspace={"auto": "auto", "on": True, "off": False}[args.subspace],
                          fused_bn={"auto": "auto", "on": True, "off": False}[args.fused_bn],
                          quantization_level=args.quantization_level, entry_budget=args.entry_budget)
    shape = input_shape(args.network, args.dataset)
    ds = SyntheticImageDataset(shape, ncls, 50000, seed=rank)
    nbatches = 8
    xs, ys = ds.materialize(args.batch_size * nbatches)
    host_x = [xs[i * args.batch_size:(i + 1) * args.batch_size].contiguous().pin_memory() for i in range(nbatches)]
    host_y = [ys[i * args.batch_size:(i + 1) * args.batch_size].contiguous().pin_memory() for i in range(nbatches)]
    torch.cuda.reset_peak_memory_stats(dev)
    base_mem = torch.cuda.memory_allocated(dev)
    eng.prepare(host_x[0], host_y[0], warmup=max(args.warmup, 3))
    state_mb = (3 * eng.plan.total_elems * 4 if engine == "fused" else 10 * eng.plan.w_total) / 2 ** 20
    work_mb = (torch.cuda.max_memory_allocated(dev) - base_mem) / 2 ** 20 + state_mb

    def barrier():
        torch.cuda.synchronize(dev)
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    def max_over_ranks(v):
        if world == 1:
            return v
        t = torch.tensor([v], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    nworkers = eng.W
    imgs_per_step = nworkers * args.batch_size

    def percentile(v, q):
        s = sorted(v)
        return s[min(len(s) - 1, int(q * len(s)))]

    def check_error(where):
        err = eng.error_code()
        if err:
            sys.stderr.write("bench.py: rank %d: device-side error code %d %s: aborting, no number reported\n"
                             % (rank, err, where))
            sys.stderr.flush()
            os._exit(3)

    # ---- device-timed: the step graph alone (inputs resident) ---------------------------------
    # Everything slow on the host (NVML init of the clock sampler, the D2H read in phase_stats, event
    # creation) happens BEFORE the barrier; the barrier sits immediately before e0.record(), so the ranks
    # enter the timed window within microseconds of each other (round-1 VERDICT: an 8-way nvmlInit skew
    # between the barrier and e0 was charged to the slowest rank's first parameter wait).
    sampler = ClockSampler(local_rank)
    sampler.start()
    for _ in range(max(args.warmup, 3)):
        eng.train_step()
    step_ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
    eng.phase_stats(reset=True)
    barrier()
    for _ in range(3):              # warm replays after the barrier: queues full, clocks up
        eng.train_step()
    eng.tstats.zero_()
    barrier()
    step_ev[0].record()
    for i in range(args.steps):
        eng.train_step()
        step_ev[i + 1].record()
    barrier()
    ms = max_over_ranks(step_ev[0].elapsed_time(step_ev[-1]))
    per_step = [step_ev[i].elapsed_time(step_ev[i + 1]) for i in range(args.steps)]
    clocks = sampler.stop()
    check_error("after the device-timed loop")
    value = imgs_per_step * args.steps / (ms / 1e3)
    step_stats = {"median_ms": round(max_over_ranks(percentile(per_step, 0.5)), 4),
                  "p99_ms": round(max_over_ranks(percentile(per_step, 0.99)), 4),
                  "max_ms": round(max_over_ranks(max(per_step)), 4),
                  "min_ms": round(-max_over_ranks(-min(per_step)), 4)}
    phases = eng.phase_stats(reset=True)
    phases["param_wait_us_max"] = max_over_ranks(phases["param_wait_us"])

    # ---- end to end: public API, pinned-host inputs every step, loss to the host every step ------
    pinned_loss = torch.zeros(3, dtype=torch.float32).pin_memory()
    copy_evt = torch.cuda.Event()
    losses = []
    e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for i in range(3):
        eng.train_step(host_x[i % nbatches], host_y[i % nbatches])
    barrier()
    e2.record()
    for i in range(args.steps):
        stats = eng.train_step(host_x[i % nbatches], host_y[i % nbatches])
        if i > 0:
            copy_evt.synchronize()          # previous step's loss has landed on the host
            losses.append(float(pinned_loss[0]))
        pinned_loss.copy_(stats, non_blocking=True)
        copy_evt.record()
    copy_evt.synchronize()
    losses.append(float(pinned_loss[0]))
    e3.record()
    barrier()
    ms_e2e = max_over_ranks(e2.elapsed_time(e3))
    e2e_value = imgs_per_step * args.steps / (ms_e2e / 1e3)
    h2d = host_x[0].numel() * host_x[0].element_size() + host_y[0].numel() * host_y[0].element_size()
    check_error("after the end-to-end loop")
    err = 0
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, stats, eng.model)

    if rank == 0:
        pm = eng.ps_mode
        par = {"sharded": "%dworkers+sharded-ps(every GPU trains and owns 1/%d of the PS)" % (nworkers, world),
               "colocated": "ps+%dworkers(colocated)" % nworkers, "dedicated": "ps+%dworkers" % nworkers}[pm]
        out = {
            "metric": metric_name(args), "value": round(value, 2), "unit": "images/s", "n_gpus": world, "steps": args.steps,
            "warmup": max(args.warmup, 3), "ms_per_step": round(ms / args.steps, 4), "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": args.dtype, "data": "synthetic",
            "impl": "atomo_b200",
            "config": {"model": args.network, "global_batch": imgs_per_step, "per_worker_batch": args.batch_size,
                       "seq_len": None, "image": list(shape), "parallelism": par, "code": args.code,
                       "svd_rank": args.svd_rank, "sampling": args.sampling, "dataset_shape": args.dataset,
                       "engine": engine, "groups": getattr(eng, "G", 1), "overlap": getattr(eng, "overlap", False),
                       "subspace_route_layers": (len(eng.plan.ext.layers) if eng.plan.ext else 0) if engine == "fused" else 0,
                       "coded_units": getattr(eng.plan, "n_coded", None),
                       "fused_bn_layers": eng.fused_bn_layers, "cuda_graph": not args.no_graph,
                       "heap": eng.heap.mode, "nvls_multicast": eng.heap.has_multicast,
                       "l2": "no explicit flush: per-step working set %.0f MB > 50 MB L2 (H100)" % work_mb,
                       "optimizer": "%s fused in PS kernel" % ("momentum-SGD" if args.optimizer == "sgd" else "Adam"), "final_loss": round(losses[-1], 4),
                       "device_error": err},
            "clocks": clocks,
            "e2e": {"value": round(e2e_value, 2), "unit": "images/s", "ms_per_step": round(ms_e2e / args.steps, 4),
                    "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 12},
            "gpu_launches": eng.launches_per_step * args.steps,
            "step_ms": step_stats,
            "phase_us": {k: round(v, 1) for k, v in phases.items()},
        }
    eng.close()
    if world > 1:
        dist.destroy_process_group()
    # ---- the same config at fp32 model precision (round-1 VERDICT: print it next to the bf16 line) --------------
    # Runs in a child process per rank (fresh CUDA context + symmetric heap; re-creating an NVLS binding inside
    # one process is avoided on purpose) through the fp32-flat engine; its JSON is nested under "fp32".
    fp32 = None
    if args.fp32_line and args.dtype == "bf16" and args.impl == "atomo_b200" and (world == 1 or args.fp32_line_multi):
        fp32 = fp32_child(args, rank, world)
    if rank == 0:
        if fp32 is not None:
            out["fp32"] = fp32
        print(json.dumps(out))


def fp32_child(args, rank, world):
    import subprocess
    import torch
    torch.cuda.empty_cache()
    env = dict(os.environ)
    env["MASTER_PORT"] = str(int(env.get("MASTER_PORT", "29500")) + 53)
    # Under torchrun every rank is a CLIENT of the elastic agent's store (TORCHELASTIC_USE_AGENT_STORE): on a new
    # port nobody would serve and the children would block in the rendezvous (this hung an 8-GPU run for the full
    # timeout).  Without the variable rank 0 of the children hosts its own TCPStore.
    env.pop("TORCHELASTIC_USE_AGENT_STORE", None)
    cmd = [sys.executable, os.path.abspath(__file__), "--gpus", str(args.gpus), "--steps", str(args.steps), "--warmup",
           str(args.warmup), "--dtype", "fp32", "--engine", "fused", "--no-fp32-line", "--network", args.network,
           "--batch-size", str(args.batch_size), "--code", args.code, "--svd-rank", str(args.svd_rank), "--dataset",
           args.dataset, "--momentum", str(args.momentum), "--lr", str(args.lr)]
    try:
        r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=150)
    except Exception as e:  # noqa
        return {"unavailable": "fp32 child failed: %r" % (e,)}
    if rank != 0:
        return None
    for line in reversed(r.stdout.splitlines()):
        if line.startswith("{") and '"metric"' in line:
            d = json.loads(line)
            return {"value": d["value"], "unit": d["unit"], "ms_per_step": d["ms_per_step"], "dtype": "fp32",
                    "e2e_value": d["e2e"]["value"], "engine": "fused (round-1 fp32-flat engine; cuDNN TF32 convs = "
                    "PyTorch default, fp32 weights / gradients / coding)", "parallelism": d["config"]["parallelism"],
                    "step_ms": d.get("step_ms"), "clocks": d.get("clocks")}
    return {"unavailable": "fp32 child printed no result (rc=%d): %s" % (r.returncode, r.stderr[-300:])}


if __name__ == "__main__":
    main()

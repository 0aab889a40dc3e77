"""Kernel timeline of one graph-replayed ShadowEngine step: which kernels run where, what is exposed after
backward.  python scripts/timeline_shadow.py [--code svd] [--groups 4] [--no-cudnn-benchmark] > timeline.txt"""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import profile, ProfilerActivity
from atomo_b200.data import SyntheticImageDataset
from atomo_b200.models import build_model, input_shape
from atomo_b200.runtime.shadow_engine import ShadowEngine


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--network", default="ResNet18")
    ap.add_argument("--code", default="svd")
    ap.add_argument("--groups", type=int, default=4)
    ap.add_argument("--no-overlap", action="store_true")
    ap.add_argument("--batch-size", type=int, default=128)
    ap.add_argument("--no-cudnn-benchmark", dest="cudnn_benchmark", action="store_false", default=True,
                    help="deterministic, heuristically chosen cuDNN algorithms, as bench.py runs them")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = args.cudnn_benchmark
    torch.backends.cudnn.deterministic = not args.cudnn_benchmark
    torch.manual_seed(0)
    eng = ShadowEngine(build_model(args.network, 10), 0, 1, code=args.code, svd_rank=3, lr=0.01, momentum=0.9,
                       use_graph=True, overlap=not args.no_overlap, groups=args.groups)
    x, y = SyntheticImageDataset(input_shape(args.network), 10, 4096).materialize(args.batch_size)
    eng.prepare(x.pin_memory(), y.pin_memory(), warmup=4)
    for _ in range(5):
        eng.train_step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            eng.train_step()
        torch.cuda.synchronize()
    evs = [e for e in prof.events() if getattr(e, "device_time", 0) and "Memcpy" not in e.name and "Memset" not in e.name]
    evs.sort(key=lambda e: e.time_range.start)
    # split into steps by the wait_params kernel
    starts = [i for i, e in enumerate(evs) if "wait_params" in e.name]
    a, b = starts[1], starts[2]
    step = evs[a:b]
    t0 = step[0].time_range.start
    end = max(e.time_range.end for e in step)
    print("step span %.1f us, %d kernels" % (end - t0, len(step)))
    ours = [e for e in step if "atomo" in e.name]
    last_lib = max(e.time_range.end for e in step if "v2_" not in e.name)
    print("last non-v2 kernel ends at +%.1f us -> exposed tail %.1f us" % (last_lib - t0, end - last_lib))
    busy = sum(e.device_time for e in step if "v2_" not in e.name)
    print("sum of non-v2 kernel time %.1f us; sum of v2 kernel time %.1f us" % (busy, sum(e.device_time for e in step if "v2_" in e.name)))
    for e in step:
        if "v2_" in e.name:
            print("  +%8.1f .. +%8.1f  (%6.1f us)  %s" % (e.time_range.start - t0, e.time_range.end - t0, e.device_time,
                                                        e.name.split("(")[0].replace("atomo::v2::", "")))
    # gaps on the main chain: idle time between consecutive non-v2 kernels
    lib = [e for e in step if "v2_" not in e.name]
    gaps = sorted(((lib[i + 1].time_range.start - lib[i].time_range.end, lib[i].name[:50], lib[i + 1].name[:50])
                   for i in range(len(lib) - 1)), reverse=True)[:8]
    print("largest gaps between consecutive main-stream kernels:")
    for g, n1, n2 in gaps:
        print("  %6.1f us  after %s  before %s" % (g, n1, n2))
    bn_chains(step)
    backward_streams(step)
    eng.close()


def bn_chains(step):
    """Fused-BN chains of the step (stats -> sum_partials -> apply, bwd_reduce -> sum_partials -> bwd_apply): kernel
    time, the gaps on the two edges of each chain, and the chain's span from first start to last end.  A kernel
    launched as a programmatic dependent can start before its predecessor ends (negative gap) and then counts its
    wait as kernel time, so the span is the figure to compare."""
    bn = [e for e in step if "bn_" in e.name]
    chains, cur = {"fwd": [], "bwd": []}, None
    for e in bn:
        if "bn_stats_kernel" in e.name or "bn_bwd_reduce_kernel" in e.name:
            cur = [e]
            chains["bwd" if "bwd" in e.name else "fwd"].append(cur)
        elif cur is not None:
            cur.append(e)
    print("fused BN: %d kernels, %.1f us of kernel time" % (len(bn), sum(e.device_time for e in bn)))
    for kind, cs in chains.items():
        cs = [c for c in cs if len(c) == 3]
        if not cs:
            continue
        busy = sum(e.device_time for c in cs for e in c)
        span = sum(c[2].time_range.end - c[0].time_range.start for c in cs)
        g1 = [c[1].time_range.start - c[0].time_range.end for c in cs]
        g2 = [c[2].time_range.start - c[1].time_range.end for c in cs]
        print("  %s: %d chains, kernel time %.1f us, span %.1f us, edge gaps %.1f + %.1f us (mean %.2f / %.2f)"
              % (kind, len(cs), busy, span, sum(g1), sum(g2), sum(g1) / len(cs), sum(g2) / len(cs)))
        for i, c in enumerate(cs):
            print("    %2d: span %6.1f  kernels %s  gaps %5.1f %5.1f"
                  % (i, c[2].time_range.end - c[0].time_range.start,
                     " ".join("%5.1f" % e.device_time for e in c),
                     c[1].time_range.start - c[0].time_range.end, c[2].time_range.start - c[1].time_range.end))


def backward_streams(step):
    """The backward's convolution and add kernels by name: cuDNN input gradients (dgrad), weight gradients (wgrad) and
    elementwise adds, with the streams they ran on (under graph replay the stream ids are the graph's), then every
    kernel that started between the end of one BN backward and the start of the next, in time order."""
    t0 = step[0].time_range.start
    short = lambda n: n.split("(")[0][:80]
    first = next((e.time_range.start for e in step if "bn_bwd_reduce" in e.name), None)
    if first is None:
        return
    bwd = [e for e in step if e.time_range.start >= first and "v2_" not in e.name]
    kinds = {"dgrad": lambda n: "dgrad" in n, "wgrad": lambda n: "wgrad" in n,
             "add": lambda n: "elementwise" in n and "add" in n.lower()}
    for kind, match in kinds.items():
        evs = [e for e in bwd if match(e.name)]
        print("backward %s kernels: %d, %.1f us of kernel time, streams %s"
              % (kind, len(evs), sum(e.device_time for e in evs), sorted({e.device_resource_id for e in evs})))
    bn_bwd = [e for e in bwd if "bn_bwd" in e.name or "bn_sum_partials" in e.name]
    print("backward span from the first BN backward kernel: %.1f us; BN backward chains:" %
          (max(e.time_range.end for e in bwd) - first))
    chain_starts = [e for e in bn_bwd if "bn_bwd_reduce" in e.name]
    applies = [e for e in bn_bwd if "bn_bwd_apply" in e.name]
    for a in applies:
        nxt = next((r for r in chain_starts if r.time_range.start > a.time_range.start), None)
        end = nxt.time_range.start if nxt is not None else float("inf")
        mid = [e for e in bwd if a.time_range.end - 1 <= e.time_range.start < end and "bn_" not in e.name]
        print("  after %s at +%.1f .. next BN backward at %s" % (short(a.name).replace("atomo::", ""),
              a.time_range.end - t0, "+%.1f" % (end - t0) if nxt is not None else "-"))
        for e in mid:
            print("      +%8.1f %6.1f us  s%-3s %s" % (e.time_range.start - t0, e.device_time, e.device_resource_id,
                                                   short(e.name)))

if __name__ == "__main__":
    main()

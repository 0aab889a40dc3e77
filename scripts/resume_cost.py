"""Size of a worker's checkpoint file (``model_step_<N>_worker<R>``) and the host time to write and to restore it, for
one bf16-engine configuration.  Prints one JSON line, with the GPU's name and power limit.

    python scripts/resume_cost.py [--net ResNet18] [--code svd] [--error-feedback 1] [--repeats 5]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from atomo_b200.data import SyntheticImageDataset  # noqa: E402
from atomo_b200.models import build_model, input_shape  # noqa: E402
from atomo_b200.runtime.shadow_engine import ShadowEngine  # noqa: E402
from atomo_b200.utils import checkpoint as ckpt  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--net", default="ResNet18")
    ap.add_argument("--code", default="svd")
    ap.add_argument("--error-feedback", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    torch.manual_seed(0)
    eng = ShadowEngine(build_model(args.net, 10), 0, 1, code=args.code, lr=0.05, momentum=0.9,
                       error_feedback=bool(args.error_feedback))
    x, y = SyntheticImageDataset(input_shape(args.net), 10, 256).materialize(32)
    eng.prepare(x.cuda(), y.cuda(), warmup=2)
    for _ in range(3):
        eng.train_step(x.cuda(), y.cuda())
    torch.cuda.synchronize()
    step = eng.step - 1
    save_s, load_s = [], []
    with tempfile.TemporaryDirectory() as d:
        d += "/"
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ckpt.save_worker_state(d, step, eng.rank, eng._worker_config(), eng._worker_tensors())
            save_s.append(time.perf_counter() - t0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            assert eng._load_worker_state(d, step)
            torch.cuda.synchronize()
            load_s.append(time.perf_counter() - t0)
        size = os.path.getsize(ckpt.worker_path(d, step, eng.rank))
    tensors = {k: [list(t.shape), str(t.dtype)] for k, t in eng._worker_tensors().items()}
    eng.close()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    print(json.dumps({"net": args.net, "code": args.code, "error_feedback": bool(args.error_feedback),
                      "bytes": size, "tensors": tensors, "save_ms": [round(1e3 * s, 2) for s in save_s],
                      "load_ms": [round(1e3 * s, 2) for s in load_s], "gpu": torch.cuda.get_device_name(0),
                      "power_limit": power}))


if __name__ == "__main__":
    main()

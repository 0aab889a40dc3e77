"""CPU checks of the bench.py driver contract: the parts that do not need a GPU (argument defaults, the reference
arm's line, the nested fp32 child's environment, the clock sampler's shape)."""
import importlib.util
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bench():
    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(ROOT, "bench.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_defaults_are_the_headline_config(monkeypatch):
    b = _bench()
    monkeypatch.setattr(sys, "argv", ["bench.py"])
    a = b.parse()
    assert (a.gpus, a.steps, a.warmup) == (1, 50, 5)
    assert (a.network, a.dataset, a.batch_size, a.code, a.svd_rank, a.dtype) == ("ResNet18", "Cifar10", 128, "svd", 3, "bf16")
    assert a.ps_mode == "sharded" and a.engine == "auto" and a.fp32_line and not a.fp32_line_multi
    assert b.metric_name(a) == b.METRIC and "ResNet-18 CIFAR-10 images/sec" in b.METRIC


def test_reference_arm_prints_one_unavailable_line_from_rank0_only():
    env = dict(os.environ, PYTHONPATH=ROOT)
    env.pop("RANK", None)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "8",
                        "--steps", "5", "--warmup", "3"], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and isinstance(d["unavailable"], str) and "\n" not in d["unavailable"]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "8"],
                       env=dict(env, RANK="3", WORLD_SIZE="8"), capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_fp32_child_gets_its_own_rendezvous(monkeypatch):
    """The nested fp32 measurement runs `bench.py --dtype fp32 --engine fused --no-fp32-line` in a child.  Under
    torchrun the child must not inherit TORCHELASTIC_USE_AGENT_STORE (it would be a client of a store nobody serves on
    the shifted port: this hung an 8-GPU run) and must not recurse."""
    b = _bench()
    seen = {}

    class R:
        returncode, stderr = 0, ""
        stdout = json.dumps({"metric": "m", "value": 1.0, "unit": "images/s", "ms_per_step": 2.0,
                             "e2e": {"value": 0.9}, "config": {"parallelism": "p"}})

    def fake_run(cmd, env=None, **kw):
        seen["cmd"], seen["env"], seen["kw"] = cmd, env, kw
        return R()

    monkeypatch.setattr(subprocess, "run", fake_run)
    monkeypatch.setenv("TORCHELASTIC_USE_AGENT_STORE", "True")
    monkeypatch.setenv("MASTER_PORT", "29500")
    monkeypatch.setattr(sys, "argv", ["bench.py", "--steps", "7", "--warmup", "3"])
    out = b.fp32_child(b.parse(), rank=0, world=1)
    assert "TORCHELASTIC_USE_AGENT_STORE" not in seen["env"] and seen["env"]["MASTER_PORT"] == "29553"
    cmd = seen["cmd"]
    assert "--no-fp32-line" in cmd and cmd[cmd.index("--dtype") + 1] == "fp32" and cmd[cmd.index("--engine") + 1] == "fused"
    assert cmd[cmd.index("--steps") + 1] == "7" and seen["kw"]["timeout"] <= 300
    assert out["value"] == 1.0 and out["dtype"] == "fp32" and out["e2e_value"] == 0.9
    # a non-zero rank runs the child (it is one rank of the child job) but reports nothing
    assert b.fp32_child(b.parse(), rank=1, world=2) is None


def test_clock_sampler_shape_without_a_gpu():
    b = _bench()
    s = b.ClockSampler(0, period=0.01)
    s.start()
    out = s.stop()
    assert set(out) == {"sm_mhz", "sm_max_mhz", "reasons"} and isinstance(out["reasons"], list)


def test_built_extension_is_the_profiled_one():
    """Evidence integrity: every kernel of the built extension is instruction-identical to the committed SASS
    manifest (profiles/sass/kernels.json, taken from the build that ran the GPU tests and the benchmark).  Skipped
    when the extension has not been built yet or cuobjdump is not on PATH."""
    import glob
    import shutil
    import pytest
    if not glob.glob(os.path.join(ROOT, "atomo_b200", "_C*.so")) or shutil.which("cuobjdump") is None:
        pytest.skip("needs the built extension and cuobjdump")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "check_sass_listings.py")], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-1500:]
    assert r.stdout.count("identical") >= 27

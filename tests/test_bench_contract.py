"""bench.py contract checks that need no GPU: the reference arm prints exactly ONE JSON line on stdout with the keys
the driver reads, also under torchrun (rank 0 only), and nothing else reaches stdout."""
import json
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
KEYS = {"impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
        "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"}


def _check(stdout: str, n_gpus: int):
    lines = [l for l in stdout.splitlines() if l.strip()]
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    assert KEYS <= set(d), KEYS - set(d)
    assert d["impl"] == "reference" and d["n_gpus"] == n_gpus and d["steps"] == 1 and d["warmup"] == 0
    assert d["unit"] == "samples/s" and d["higher_is_better"] is True and d["vs_baseline"] is None
    # N = 1 with oracle/_ref present (oracle/make_ref.py): the unmodified reference generate(); otherwise its torch-operator port
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_ref", ROOT / "oracle" / "make_ref.py")
    make_ref = importlib.util.module_from_spec(spec); spec.loader.exec_module(make_ref)
    want_kind = "reference" if (n_gpus == 1 and make_ref.verify()) else "port"
    assert d["value"] > 0 and d["cpu_baseline"]["kind"] == want_kind and d["cpu_baseline"]["cores"] >= 1
    spec = importlib.util.spec_from_file_location("bench", ROOT / "bench.py")
    bench = importlib.util.module_from_spec(spec); spec.loader.exec_module(bench)
    assert d["config"] == bench.workload_config(n_gpus, "cfg2")          # the SAME config object the GPU arm prints
    assert d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert "workload" in d["config"] and "sample" in d["cpu_baseline"]


def test_reference_arm_prints_one_json_line():
    r = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    _check(r.stdout, 1)


def test_reference_arm_under_torchrun_prints_one_line_from_rank0():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29571", str(ROOT / "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "0"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    _check(r.stdout, 2)


@pytest.mark.gpu
def test_gpu_bench_line_carries_the_contract_keys(tmp_path):
    """The GPU arm (bench.py on the GPU, a short run): one JSON line with every key a reader of the bench line needs --
    incl. roofline, clocks, gpu_launches and a real e2e --, `--steps` is the number of timed steps, and
    `--dump-outputs` writes the timed path's last results."""
    gpu_keys = (KEYS - {"impl", "cpu_baseline"}) | {"roofline", "clocks", "gpu_launches"}
    dump = tmp_path / "dump"
    r = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--gpus", "1", "--steps", "2", "--warmup", "1", "--no-cpu-baseline",
                        "--dump-outputs", str(dump)], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    missing = gpu_keys - set(d)
    assert not missing, missing
    assert d["unit"] == "samples/s" and d["value"] > 0 and d["gpu_launches"] > 0 and d["higher_is_better"] is True
    assert d["steps"] == 2 and d["warmup"] == 1
    spec = __import__("importlib.util").util.spec_from_file_location("bench", ROOT / "bench.py")
    bench = __import__("importlib.util").util.module_from_spec(spec); spec.loader.exec_module(bench)
    assert d["config"] == bench.workload_config(1, "cfg2")
    r_ = d["roofline"]
    assert r_["bound"] == "tensor" and abs(r_["frac"] - r_["achieved"] / r_["peak"]) < 1e-9 and r_["unit"] == "TFLOP/s"
    assert d["e2e"]["value"] > 0 and d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0
    assert d["e2e"]["value"] <= d["value"] * 1.0001          # host copies inside: never faster than the device-resident leg
    import numpy as np
    samples, wav = np.load(dump / "samples.npy"), np.load(dump / "wav.npy")
    cfg = bench.workload_config(1, "cfg2")
    assert samples.dtype == np.float32 and samples.shape == (cfg["folds"], cfg["steps_per_fold"]) and np.isfinite(samples).all()
    assert wav.dtype == np.float64 and wav.shape == ((bench.frames_for(1) - 1) * bench.HOP,)

"""bench.py's contract on the CPU side: the reference arm prints one JSON line with the keys the driver reads, its
`ms_per_step` is the timed region that `value` is computed from, and the module's helpers that need no GPU behave."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(*args):
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], capture_output=True, text=True, timeout=600,
                       cwd=ROOT, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.strip().splitlines() if ln.startswith("{")]
    assert len(lines) == 1, r.stdout[-500:]
    return json.loads(lines[0])


def test_reference_arm_line():
    d = _run("--impl", "reference", "--steps", "2", "--warmup", "1", "--blocks", "512")
    assert d["impl"] == "reference" and d["unit"] == "MiB/s" and d["higher_is_better"] is True and d["n_gpus"] == 1
    assert d["steps"] == 2 and d["gpu_launches"] == 0 and d["vs_baseline"] is None and d["dtype"] == "u8"
    assert d["config"]["blocks_per_gpu"] == 512 and "workload" in d["config"]
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["threads"] >= cb["cores"] and cb["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "MiB/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    # value and ms_per_step describe the same timed region: 512 blocks of 64 KiB = 32 MiB per step
    assert abs(d["value"] * d["ms_per_step"] / 1e3 - 32.0) < 0.01 * 32.0
    assert d["wall_ms_per_step"] >= d["ms_per_step"]


def test_reference_arm_is_silent_on_other_ranks():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1",
                        "--warmup", "1", "--blocks", "64"], capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_workload_is_the_tiled_fixture():
    sys.path.insert(0, ROOT)
    import bench
    from lz4_flex_b200 import corpus
    w = bench.build_workload(8, 0)
    assert w.dtype == np.uint8 and w.size == 8 * 65536
    assert np.array_equal(w, corpus.tiled("compression_66k_JSON.txt", 8 * 65536))

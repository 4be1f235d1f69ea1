"""CPU tests of bench.py's contract: the reference arm prints one JSON line with the agreed keys, and our arm refuses to
run without a GPU instead of falling back to anything."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_json_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    line = [l for l in out.stdout.splitlines() if l.startswith("{")][-1]
    d = json.loads(line)
    assert d["impl"] == "reference" and d["unit"] == "images/sec" and d["higher_is_better"] is True
    assert d["metric"].startswith("64x64 images/sec IAN encode->decode")
    assert d["value"] > 0 and d["gpu_launches"] == 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert "workload" in d["config"] and "model" not in d["config"]


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_our_arm_has_no_cpu_fallback():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "3"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode != 0
    assert "no CPU fallback" in (out.stderr + out.stdout)


def test_reference_arm_nonzero_ranks_do_no_work():
    env = dict(os.environ, RANK="1", LOCAL_RANK="1", WORLD_SIZE="2")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1",
                          "--warmup", "0"], capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    assert out.returncode == 0 and not [l for l in out.stdout.splitlines() if l.startswith("{")]


def _bench():
    sys.path.insert(0, ROOT)
    import importlib
    return importlib.import_module("bench")


def test_dump_outputs_size_rule(tmp_path):
    """--dump-outputs keeps z and x_hat within 64 MB together: all rows when they fit, else the same fixed, sorted, seeded
    sample of rows in every array, depending only on the batch size (two builds dump the same samples)."""
    import numpy as np
    bench = _bench()
    row = 100 * 4 + 3 * 64 * 64 * 4                               # one sample of z + one of x_hat, float32
    assert np.array_equal(bench.dump_rows(256, row), np.arange(256))   # 12.7 MB: everything
    big = bench.dump_rows(4096, row)                               # 201 MB: a sample
    assert len(big) * row <= bench.DUMP_MAX_BYTES < (len(big) + 1) * row
    assert np.all(np.diff(big) > 0) and big[0] >= 0 and big[-1] < 4096
    assert np.array_equal(big, bench.dump_rows(4096, row))
    n = 3000                                                       # end to end with small arrays and a small cap
    z = np.arange(n * 2, dtype=np.float64).reshape(n, 2)
    x = -np.arange(n * 6, dtype=np.float32).reshape(n, 3, 2)
    rows = bench.write_dump(str(tmp_path), {"z": z, "xhat": x}, max_bytes=1000 * (2 + 6) * 4)
    zd, xd = np.load(tmp_path / "z.npy"), np.load(tmp_path / "xhat.npy")
    assert len(rows) == 1000 and zd.dtype == np.float32 and xd.dtype == np.float32
    assert np.array_equal(zd, z[rows].astype(np.float32)) and np.array_equal(xd, x[rows])
    assert zd.nbytes + xd.nbytes <= 1000 * (2 + 6) * 4


def test_committed_h100_bench_line():
    """the bench line committed beside the docs (profiles/h100_bench_n1.json) carries its card, a sane roofline fraction
    and the launch count of the IAN_simple step: conv1, 3 convs, fc1 + finalize, head + finalize, sample, fc2, 3 deconvs,
    dec_out"""
    line = [l for l in open(os.path.join(ROOT, "profiles", "h100_bench_n1.json")) if l.startswith("{")][-1]
    d = json.loads(line)
    assert "H100" in d["gpu"]["name"] and d["gpu"]["power_limit_w"] > 0
    assert d["roofline"]["frac"] == d["roofline"]["frac_burst"] and 0.1 < d["roofline"]["frac_burst"] <= 1.0
    assert d["gpu_launches"] == 14 * d["steps"]
    assert d["n_gpus"] == 1 and d["value"] > 0 and d["unit"] == "images/sec"

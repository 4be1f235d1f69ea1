"""The shipped library IS the wgmma / TMA / PDL code the design describes: SASS of the in-tree libian_b200.so, read with
cuobjdump (no GPU needed).  Guards against a silent rebuild onto another code path (a recompiled mma.sync kernel, a plain
store epilogue, plain launches) and keeps profiles/r2_sass_summary.txt -- the evidence file the docs cite -- in step with
the build that is tested."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "neural-photo-editor_b200", "libian_b200.so")


def _summary():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_summary.py")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    rows = {}
    for line in out.stdout.splitlines():
        if line.startswith("#"):
            continue
        f = [c.strip() for c in line.split("|")]
        rows[f[0]] = dict(kv.rsplit(" x", 1) for kv in f[4].split(", ") if " x" in kv)
    return out.stdout, rows


def test_tensor_core_kernels_are_wgmma_tma_pdl():
    text, rows = _summary()
    one = [k for k in rows if k.startswith("tapgemm_tc_kernel<")]
    assert len(one) >= 4, sorted(rows)

    def wgmma(r):
        return any(m.startswith("HGMMA.") for m in r) and "WARPGROUP.ARRIVE" in r and "WARPGROUP.DEPBAR" in r

    for k in one:
        r = rows[k]
        assert wgmma(r) and any(m.startswith("UTMALDG") for m in r), (k, r)
        assert "PREEXIT" in r and "ACQBULK" in r, (k, r)      # griddepcontrol.launch_dependents / .wait
    c1 = rows["conv1_tc_kernel"]
    assert wgmma(c1) and "UTMASTG" in c1, c1                  # epilogue leaves through TMA stores
    for k in ("decout_tc_kernel", "head_tc_kernel<1>", "head_tc_kernel<3>"):
        assert wgmma(rows[k]) and any(m.startswith("UTMALDG") for m in rows[k]), (k, rows[k])
    assert not any(m == "HMMA" for r in rows.values() for m in r), "an mma.sync kernel is in the library"
    for k in ("splitk_finalize_kernel", "splitk_finalize8_kernel", "brush_seed_bwd_kernel", "brush_update_kernel", "sample_kernel"):
        assert "PREEXIT" in rows[k] and "ACQBULK" in rows[k], (k, rows[k])


def test_committed_sass_summary_matches_the_build():
    text, _ = _summary()
    path = os.path.join(ROOT, "profiles", "r2_sass_summary.txt")
    committed = open(path).read()

    def key(t):                                              # kernel | Hopper mnemonics (registers may differ across toolkits)
        out = []
        for line in t.splitlines():
            if line.startswith("#"):
                continue
            f = [c.strip() for c in line.split("|")]
            out.append((f[0], f[4]))
        return out
    assert key(text) == key(committed), "profiles/r2_sass_summary.txt is stale: run `python tools/sass_summary.py > profiles/r2_sass_summary.txt`"

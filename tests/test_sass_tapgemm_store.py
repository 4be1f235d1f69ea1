"""The float32-mode tap-GEMM writes plain tiles with TMA stores and keeps its main loop as it was: SASS of the in-tree
libian_b200.so (tools/sass_summary.py) and ptxas' own resource report of csrc/tapgemm_tc.cu (no GPU needed)."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from test_sass import _summary

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "neural-photo-editor_b200", "csrc")
KERNELS = ("tapgemm_tc_kernel<128, 3, false>", "tapgemm_tc_kernel<128, 3, true>")


def test_float32_tapgemm_stores_through_tma():
    _, rows = _summary()
    for k in KERNELS:
        r = rows[k]
        assert "UTMASTG" in r, (k, r)                                 # the TMA-store epilogue
        assert r.get("HGMMA.64x128x16.F32.BF16") == "12", (k, r)      # 4 K slices x (hi*hi, lo*hi, hi*lo) per stage
        assert r.get("UTMALDG.5D") == "1" and r.get("UTMALDG.3D") == "1", (k, r)
    for k in ("tapgemm_tc_kernel<128, 1, false>", "tapgemm_tc_kernel<16, 3, false>"):
        assert "UTMASTG" not in rows[k], (k, rows[k])                 # bf16 mode and the head tiles keep thread stores


def test_float32_tapgemm_does_not_spill():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc) and shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    nvcc = nvcc if os.path.exists(nvcc) else shutil.which("nvcc")
    with tempfile.TemporaryDirectory(prefix="ian_ptxas_") as tmp:
        p = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-cubin",
                            os.path.join(CSRC, "tapgemm_tc.cu"), "-o", os.path.join(tmp, "t.cubin")],
                           capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    # ptxas prints "Compiling entry function '<mangled>'", then "N bytes stack frame, S bytes spill stores, L bytes spill loads"
    report = re.findall(r"Compiling entry function '(\S+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads\s+"
                        r"ptxas info\s+: Used (\d+) registers", p.stderr, re.S)
    found = {}
    for name, st, ld, regs in report:
        m = re.search(r"tapgemm_tc_kernelILi(\d+)ELi(\d+)ELb([01])E", name)
        if m:
            found[(int(m.group(1)), int(m.group(2)), m.group(3) == "1")] = (int(st), int(ld), int(regs))
    for sk in (False, True):
        st, ld, regs = found[(128, 3, sk)]
        assert st == 0 and ld == 0, ("spills", sk, st, ld)
        # 288 threads = 9 warps: three share one SM sub-partition's 16 384 registers
        assert regs <= 168, ("registers", sk, regs)

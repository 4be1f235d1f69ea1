"""The decoder JVP's new kernels are the wgmma / TMA / PDL code DESIGN.md section 5.6f describes: SASS of the in-tree
libian_b200.so read with cuobjdump (tools/sass_summary.py; no GPU needed)."""
import os
import re
import subprocess

from test_sass import ROOT, _summary


def test_decout_jvp_tc_kernel_is_wgmma_tma_pdl():
    _, rows = _summary()
    r = rows["decout_jvp_tc_kernel"]
    assert any(m.startswith("HGMMA.64x80x16.F32.BF16") for m in r), r
    assert "WARPGROUP.ARRIVE" in r and "WARPGROUP.DEPBAR" in r, r
    assert "UTMALDG.5D" in r and "UTMALDG.3D" in r, r
    assert "PREEXIT" in r and "ACQBULK" in r, r
    assert "HMMA" not in r, r
    assert "PREEXIT" in rows["dec_out_jvp_kernel"] and "ACQBULK" in rows["dec_out_jvp_kernel"], rows["dec_out_jvp_kernel"]
    for k in ("head_jvp_r_kernel", "head_jvp_g_kernel", "head_jvp_b_out_kernel"):
        assert k in rows, k


def test_new_kernels_do_not_spill():
    lib = os.path.join(ROOT, "neural-photo-editor_b200", "libian_b200.so")
    res = subprocess.run(["cuobjdump", "--dump-resource-usage", lib], capture_output=True, text=True, check=True).stdout
    cur, seen = None, 0
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = m.group(1)
        m = re.search(r"STACK:(\d+).*LOCAL:(\d+)", line)
        if m and cur and "jvp" in cur:
            seen += 1
            assert m.group(1) == "0" and m.group(2) == "0", (cur, line)
    assert seen == 5, seen

"""The encoder JVP's new kernels (DESIGN.md section 5.6g): enc_conv1's tangent on the tensor cores is the wgmma / TMA / PDL
code of conv1_tc_kernel, and none of the four new kernels spills.  SASS of the in-tree libian_b200.so read with cuobjdump
(tools/sass_summary.py; no GPU needed)."""
import os
import re
import subprocess

from test_sass import ROOT, _summary

NEW = ("conv1_tangent_tc_kernel", "conv1_tangent_kernel", "sample_tangent_kernel", "made_iaf_tangent_kernel")


def test_conv1_tangent_tc_kernel_is_wgmma_tma_pdl():
    _, rows = _summary()
    r = rows["conv1_tangent_tc_kernel"]
    assert any(m.startswith("HGMMA.64x64x16.F32.BF16") for m in r), r
    assert "WARPGROUP.ARRIVE" in r and "WARPGROUP.DEPBAR" in r, r
    assert "UTMALDG.3D" in r and "UTMASTG" in r, r
    assert "PREEXIT" in r and "ACQBULK" in r, r
    assert "HMMA" not in r, r
    for k in ("sample_tangent_kernel", "made_iaf_tangent_kernel"):
        assert "PREEXIT" in rows[k] and "ACQBULK" in rows[k], (k, rows[k])
    assert "conv1_tangent_kernel" in rows


def _usage():
    lib = os.path.join(ROOT, "neural-photo-editor_b200", "libian_b200.so")
    res = subprocess.run(["cuobjdump", "--dump-resource-usage", lib], capture_output=True, text=True, check=True).stdout
    cur, out = None, {}
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = m.group(1)
        m = re.search(r"STACK:(\d+).*LOCAL:(\d+)", line)
        if m and cur:
            out[cur] = (int(m.group(1)), int(m.group(2)))
    return out


def test_new_kernels_do_not_spill():
    usage = _usage()
    for k in NEW:
        hits = [(name, u) for name, u in usage.items() if re.search(r"\d%s" % k, name)]
        assert len(hits) == 1, (k, hits)
        assert hits[0][1] == (0, 0), hits


def test_only_the_decoder_jvp_kernels_carry_jvp_in_their_names():
    names = [n for n in _usage() if "jvp" in n]
    assert len(names) == 5, names

"""The parameter VJP's weight-gradient kernel is the wgmma / TMA / PDL code DESIGN.md section 5.6e describes: SASS of the
in-tree libian_b200.so read with cuobjdump (tools/sass_summary.py; no GPU needed)."""
from test_sass import _summary


def test_wgrad_tc_kernel_is_wgmma_tma_pdl():
    _, rows = _summary()
    r = rows["wgrad_tc_kernel"]
    assert any(m.startswith("HGMMA.64x128x16.F32.BF16") for m in r), r
    assert "WARPGROUP.ARRIVE" in r and "WARPGROUP.DEPBAR" in r, r
    assert r.get("UTMALDG.5D") == "4", r                  # two output-gradient boxes + two activation boxes per K step
    assert "PREEXIT" in r and "ACQBULK" in r, r           # griddepcontrol.launch_dependents / .wait
    assert "HMMA" not in r, r
    for k in ("wgrad_simt_kernel", "wgrad_finalize_kernel", "decout_wgrad_kernel", "bn_param_bwd_kernel",
              "brush_param_seed_bwd_kernel"):
        assert "PREEXIT" in rows[k] and "ACQBULK" in rows[k], (k, rows[k])

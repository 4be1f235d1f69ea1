"""The features' vector-Jacobian product (DESIGN.md section 5.6l): its one new kernel, feat_cotangent_kernel, sits on the
PDL chain (griddepcontrol -> PREEXIT / ACQBULK), does not spill, and keeps "jvp" out of its name.  SASS of the in-tree
libian_b200.so read with cuobjdump (tools/sass_summary.py; no GPU needed)."""
import re

from test_sass import _summary
from test_sass_encode_tangent import _usage

KERNEL = "feat_cotangent_kernel"


def test_feat_cotangent_kernel_is_on_the_pdl_chain():
    _, rows = _summary()
    r = rows[KERNEL]
    assert "PREEXIT" in r and "ACQBULK" in r, r


def test_feat_cotangent_kernel_does_not_spill():
    hits = [(name, u) for name, u in _usage().items() if re.search(r"\d%s" % KERNEL, name)]
    assert len(hits) == 1, hits
    assert hits[0][1] == (0, 0), hits
    assert "jvp" not in hits[0][0]

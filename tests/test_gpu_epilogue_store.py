"""The two epilogue forms of the float32-mode tap-GEMM compute the same bits.

Plain whole tiles (scale/shift and none/LReLU/ReLU/ELU into one split-plane output) leave through TMA stores from the
accumulator fragments by default; IAN_EPI_TMA=0 sends them through the float32 staging tile and per-thread stores like
every other epilogue.  Every batch entry point, in its host and its device form (the calls of test_gpu_launch_forms.py),
must agree bit for bit between the two: on IAN_simple, IAN.py and IANv1.py under every stream-K setting, in bf16 mode on
IAN.py (which never takes the TMA-store form), at batches that give partial last m-tiles, graph replay, split-K and
chunking."""
import numpy as np
import pytest

from test_gpu_launch_forms import _inputs, _pairs, handle  # noqa: F401  (handle is a fixture)

pytestmark = pytest.mark.gpu
SIZES = (1, 3, 47, 130, 256, 513)
CASES = [(g, "fp32", s) for g in ("simple", "full", "v1") for s in (0, 1, 2)]
CASES += [("full", "bf16", 1)]


@pytest.mark.parametrize("graph,precision,streamk", CASES, ids=["%s-%s-streamk%d" % c for c in CASES])
def test_tma_store_epilogue_is_bit_identical(handle, npe, graph, precision, streamk):  # noqa: F811
    tma = handle(graph, "tc", precision, IAN_STREAMK=streamk)
    plain = handle(graph, "tc", precision, IAN_STREAMK=streamk, IAN_EPI_TMA=0)
    for n in SIZES:
        inp = _inputs(n, 8100 + n)
        for (name, th, td), (name2, ph, pd) in zip(_pairs(tma, npe, inp), _pairs(plain, npe, inp)):
            assert name == name2
            assert np.isfinite(th).all(), (name, n)
            for form, a, b in (("host", th, ph), ("dev", td, pd)):
                assert a.shape == b.shape and np.array_equal(a, b), (name, form, n, float(np.abs(a.astype(np.float64) - b).max()))

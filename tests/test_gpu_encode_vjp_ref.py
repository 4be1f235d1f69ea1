"""GPU encoder VJP (ian_encode_vjp_*) against the EXECUTED reference, and its argument checks.

  * <dx_gpu, v> against every directional derivative of the reference's own Z_hat in tests/golden/ref_exec_encvjp.npz
    (two golden images per graph, without and with eps), on both CUDA paths.  The bound is what the per-sample rule of
    tests/test_gpu_encode_vjp.py (max|dx_gpu - dx_ref| <= 1e-1 max|dx_ref|) implies for an inner product:
    |<dx_gpu, v> - d| <= 1e-1 max|dx_ref| sum|v|, with dx_ref the float64 oracle (itself held to d at 1e-7 by
    tests/test_ref_exec_encvjp.py).  The measured error relative to sum|dx_ref v| is recorded.
  * n = 0 and n = -1, on the host and the device-pointer entry points, return IAN_ERR_INVALID."""
import json
import os

import numpy as np
import pytest

from oracle import ian_full_numpy as fn
from oracle import weights as ow

import encode_vjp_oracle as eo
from test_ref_exec_encvjp import fixture

pytestmark = pytest.mark.gpu
IAN_ERR_INVALID = -1
CONFIG = {"simple": "IAN_simple.py", "full": "IAN.py", "v1": "IANv1.py"}
MAKE = {"simple": ow.make_simple_weights, "full": ow.make_full_weights, "v1": ow.make_v1_weights}


@pytest.mark.parametrize("g", ["simple", "full", "v1"])
def test_gpu_matches_executed_reference(npe, g):
    x, seed, (v, dz, eps), dd = fixture()[g]
    P = MAKE[g](seed)
    m = npe.IAN(CONFIG[g], True, weights=P)
    rec = {}
    try:
        for path in ("tc", "simt"):
            m.set_path(path)
            for j, e in enumerate((None, eps.astype(np.float32))):
                dx = m.encode_vjp(x, dz.astype(np.float32), e)
                for k in range(len(x)):
                    ek = None if e is None else eps[k:k + 1]
                    if g == "simple":
                        ref = eo.simple_encode_vjp(P, x[k:k + 1], dz[k:k + 1], ek)[0]
                    else:
                        ref = eo.full_encode_vjp(P, x[k:k + 1], fn.made_masks(m.made_ordering.astype(np.float32)), dz[k:k + 1], ek)[0]
                    got = float((dx[k].astype(np.float64) * v[k]).sum())
                    err = abs(got - dd[j, k])
                    rec["%s_eps%d_img%d" % (path, j, k)] = err / float(np.abs(ref * v[k]).sum())
                    assert err <= 1e-1 * np.abs(ref).max() * np.abs(v[k]).sum(), (g, path, j, k, got, dd[j, k])
    finally:
        m.close()
    if os.environ.get("IAN_TEST_RECORD"):
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "encvjp_ref_%s.json" % g), "w") as f:
            json.dump(rec, f, indent=1, sort_keys=True)


def test_nonpositive_batch_is_invalid(npe, weights):
    import torch
    m = npe.IAN("IAN_simple.py", True, weights=weights)
    try:
        lib, h = m._lib, m._h
        x = np.zeros((1, 3, 64, 64), np.float32)
        dz = np.zeros((1, 100), np.float32)
        dx = np.zeros_like(x)
        fp = lambda a: a.ctypes.data_as(lib.ian_encode_vjp_host.argtypes[1])
        xd, dzd = torch.zeros(1, 3, 64, 64, device="cuda"), torch.zeros(1, 100, device="cuda")
        dxd = torch.zeros_like(xd)
        for n in (0, -1):
            assert lib.ian_encode_vjp_host(h, fp(x), n, None, fp(dz), fp(dx)) == IAN_ERR_INVALID
            assert lib.ian_encode_vjp_dev(h, xd.data_ptr(), n, None, dzd.data_ptr(), dxd.data_ptr(), None) == IAN_ERR_INVALID
    finally:
        m.close()

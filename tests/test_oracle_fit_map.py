"""The float64 references of the masked latent fit under the prior (tests/fit_map_oracle.py), on the CPU:
  * torch jacfwd of decode . flow (J_u, and from it A, g, e) against central differences of the independent numpy
    oracle's E and x_hat, with random weights in [0, 1], a zero-weight hole whose target pixels are NaN, and beta > 0;
  * the inpainting targets of tests/test_gpu_fit_map.py: F(u*) lands on the margin-weight pool's latents, the decoder is
    certified there, and W^1/2 J_u at u* is well-conditioned for both holes (the fit can recover u* from the visible
    pixels alone).  Measured sigma_min / sigma_max: 0.016 on every graph and hole."""
import numpy as np
import pytest

import fit_map_oracle as fo
from test_ref_exec_decjvp import MAKE, weight_seed

H = 1e-7
BETA = 0.3
COND_MIN = 5e-3


def _case(g, n=1):
    rng = np.random.default_rng({"simple": 21, "full": 22, "v1": 23}[g])
    u = rng.standard_normal((n, 100))
    x = np.tanh(rng.standard_normal((n, 3, 64, 64)))
    w = rng.uniform(0, 1, (n, 3, 64, 64)) * fo.masks(n)["square"]
    x[w == 0] = np.nan
    return u, x, w, rng.standard_normal((2, n, 100))


@pytest.mark.parametrize("g", ["simple", "full", "v1"])
def test_jacfwd_matches_numpy_central_differences(g):
    P = MAKE[g](weight_seed(g))
    u, x, w, vs = _case(g)
    J, r = fo.jacobians64(g, P, u, x)
    A, gv, e = fo.gram64(J, r, w, u, BETA)
    E = lambda uu: fo.energy_np(g, P, uu, x, w, BETA)
    assert np.all(np.isfinite(A)) and np.all(np.isfinite(gv))
    assert np.allclose(e, E(u), rtol=1e-12, atol=0), (e, E(u))
    assert np.array_equal(A, np.swapaxes(A, 1, 2)) or np.abs(A - np.swapaxes(A, 1, 2)).max() <= 1e-12 * np.abs(A).max()
    wf = w.reshape(len(u), -1)
    for v in vs:
        xh = lambda uu: fo.DECODE_NP[g](P, fo.flow_np(g, P, uu)).reshape(len(u), -1)
        fd_x = (xh(u + H * v) - xh(u - H * v)) / (2 * H)
        jv = np.einsum("kip,ki->kp", J, v)
        # E sums 12288 terms: its central difference loses their magnitude's rounding, so the scale is the terms' L1 norm
        fd_e = (E(u + H * v) - E(u - H * v)) / (2 * H)
        scale = np.abs(2 * wf * np.where(wf != 0, r, 0) * jv).sum(1) + np.abs(2 * BETA * u * v).sum(1)
        assert np.all(np.abs(2 * (gv * v).sum(1) - fd_e) <= 1e-6 * scale), (2 * (gv * v).sum(1), fd_e, scale)
        assert np.abs(jv - fd_x).max() <= 1e-6 * np.abs(fd_x).max(), np.abs(jv - fd_x).max()
        # the Gauss-Newton curvature along v is the weighted norm of J_u v plus the prior's
        vAv = np.einsum("ki,kij,kj->k", v, A, v)
        want = (w.reshape(len(u), -1) * fd_x ** 2).sum(1) + BETA * (v * v).sum(1)
        assert np.allclose(vAv, want, rtol=1e-6, atol=0), (vAv, want)


@pytest.mark.parametrize("g", ["simple", "full", "v1"])
def test_inpainting_targets_are_certified_and_well_conditioned(g):
    import margin_weights as mw
    P = mw.weights(g)
    u, res = fo.recovery_targets(g, P)
    z = fo.flow_np(g, P, u.astype(np.float64))
    assert res <= 1e-6 * np.abs(z).max(), res
    for k in range(len(u)):
        assert mw.decoder_margin(g, P, z[k:k + 1])[0] > 0, k
    J, _ = fo.jacobians64(g, P, u, fo.DECODE_NP[g](P, z))
    for name, w in fo.masks(len(u)).items():
        for k in range(len(u)):
            s = np.linalg.svd(J[k] * np.sqrt(w[k].reshape(1, -1)), compute_uv=False)
            assert s.min() >= COND_MIN * s.max(), (name, k, s.min() / s.max())

"""The float64 references of the robust latent fit (tests/fit_robust_oracle.py), on the CPU:
  * rho and rho' of both losses: the quadratic limit, continuity at Huber's knee, rho' against central differences of rho;
  * g = grad E / 2 of the reweighted normal equations against central differences of the numpy oracle's E, on every graph,
    with random weights, a zero-weight hole with NaN targets and beta > 0; Huber at delta -> inf is fit_map_oracle's E;
  * the majorisation that makes the reweighted Gauss-Newton step sound: sum omega r'^2 - sum omega r^2 >= E' - E (pixel
    terms) at random points, since rho is concave in s;
  * the automatic scale rule against a plain sort, with ties, all-equal residuals, one weighted pixel and none;
  * the corruption generator: seeded, the block and the salt within [-1, 1], and about 2 % salt."""
import numpy as np
import pytest

import fit_map_oracle as fo
import fit_robust_oracle as ro
from test_ref_exec_decjvp import MAKE, weight_seed

H = 1e-6
BETA = 0.3


@pytest.mark.parametrize("kind", ro.KINDS)
def test_rho_and_its_derivative(kind):
    rng = np.random.default_rng(1)
    s = rng.uniform(0, 4, 1000) ** 2
    d = 0.3
    assert np.allclose(ro.rho(kind, s, 1e8), s, rtol=1e-9, atol=0)
    assert np.allclose(ro.drho(kind, s, 1e8), 1.0, rtol=1e-9, atol=0)
    hs = 1e-6 * np.maximum(s, 1e-3)
    fd = (ro.rho(kind, s + hs, d) - ro.rho(kind, s - hs, d)) / (2 * hs)
    knee = np.abs(s - d * d) < 2 * hs
    assert np.allclose(fd[~knee], ro.drho(kind, s, d)[~knee], rtol=1e-6, atol=0)
    assert np.all(ro.drho(kind, s, d) <= 1.0) and np.all(np.diff(ro.drho(kind, np.sort(s), d)) <= 0)   # concave in s
    if kind == "huber":
        assert ro.rho(kind, d * d, d) == d * d and np.isclose(ro.rho(kind, d * d * (1 + 1e-12), d), d * d, rtol=1e-11)
        assert np.array_equal(ro.rho(kind, s, np.inf), s) and np.all(ro.drho(kind, s, np.inf) == 1.0)


def _case(g, n=1):
    rng = np.random.default_rng({"simple": 31, "full": 32, "v1": 33}[g])
    u = rng.standard_normal((n, 100))
    x = np.tanh(rng.standard_normal((n, 3, 64, 64)))
    w = rng.uniform(0, 1, (n, 3, 64, 64)) * fo.masks(n)["square"]
    x[w == 0] = np.nan
    return u, x, w, rng.standard_normal((2, n, 100))


@pytest.mark.parametrize("g", ["simple", "full", "v1"])
def test_gradient_is_half_the_central_difference_of_E(g):
    P = MAKE[g](weight_seed(g))
    u, x, w, vs = _case(g)
    J, r = fo.jacobians64(g, P, u, x)
    rr = np.where(w.reshape(1, -1) != 0, r, 0.0)
    for kind in ro.KINDS:
        delta = np.array([0.5 * np.median(np.abs(rr[w.reshape(1, -1) != 0]))])
        A, gv, e = ro.gram64(J, r, w, u, BETA, kind, delta)
        E = lambda uu: ro.energy_np(g, P, uu, x, w, BETA, kind, delta)
        assert np.allclose(e, E(u), rtol=1e-12, atol=0), (kind, e, E(u))
        om = np.where(w.reshape(1, -1) != 0, w.reshape(1, -1) * ro.drho(kind, rr * rr, delta[:, None]), 0.0)
        jv_all = [np.einsum("kip,ki->kp", J, v) for v in vs]
        for v, jv in zip(vs, jv_all):
            fd_e = (E(u + H * v) - E(u - H * v)) / (2 * H)
            scale = np.abs(2 * om * rr * jv).sum(1) + np.abs(2 * BETA * u * v).sum(1)
            # 1e-5: rounding of E over 2H, and pixels whose residual crosses Huber's knee (rho is C1 there, not C2)
            assert np.all(np.abs(2 * (gv * v).sum(1) - fd_e) <= 1e-5 * scale), (kind, 2 * (gv * v).sum(1), fd_e, scale)
    # Huber with delta = inf is the masked fit's objective and normal equations
    got = ro.gram64(J, r, w, u, BETA, "huber", np.array([np.inf]))
    want = fo.gram64(J, r, w, u, BETA)
    assert all(np.array_equal(a, b) for a, b in zip(got[:2], want[:2])) and np.allclose(got[2], want[2], rtol=1e-14)
    assert np.allclose(ro.energy_np(g, P, u, x, w, BETA, "huber", [np.inf]), fo.energy_np(g, P, u, x, w, BETA), rtol=1e-14)


@pytest.mark.parametrize("kind", ro.KINDS)
def test_reweighted_squares_majorise_the_robust_loss(kind):
    """rho concave in s: rho(s') <= rho(s) + rho'(s) (s' - s), so the IRLS surrogate bounds E from above, equal at s"""
    rng = np.random.default_rng(2)
    for _ in range(20):
        delta = rng.uniform(0.01, 1)
        r0 = rng.standard_normal(4096) * rng.uniform(0.01, 2)
        r1 = r0 + rng.standard_normal(4096) * rng.uniform(0.001, 2)
        w = rng.uniform(0, 1, 4096)
        om = w * ro.drho(kind, r0 * r0, delta)
        lhs = (w * ro.rho(kind, r1 * r1, delta)).sum() - (w * ro.rho(kind, r0 * r0, delta)).sum()
        rhs = (om * r1 * r1).sum() - (om * r0 * r0).sum()
        assert lhs <= rhs + 1e-12 * np.abs(w * r1 * r1).sum(), (lhs, rhs)


@pytest.mark.parametrize("kind", ro.KINDS)
def test_scale_rule(kind):
    rng = np.random.default_rng(3)
    n = 6
    x = rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)
    xh = rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)
    x[1], xh[1] = 0.5, 0.75                                          # all-equal residuals
    xh[2].reshape(-1)[:6000] = x[2].reshape(-1)[:6000] + np.float32(0.5)   # many ties around the median
    w = np.ones_like(x)
    w[3] = 0
    w[3, 1, 7, 9] = 2.0                                              # a single weighted pixel
    w[4] = 0                                                         # none
    w[5, :, :, :32] = 0
    got = ro.scale_np(kind, xh, x, w)
    a = np.abs(xh - x).reshape(n, -1)
    for k in range(n):
        v = np.sort(a[k][w[k].reshape(-1) != 0])
        want = ro.FLOOR if v.size == 0 else max(float(v[(v.size - 1) // 2]) * ro.C_SCALE[kind], ro.FLOOR)
        assert got[k] == want, (k, got[k], want)
    assert got[4] == ro.FLOOR
    assert got[1] == 0.25 * ro.C_SCALE[kind]
    assert got[3] == max(float(np.abs(xh[3, 1, 7, 9] - x[3, 1, 7, 9])) * ro.C_SCALE[kind], ro.FLOOR)
    tiny = ro.scale_np(kind, x[:1] + np.float32(1e-4), x[:1])
    assert tiny[0] == ro.FLOOR                                      # below half an 8-bit level: the floor
    assert ro.scale_np(kind, xh, x)[0] == ro.scale_np(kind, xh[:1], x[:1])[0]


def test_corruption_is_seeded_and_bounded():
    x = np.zeros((4, 3, 64, 64), np.float32)
    y, bad = ro.corrupt(x, 5)
    y2, bad2 = ro.corrupt(x, 5)
    assert np.array_equal(y, y2) and np.array_equal(bad, bad2)
    assert np.all(np.abs(y) <= 1) and np.all(y[~bad] == 0)
    for k in range(4):
        salt = (np.abs(y[k]) == 1).all(0)
        assert 0.01 < salt.mean() < 0.03, salt.mean()
        assert 256 <= bad[k, 0].sum() <= 256 + 0.03 * 4096
    assert not np.array_equal(bad[0], bad[1])

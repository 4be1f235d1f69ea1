"""GPU tests of the masked latent fit under the prior (include/ian_b200.h ian_map_gauss_newton_* / ian_fit_latent_map_*,
API.IAN.gauss_newton_map / fit_latent_map) on all three graphs, on the tensor-core and SIMT paths and, on IAN.py, in bf16
mode.  u is the fit-space latent (l_Z on IAN_simple, l_Z_IAF on IAN.py / IANv1.py); tests/fit_map_oracle.py holds the
float64 references and the targets.

  A. reductions, bit for bit: IAN_simple with w = None and prior 0 is ian_decode_gauss_newton_* / ian_fit_latent_*; w of
     all ones is w = None on every graph; with prior 0, A, g and e are a float64 Gram of J_u's own bits (decode_jvp of
     flow_jvp's identity columns) to 1e-10.
  B. A, g, e against float64 torch (jacfwd of decode . flow) on margin weights: random w in [0, 1] with beta > 0, and a 0/1
     mask with NaN targets in the hole; per-sample relative Frobenius / L2.  The float32 bound has 2x headroom over the
     measured worst and is checked to be at most a third of the floor that rounding J_u to bf16 moves the float64 A and g by.
  C. the solver: fit_latent_map(iters=1) against u0 + delta, delta solved in numpy float64 from gauss_newton_map(u0)'s own A
     and g with lambda_0 D, where that step lowers E; u0 bit for bit where it does not.
  D. inpainting: targets x = sample(u*) with F(u*) certified, a 24 x 24 square or the left half at weight 0 and NaN in x
     there, starts 5 % away; after 10 steps u is u* and the decoded hole the target's, within bounds set from measurement;
     fit_latent on the same image with the hole filled with 0 misses the hole by at least 10x more.  The loss history never
     increases; with every weight 0 the prior alone pulls u towards 0.
  E. bits: reruns, device form = host form, IAN_PDL=0, IAN_CHUNK=16 within D's bounds, and one sample's u and z are
     bit-unchanged when another sample's x, w or start changes (NaN at a weighted pixel included).
  F. errors: NULL pointers, a negative or non-finite prior or weight, iters < 0, n < 0, n = 0, an unfinalized handle.
Measured values go to fit_map.json when IAN_TEST_RECORD names a directory."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import fit_map_oracle as fo
import margin_weights as mw
from test_ref_exec_decjvp import MAKE, weight_seed

pytestmark = pytest.mark.gpu
CONFIG = {"simple": "IAN_simple.py", "full": "IAN.py", "v1": "IANv1.py"}
GRAPHS = ["simple", "full", "v1"]
ENV = ("IAN_STREAMK", "IAN_SPLITK", "IAN_GRAPHS", "IAN_PDL", "IAN_FINALIZE8", "IAN_CHUNK", "IAN_PATH")
LAMBDA0, DAMP_FLOOR = 1e-3, 1e-9
BETA = 1e-2
# Bounds set from one run on an H100 80GB HBM3 at 700 W (the results are the same bits on every rerun).
# B. per-sample relative error of (A, g, e) against float64 at certified targets against the pool's images.  Float32 mode,
# both paths, both weight cases: worst 3.8e-5 / 3.4e-5 / 5.6e-7 (IAN.py, tensor cores, the 0/1 mask).  Rounding J_u to bf16
# moves the float64 A and g by at least 1.4e-4 / 9.1e-4 (IAN.py), so the A bound cannot have both 2x headroom and sit below
# a third of that floor: it has 1.2x; the g and e bounds have 2x.  bf16 mode on IAN.py: worst 4.3e-3 / 8.3e-3 / 7.6e-5, at
# the level of the floor, as expected of single-pass bf16 (bounds 2x over).
NE_BOUND = (4.5e-5, 7e-5, 1.2e-6)
NE_BF16 = (9e-3, 1.7e-2, 1.6e-4)
# D. after 10 steps from 5 % away, float32 mode: |u - u*| / |u*| and the hole's max |x_hat - x*| (x in [-1, 1]).
# Measured worst over both paths, both holes, 3 targets and 20 targets in chunks of 16: 3.2e-4 (IAN.py; <= 4.4e-5 on the
# other graphs) and 1.95e-5 (IAN_simple); fit_latent on the hole filled with 0 misses it by at least 6.5e3x more.
RECOVERY = (7e-4, 4e-5)
RECORD = {}


def _record(key, value):
    RECORD[key] = value
    if os.environ.get("IAN_TEST_RECORD"):
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "fit_map.json"), "w") as f:
            json.dump(RECORD, f, indent=1, sort_keys=True)


def _margin(g):
    return mw.weights(g, device="cuda")


_TARGETS = {}


def _targets(g, n=3):
    if (g, n) not in _TARGETS:
        _TARGETS[(g, n)] = fo.recovery_targets(g, _margin(g), n)[0]
    return _TARGETS[(g, n)]


@pytest.fixture
def handles(npe, monkeypatch):
    """make(graph, weights, **env): a handle with exactly `env` among the schedule variables, closed at test end"""
    made = []

    def make(graph, weights, **env):
        for k in ENV:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, str(v))
        try:
            m = npe.IAN(CONFIG[graph], True, weights=weights)
        finally:
            for k in env:
                monkeypatch.delenv(k, raising=False)
        made.append(m)
        return m
    try:
        yield make
    finally:
        for m in made:
            m.close()


def _rel(got, ref):
    """per-sample ||got - ref|| / ||ref|| (Frobenius for A)"""
    n = len(ref)
    d = (np.asarray(got, np.float64) - ref).reshape(n, -1)
    return np.linalg.norm(d, axis=1) / np.linalg.norm(np.asarray(ref, np.float64).reshape(n, -1), axis=1)


def _start(us, seed):
    d = np.random.default_rng(seed).standard_normal(us.shape)
    d *= 0.05 * np.linalg.norm(us, axis=1, keepdims=True) / np.linalg.norm(d, axis=1, keepdims=True)
    return (us + d).astype(np.float32)


def _holed(x, w):
    x = x.copy()
    x[w == 0] = np.nan
    return x


def _cases(g, x):
    """(name, w, images, beta): random weights in [0, 1] with the prior, and a 0/1 mask with NaN targets in its hole"""
    n = len(x)
    w = np.random.default_rng(40).uniform(0, 1, x.shape).astype(np.float32)
    sq = fo.masks(n)["square"]
    return [("random", w, x, BETA), ("mask", sq, _holed(x, sq), 0.0)]


# ---- A. reductions ----------------------------------------------------------------------------------------------------------
def test_simple_reduces_to_the_fit_bit_for_bit(handles):
    m = handles("simple", _margin("simple"))
    us = _targets("simple")
    u0 = _start(us, 1)
    x = m.sample(us)
    ne = m.gauss_newton(u0, x)
    for w in (None, np.ones_like(x)):
        got = m.gauss_newton_map(u0, x, w, 0.0)
        assert all(np.array_equal(a, b) for a, b in zip(got, ne))
    z1, l1 = m.fit_latent(x, u0, iters=3, return_loss=True)
    u2, z2, l2 = m.fit_latent_map(x, None, 0.0, u0, iters=3, return_loss=True)
    assert np.array_equal(u2, z1) and np.array_equal(z2, z1) and np.array_equal(l2, l1)


@pytest.mark.parametrize("g", GRAPHS)
def test_gram_of_the_same_bits_and_unit_weights(handles, g):
    m = handles(g, _margin(g))
    us = _targets(g)
    u0 = _start(us, 2)
    x = m.sample(us)
    got = m.gauss_newton_map(u0, x)
    assert all(np.array_equal(a, b) for a, b in zip(got, m.gauss_newton_map(u0, x, np.ones_like(x), 0.0)))
    assert np.array_equal(got[0], np.swapaxes(got[0], 1, 2))
    J = []
    for k in range(len(u0)):
        zr, tan = m.flow_jvp(np.repeat(u0[k:k + 1], 100, 0), np.eye(100, dtype=np.float32), return_z=True)
        J.append(m.decode_jvp(zr, tan).reshape(100, -1))
    J = np.stack(J).astype(np.float64)
    xh = m.sample(u0).astype(np.float64)
    err = {}
    for name, w, xx, beta in [("none", None, x, 0.0)] + _cases(g, x):
        ref = fo.gram64(J, (xh - xx).reshape(len(u0), -1), w, u0, beta)
        out = m.gauss_newton_map(u0, xx, w, beta)
        err[name] = [float(_rel(a, b).max()) for a, b in zip(out, ref)]
    _record("A_%s" % g, err)
    assert max(max(v) for v in err.values()) <= 1e-10, err


# ---- B. against float64 ------------------------------------------------------------------------------------------------------
_REF = {}


def _ref64(g):
    """u* and per weight case (w, images, beta, float64 A, g, e, the same from J_u rounded to bf16); the images are the
    margin-weight pool's own, so r is of the order of the image"""
    if g not in _REF:
        u = _targets(g, 6)
        x = mw.pool()["x"][np.linspace(0, mw.POOL - 1, 6).astype(int)]
        J, xh = fo.jacobians64(g, _margin(g), u, np.zeros_like(x), device="cuda")
        Jb = mw.bf16_round(J.astype(np.float32)).astype(np.float64)
        out = {}
        for name, w, xx, beta in _cases(g, x):
            r = xh - xx.reshape(len(u), -1).astype(np.float64)
            out[name] = (w, xx, beta, fo.gram64(J, r, w, u, beta), fo.gram64(Jb, r, w, u, beta))
        _REF[g] = (u, out)
    return _REF[g]


@pytest.mark.parametrize("g", GRAPHS)
def test_normal_equations_against_float64(handles, g):
    u, cases = _ref64(g)
    # the floor is taken where the normal equations are J_u's alone (prior 0): beta I and beta u hold no J
    _, _, _, ref, slip = cases["mask"]
    floor = [float(_rel(s, rf).min()) for s, rf in zip(slip[:2], ref[:2])]
    rec, worst = {"bf16_J_floor": floor}, []
    for name, (w, xx, beta, ref, _) in cases.items():
        for mode in ["tc", "simt"] + (["bf16"] if g == "full" else []):
            m = handles(g, _margin(g))
            if mode == "simt":
                m.set_path("simt")
            if mode == "bf16":
                m.set_precision("bf16")
            err = [float(_rel(a, b).max()) for a, b in zip(m.gauss_newton_map(u, xx, w, beta), ref)]
            rec["%s_%s" % (name, mode)] = err
            worst.append((name, mode, err, NE_BF16 if mode == "bf16" else NE_BOUND))
    _record("B_%s" % g, rec)
    for name, mode, err, bound in worst:
        assert all(e <= b for e, b in zip(err, bound)), (name, mode, err, bound)
    for nm, b, f in zip("Ag", NE_BOUND, floor):
        assert b <= f / 3, (nm, b, f)


# ---- C. the solver -------------------------------------------------------------------------------------------------------------
def _lm_step(A, g, lam=LAMBDA0):
    d = np.diagonal(A, axis1=1, axis2=2)
    D = np.maximum(d, DAMP_FLOOR * d.max(axis=1, keepdims=True))
    M = A + lam * np.einsum("ki,ij->kij", D, np.eye(100))
    return np.linalg.solve(M, -g[..., None])[..., 0]


@pytest.mark.parametrize("mode", ["tc", "simt"])
@pytest.mark.parametrize("g", GRAPHS)
def test_one_step_is_the_float64_solve(handles, g, mode):
    m = handles(g, _margin(g))
    m.set_path(mode)
    us = _targets(g, 6)
    u0 = _start(us, 4)
    x = m.sample(us)
    rec = {}
    for name, w, xx, beta in _cases(g, x):
        A, gv, e = m.gauss_newton_map(u0, xx, w, beta)
        u1, z1, loss = m.fit_latent_map(xx, w, beta, u0, iters=1, return_loss=True)
        assert np.allclose(loss[:, 0], e / 12288, rtol=1e-6, atol=0), (loss[:, 0], e / 12288)
        assert np.array_equal(z1, m.Z_IAF_fn(u1))
        delta = _lm_step(A, gv)
        want = u0.astype(np.float64) + delta
        took = loss[:, 1] < loss[:, 0]
        ulps = []
        for k in range(len(u0)):
            if not took[k]:
                assert np.array_equal(u1[k], u0[k]) and loss[k, 1] == loss[k, 0], k
                continue
            tol = np.spacing(np.abs(want[k]).astype(np.float32)).astype(np.float64) + 1e-9 * np.abs(delta[k]).max()
            err = np.abs(u1[k] - want[k])
            ulps.append(float((err / tol).max()))
            assert np.all(err <= tol), (name, k, (err / tol).max())
        rec[name] = {"accepted": took.tolist(), "err_ulps": ulps}
        _record("C_%s_%s" % (g, mode), rec)
        assert took.any()


# ---- D. inpainting ------------------------------------------------------------------------------------------------------------------
def _inpaint(m, g, us, u0, hole, key):
    """fit_latent_map with the hole at weight 0 and NaN in it, and fit_latent with the hole filled with 0"""
    x = m.sample(us)
    w = fo.masks(len(us))[hole]
    u, z, loss = m.fit_latent_map(_holed(x, w), w, 0.0, u0, iters=10, return_loss=True)
    du = np.linalg.norm(u.astype(np.float64) - us, axis=1) / np.linalg.norm(us.astype(np.float64), axis=1)
    inside = (w == 0)
    miss = np.abs(m.sample(u) - x)[inside].reshape(len(us), -1).max(1)
    zf = m.fit_latent(np.where(inside, np.float32(0), x), m.Z_IAF_fn(u0), iters=10)
    miss_plain = np.abs(m.sample_at(zf) - x)[inside].reshape(len(us), -1).max(1)
    _record(key, {"du": du.tolist(), "hole_miss": miss.tolist(), "hole_miss_fit_latent": miss_plain.tolist(),
                  "loss_first": loss[:, 0].tolist(), "loss_last": loss[:, -1].tolist()})
    assert np.all(np.diff(loss.astype(np.float64), axis=1) <= 0), loss
    assert du.max() <= RECOVERY[0] and miss.max() <= RECOVERY[1], (du, miss)
    assert np.all(miss_plain >= 10 * miss), (miss_plain, miss)
    assert np.array_equal(z, m.Z_IAF_fn(u))


@pytest.mark.parametrize("hole", ["square", "left"])
@pytest.mark.parametrize("mode", ["tc", "simt"])
@pytest.mark.parametrize("g", GRAPHS)
def test_inpainting_recovers_the_latent(handles, g, mode, hole):
    m = handles(g, _margin(g))
    m.set_path(mode)
    us = _targets(g)
    _inpaint(m, g, us, _start(us, 5), hole, "D_%s_%s_%s" % (g, mode, hole))


@pytest.mark.parametrize("g", GRAPHS)
def test_prior_alone_pulls_towards_zero(handles, g):
    m = handles(g, synth(g))
    rng = np.random.default_rng(50)
    u0 = rng.standard_normal((4, 100)).astype(np.float32)
    x = np.full((4, 3, 64, 64), np.nan, np.float32)
    w = np.zeros_like(x)
    u, z, loss = m.fit_latent_map(x, w, 0.5, u0, iters=5, return_loss=True)
    assert np.all(np.diff(loss.astype(np.float64), axis=1) <= 0), loss
    assert np.allclose(loss[:, 0], 0.5 * (u0.astype(np.float64) ** 2).sum(1) / 12288, rtol=1e-6)
    shrink = np.linalg.norm(u, axis=1) / np.linalg.norm(u0, axis=1)
    _record("D_prior_%s" % g, shrink.tolist())
    assert np.all(shrink < 0.5), shrink
    assert np.all(np.isfinite(z))


_SYNTH = {}


def synth(g):
    if g not in _SYNTH:
        _SYNTH[g] = MAKE[g](weight_seed(g))
    return _SYNTH[g]


# ---- E. bits ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_bits_forms_and_schedules(handles, g):
    import torch
    m = handles(g, _margin(g))
    us = _targets(g)
    u0 = _start(us, 6)
    w = np.random.default_rng(41).uniform(0, 1, (3, 3, 64, 64)).astype(np.float32) * fo.masks(3)["square"]
    x = _holed(m.sample(us), w)
    u1, z1, l1 = m.fit_latent_map(x, w, BETA, u0, iters=3, return_loss=True)
    u2, z2, l2 = m.fit_latent_map(x, w, BETA, u0, iters=3, return_loss=True)
    assert np.array_equal(u1, u2) and np.array_equal(z1, z2) and np.array_equal(l1, l2)
    ne = m.gauss_newton_map(u0, x, w, BETA)
    assert all(np.array_equal(a, b) for a, b in zip(ne, m.gauss_newton_map(u0, x, w, BETA)))
    # device form
    ud, xd, wd = (torch.from_numpy(a).cuda() for a in (u0, x, w))
    Ad = torch.empty(3, 100, 100, dtype=torch.float64, device="cuda")
    gd = torch.empty(3, 100, dtype=torch.float64, device="cuda")
    ed = torch.empty(3, dtype=torch.float64, device="cuda")
    m.gauss_newton_map_dev(ud.data_ptr(), xd.data_ptr(), wd.data_ptr(), BETA, 3, Ad.data_ptr(), gd.data_ptr(), ed.data_ptr())
    zd = torch.empty(3, 100, device="cuda")
    ld = torch.empty(3, 4, device="cuda")
    m.fit_latent_map_dev(xd.data_ptr(), wd.data_ptr(), BETA, 3, ud.data_ptr(), 3, zd.data_ptr(), ld.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(Ad.cpu().numpy(), ne[0]) and np.array_equal(gd.cpu().numpy(), ne[1])
    assert np.array_equal(ed.cpu().numpy(), ne[2])
    assert np.array_equal(ud.cpu().numpy(), u1) and np.array_equal(zd.cpu().numpy(), z1)
    assert np.array_equal(ld.cpu().numpy(), l1)
    ud.copy_(torch.from_numpy(u0))
    m.fit_latent_map_dev(xd.data_ptr(), wd.data_ptr(), BETA, 3, ud.data_ptr(), 3)         # z and loss left out
    m.gauss_newton_map_dev(ud.data_ptr(), xd.data_ptr(), 0, 0.0, 0, 0, 0)                 # n = 0
    torch.cuda.synchronize()
    assert np.array_equal(ud.cpu().numpy(), u1)
    # PDL off
    m0 = handles(g, _margin(g), IAN_PDL=0)
    u3, z3, l3 = m0.fit_latent_map(x, w, BETA, u0, iters=3, return_loss=True)
    assert np.array_equal(u3, u1) and np.array_equal(z3, z1) and np.array_equal(l3, l1)
    assert all(np.array_equal(a, b) for a, b in zip(ne, m0.gauss_newton_map(u0, x, w, BETA)))
    # chunked: 20 samples in chunks of 16 and 4
    mc = handles(g, _margin(g), IAN_CHUNK=16)
    us = _targets(g, 20)
    _inpaint(mc, g, us, _start(us, 7), "square", "E_chunk_%s" % g)


@pytest.mark.parametrize("g", GRAPHS)
def test_samples_stay_apart(handles, g):
    m = handles(g, _margin(g))
    us = _targets(g, 4)
    u0 = _start(us, 8)
    w = fo.masks(4)["left"]
    x = _holed(m.sample(us), w)
    u1, z1, l1 = m.fit_latent_map(x, w, BETA, u0, iters=3, return_loss=True)
    x2, w2, u2 = x.copy(), w.copy(), u0.copy()
    x2[1] = np.float32(0.25)
    x2[2, :, 10, 40] = np.nan                                 # NaN at a weighted pixel: sample 2 alone goes bad
    w2[3] = np.float32(0.5)
    u2[3] += np.float32(0.1)
    v1, y1, k1 = m.fit_latent_map(x2, w2, BETA, u2, iters=3, return_loss=True)
    assert np.array_equal(v1[0], u1[0]) and np.array_equal(y1[0], z1[0]) and np.array_equal(k1[0], l1[0])
    assert not np.array_equal(v1[1], u1[1]) and not np.array_equal(v1[3], u1[3])


# ---- F. errors ---------------------------------------------------------------------------------------------------------------------
def test_errors(npe, model):
    lib, h = model._lib, model._h
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    u = np.zeros((2, 100), np.float32)
    x = np.zeros((2, 3, 64, 64), np.float32)
    w = np.ones((2, 3, 64, 64), np.float32)
    A, g, e = np.full((2, 100, 100), 7.0), np.full((2, 100), 7.0), np.full(2, 7.0)
    z = np.full((2, 100), 7, np.float32)
    loss = np.full((2, 4), 7, np.float32)
    gn = lambda *a: lib.ian_map_gauss_newton_host(h, *a)
    fit = lambda *a: lib.ian_fit_latent_map_host(h, *a)
    assert gn(None, fp(x), fp(w), 0.0, 2, dp(A), dp(g), dp(e)) == -1
    assert gn(fp(u), None, fp(w), 0.0, 2, dp(A), dp(g), dp(e)) == -1
    assert gn(fp(u), fp(x), fp(w), 0.0, 2, None, dp(g), dp(e)) == -1
    assert gn(fp(u), fp(x), fp(w), 0.0, 2, dp(A), None, dp(e)) == -1
    assert gn(fp(u), fp(x), fp(w), 0.0, -1, dp(A), dp(g), dp(e)) == -1
    for bad in (-1.0, float("nan"), float("inf")):
        assert gn(fp(u), fp(x), fp(w), bad, 2, dp(A), dp(g), dp(e)) == -1
        assert fit(fp(x), fp(w), bad, 2, fp(u), fp(z), 3, fp(loss)) == -1
        assert lib.ian_map_gauss_newton_dev(h, None, None, None, bad, 2, None, None, None, None) == -1
    for bad in (-1.0, float("nan"), float("inf")):
        wb = w.copy()
        wb[1, 2, 3, 4] = bad
        assert gn(fp(u), fp(x), fp(wb), 0.0, 2, dp(A), dp(g), dp(e)) == -1
        assert fit(fp(x), fp(wb), 0.0, 2, fp(u), fp(z), 3, fp(loss)) == -1
    assert lib.ian_map_gauss_newton_dev(h, None, None, None, 0.0, -1, None, None, None, None) == -1
    assert fit(None, fp(w), 0.0, 2, fp(u), fp(z), 3, fp(loss)) == -1
    assert fit(fp(x), fp(w), 0.0, 2, None, fp(z), 3, fp(loss)) == -1
    assert fit(fp(x), fp(w), 0.0, 2, fp(u), fp(z), -1, fp(loss)) == -1
    assert fit(fp(x), fp(w), 0.0, -1, fp(u), fp(z), 3, fp(loss)) == -1
    assert lib.ian_fit_latent_map_dev(h, None, None, 0.0, -1, None, None, 3, None, None) == -1
    assert gn(fp(u), fp(x), fp(w), 0.0, 0, dp(A), dp(g), dp(e)) == 0 and np.all(A == 7) and np.all(g == 7)
    assert fit(fp(x), fp(w), 0.0, 0, fp(u), fp(z), 3, fp(loss)) == 0 and np.all(loss == 7) and np.all(z == 7)
    assert np.all(u == 0) and np.all(e == 7)
    A0, g0, e0 = model.gauss_newton_map(np.zeros((0, 100), np.float32), np.zeros((0, 3, 64, 64), np.float32))
    assert A0.shape == (0, 100, 100) and g0.shape == (0, 100) and e0.shape == (0,)
    u0, z0, l0 = model.fit_latent_map(np.zeros((0, 3, 64, 64), np.float32), u0=np.zeros((0, 100), np.float32),
                                      return_loss=True)
    assert u0.shape == (0, 100) and z0.shape == (0, 100) and l0.shape == (0, 11)
    with pytest.raises(ValueError):
        model.gauss_newton_map(u, x[:1])
    with pytest.raises(ValueError):
        model.gauss_newton_map(u, x, w[:1])
    with pytest.raises(ValueError):
        model.fit_latent_map(x, prior=-1.0)
    with pytest.raises(ValueError):
        model.fit_latent_map(x, u0=u, iters=-1)
    with pytest.raises(TypeError):
        model.fit_latent_map(x, u0=u.astype(np.float64))
    raw = C.c_void_p()
    assert lib.ian_create(0, 0, C.byref(raw)) == 0
    try:
        assert lib.ian_map_gauss_newton_host(raw, fp(u), fp(x), fp(w), 0.0, 2, dp(A), dp(g), dp(e)) == -3
        assert lib.ian_fit_latent_map_host(raw, fp(x), fp(w), 0.0, 2, fp(u), fp(z), 3, fp(loss)) == -3
    finally:
        lib.ian_destroy(raw)


def test_default_start_ignores_the_hole(handles):
    """the default start is Zfn of the images with zero-weight pixels set to 0: NaN there never reaches it"""
    m = handles("full", _margin("full"))
    us = _targets("full")
    x = m.sample(us)
    w = fo.masks(3)["square"]
    u, z = m.fit_latent_map(_holed(x, w), w, 0.0, iters=0)
    assert np.array_equal(u, m.Zfn(np.where(w == 0, np.float32(0), x))) and np.all(np.isfinite(u))
    assert np.array_equal(z, m.Z_IAF_fn(u))

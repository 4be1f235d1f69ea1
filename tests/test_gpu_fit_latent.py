"""GPU tests of the latent fit (include/ian_b200.h ian_decode_gauss_newton_* / ian_fit_latent_*, API.IAN.gauss_newton /
fit_latent) on all three graphs, on the tensor-core and SIMT paths and, on IAN.py, in bf16 mode.

  A. the normal equations A = J^T J, g = J^T r, e = r^T r against float64 torch (J from torch.func.jacfwd of
     oracle/ian_torch.py's decoders) on 13 samples spread over the margin-weight pool, per-sample relative Frobenius / L2.
     The float32 bound has 2x headroom over the measured worst and is checked to be at most a third of the floor that
     rounding J to bf16 moves the float64 normal equations by.
  B. the Gram alone: against a float64 Gram of decoder_jacobian(z) and of sample_at(z) - x, the same bits summed in
     another order: <= 1e-10 relative.
  C. the solver alone: fit_latent(iters=1) against z0 + delta, delta solved in numpy float64 from gauss_newton(z0)'s own A
     and g with lambda_0 D, where that step lowers e; z0 bit for bit where it does not.
  D. Levenberg-Marquardt properties on synthetic weights and random targets, 10 steps: the loss history never increases,
     z is bit-unchanged across a flat entry, the reject path runs, and every sample ends below its start.
  E. recovery: targets decoded from certified pool latents z*, starts 5 % away; after 10 steps |z - z*| / |z*| and the MSE
     are below bounds set from measurement (bf16 mode: the MSE only, see the bounds below).
  F. bits: reruns, device form = host form, IAN_PDL=0, and IAN_CHUNK=16 within E's bounds.
  G. errors: NULL pointers, iters < 0, n < 0, n = 0, an unfinalized handle.
Measured values go to fit_latent.json when IAN_TEST_RECORD names a directory."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import margin_weights as mw
from test_ref_exec_decjvp import MAKE, weight_seed

pytestmark = pytest.mark.gpu
CONFIG = {"simple": "IAN_simple.py", "full": "IAN.py", "v1": "IANv1.py"}
GRAPHS = ["simple", "full", "v1"]
ENV = ("IAN_STREAMK", "IAN_SPLITK", "IAN_GRAPHS", "IAN_PDL", "IAN_FINALIZE8", "IAN_CHUNK", "IAN_PATH")
LAMBDA0, DAMP_FLOOR = 1e-3, 1e-9
# Bounds set from one run on an H100 80GB HBM3 at 700 W (the results are the same bits on every rerun).
# A. per-sample relative error of (A, g, e) against float64.  Float32 mode, both paths: worst 3.6e-5 / 2.6e-5 / 6.6e-7
# (IAN.py, tensor cores); rounding J to bf16 moves the float64 A and g by at least 2.5e-4 / 9.8e-4 (IAN.py), so the A and g
# bounds are >= 2x over the worst and <= a third of that floor.  e holds no J: its bound is 3x over its worst alone.
# bf16 mode on IAN.py: worst 1.8e-3 / 7.3e-3 / 9.0e-5, at the level of that floor, as expected of single-pass bf16.
NE_BOUND = (8e-5, 6e-5, 2e-6)
NE_BF16 = (4e-3, 1.5e-2, 2e-4)
# E. after 10 steps from 5 % away, float32 mode: |z - z*| / |z*| worst 2.3e-4 (IAN.py; 2.3e-5 on the other graphs) and MSE
# worst 6.5e-12 (IAN_simple), from start MSEs of 1e-7 to 9e-7 (IAN.py: 2e-9).  In bf16 mode the decoder's own rounding moves
# x_hat more than the 5 % move of z does (start MSE 1.1e-6 against 2e-9 in float32), so z is not recovered there: the bf16
# case checks only that the MSE stays at that level (worst 1.16e-6) and does not rise.
RECOVERY = (5e-4, 1.5e-11)
RECOVERY_BF16_MSE = 2.5e-6
RECORD = {}


def _record(key, value):
    RECORD[key] = value
    if os.environ.get("IAN_TEST_RECORD"):
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "fit_latent.json"), "w") as f:
            json.dump(RECORD, f, indent=1, sort_keys=True)


_SYNTH = {}


def synth(g):
    if g not in _SYNTH:
        _SYNTH[g] = MAKE[g](weight_seed(g))
    return _SYNTH[g]


def _margin(g):
    return mw.weights(g, device="cuda")


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


def _gram64(J, r):
    """J (n,100,12288), r (n,12288) float64 -> A, g, e"""
    return np.einsum("kip,kjp->kij", J, J), np.einsum("kip,kp->ki", J, r), np.einsum("kp,kp->k", r, r)


# ---- A. normal equations against float64 ------------------------------------------------------------------------------
SPREAD = np.linspace(0, mw.POOL - 1, 13).astype(int)
_REF = {}


def _ref64(g):
    """float64 A, g, e at the spread pool latents against the pool's images, and the same from J rounded to bf16"""
    if g not in _REF:
        import torch
        from oracle import ian_torch as ot
        dec = mw.DECODER[g]
        Q = {k: t.cuda() for k, t in ot.to_torch(_margin(g), torch.float64).items()}
        p = mw.pool()
        z, x = p["z"][SPREAD], p["x"][SPREAD]
        J, r = [], []
        for k in range(len(SPREAD)):
            zk = torch.from_numpy(z[k].astype(np.float64)).cuda()
            jac = torch.func.jacfwd(lambda zz: dec(Q, zz[None])[0])(zk)            # (3,64,64,100)
            J.append(jac.reshape(-1, 100).T.cpu().numpy())
            r.append((dec(Q, zk[None])[0] - torch.from_numpy(x[k].astype(np.float64)).cuda()).reshape(-1).cpu().numpy())
        J, r = np.stack(J), np.stack(r)
        Jb = mw.bf16_round(J.astype(np.float32)).astype(np.float64)
        _REF[g] = (z, x, _gram64(J, r), _gram64(Jb, r))
    return _REF[g]


@pytest.mark.parametrize("g", GRAPHS)
def test_normal_equations_against_float64(handles, g):
    z, x, ref, slip = _ref64(g)
    floor = [float(_rel(s, rf).min()) for s, rf in zip(slip, ref)]
    rec = {"bf16_J_floor": floor}
    modes = ["tc", "simt"] + (["bf16"] if g == "full" else [])
    for mode in modes:
        m = handles(g, _margin(g))
        if mode == "simt":
            m.set_path("simt")
        if mode == "bf16":
            m.set_precision("bf16")
        got = m.gauss_newton(z, x)
        err = [_rel(a, b) for a, b in zip(got, ref)]
        rec[mode] = [float(e.max()) for e in err]
        _record("A_%s" % g, rec)
        bound = NE_BF16 if mode == "bf16" else NE_BOUND
        for name, e, b in zip("Age", err, bound):
            assert e.max() <= b, (mode, name, e)
    for name, b, f in zip("Ag", NE_BOUND, floor):
        assert b <= f / 3, (name, b, f)


# ---- B. the Gram alone ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_gram_against_float64_gram_of_the_same_bits(handles, g):
    m = handles(g, _margin(g))
    p = mw.pool()
    z, x = p["z"][:3], p["x"][:3]
    J = m.decoder_jacobian(z).reshape(3, 100, -1).astype(np.float64)
    r = (m.sample_at(z).astype(np.float64) - x.astype(np.float64)).reshape(3, -1)
    ref = _gram64(J, r)
    got = m.gauss_newton(z, x)
    err = [float(_rel(a, b).max()) for a, b in zip(got, ref)]
    _record("B_%s" % g, err)
    assert max(err) <= 1e-10, err
    assert np.array_equal(got[0], np.swapaxes(got[0], 1, 2))            # both triangles, the same sums


# ---- C. the solver alone -------------------------------------------------------------------------------------------------
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
    p = mw.pool()
    idx = SPREAD[:6]
    z0 = (p["z"][idx] + 0.05 * np.random.default_rng(11).standard_normal((6, 100))).astype(np.float32)
    x = m.sample_at(p["z"][idx])
    A, gv, e = m.gauss_newton(z0, x)
    z1, loss = m.fit_latent(x, z0, iters=1, return_loss=True)
    assert np.allclose(loss[:, 0], e / 12288, rtol=1e-6, atol=0), (loss[:, 0], e / 12288)
    delta = _lm_step(A, gv)
    want = z0.astype(np.float64) + delta
    took = loss[:, 1] < loss[:, 0]
    rec = {"accepted": took.tolist(), "err_ulps": []}
    for k in range(6):
        if not took[k]:
            assert np.array_equal(z1[k], z0[k]) and loss[k, 1] == loss[k, 0], k
            continue
        tol = np.spacing(np.abs(want[k]).astype(np.float32)).astype(np.float64) + 1e-9 * np.abs(delta[k]).max()
        err = np.abs(z1[k] - want[k])
        rec["err_ulps"].append(float((err / tol).max()))
        _record("C_%s_%s" % (g, mode), rec)
        assert np.all(err <= tol), (k, (err / tol).max())
    assert took.any()
    _record("C_%s_%s" % (g, mode), rec)


# ---- D. Levenberg-Marquardt properties ------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_lm_properties_on_random_targets(handles, g):
    m = handles(g, synth(g))
    n, iters = 8, 10
    rng = np.random.default_rng(500)
    z0 = rng.standard_normal((n, 100)).astype(np.float32)
    x = rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)
    zs = [z0] + [m.fit_latent(x, z0, iters=k) for k in range(1, iters + 1)]
    z, loss = m.fit_latent(x, z0, iters=iters, return_loss=True)
    assert np.array_equal(z, zs[-1])
    step = np.diff(loss.astype(np.float64), axis=1)
    flat = step == 0
    _record("D_%s" % g, {"rejected": int(flat.sum()), "first": loss[:, 0].tolist(), "last": loss[:, -1].tolist()})
    assert np.all(step <= 0), loss
    for k in range(n):
        for i in range(iters):
            if flat[k, i]:
                assert np.array_equal(zs[i + 1][k], zs[i][k]), (k, i)
            else:
                assert not np.array_equal(zs[i + 1][k], zs[i][k]), (k, i)
    assert flat.sum() >= 1
    assert np.all(loss[:, -1] < loss[:, 0])


# ---- E. recovery of a decoded latent ----------------------------------------------------------------------------------------
def _recovery_case(g, n):
    p = mw.pool()
    idx = np.linspace(0, mw.POOL - 1, n).astype(int)
    zs = p["z"][idx]
    u = np.random.default_rng(600 + n).standard_normal((n, 100))
    u *= 0.05 * np.linalg.norm(zs, axis=1, keepdims=True) / np.linalg.norm(u, axis=1, keepdims=True)
    return zs, (zs + u).astype(np.float32)


def _recovery(m, g, zs, z0, key, bf16=False):
    x = m.sample_at(zs)
    z, loss = m.fit_latent(x, z0, iters=10, return_loss=True)
    dz = np.linalg.norm(z.astype(np.float64) - zs, axis=1) / np.linalg.norm(zs.astype(np.float64), axis=1)
    margin = [mw.decoder_margin(g, _margin(g), zs[k:k + 1], device="cuda")[0] for k in range(len(zs))]
    _record(key, {"dz": dz.tolist(), "mse": loss[:, -1].tolist(), "start_mse": loss[:, 0].tolist(), "margin": margin})
    assert min(margin) > 0, margin
    assert np.all(loss[:, -1] <= loss[:, 0])
    if bf16:
        assert loss[:, -1].max() <= RECOVERY_BF16_MSE, loss[:, -1]
    else:
        assert dz.max() <= RECOVERY[0] and loss[:, -1].max() <= RECOVERY[1], (dz, loss[:, -1])


@pytest.mark.parametrize("mode", ["tc", "simt", "bf16"])
@pytest.mark.parametrize("g", GRAPHS)
def test_recovery(handles, g, mode):
    if mode == "bf16" and g != "full":
        pytest.skip("bf16 mode is tested on IAN.py")
    m = handles(g, _margin(g))
    if mode == "simt":
        m.set_path("simt")
    if mode == "bf16":
        m.set_precision("bf16")
    zs, z0 = _recovery_case(g, 8)
    _recovery(m, g, zs, z0, "E_%s_%s" % (g, mode), bf16=mode == "bf16")


# ---- F. bits -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_bits_forms_and_schedules(handles, g):
    import torch
    m = handles(g, _margin(g))
    zs, z0 = _recovery_case(g, 3)
    x = m.sample_at(zs)
    z1, l1 = m.fit_latent(x, z0, iters=3, return_loss=True)
    z2, l2 = m.fit_latent(x, z0, iters=3, return_loss=True)
    assert np.array_equal(z1, z2) and np.array_equal(l1, l2)
    ne = m.gauss_newton(z0, x)
    assert all(np.array_equal(a, b) for a, b in zip(ne, m.gauss_newton(z0, x)))
    # device form
    zd, xd = torch.from_numpy(z0).cuda(), torch.from_numpy(x).cuda()
    Ad = torch.empty(3, 100, 100, dtype=torch.float64, device="cuda")
    gd = torch.empty(3, 100, dtype=torch.float64, device="cuda")
    ed = torch.empty(3, dtype=torch.float64, device="cuda")
    m.gauss_newton_dev(zd.data_ptr(), xd.data_ptr(), 3, Ad.data_ptr(), gd.data_ptr(), ed.data_ptr())
    ld = torch.empty(3, 4, device="cuda")
    m.fit_latent_dev(xd.data_ptr(), 3, zd.data_ptr(), 3, ld.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(Ad.cpu().numpy(), ne[0]) and np.array_equal(gd.cpu().numpy(), ne[1])
    assert np.array_equal(ed.cpu().numpy(), ne[2])
    assert np.array_equal(zd.cpu().numpy(), z1) and np.array_equal(ld.cpu().numpy(), l1)
    zd.copy_(torch.from_numpy(z0))
    m.fit_latent_dev(xd.data_ptr(), 3, zd.data_ptr(), 3)                     # loss left out
    m.gauss_newton_dev(zd.data_ptr(), xd.data_ptr(), 0, 0, 0)                # n = 0
    torch.cuda.synchronize()
    assert np.array_equal(zd.cpu().numpy(), z1)
    # PDL off
    m0 = handles(g, _margin(g), IAN_PDL=0)
    z3, l3 = m0.fit_latent(x, z0, iters=3, return_loss=True)
    assert np.array_equal(z3, z1) and np.array_equal(l3, l1)
    assert all(np.array_equal(a, b) for a, b in zip(ne, m0.gauss_newton(z0, x)))
    # chunked: 20 samples in chunks of 16 and 4
    mc = handles(g, _margin(g), IAN_CHUNK=16)
    zs, z0 = _recovery_case(g, 20)
    _recovery(mc, g, zs, z0, "F_chunk_%s" % g)


# ---- G. errors -------------------------------------------------------------------------------------------------------------
def test_errors(npe, model):
    lib, h = model._lib, model._h
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    z = np.zeros((2, 100), np.float32)
    x = np.zeros((2, 3, 64, 64), np.float32)
    A, g, e = np.full((2, 100, 100), 7.0), np.full((2, 100), 7.0), np.full(2, 7.0)
    loss = np.full((2, 4), 7, np.float32)
    assert lib.ian_decode_gauss_newton_host(h, None, fp(x), 2, dp(A), dp(g), dp(e)) == -1
    assert lib.ian_decode_gauss_newton_host(h, fp(z), None, 2, dp(A), dp(g), dp(e)) == -1
    assert lib.ian_decode_gauss_newton_host(h, fp(z), fp(x), 2, None, dp(g), dp(e)) == -1
    assert lib.ian_decode_gauss_newton_host(h, fp(z), fp(x), 2, dp(A), None, dp(e)) == -1
    assert lib.ian_decode_gauss_newton_host(h, fp(z), fp(x), -1, dp(A), dp(g), dp(e)) == -1
    assert lib.ian_decode_gauss_newton_dev(h, None, None, -1, None, None, None, None) == -1
    assert lib.ian_fit_latent_host(h, None, 2, fp(z), 3, fp(loss)) == -1
    assert lib.ian_fit_latent_host(h, fp(x), 2, None, 3, fp(loss)) == -1
    assert lib.ian_fit_latent_host(h, fp(x), 2, fp(z), -1, fp(loss)) == -1
    assert lib.ian_fit_latent_host(h, fp(x), -1, fp(z), 3, fp(loss)) == -1
    assert lib.ian_fit_latent_dev(h, None, -1, None, 3, None, None) == -1
    assert lib.ian_decode_gauss_newton_host(h, fp(z), fp(x), 0, dp(A), dp(g), dp(e)) == 0 and np.all(A == 7)
    assert lib.ian_fit_latent_host(h, fp(x), 0, fp(z), 3, fp(loss)) == 0 and np.all(loss == 7) and np.all(z == 0)
    assert np.all(np.isfinite(g)) and np.all(e == 7)
    A0, g0, e0 = model.gauss_newton(np.zeros((0, 100), np.float32), np.zeros((0, 3, 64, 64), np.float32))
    assert A0.shape == (0, 100, 100) and g0.shape == (0, 100) and e0.shape == (0,)
    z0, l0 = model.fit_latent(np.zeros((0, 3, 64, 64), np.float32), np.zeros((0, 100), np.float32), return_loss=True)
    assert z0.shape == (0, 100) and l0.shape == (0, 11)
    with pytest.raises(ValueError):
        model.gauss_newton(z, x[:1])
    with pytest.raises(ValueError):
        model.fit_latent(x, z, iters=-1)
    with pytest.raises(TypeError):
        model.fit_latent(x, z.astype(np.float64))
    raw = C.c_void_p()
    assert lib.ian_create(0, 0, C.byref(raw)) == 0
    try:
        assert lib.ian_decode_gauss_newton_host(raw, fp(z), fp(x), 2, dp(A), dp(g), dp(e)) == -3
        assert lib.ian_fit_latent_host(raw, fp(x), 2, fp(z), 3, fp(loss)) == -3
    finally:
        lib.ian_destroy(raw)

"""GPU tests of the IAN's introspection features and the latent fit under its feature-wise loss (include/ian_b200.h
ian_introspect_*, ian_introspect_jvp_*, ian_feature_gauss_newton_*, ian_fit_latent_features_*; API.IAN.introspect,
introspect_jvp, feature_loss, gauss_newton_features, fit_latent_features) on all three graphs, on the tensor-core and SIMT
paths and, on IAN.py, in bf16 mode.

  1. introspect against the float64 restatement (tests/introspect_oracle.py) and introspect_jvp against torch.func.jvp of
     it, on the margin-weight pool's images; feature_loss against the formula; both against the executed reference's
     features and central differences (tests/golden/ref_exec_introspect.npz) on the golden images and weights.
  2. the normal equations against float64 (J and J_i from torch.func.jacfwd of features . decode) at pool latents; the
     float32 bounds are <= a third of the floor that rounding J and J_i to bf16 moves the float64 A and g by.
  3. the Gram alone: J_i's bits rebuilt from the public entries (introspect_jvp of sample_at(z) rows along
     decoder_jacobian(z) at batch 100) and r_i from introspect at the call's batch size: <= 1e-10 relative.
  4. reductions: a = 1, b = 0 gives gauss_newton / fit_latent's bits, history included; b = 0 with a = 2 (the feature
     entries' own pixel-only path) gives twice gauss_newton's bits and fit_latent's decisions at twice its history.
  5. the solver: one step is z0 + delta, delta solved in numpy float64 from the entry's own A and g.
  6. Levenberg-Marquardt properties over 10 steps: the history never rises, a flat entry leaves z bit-unchanged, and the
     reject path runs.
  7. recovery: a pure feature fit (a = 0) from 5 % away recovers decoded certified latents, with the conditioning of the
     feature Gram at z* recorded; on an out-of-range target each fit wins on its own objective.
  8. bits: reruns, device form = host form, IAN_PDL=0, IAN_CHUNK=16, and one sample's inputs never change another's bits.
  9. errors.
Measured values go to fit_features.json when IAN_TEST_RECORD names a directory."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import introspect_oracle as io
import margin_weights as mw
from test_ref_exec_decjvp import MAKE, weight_seed

pytestmark = pytest.mark.gpu
CONFIG = {"simple": "IAN_simple.py", "full": "IAN.py", "v1": "IANv1.py"}
GRAPHS = ["simple", "full", "v1"]
ENV = ("IAN_STREAMK", "IAN_SPLITK", "IAN_GRAPHS", "IAN_PDL", "IAN_FINALIZE8", "IAN_CHUNK", "IAN_PATH")
LAMBDA0, DAMP_FLOOR = 1e-3, 1e-9
# Bounds set from one run on an H100 80GB HBM3 at 700 W (the results are the same bits on every rerun); per-sample relative
# L2 against float64.
# 1. features / tangents / feature_loss, float32 mode: worst 6.4e-6 / 9.5e-6 / 1.1e-6 (tensor cores; the encoder is the same
#    on every graph's margin weights); bf16 mode on IAN.py: 3.5e-3 / 4.4e-3 / 1.6e-3.  Bounds >= 2x over the worst.
FEAT_BOUND, TAN_BOUND, LOSS_BOUND = 1.5e-5, 2e-5, 3e-6
FEAT_BF16, TAN_BF16, LOSS_BF16 = 8e-3, 1e-2, 4e-3
# against the executed reference (synthetic golden weights, two golden images): relative L2 of the channel subset and of the
# probe projections, features / tangents.  Float32 mode: worst 1.25e-5 / 7.5e-6 (features, IAN_simple on the tensor cores)
# and 1.3e-4 / 1.4e-4 (tangents, IAN_simple on the SIMT path: on these weights some rectifier sits near its kink; 1.3e-5 or
# better elsewhere).  bf16 mode on IAN.py: 5.7e-3 / 5.1e-3 and 3.4e-2 / 5.3e-2.  Bounds >= 2x over the worst.
REF_BOUND = {"f": 3e-5, "p": 2e-5, "df": 3e-4, "dp": 3e-4}
REF_BF16 = {"f": 1.2e-2, "p": 1.2e-2, "df": 7e-2, "dp": 0.11}
# 2. A, g, e at a = 0.5, b = 2: worst 4.2e-5 / 3.7e-5 / 9.0e-7 (A: IAN.py, tensor cores; the SIMT path 2.8e-6).  Rounding J
#    and J_i to bf16 moves the float64 A and g by at least 1.37e-4 / 5.7e-4 (IAN.py), so A's bound, a third of that floor,
#    has only 1.1x headroom over the tensor-core worst; g's and e's have >= 2x.  bf16 mode on IAN.py: 1.9e-3 / 1.1e-2 / 7.9e-4.
NE_BOUND = (4.5e-5, 7.5e-5, 2e-6)
NE_BF16 = (4e-3, 2.5e-2, 2e-3)
# 7. a pure feature fit (a = 0, b = 1) from 5 % away, 10 steps: |z - z*| / |z*| worst 1.8e-3 (IAN.py; 2.4e-4 on IANv1.py,
#    1e-4 on IAN_simple) and l_f worst 1.24e-10, the float32 level of the features (IAN.py starts at only 7e-10: its decoder
#    moves the image little when z moves 5 %).
RECOVERY = (4e-3, 2.5e-10)
RECORD = {}


def _record(key, value):
    RECORD[key] = value
    if os.environ.get("IAN_TEST_RECORD"):
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "fit_features.json"), "w") as f:
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
    """make(graph, weights, mode="tc", **env): a handle with exactly `env` among the schedule variables, closed at test end"""
    made = []

    def make(graph, weights, mode="tc", **env):
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
        if mode == "simt":
            m.set_path("simt")
        if mode == "bf16":
            m.set_precision("bf16")
        return m
    try:
        yield make
    finally:
        for m in made:
            m.close()


MODES = [(g, m) for g in GRAPHS for m in ("tc", "simt", "bf16") if m != "bf16" or g == "full"]


def _rel(got, ref):
    n = len(ref)
    d = (np.asarray(got, np.float64) - ref).reshape(n, -1)
    return np.linalg.norm(d, axis=1) / np.linalg.norm(np.asarray(ref, np.float64).reshape(n, -1), axis=1)


def _flat(f):
    """feature list (n, ...) x 4 -> (n, 245760) float64, NCHW layer after layer"""
    n = len(f[0])
    return np.concatenate([np.asarray(a, np.float64).reshape(n, -1) for a in f], axis=1)


# ---- 1. the features and their tangents --------------------------------------------------------------------------------
@pytest.mark.parametrize("g,mode", MODES)
def test_introspect_against_float64(handles, g, mode):
    import torch
    m = handles(g, _margin(g), mode)
    p = mw.pool()
    x = p["x"][:6]
    v = np.random.default_rng(3).standard_normal(x.shape).astype(np.float32)
    Q = io.weights64(_margin(g), "cuda")
    xt = torch.from_numpy(x.astype(np.float64)).cuda()
    vt = torch.from_numpy(v.astype(np.float64)).cuda()
    ref, tref = torch.func.jvp(lambda a: tuple(io.features(Q, a)), (xt,), (vt,))
    ref = [r.cpu().numpy() for r in ref]
    tref = [t.cpu().numpy() for t in tref]
    f = m.introspect(x)
    f2, t = m.introspect_jvp(x, v, return_features=True)
    assert all(a.shape == b.shape for a, b in zip(f, ref))
    assert all(np.array_equal(a, b) for a, b in zip(f, f2))
    ef = [float(_rel(a, b).max()) for a, b in zip(f, ref)]
    et = [float(_rel(a, b).max()) for a, b in zip(t, tref)]
    lf = m.feature_loss(x[::-1].copy(), x)
    lref = io.feature_loss([r[::-1] for r in ref], ref)
    el = float(np.abs(lf / lref - 1).max())
    _record("1_%s_%s" % (g, mode), {"features": ef, "tangents": et, "feature_loss": el})
    fb, tb, lb = (FEAT_BF16, TAN_BF16, LOSS_BF16) if mode == "bf16" else (FEAT_BOUND, TAN_BOUND, LOSS_BOUND)
    assert max(ef) <= fb and max(et) <= tb and el <= lb, (ef, et, el)


@pytest.mark.parametrize("g,mode", MODES)
def test_introspect_against_the_executed_reference(handles, g, mode):
    x, seed, v, probes, stored = io.fixture()[g]
    m = handles(g, MAKE[g](seed), mode)
    f, t = m.introspect_jvp(x, v.astype(np.float32), return_features=True)
    assert all(np.array_equal(a, b) for a, b in zip(f, m.introspect(x)))
    err = io.against_fixture(f, t, probes, stored)
    _record("1_ref_%s_%s" % (g, mode), err)
    bound = REF_BF16 if mode == "bf16" else REF_BOUND
    assert all(err[k] <= bound[k] for k in err), err


# ---- 2. the normal equations against float64 -----------------------------------------------------------------------------
SPREAD = np.linspace(0, mw.POOL - 1, 3).astype(int)
_REF = {}


def _ref64(g):
    if g not in _REF:
        p = mw.pool()
        z, x = p["z"][SPREAD], p["x"][SPREAD]
        parts = io.jacobians64(g, _margin(g), z, x, device="cuda")
        _REF[g] = (z, x, parts)
    return _REF[g]


@pytest.mark.parametrize("g", GRAPHS)
def test_normal_equations_against_float64(handles, g):
    z, x, parts = _ref64(g)
    a, b = 0.5, 2.0
    ref = [np.stack(t) for t in zip(*[io.gram64(J, Jf, r, rf, a, b) for J, Jf, r, rf in parts])]
    bf = lambda J: mw.bf16_round(J.astype(np.float32)).astype(np.float64)
    slip = [np.stack(t) for t in zip(*[io.gram64(bf(J), bf(Jf), r, rf, a, b) for J, Jf, r, rf in parts])]
    floor = [float(_rel(s, rf).min()) for s, rf in zip(slip, ref)]
    rec = {"bf16_J_floor": floor}
    for mode in ["tc", "simt"] + (["bf16"] if g == "full" else []):
        m = handles(g, _margin(g), mode)
        got = m.gauss_newton_features(z, x, a, b)
        err = [_rel(u, w) for u, w in zip(got, ref)]
        rec[mode] = [float(e.max()) for e in err]
        _record("2_%s" % g, rec)
        bound = NE_BF16 if mode == "bf16" else NE_BOUND
        for name, e, bd in zip("Age", err, bound):
            assert e.max() <= bd, (mode, name, e)
    for name, bd, fl in zip("Ag", NE_BOUND, floor):
        assert bd <= fl / 3, (name, bd, fl)


# ---- 3. the Gram alone ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g,mode", MODES)
def test_gram_against_float64_gram_of_the_same_bits(handles, g, mode):
    m = handles(g, _margin(g), mode)
    p = mw.pool()
    z, x = p["z"][:2], p["x"][:2]
    a, b = 0.7, 1.3
    xh = m.sample_at(z)
    r = (xh.astype(np.float64) - x).reshape(2, -1)
    rf = _flat(m.introspect(xh)) - _flat(m.introspect(x))
    Jall = m.decoder_jacobian(z)
    ref = []
    for k in range(2):
        rows = m.sample_at(np.ascontiguousarray(np.repeat(z[k:k + 1], 100, 0)))
        Jf = _flat(m.introspect_jvp(rows, np.ascontiguousarray(Jall[k])))
        ref.append(io.gram64(Jall[k].reshape(100, -1).astype(np.float64), Jf, r[k], rf[k], a, b))
    ref = [np.stack(t) for t in zip(*ref)]
    got = m.gauss_newton_features(z, x, a, b)
    err = [float(_rel(u, w).max()) for u, w in zip(got, ref)]
    _record("3_%s_%s" % (g, mode), err)
    assert max(err) <= 1e-10, err
    assert np.array_equal(got[0], np.swapaxes(got[0], 1, 2))


# ---- 4. reductions -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_pixel_only_is_the_latent_fit(handles, g):
    m = handles(g, _margin(g))
    p = mw.pool()
    z0, x = p["z"][:3], m.sample_at(p["z"][3:6])
    assert all(np.array_equal(u, w) for u, w in zip(m.gauss_newton_features(z0, x, 1.0, 0.0), m.gauss_newton(z0, x)))
    za, la = m.fit_latent_features(x, z0, iters=3, pixel_weight=1.0, feature_weight=0.0, return_loss=True)
    zb, lb = m.fit_latent(x, z0, iters=3, return_loss=True)
    assert np.array_equal(za, zb) and np.array_equal(la, lb)
    # the feature entries' own pixel term (a != 1, b = 0) is the pixel Gram scaled
    A2, g2, e2 = m.gauss_newton_features(z0, x, 2.0, 0.0)
    A1, g1, e1 = m.gauss_newton(z0, x)
    assert np.array_equal(A2, 2 * A1) and np.array_equal(g2, 2 * g1) and np.array_equal(e2, 2 * e1)
    # ... and its fit: 2E has fit_latent's minimiser and decisions; the start's history is exactly twice fit_latent's, and
    # the solve of 2A + lambda 2D against 2g moves z within rounding of fit_latent's step (measured: the same bits, and
    # exactly twice the history, on every graph)
    z2, l2 = m.fit_latent_features(x, z0, iters=6, pixel_weight=2.0, feature_weight=0.0, return_loss=True)
    z1, l1 = m.fit_latent(x, z0, iters=6, return_loss=True)
    assert np.array_equal(l2[:, 0], 2 * l1[:, 0])
    assert np.array_equal(np.diff(l2, axis=1) == 0, np.diff(l1, axis=1) == 0)
    rel = np.abs(l2.astype(np.float64) / (2 * l1.astype(np.float64)) - 1).max()
    dz = float((np.linalg.norm(z2.astype(np.float64) - z1, axis=1) / np.linalg.norm(z1.astype(np.float64) - z0, axis=1)).max())
    _record("4_a2_%s" % g, {"history_rel": float(rel), "dz_rel_to_move": dz})
    assert rel <= 1e-4 and dz <= 1e-3, (rel, dz)


# ---- 5. the solver alone -------------------------------------------------------------------------------------------------
def _lm_step(A, g, lam=LAMBDA0):
    d = np.diagonal(A, axis1=1, axis2=2)
    D = np.maximum(d, DAMP_FLOOR * d.max(axis=1, keepdims=True))
    M = A + lam * np.einsum("ki,ij->kij", D, np.eye(100))
    return np.linalg.solve(M, -g[..., None])[..., 0]


# bf16 mode: the decoder's and encoder's own rounding outweighs the step, which is then rejected (as for fit_latent)
@pytest.mark.parametrize("g,mode", [c for c in MODES if c[1] != "bf16"])
def test_one_step_is_the_float64_solve(handles, g, mode):
    m = handles(g, _margin(g), mode)
    p = mw.pool()
    idx = SPREAD
    z0 = (p["z"][idx] + 0.05 * np.random.default_rng(11).standard_normal((3, 100))).astype(np.float32)
    x = m.sample_at(p["z"][idx])
    a, b = 0.25, 1.0
    A, gv, e = m.gauss_newton_features(z0, x, a, b)
    z1, loss = m.fit_latent_features(x, z0, iters=1, pixel_weight=a, feature_weight=b, return_loss=True)
    assert np.allclose(loss[:, 0], e / 12288, rtol=1e-6, atol=0), (loss[:, 0], e / 12288)
    delta = _lm_step(A, gv)
    want = z0.astype(np.float64) + delta
    took = loss[:, 1] < loss[:, 0]
    rec = {"accepted": took.tolist(), "err_ulps": []}
    for k in range(3):
        if not took[k]:
            assert np.array_equal(z1[k], z0[k]) and loss[k, 1] == loss[k, 0], k
            continue
        tol = np.spacing(np.abs(want[k]).astype(np.float32)).astype(np.float64) + 1e-9 * np.abs(delta[k]).max()
        err = np.abs(z1[k] - want[k])
        rec["err_ulps"].append(float((err / tol).max()))
        assert np.all(err <= tol), (k, (err / tol).max())
    _record("5_%s_%s" % (g, mode), rec)
    assert took.any()


# ---- 6. Levenberg-Marquardt properties ------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_lm_properties_on_random_targets(handles, g):
    m = handles(g, synth(g))
    n, iters = 6, 10
    rng = np.random.default_rng(500)
    z0 = rng.standard_normal((n, 100)).astype(np.float32)
    x = rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)
    fit = lambda k: m.fit_latent_features(x, z0, iters=k, pixel_weight=0.5, feature_weight=1.0, return_loss=True)
    zs = [z0] + [fit(k)[0] for k in range(1, iters + 1)]
    z, loss = fit(iters)
    assert np.array_equal(z, zs[-1])
    step = np.diff(loss.astype(np.float64), axis=1)
    flat = step == 0
    _record("6_%s" % g, {"rejected": int(flat.sum()), "first": loss[:, 0].tolist(), "last": loss[:, -1].tolist()})
    assert np.all(step <= 0), loss
    for k in range(n):
        for i in range(iters):
            if flat[k, i]:
                assert np.array_equal(zs[i + 1][k], zs[i][k]), (k, i)
            else:
                assert not np.array_equal(zs[i + 1][k], zs[i][k]), (k, i)
    assert flat.sum() >= 1
    assert np.all(loss[:, -1] < loss[:, 0])


# ---- 7. recovery ----------------------------------------------------------------------------------------------------------
def _recovery_case(n):
    p = mw.pool()
    idx = np.linspace(0, mw.POOL - 1, n).astype(int)
    zs = p["z"][idx]
    u = np.random.default_rng(600 + n).standard_normal((n, 100))
    u *= 0.05 * np.linalg.norm(zs, axis=1, keepdims=True) / np.linalg.norm(u, axis=1, keepdims=True)
    return zs, (zs + u).astype(np.float32)


def _recovery(m, g, zs, z0, key):
    x = m.sample_at(zs)
    z, loss = m.fit_latent_features(x, z0, iters=10, pixel_weight=0.0, feature_weight=1.0, return_loss=True)
    dz = np.linalg.norm(z.astype(np.float64) - zs, axis=1) / np.linalg.norm(zs.astype(np.float64), axis=1)
    lf = m.feature_loss(m.sample_at(z), x)
    _record(key, {"dz": dz.tolist(), "l_f": lf.tolist(), "start": loss[:, 0].tolist(), "last": loss[:, -1].tolist()})
    assert np.all(loss[:, -1] < loss[:, 0]), loss
    assert dz.max() <= RECOVERY[0] and lf.max() <= RECOVERY[1], (dz, lf)


@pytest.mark.parametrize("g,mode", [c for c in MODES if c[1] != "bf16"])
def test_feature_fit_recovers_the_latent(handles, g, mode):
    m = handles(g, _margin(g), mode)
    zs, z0 = _recovery_case(6)
    x = m.sample_at(zs)
    A = m.gauss_newton_features(zs, x, 0.0, 1.0)[0]
    ev = np.linalg.eigvalsh(A)
    margin = [mw.decoder_margin(g, _margin(g), zs[k:k + 1], device="cuda")[0] for k in range(len(zs))]
    _record("7_cond_%s_%s" % (g, mode), {"cond": (ev[:, -1] / ev[:, 0]).tolist(), "decoder_margin": margin})
    assert min(margin) > 0 and np.all(ev[:, 0] > 0)
    _recovery(m, g, zs, z0, "7_%s_%s" % (g, mode))


@pytest.mark.parametrize("g", GRAPHS)
def test_each_fit_wins_on_its_own_objective(handles, g):
    m = handles(g, _margin(g))
    zs, z0 = _recovery_case(4)
    x = m.sample_at(zs)
    x = np.clip(x + 0.1 * np.random.default_rng(9).standard_normal(x.shape), -1, 1).astype(np.float32)
    zf = m.fit_latent_features(x, z0, iters=10, pixel_weight=0.0, feature_weight=1.0)
    zp = m.fit_latent(x, z0, iters=10)
    xf, xp = m.sample_at(zf), m.sample_at(zp)
    lf = (m.feature_loss(xf, x), m.feature_loss(xp, x))
    mse = [((a.astype(np.float64) - x) ** 2).reshape(4, -1).mean(1) for a in (xf, xp)]
    _record("7_out_of_range_%s" % g, {"l_f": [t.tolist() for t in lf], "mse": [t.tolist() for t in mse]})
    assert np.all(lf[0] < lf[1]) and np.all(mse[1] < mse[0]), (lf, mse)


# ---- 8. bits ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_bits_forms_and_schedules(handles, g):
    import torch
    m = handles(g, _margin(g))
    zs, z0 = _recovery_case(3)
    x = m.sample_at(zs)
    a, b = 0.5, 1.0
    fit = lambda mm: mm.fit_latent_features(x, z0, iters=3, pixel_weight=a, feature_weight=b, return_loss=True)
    z1, l1 = fit(m)
    z2, l2 = fit(m)
    assert np.array_equal(z1, z2) and np.array_equal(l1, l2)
    ne = m.gauss_newton_features(z0, x, a, b)
    assert all(np.array_equal(u, w) for u, w in zip(ne, m.gauss_newton_features(z0, x, a, b)))
    f, t = m.introspect_jvp(x, x[::-1].copy(), return_features=True)
    # device forms
    zd, xd = torch.from_numpy(z0).cuda(), torch.from_numpy(x).cuda()
    vd = torch.from_numpy(x[::-1].copy()).cuda()
    Ad = torch.empty(3, 100, 100, dtype=torch.float64, device="cuda")
    gd = torch.empty(3, 100, dtype=torch.float64, device="cuda")
    ed = torch.empty(3, dtype=torch.float64, device="cuda")
    fd = [torch.empty((3,) + s, device="cuda") for s in io_shapes()]
    td = [torch.empty((3,) + s, device="cuda") for s in io_shapes()]
    m.introspect_dev(xd.data_ptr(), 3, [a_.data_ptr() for a_ in fd])
    fj = [torch.empty((3,) + s, device="cuda") for s in io_shapes()]
    m.introspect_jvp_dev(xd.data_ptr(), vd.data_ptr(), 3, [a_.data_ptr() for a_ in td], [a_.data_ptr() for a_ in fj])
    m.gauss_newton_features_dev(zd.data_ptr(), xd.data_ptr(), 3, Ad.data_ptr(), gd.data_ptr(), ed.data_ptr(), a, b)
    ld = torch.empty(3, 4, device="cuda")
    m.fit_latent_features_dev(xd.data_ptr(), 3, zd.data_ptr(), 3, ld.data_ptr(), a, b)
    torch.cuda.synchronize()
    assert all(np.array_equal(u.cpu().numpy(), w) for u, w in zip(fd, f))
    assert all(np.array_equal(u.cpu().numpy(), w) for u, w in zip(fj, f))
    assert all(np.array_equal(u.cpu().numpy(), w) for u, w in zip(td, t))
    assert np.array_equal(Ad.cpu().numpy(), ne[0]) and np.array_equal(gd.cpu().numpy(), ne[1])
    assert np.array_equal(ed.cpu().numpy(), ne[2])
    assert np.array_equal(zd.cpu().numpy(), z1) and np.array_equal(ld.cpu().numpy(), l1)
    # PDL off
    m0 = handles(g, _margin(g), IAN_PDL=0)
    z3, l3 = fit(m0)
    assert np.array_equal(z3, z1) and np.array_equal(l3, l1)
    assert all(np.array_equal(u, w) for u, w in zip(ne, m0.gauss_newton_features(z0, x, a, b)))
    # chunked: 20 samples in chunks of 16 and 4
    mc = handles(g, _margin(g), IAN_CHUNK=16)
    zs, z0 = _recovery_case(20)
    _recovery(mc, g, zs, z0, "8_chunk_%s" % g)


def io_shapes():
    return [(128, 32, 32), (256, 16, 16), (512, 8, 8), (1024, 4, 4)]


@pytest.mark.parametrize("g", GRAPHS)
def test_samples_stay_apart(handles, g):
    m = handles(g, synth(g))
    rng = np.random.default_rng(77)
    n = 4
    x = rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)
    v = rng.standard_normal((n, 3, 64, 64)).astype(np.float32)
    z0 = rng.standard_normal((n, 100)).astype(np.float32)

    def run(xx, zz):
        out = list(m.introspect(xx)) + list(m.introspect_jvp(xx, v))
        out += list(m.gauss_newton_features(zz, xx, 0.5, 1.0))
        out += list(m.fit_latent_features(xx, zz, iters=2, pixel_weight=0.5, feature_weight=1.0, return_loss=True))
        return out
    base = run(x, z0)
    x1 = x.copy()
    x1[1] = rng.uniform(-1, 1, (3, 64, 64))
    z1 = z0.copy()
    z1[1] = rng.standard_normal(100)
    x2 = x.copy()
    x2[1, 0, 5, 7] = np.nan
    for xx, zz in ((x1, z0), (x, z1), (x2, z0)):
        out = run(xx, zz)
        for u, w in zip(out, base):
            keep = [0, 2, 3]
            assert np.array_equal(u[keep], w[keep])


# ---- 9. errors -------------------------------------------------------------------------------------------------------------
def test_errors(npe, model):
    lib, h = model._lib, model._h
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    z = np.zeros((2, 100), np.float32)
    x = np.zeros((2, 3, 64, 64), np.float32)
    A, g, e = np.full((2, 100, 100), 7.0), np.full((2, 100), 7.0), np.full(2, 7.0)
    loss = np.full((2, 4), 7, np.float32)
    t = [np.zeros((2,) + s, np.float32) for s in io_shapes()]
    for a, b in ((-1.0, 1.0), (1.0, -1.0), (float("nan"), 1.0), (1.0, float("inf")), (0.0, 0.0)):
        assert lib.ian_feature_gauss_newton_host(h, fp(z), fp(x), 2, a, b, dp(A), dp(g), dp(e)) == -1
        assert lib.ian_fit_latent_features_host(h, fp(x), 2, fp(z), 3, a, b, fp(loss)) == -1
    assert lib.ian_feature_gauss_newton_host(h, None, fp(x), 2, 1.0, 1.0, dp(A), dp(g), dp(e)) == -1
    assert lib.ian_feature_gauss_newton_host(h, fp(z), None, 2, 1.0, 1.0, dp(A), dp(g), dp(e)) == -1
    assert lib.ian_feature_gauss_newton_host(h, fp(z), fp(x), 2, 1.0, 1.0, None, dp(g), dp(e)) == -1
    assert lib.ian_feature_gauss_newton_host(h, fp(z), fp(x), 2, 1.0, 1.0, dp(A), None, dp(e)) == -1
    assert lib.ian_feature_gauss_newton_host(h, fp(z), fp(x), -1, 1.0, 1.0, dp(A), dp(g), dp(e)) == -1
    assert lib.ian_fit_latent_features_host(h, None, 2, fp(z), 3, 1.0, 1.0, fp(loss)) == -1
    assert lib.ian_fit_latent_features_host(h, fp(x), 2, None, 3, 1.0, 1.0, fp(loss)) == -1
    assert lib.ian_fit_latent_features_host(h, fp(x), 2, fp(z), -1, 1.0, 1.0, fp(loss)) == -1
    assert lib.ian_fit_latent_features_host(h, fp(x), -1, fp(z), 3, 1.0, 1.0, fp(loss)) == -1
    assert lib.ian_introspect_host(h, None, 2, *[fp(a) for a in t]) == -1
    assert lib.ian_introspect_host(h, fp(x), -1, *[fp(a) for a in t]) == -1
    assert lib.ian_introspect_jvp_host(h, fp(x), None, 2, None, None, None, None, *[fp(a) for a in t]) == -1
    assert lib.ian_introspect_jvp_host(h, fp(x), fp(x), 2, None, None, None, None, fp(t[0]), fp(t[1]), fp(t[2]), None) == -1
    assert lib.ian_feature_gauss_newton_host(h, fp(z), fp(x), 0, 1.0, 1.0, dp(A), dp(g), dp(e)) == 0 and np.all(A == 7)
    assert lib.ian_fit_latent_features_host(h, fp(x), 0, fp(z), 3, 1.0, 1.0, fp(loss)) == 0 and np.all(loss == 7)
    assert lib.ian_introspect_host(h, fp(x), 0, None, None, None, None) == 0
    assert lib.ian_introspect_host(h, fp(x), 2, None, None, None, None) == 0              # every output left out
    f0 = model.introspect(np.zeros((0, 3, 64, 64), np.float32))
    assert [a.shape for a in f0] == [(0,) + s for s in io_shapes()]
    with pytest.raises(ValueError):
        model.fit_latent_features(x, z, pixel_weight=0.0, feature_weight=0.0)
    with pytest.raises(ValueError):
        model.gauss_newton_features(z, x, feature_weight=-1.0)
    raw = C.c_void_p()
    assert lib.ian_create(0, 0, C.byref(raw)) == 0
    try:
        assert lib.ian_feature_gauss_newton_host(raw, fp(z), fp(x), 2, 1.0, 1.0, dp(A), dp(g), dp(e)) == -3
        assert lib.ian_fit_latent_features_host(raw, fp(x), 2, fp(z), 3, 1.0, 1.0, fp(loss)) == -3
        assert lib.ian_introspect_host(raw, fp(x), 2, *[fp(a) for a in t]) == -3
    finally:
        lib.ian_destroy(raw)

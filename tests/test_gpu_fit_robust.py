"""GPU tests of the robust latent fit (include/ian_b200.h ian_robust_gauss_newton_* / ian_fit_latent_robust_*,
API.IAN.gauss_newton_robust / fit_latent_robust) on all three graphs, on the tensor-core and SIMT paths and, on IAN.py, in
bf16 mode.  tests/fit_robust_oracle.py holds the float64 references, the scale rule and the corruption.

  A. reductions, bit for bit: Huber with scale +inf is ian_map_gauss_newton_*'s A and g and ian_fit_latent_map_*'s u, z and
     loss, for w None, random w with beta > 0 and a 0/1 mask with NaN in the hole; e is the fit's init reduction and within
     1e-14 of map's e.  Both kinds' A, g and e are a float64 Gram of J_u's own bits with omega from the entry's own x_hat.
  B. A, g, e against float64 (jacfwd of decode . flow) at certified targets, bounds set as in test_gpu_fit_map.py.
  C. the scale: automatic is the numpy rule on sample(u0) bit for bit (no weighted pixel and a single one included); a
     passed scale comes back unchanged; one step is u0 + the numpy float64 LM step of the entry's own A and g.
  D. outliers: x = the float64 decode of F(u*) corrupted by a 16 x 16 noise block and 2 % salt and pepper, no mask, start 5 %
     away, the scale the automatic rule gives at the float64 start, one problem for both paths.  After CONVERGE_ITERS steps
     the float64 gradient has fallen by 1e3 and u is the float64 IRLS-LM loop's converged minimiser; Cauchy lands at least
     10x closer to u* than fit_latent_map, Huber closer; the outlier map separates corrupted from clean pixels.  A Cauchy fit
     with a NaN hole at weight 0 fills the hole.
  E. bits: reruns, device form = host form, IAN_PDL=0, IAN_CHUNK=16, and samples kept apart.
  F. errors.
Measured values go to fit_robust.json when IAN_TEST_RECORD names a directory."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import fit_map_oracle as fo
import fit_robust_oracle as ro
import margin_weights as mw
from test_gpu_fit_map import CONFIG, GRAPHS, _holed, _margin, _rel, _start, _targets, handles  # noqa: F401
from test_gpu_fit_map import _lm_step

pytestmark = pytest.mark.gpu
BETA = 1e-2
INF = float("inf")
# Bounds set from one run on an H100 80GB HBM3 at 700 W (the results are the same bits on every rerun).
# B. per-sample relative error of (A, g, e) against float64, both kinds, every weight case.  Float32 mode, both paths: worst
# 3.9e-5 / 3.7e-5 / 3.5e-7 (A and g: IAN.py and IAN_simple on tensor cores).  Rounding J_u to bf16 moves the float64 A and g
# by at least 1.55e-4 / 1.03e-3 (IAN.py), so the A bound sits at a third of that floor with 1.3x headroom; the g and e
# bounds have 2x.  bf16 mode on IAN.py: worst 4.5e-3 / 1.0e-2 / 4.6e-5, at the floor (bounds 2x over).
NE_BOUND = (5e-5, 7.5e-5, 7e-7)
NE_BF16 = (9e-3, 2e-2, 1e-4)
# D. The float64 loop, started at the GPU's fit, runs until its gradient has fallen by REF_GTOL (it takes 1-2 steps): its
# u is the converged minimiser.  The fit runs CONVERGE_ITERS steps, past its plateau: it converges to the minimiser of its
# own objective, whose x_hat and J_u are the float32 decoder's, so the float64 |grad E| at its u stops at a floor set by the
# decoder's float32 error, not by the step count: the float32 loss after PLATEAU_CHECK steps is already the final one.
# GRAD_DROP (float64 |grad E| at u over its value at u0) and FIDELITY (|u - u_ref| / |u*|) per graph, both kinds and paths,
# 2x over the measured worst: IAN_simple 2.4e-3 / 1.3e-4, IAN.py 5.0e-3 / 1.3e-3, IANv1.py 1.8e-4 / 4.2e-5 (Huber the worse
# kind on each).  The issue's 1e-3 gradient drop holds on IANv1.py only; the floor is the float32 decoder's.
# OUTLIER_MAP: the least fraction of corrupted elements with rho' < 0.1 and of clean ones with rho' > 0.9; measured worst
# 0.945 and 1.0 (Huber), 0.984 and 1.0 (Cauchy).
CONVERGE_ITERS, PLATEAU_CHECK = 50, 20
REF_GTOL, REF_MAX = 1e-5, 40
GRAD_DROP = {"simple": 5e-3, "full": 1e-2, "v1": 4e-4}
FIDELITY = {"simple": 3e-4, "full": 3e-3, "v1": 1e-4}
OUTLIER_MAP = {"huber": (0.9, 0.99), "cauchy": (0.95, 0.99)}
# the hole test after ITERS steps (Cauchy): |u - u*| / |u*| and the hole's max |x_hat - x*|; measured worst 1.27e-2 (IAN.py)
# and 5.9e-5
ITERS = 20
HOLE = (2.5e-2, 1.2e-4)
RECORD = {}


def _record(key, value):
    RECORD[key] = value
    if os.environ.get("IAN_TEST_RECORD"):
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "fit_robust.json"), "w") as f:
            json.dump(RECORD, f, indent=1, sort_keys=True)


def _cases(x):
    """(name, w, images, beta): no weights, random weights in [0, 1] with the prior, a 0/1 mask with NaN in its hole"""
    n = len(x)
    w = np.random.default_rng(40).uniform(0, 1, x.shape).astype(np.float32)
    sq = fo.masks(n)["square"]
    return [("none", None, x, 0.0), ("random", w, x, BETA), ("mask", sq, _holed(x, sq), 0.0)]


def _modes(g):
    return ["tc", "simt"] + (["bf16"] if g == "full" else [])


def _set(m, mode):
    if mode == "simt":
        m.set_path("simt")
    if mode == "bf16":
        m.set_precision("bf16")
    return m


# ---- A. reductions ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_huber_at_infinite_scale_is_the_map_fit(handles, g):
    us = _targets(g)
    u0 = _start(us, 1)
    for mode in _modes(g):
        m = _set(handles(g, _margin(g)), mode)
        x = m.sample(us)
        for name, w, xx, beta in _cases(x):
            A, gv, e = m.gauss_newton_map(u0, xx, w, beta)
            Ar, gr, er, sr = m.gauss_newton_robust(u0, xx, "huber", INF, w, beta)
            assert np.array_equal(Ar, A) and np.array_equal(gr, gv), (mode, name)
            assert np.all(sr == INF) and np.all(np.abs(er - e) <= 1e-14 * np.abs(e)), (mode, name, er, e)
            u1, z1, l1 = m.fit_latent_map(xx, w, beta, u0, iters=3, return_loss=True)
            u2, z2, s2, l2 = m.fit_latent_robust(xx, "huber", INF, w, beta, u0, iters=3, return_loss=True)
            assert np.array_equal(u2, u1) and np.array_equal(z2, z1) and np.array_equal(l2, l1), (mode, name)
            assert np.array_equal(l2[:, 0], (er / 12288).astype(np.float32)), (mode, name)


@pytest.mark.parametrize("g", GRAPHS)
def test_gram_of_the_same_bits(handles, g):
    m = handles(g, _margin(g))
    us = _targets(g)
    u0 = _start(us, 2)
    x, _ = ro.corrupt(m.sample(us), 11)
    J = []
    for k in range(len(u0)):
        zr, tan = m.flow_jvp(np.repeat(u0[k:k + 1], 100, 0), np.eye(100, dtype=np.float32), return_z=True)
        J.append(m.decode_jvp(zr, tan).reshape(100, -1))
    J = np.stack(J).astype(np.float64)
    xh = m.sample(u0).astype(np.float64)
    err = {}
    for kind in ro.KINDS:
        for name, w, xx, beta in _cases(x):
            A, gv, e, s = m.gauss_newton_robust(u0, xx, kind, None, w, beta)
            assert np.array_equal(A, np.swapaxes(A, 1, 2))
            ref = ro.gram64(J, (xh - xx).reshape(len(u0), -1), w, u0, beta, kind, s)
            err["%s_%s" % (kind, name)] = [float(_rel(a, b).max()) for a, b in zip((A, gv, e), ref)]
    _record("A_%s" % g, err)
    assert max(max(v) for v in err.values()) <= 1e-10, err


# ---- B. against float64 ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_normal_equations_against_float64(handles, g):
    u = _targets(g, 6)
    x, _ = ro.corrupt(mw.pool()["x"][np.linspace(0, mw.POOL - 1, 6).astype(int)], 12)
    J, xh = fo.jacobians64(g, _margin(g), u, np.zeros_like(x), device="cuda")
    Jb = mw.bf16_round(J.astype(np.float32)).astype(np.float64)
    rec, worst, floor = {}, [], [1.0, 1.0]
    for kind in ro.KINDS:
        for name, w, xx, beta in _cases(x):
            r = xh - xx.reshape(len(u), -1).astype(np.float64)
            dl = np.full(len(u), 0.2)
            ref = ro.gram64(J, r, w, u, beta, kind, dl)
            if beta == 0:
                slip = ro.gram64(Jb, r, w, u, beta, kind, dl)
                floor = [min(f, float(_rel(a, b).min())) for f, a, b in zip(floor, slip[:2], ref[:2])]
            for mode in _modes(g):
                m = _set(handles(g, _margin(g)), mode)
                err = [float(_rel(a, b).max()) for a, b in zip(m.gauss_newton_robust(u, xx, kind, dl, w, beta)[:3], ref)]
                rec["%s_%s_%s" % (kind, name, mode)] = err
                worst.append((kind, name, mode, err, NE_BF16 if mode == "bf16" else NE_BOUND))
    rec["bf16_J_floor"] = floor
    _record("B_%s" % g, rec)
    for kind, name, mode, err, bound in worst:
        assert all(e <= b for e, b in zip(err, bound)), (kind, name, mode, err, bound)
    for nm, b, f in zip("Ag", NE_BOUND, floor):
        assert b <= f / 3, (nm, b, f)


# ---- C. scale and solver ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_scale_rule_and_one_step(handles, g):
    m = handles(g, _margin(g))
    us = _targets(g, 6)
    u0 = _start(us, 4)
    x, _ = ro.corrupt(m.sample(us), 13)
    xh = m.sample(u0)
    w = np.random.default_rng(42).uniform(0, 1, x.shape).astype(np.float32)
    w[1] = 0                                                  # no weighted pixel
    w[2] = 0
    w[2, 0, 5, 6] = 0.5                                       # a single one
    w[3, :, 20:44, 20:44] = 0
    rec = {}
    for kind in ro.KINDS:
        for ww in (None, w):
            _, _, _, s = m.gauss_newton_robust(u0, x, kind, None, ww, BETA)
            assert np.array_equal(s, ro.scale_np(kind, xh, x, ww)), (kind, s, ro.scale_np(kind, xh, x, ww))
            u1, z1, s1, loss = m.fit_latent_robust(x, kind, None, ww, BETA, u0, iters=1, return_loss=True)
            assert np.array_equal(s1, s)
        passed = np.linspace(0.05, 0.3, 6)
        assert np.array_equal(m.gauss_newton_robust(u0, x, kind, passed, w)[3], passed)
        assert np.array_equal(m.fit_latent_robust(x, kind, 0.125, w, iters=0, u0=u0)[2], np.full(6, 0.125))
        # one step from the entry's own A and g
        A, gv, e, s = m.gauss_newton_robust(u0, x, kind, None, None, BETA)
        u1, z1, s1, loss = m.fit_latent_robust(x, kind, None, None, BETA, u0, iters=1, return_loss=True)
        assert np.array_equal(loss[:, 0], (e / 12288).astype(np.float32))
        assert np.array_equal(z1, m.Z_IAF_fn(u1))
        delta = _lm_step(A, gv)
        want = u0.astype(np.float64) + delta
        took = loss[:, 1] < loss[:, 0]
        ulps = []
        for k in range(len(u0)):
            if not took[k]:
                assert np.array_equal(u1[k], u0[k]) and loss[k, 1] == loss[k, 0], k
                continue
            tol = 0.5 * np.spacing(np.abs(want[k]).astype(np.float32)).astype(np.float64) + 1e-9 * np.abs(delta[k]).max()
            err = np.abs(u1[k] - want[k])
            ulps.append(float((err / tol).max()))
            assert np.all(err <= tol), (kind, k, (err / tol).max())
        rec[kind] = {"accepted": took.tolist(), "err_ulps": ulps, "scale": s.tolist()}
        assert took.any()
    _record("C_%s" % g, rec)


# ---- D. outliers ----------------------------------------------------------------------------------------------------------------
_PROBLEMS = {}


def _problem(g):
    """per graph, one problem for both paths: u*, the start u0, x = the float64 decode of F(u*) as float32 with the corruption,
    the corruption map, and per kind the scale (the automatic rule at the float64 decode of F(u0)) and |grad E(u0)| there"""
    if g not in _PROBLEMS:
        P = _margin(g)
        us = _targets(g)
        u0 = _start(us, 5)
        _, xs = fo.jacobians64(g, P, us, np.zeros((3, 3, 64, 64)), device="cuda")
        x, bad = ro.corrupt(xs.reshape(3, 3, 64, 64).astype(np.float32), 21)
        J0, r0 = fo.jacobians64(g, P, u0, x, device="cuda")
        xh0 = (r0 + x.reshape(3, -1).astype(np.float64)).astype(np.float32)
        per = {}
        for kind in ro.KINDS:
            dl = ro.scale_np(kind, xh0, x)
            per[kind] = (dl, np.linalg.norm(ro.gram64(J0, r0, None, u0, 0.0, kind, dl)[1], axis=1))
        _PROBLEMS[g] = (us, u0, x, bad, per)
    return _PROBLEMS[g]


_REFS = {}


def _minimiser(g, kind, x, dl, g0, u_start):
    """the float64 loop's converged minimiser: from u_start (the first path's fit) until |grad E| <= REF_GTOL |grad E(u0)|"""
    if (g, kind) not in _REFS:
        _REFS[(g, kind)] = ro.irls_lm64(g, _margin(g), x, None, 0.0, kind, dl, u_start, REF_MAX, device="cuda",
                                        gstop=REF_GTOL * g0)
    return _REFS[(g, kind)]


@pytest.mark.parametrize("mode", ["tc", "simt"])
@pytest.mark.parametrize("g", GRAPHS)
def test_outliers_lose_their_pull(handles, g, mode):
    m = handles(g, _margin(g))
    m.set_path(mode)
    us, u0, x, bad, per = _problem(g)
    n = len(us)
    nu = np.linalg.norm(us.astype(np.float64), axis=1)
    zm = m.fit_latent_map(x, None, 0.0, u0, iters=CONVERGE_ITERS)[0]
    du_l2 = np.linalg.norm(zm.astype(np.float64) - us, axis=1) / nu
    rec = {"du_l2": du_l2.tolist()}
    key = "D_%s_%s" % (g, mode)
    for kind in ro.KINDS:
        dl, g0 = per[kind]
        u, z, s, loss, ow = m.fit_latent_robust(x, kind, dl, None, 0.0, u0, iters=CONVERGE_ITERS, return_loss=True,
                                                return_outliers=True)
        assert np.all(np.diff(loss.astype(np.float64), axis=1) <= 0), loss
        assert np.array_equal(z, m.Z_IAF_fn(u)) and np.array_equal(s, dl)
        J, r = fo.jacobians64(g, _margin(g), u, x, device="cuda")
        drop = np.linalg.norm(ro.gram64(J, r, None, u, 0.0, kind, dl)[1], axis=1) / g0
        uref, hist, gref = _minimiser(g, kind, x, dl, g0, u)
        du = np.linalg.norm(u.astype(np.float64) - us, axis=1) / nu
        low = [float((ow[k][bad[k]] < 0.1).mean()) for k in range(n)]
        high = [float((ow[k][~bad[k]] > 0.9).mean()) for k in range(n)]
        rec[kind] = {"du": du.tolist(), "ratio_l2": (du_l2 / du).tolist(), "outlier_low_on_bad": low,
                     "outlier_high_on_clean": high, "scale": dl.tolist(), "grad_drop": drop.tolist(),
                     "fidelity": (np.linalg.norm(u - uref, axis=1) / nu).tolist(), "ref_steps": hist.shape[1] - 1,
                     "ref_grad_drop": (gref / g0).tolist(), "steps_accepted": int((np.diff(loss, axis=1) < 0).sum(1).min())}
        rec[kind]["loss_at_%d" % PLATEAU_CHECK] = loss[:, PLATEAU_CHECK].tolist()
        rec[kind]["loss_last"] = loss[:, -1].tolist()
        _record(key, rec)
    for kind in ro.KINDS:
        r = rec[kind]
        assert max(r["ref_grad_drop"]) <= REF_GTOL, r            # the reference has converged
        assert r["loss_at_%d" % PLATEAU_CHECK] == r["loss_last"], r    # and the fit has stopped on its own objective
        assert max(r["grad_drop"]) <= GRAD_DROP[g] and max(r["fidelity"]) <= FIDELITY[g], (kind, r)
        assert min(r["outlier_high_on_clean"]) >= OUTLIER_MAP[kind][1], (kind, r)
        assert min(r["outlier_low_on_bad"]) >= OUTLIER_MAP[kind][0], (kind, r)
        if kind == "cauchy":
            assert np.all(du_l2 >= 10 * np.array(r["du"])), (kind, r["ratio_l2"])
        else:
            assert np.all(np.array(r["du"]) < du_l2), (kind, r["du"], du_l2)


@pytest.mark.parametrize("g", GRAPHS)
def test_robust_fit_fills_a_hole(handles, g):
    m = handles(g, _margin(g))
    us = _targets(g)
    u0 = _start(us, 5)
    x, _ = ro.corrupt(m.sample(us), 22)
    w = fo.masks(3)["square"]
    u, z, s, loss = m.fit_latent_robust(_holed(x, w), "cauchy", None, w, 0.0, u0, iters=ITERS, return_loss=True)
    assert np.all(np.isfinite(u)) and np.all(np.diff(loss.astype(np.float64), axis=1) <= 0)
    du = np.linalg.norm(u.astype(np.float64) - us, axis=1) / np.linalg.norm(us.astype(np.float64), axis=1)
    miss = np.abs(m.sample(u) - m.sample(us))[w == 0].reshape(3, -1).max(1)
    _record("D_hole_%s" % g, {"du": du.tolist(), "hole_miss": miss.tolist()})
    assert du.max() <= HOLE[0] and miss.max() <= HOLE[1], (du, miss)


# ---- E. bits ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_bits_forms_and_schedules(handles, g):
    import torch
    m = handles(g, _margin(g))
    us = _targets(g)
    u0 = _start(us, 6)
    w = np.random.default_rng(41).uniform(0, 1, (3, 3, 64, 64)).astype(np.float32) * fo.masks(3)["square"]
    x = _holed(ro.corrupt(m.sample(us), 23)[0], w)
    for kind in ro.KINDS:
        r1 = m.fit_latent_robust(x, kind, None, w, BETA, u0, iters=3, return_loss=True, return_outliers=True)
        r2 = m.fit_latent_robust(x, kind, None, w, BETA, u0, iters=3, return_loss=True, return_outliers=True)
        assert all(np.array_equal(a, b) for a, b in zip(r1, r2))
        ne = m.gauss_newton_robust(u0, x, kind, None, w, BETA)
        assert all(np.array_equal(a, b) for a, b in zip(ne, m.gauss_newton_robust(u0, x, kind, None, w, BETA)))
        # device form
        ud, xd, wd = (torch.from_numpy(a).cuda() for a in (u0, x, w))
        Ad = torch.empty(3, 100, 100, dtype=torch.float64, device="cuda")
        gd = torch.empty(3, 100, dtype=torch.float64, device="cuda")
        ed = torch.empty(3, dtype=torch.float64, device="cuda")
        sd = torch.empty(3, dtype=torch.float64, device="cuda")
        m.gauss_newton_robust_dev(ud.data_ptr(), xd.data_ptr(), wd.data_ptr(), BETA, kind, 0, 3, Ad.data_ptr(), gd.data_ptr(),
                                  ed.data_ptr(), sd.data_ptr())
        zd = torch.empty(3, 100, device="cuda")
        ld = torch.empty(3, 4, device="cuda")
        s2 = torch.empty(3, dtype=torch.float64, device="cuda")
        od = torch.empty(3, 3, 64, 64, device="cuda")
        m.fit_latent_robust_dev(xd.data_ptr(), wd.data_ptr(), BETA, kind, 0, 3, ud.data_ptr(), 3, zd.data_ptr(), ld.data_ptr(),
                                s2.data_ptr(), od.data_ptr())
        torch.cuda.synchronize()
        for a, b in zip((Ad, gd, ed, sd), ne):
            assert np.array_equal(a.cpu().numpy(), b)
        for a, b in zip((ud, zd, s2, ld, od), r1):
            assert np.array_equal(a.cpu().numpy(), b)
        # a passed scale on the device, scale_out a copy of it
        ud.copy_(torch.from_numpy(u0))
        sc = torch.from_numpy(r1[2]).cuda()
        s3 = torch.empty(3, dtype=torch.float64, device="cuda")
        m.fit_latent_robust_dev(xd.data_ptr(), wd.data_ptr(), BETA, kind, sc.data_ptr(), 3, ud.data_ptr(), 3, 0, 0,
                                s3.data_ptr())
        torch.cuda.synchronize()
        assert np.array_equal(ud.cpu().numpy(), r1[0]) and np.array_equal(s3.cpu().numpy(), r1[2])
        # PDL off
        m0 = handles(g, _margin(g), IAN_PDL=0)
        r3 = m0.fit_latent_robust(x, kind, None, w, BETA, u0, iters=3, return_loss=True, return_outliers=True)
        assert all(np.array_equal(a, b) for a, b in zip(r3, r1))
    # chunked: 20 samples in chunks of 16 and 4, against the unchunked handle's bits
    mc = handles(g, _margin(g), IAN_CHUNK=16)
    us = _targets(g, 20)
    u0 = _start(us, 7)
    x = ro.corrupt(m.sample(us), 24)[0]
    a = mc.fit_latent_robust(x, "cauchy", None, None, 0.0, u0, iters=3, return_loss=True, return_outliers=True)
    b = m.fit_latent_robust(x, "cauchy", None, None, 0.0, u0, iters=3, return_loss=True, return_outliers=True)
    du = np.abs(a[0].astype(np.float64) - b[0]).max() / np.abs(b[0]).max()
    _record("E_chunk_%s" % g, float(du))
    assert du <= 1e-3 and np.all(np.diff(a[3].astype(np.float64), axis=1) <= 0), du


@pytest.mark.parametrize("g", GRAPHS)
def test_samples_stay_apart(handles, g):
    m = handles(g, _margin(g))
    us = _targets(g, 4)
    u0 = _start(us, 8)
    w = fo.masks(4)["left"]
    x = _holed(ro.corrupt(m.sample(us), 25)[0], w)
    for kind in ro.KINDS:
        s = np.array([0.1, 0.2, 0.3, 0.4])
        for scale in (None, s):
            r1 = m.fit_latent_robust(x, kind, scale, w, BETA, u0, iters=3, return_loss=True, return_outliers=True)
            x2, w2, u2 = x.copy(), w.copy(), u0.copy()
            x2[1] = np.float32(0.25)
            x2[2, :, 10, 40] = np.nan                         # NaN at a weighted pixel: sample 2 alone goes bad
            w2[3] = np.float32(0.5)
            u2[3] += np.float32(0.1)
            s2 = None if scale is None else s * np.array([1, 1, 1, 2])
            r2 = m.fit_latent_robust(x2, kind, s2, w2, BETA, u2, iters=3, return_loss=True, return_outliers=True)
            assert all(np.array_equal(a[0], b[0]) for a, b in zip(r1, r2)), (kind, scale)
            assert not np.array_equal(r2[0][1], r1[0][1]) and not np.array_equal(r2[0][3], r1[0][3])


# ---- F. errors ---------------------------------------------------------------------------------------------------------------------
def test_errors(npe, model):
    lib, h = model._lib, model._h
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    u = np.zeros((2, 100), np.float32)
    x = np.zeros((2, 3, 64, 64), np.float32)
    w = np.ones((2, 3, 64, 64), np.float32)
    A, g, e, s = np.full((2, 100, 100), 7.0), np.full((2, 100), 7.0), np.full(2, 7.0), np.full(2, 7.0)
    z = np.full((2, 100), 7, np.float32)
    loss = np.full((2, 4), 7, np.float32)
    ow = np.full((2, 3, 64, 64), 7, np.float32)
    sc = np.array([0.1, 0.2])
    gn = lambda kind, scale, *a: lib.ian_robust_gauss_newton_host(h, *a[:4], kind, scale, *a[4:])
    fit = lambda kind, scale, *a: lib.ian_fit_latent_robust_host(h, *a[:3], kind, scale, *a[3:])
    ok_gn = (fp(u), fp(x), fp(w), 0.0, 2, dp(A), dp(g), dp(e), dp(s))
    ok_fit = (fp(x), fp(w), 0.0, 2, fp(u), fp(z), 3, fp(loss), dp(s), fp(ow))
    for kind in (0, 3, -1):
        assert gn(kind, dp(sc), *ok_gn) == -1 and fit(kind, dp(sc), *ok_fit) == -1
    for kind, bad in ((1, 0.0), (1, -1.0), (1, float("nan")), (1, -INF), (2, INF), (2, 0.0), (2, float("nan"))):
        sb = np.array([0.1, bad])
        assert gn(kind, dp(sb), *ok_gn) == -1 and fit(kind, dp(sb), *ok_fit) == -1, (kind, bad)
    assert gn(1, None, None, fp(x), fp(w), 0.0, 2, dp(A), dp(g), dp(e), dp(s)) == -1
    assert gn(1, None, fp(u), None, fp(w), 0.0, 2, dp(A), dp(g), dp(e), dp(s)) == -1
    assert gn(1, None, fp(u), fp(x), fp(w), 0.0, 2, None, dp(g), dp(e), dp(s)) == -1
    assert gn(1, None, fp(u), fp(x), fp(w), 0.0, 2, dp(A), None, dp(e), dp(s)) == -1
    assert gn(1, None, fp(u), fp(x), fp(w), 0.0, -1, dp(A), dp(g), dp(e), dp(s)) == -1
    for bad in (-1.0, float("nan"), INF):
        assert gn(1, None, fp(u), fp(x), fp(w), bad, 2, dp(A), dp(g), dp(e), dp(s)) == -1
        assert fit(2, None, fp(x), fp(w), bad, 2, fp(u), fp(z), 3, fp(loss), dp(s), fp(ow)) == -1
        wb = w.copy()
        wb[1, 2, 3, 4] = bad
        assert gn(1, None, fp(u), fp(x), fp(wb), 0.0, 2, dp(A), dp(g), dp(e), dp(s)) == -1
        assert fit(2, None, fp(x), fp(wb), 0.0, 2, fp(u), fp(z), 3, fp(loss), dp(s), fp(ow)) == -1
    assert fit(1, None, None, fp(w), 0.0, 2, fp(u), fp(z), 3, fp(loss), dp(s), fp(ow)) == -1
    assert fit(1, None, fp(x), fp(w), 0.0, 2, None, fp(z), 3, fp(loss), dp(s), fp(ow)) == -1
    assert fit(1, None, fp(x), fp(w), 0.0, 2, fp(u), fp(z), -1, fp(loss), dp(s), fp(ow)) == -1
    assert fit(1, None, fp(x), fp(w), 0.0, -1, fp(u), fp(z), 3, fp(loss), dp(s), fp(ow)) == -1
    assert lib.ian_robust_gauss_newton_dev(h, None, None, None, 0.0, 1, None, -1, None, None, None, None, None) == -1
    assert lib.ian_fit_latent_robust_dev(h, None, None, 0.0, 5, None, 2, None, None, 3, None, None, None, None) == -1
    assert gn(1, None, fp(u), fp(x), fp(w), 0.0, 0, dp(A), dp(g), dp(e), dp(s)) == 0 and np.all(A == 7) and np.all(s == 7)
    assert fit(2, None, fp(x), fp(w), 0.0, 0, fp(u), fp(z), 3, fp(loss), dp(s), fp(ow)) == 0
    assert np.all(loss == 7) and np.all(z == 7) and np.all(ow == 7) and np.all(u == 0) and np.all(e == 7)
    out = model.gauss_newton_robust(np.zeros((0, 100), np.float32), np.zeros((0, 3, 64, 64), np.float32))
    assert [a.shape for a in out] == [(0, 100, 100), (0, 100), (0,), (0,)]
    out = model.fit_latent_robust(np.zeros((0, 3, 64, 64), np.float32), u0=np.zeros((0, 100), np.float32), return_loss=True,
                                  return_outliers=True)
    assert [a.shape for a in out] == [(0, 100), (0, 100), (0,), (0, 11), (0, 3, 64, 64)]
    with pytest.raises(ValueError):
        model.gauss_newton_robust(u, x, "l1")
    with pytest.raises(ValueError):
        model.gauss_newton_robust_dev(0, 0, 0, 0.0, "l1", 0, 2, 0, 0)
    with pytest.raises(ValueError):
        model.fit_latent_robust_dev(0, 0, 0.0, "tukey", 0, 2, 0, 3)
    with pytest.raises(ValueError):
        model.gauss_newton_robust(u, x, "cauchy", INF)
    with pytest.raises(ValueError):
        model.fit_latent_robust(x, "huber", [0.1, -0.1], u0=u)
    with pytest.raises(ValueError):
        model.fit_latent_robust(x, prior=-1.0, u0=u)
    with pytest.raises(ValueError):
        model.fit_latent_robust(x, u0=u, iters=-1)
    raw = C.c_void_p()
    assert lib.ian_create(0, 0, C.byref(raw)) == 0
    try:
        assert lib.ian_robust_gauss_newton_host(raw, fp(u), fp(x), fp(w), 0.0, 1, None, 2, dp(A), dp(g), dp(e), dp(s)) == -3
        assert lib.ian_fit_latent_robust_host(raw, fp(x), fp(w), 0.0, 1, None, 2, fp(u), fp(z), 3, fp(loss), dp(s),
                                              fp(ow)) == -3
    finally:
        lib.ian_destroy(raw)

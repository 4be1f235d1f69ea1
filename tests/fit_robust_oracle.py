"""float64 references of the robust latent fit (include/ian_b200.h ian_robust_gauss_newton_* / ian_fit_latent_robust_*),
built on tests/fit_map_oracle.py.  With u the fit-space latent, r = decode(F(u)) - x, weights w >= 0, s = r^2 and a
per-sample scale delta:
    E(u) = sum_{w_p > 0} w_p rho(r_p^2) + beta |u|^2,   omega = w rho'(r^2),
    A = J_u^T Omega J_u + beta I,   g = J_u^T Omega r + beta u (= grad E / 2),   e = E(u).
  rho, drho:      Huber and Cauchy rho(s) and rho'(s), float64;
  energy_np:      E from the independent numpy oracle, for central differences;
  gram64:         A, g, e from J_u and r;
  scale_np:       the automatic scale from x_hat and x, the library's rule bit for bit;
  corrupt:        a seeded corruption of target images: a 16 x 16 block of uniform noise and 2 % salt and pepper;
  irls_lm64:      the fit in float64 (IRLS with the library's Levenberg-Marquardt constants and rule), J_u by jacfwd."""
import numpy as np

import fit_map_oracle as fo

KINDS = ("huber", "cauchy")
C_SCALE = {"huber": 1.345 * 1.4826, "cauchy": 2.3849 * 1.4826}   # one double each, as in edge.h
FLOOR = 1.0 / 255.0
LAMBDA0, LAMBDA_MIN, LAMBDA_MAX, FACTOR, DAMP_FLOOR = 1e-3, 1e-7, 1e10, 10.0, 1e-9


def rho(kind, s, delta):
    s = np.asarray(s, np.float64)
    d = np.asarray(delta, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        if kind == "huber":
            return np.where(s <= d * d, s, 2 * d * np.sqrt(s) - d * d)
        return d * d * np.log1p(s / (d * d))


def drho(kind, s, delta):
    s = np.asarray(s, np.float64)
    d = np.asarray(delta, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        if kind == "huber":
            return np.where(s <= d * d, 1.0, d / np.sqrt(s))
        return 1.0 / (1.0 + s / (d * d))


def _flat(a, n):
    return np.asarray(a, np.float64).reshape(n, -1)


def energy_np(g, P, u, x, w, beta, kind, delta):
    """E(u) per sample, float64; u (n,100), x and w (n,3,64,64) (w None: all ones), delta (n,)"""
    u = np.asarray(u, np.float64)
    n = len(u)
    r = _flat(fo.DECODE_NP[g](P, fo.flow_np(g, P, u)), n) - _flat(x, n)
    w = np.ones_like(r) if w is None else _flat(w, n)
    term = np.where(w != 0, w * rho(kind, np.where(w != 0, r, 0.0) ** 2, np.asarray(delta, np.float64)[:, None]), 0.0)
    return term.sum(1) + beta * (u * u).sum(1)


def gram64(J, r, w, u, beta, kind, delta):
    """A, g, e of J (n,100,12288), r (n,12288), w (n,...) or None, u (n,100), beta, delta (n,)"""
    n = len(J)
    w = np.ones_like(r) if w is None else _flat(w, n)
    r = np.where(w != 0, r, 0.0)
    dl = np.asarray(delta, np.float64)[:, None]
    om = np.where(w != 0, w * drho(kind, r * r, dl), 0.0)
    u = np.asarray(u, np.float64)
    A = np.einsum("kip,kp,kjp->kij", J, om, J) + beta * np.eye(100)
    gv = np.einsum("kip,kp->ki", J, om * r) + beta * u
    e = np.where(w != 0, w * rho(kind, r * r, dl), 0.0).sum(1) + beta * (u * u).sum(1)
    return A, gv, e


def scale_np(kind, xh, x, w=None):
    """delta (n,) float64: max(m c, 1/255), m the lower median of float32 |xh - x| over w != 0 (1/255 with none)"""
    n = len(xh)
    a = np.abs(np.asarray(xh, np.float32).reshape(n, -1) - np.asarray(x, np.float32).reshape(n, -1))
    out = np.empty(n)
    for k in range(n):
        v = a[k] if w is None else a[k][np.asarray(w).reshape(n, -1)[k] != 0]
        if v.size == 0:
            out[k] = FLOOR
            continue
        m = np.partition(v, (v.size - 1) // 2)[(v.size - 1) // 2]
        out[k] = max(float(m) * C_SCALE[kind], FLOOR)
    return out


def corrupt(x, seed):
    """x (n,3,64,64) with, per sample, a 16 x 16 block of uniform noise in [-1, 1] at a random place and 2 % of the pixels
    (all three channels) set to -1 or +1; returns (float32 images, bool (n,3,64,64) map of the corrupted elements)"""
    rng = np.random.default_rng(seed)
    y = np.array(x, np.float32, copy=True)
    bad = np.zeros(y.shape, bool)
    for k in range(len(y)):
        i, j = rng.integers(0, 64 - 16 + 1, 2)
        y[k, :, i:i + 16, j:j + 16] = rng.uniform(-1, 1, (3, 16, 16))
        bad[k, :, i:i + 16, j:j + 16] = True
        salt = rng.random((64, 64)) < 0.02
        y[k][:, salt] = rng.choice(np.array([-1.0, 1.0], np.float32), int(salt.sum()))
        bad[k][:, salt] = True
    return y, bad


def lm_step(A, g, lam):
    d = np.diagonal(A, axis1=1, axis2=2)
    D = np.maximum(d, DAMP_FLOOR * d.max(axis=1, keepdims=True))
    M = A + lam[:, None, None] * np.einsum("ki,ij->kij", D, np.eye(100))
    return np.linalg.solve(M, -g[..., None])[..., 0]


def irls_lm64(g, P, x, w, beta, kind, delta, u0, iters, device="cpu", gstop=None):
    """the fit in float64 from u0 at the fixed scale delta: per step A, g from J_u by jacfwd at u, the damped solve, and
    acceptance when the true E falls.  At most `iters` steps; with gstop (n,) it stops once every |g| <= gstop.  Returns
    (u (n,100) float64, E history (n, steps+1), |g| (n,) at the returned u)"""
    u = np.array(u0, np.float64)
    n = len(u)
    lam = np.full(n, LAMBDA0)
    E = lambda uu: energy_np(g, P, uu, x, w, beta, kind, delta)
    e = E(u)
    hist = [e.copy()]
    for it in range(iters + 1):
        J, r = fo.jacobians64(g, P, u, x, device=device)
        A, gv, _ = gram64(J, r, w, u, beta, kind, delta)
        gn = np.linalg.norm(gv, axis=1)
        if it == iters or (gstop is not None and np.all(gn <= gstop)):
            break
        ut = u + lm_step(A, gv, lam)
        et = E(ut)
        take = et < e
        u[take], e[take] = ut[take], et[take]
        lam = np.where(take, np.maximum(lam / FACTOR, LAMBDA_MIN), np.minimum(lam * FACTOR, LAMBDA_MAX))
        hist.append(e.copy())
    return u, np.stack(hist, 1), gn

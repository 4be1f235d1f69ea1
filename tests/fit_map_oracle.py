"""float64 references of the masked latent fit under the prior (include/ian_b200.h ian_map_gauss_newton_* /
ian_fit_latent_map_*).  With u the fit-space latent (l_Z on IAN_simple, l_Z_IAF on IAN.py / IANv1.py), F the MADE/IAF flow
(the identity on IAN_simple), r = decode(F(u)) - x and per-pixel weights w >= 0:
    E(u) = sum_{w_p != 0} w_p r_p^2 + beta |u|^2,   J_u = d decode(F(u)) / d u,
    A = J_u^T W J_u + beta I,   g = J_u^T W r + beta u,   e = E(u).
Pixels with w_p == 0 are left out, so x may be NaN there.
  jacobians64: J_u and r by torch.func.jacfwd of oracle/ian_torch.py's decode . flow (float64, any device);
  gram64:      A, g, e from J_u and r;
  energy_np:   E from the independent numpy oracle (oracle/ian_numpy.py, oracle/ian_full_numpy.py), for central differences;
  targets:     fit-space latents u* with F(u*) = the margin-weight pool's latents (Newton on the float64 flow), so the decoder
               is certified at F(u*) on tests/margin_weights.py's weights;
  masks:       the two inpainting holes, a 24 x 24 square and the left half, as 0/1 weights."""
import numpy as np

from oracle import ian_full_numpy as fn
from oracle import ian_numpy as on

DECODE_NP = {"simple": on.simple_decode, "full": fn.full_decode, "v1": fn.v1_decode}


def flow_np(g, P, u):
    return u if g == "simple" else fn.full_latent(P, u, fn.made_masks(fn.made_ordering()))


def energy_np(g, P, u, x, w, beta):
    """E(u) per sample, float64; u (n,100), x and w (n,3,64,64)"""
    u = np.asarray(u, np.float64)
    n = len(u)
    r = (DECODE_NP[g](P, flow_np(g, P, u)) - np.asarray(x, np.float64)).reshape(n, -1)
    w = np.asarray(w, np.float64).reshape(n, -1)
    r = np.where(w != 0, r, 0.0)
    return (w * r * r).sum(1) + beta * (u * u).sum(1)


def _torch_parts(g, P, device):
    import torch
    from oracle import ian_torch as ot
    Q = {k: t.to(device) for k, t in ot.to_torch(P, torch.float64).items()}
    masks = [torch.from_numpy(np.asarray(m, np.float64)).to(device) for m in fn.made_masks(fn.made_ordering())]
    dec = {"simple": ot.decode, "full": ot.full_decode, "v1": ot.v1_decode}[g]
    flow = (lambda u: u) if g == "simple" else (lambda u: ot.full_latent(Q, u, masks))
    return Q, dec, flow


def jacobians64(g, P, u, x, device="cpu"):
    """J_u (n,100,12288) -- row i is d x_hat / d u_i -- and r (n,12288), float64 numpy"""
    import torch
    Q, dec, flow = _torch_parts(g, P, device)
    J, r = [], []
    for k in range(len(u)):
        uk = torch.from_numpy(np.asarray(u[k], np.float64)).to(device)
        f = lambda v: dec(Q, flow(v[None]))[0]
        J.append(torch.func.jacfwd(f)(uk).reshape(-1, 100).T.cpu().numpy())
        r.append((f(uk).cpu().numpy() - np.asarray(x[k], np.float64)).reshape(-1))
    return np.stack(J), np.stack(r)


def gram64(J, r, w, u, beta):
    """A, g, e of J (n,100,12288), r (n,12288), w (n,...) or None, u (n,100), beta"""
    n = len(J)
    w = np.ones_like(r) if w is None else np.asarray(w, np.float64).reshape(n, -1)
    r = np.where(w != 0, r, 0.0)
    u = np.asarray(u, np.float64)
    A = np.einsum("kip,kp,kjp->kij", J, w, J) + beta * np.eye(100)
    gv = np.einsum("kip,kp->ki", J, w * r) + beta * u
    e = (w * r * r).sum(1) + beta * (u * u).sum(1)
    return A, gv, e


def targets(g, P, z, iters=30):
    """u (n,100) float32 with F(u) = z on weights P (float64 Newton from u = z; IAN_simple: u = z) and the float64
    max |F(u) - z| of the float32 u"""
    z = np.asarray(z, np.float64)
    if g == "simple":
        return z.astype(np.float32), 0.0
    import torch
    _, _, flow = _torch_parts(g, P, "cpu")
    u = torch.from_numpy(z.copy())
    zt = torch.from_numpy(z)
    for _ in range(iters):
        res = flow(u) - zt
        Jf = torch.func.vmap(torch.func.jacfwd(lambda v: flow(v[None])[0]))(u)          # (n,100,100)
        u = u - torch.linalg.solve(Jf, res[..., None])[..., 0]
    u32 = u.numpy().astype(np.float32)
    return u32, float(np.abs(flow(torch.from_numpy(u32.astype(np.float64))).numpy() - z).max())


def masks(n):
    """{"square": a 24 x 24 hole at rows / columns 20..43, "left": the left half} as (n,3,64,64) float32 0/1 weights"""
    sq = np.ones((n, 3, 64, 64), np.float32)
    sq[:, :, 20:44, 20:44] = 0
    left = np.ones((n, 3, 64, 64), np.float32)
    left[:, :, :, :32] = 0
    return {"square": sq, "left": left}


def recovery_targets(g, P, n=3):
    """the inpainting tests' targets: u* = targets() of n latents spread over the margin-weight pool, and the residual"""
    import margin_weights as mw
    return targets(g, P, mw.pool()["z"][np.linspace(0, mw.POOL - 1, n).astype(int)])

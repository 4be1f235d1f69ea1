"""The prior-space derivatives' float64 oracle -- torch forward-mode autograd on oracle/ian_torch.py's full_latent (the
MADE/IAF flow, Z_IAF_fn) and full_encode_mu_ls (mu = Zfn) -- against the EXECUTED reference: every central difference of
the reference's own compiled Zfn and Z_IAF_fn (sample_IAN.py:91-94) in tests/golden/ref_exec_flowjvp.npz
(tests/golden/make_golden_flowjvp.py; IAN.py and IANv1.py, two golden images each, the flow at Zfn(x) and at an N(0,1) prior
draw) equals the oracle's Jacobian-vector product.  The GPU tests (tests/test_gpu_flow_grad.py) hold ian_flow_*_vjp/jvp and
ian_encode_pre_*_vjp/jvp to this oracle; their reverse-mode twins here are torch autograd of the same functions."""
import os

import numpy as np
import pytest

from oracle import ian_full_numpy as fn
from oracle import ian_numpy as on

from test_ref_exec_encjvp import MAKE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRAPHS = ["full", "v1"]


def fixture():
    """{graph: dict(x, seed, vx, z_prior, vz, z_zfn, jv_zfn, jv_flow_zfn, jv_flow_prior)}: the stored central differences and
    the images / directions / points they were taken at"""
    f = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_exec_flowjvp.npz")))
    rng = np.random.RandomState(int(f["seed"]))
    n = int(f["n_img"])
    draws = {g: (rng.standard_normal((n, 3, 64, 64)), rng.standard_normal((n, 100)), rng.standard_normal((n, 100)))
             for g in GRAPHS}
    out = {}
    for g in GRAPHS:
        gold = np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % g))
        x = on.to_tanh(gold["images"][:n].astype(np.float64)).astype(np.float32)   # as the generator stages them
        vx, zp, vz = draws[g]
        out[g] = {"x": x, "seed": int(gold["weight_seed"]), "vx": vx, "z_prior": zp, "vz": vz, "z_zfn": f["z_zfn_" + g]}
        for k in ("zfn", "flow_zfn", "flow_prior"):
            out[g]["jv_" + k] = f["jv_%s_%s" % (k, g)]
    return out


def _setup(P, device):
    import torch
    from oracle import ian_torch as ot
    Q = {k: t.to(device) for k, t in ot.to_torch(P, torch.float64).items()}
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64)).to(device)
    masks = [t(m) for m in fn.made_masks(fn.made_ordering())]
    return ot, Q, t, masks


def _zfn(ot, g, Q):
    return (lambda x: ot.encode_mu_ls(Q, x)[0]) if g == "simple" else (lambda x: ot.full_encode_mu_ls(Q, x)[0])


def _jvp(f, a, v):
    import torch
    import torch.autograd.forward_ad as fwAD
    with torch.no_grad(), fwAD.dual_level():
        return fwAD.unpack_dual(f(fwAD.make_dual(a, v))).tangent.cpu().numpy()


def _vjp(f, a, u):
    import torch
    a = a.clone().requires_grad_(True)
    (g,) = torch.autograd.grad((f(a) * u).sum(), a)
    return g.cpu().numpy()


def flow_jvp64(P, z_iaf, v, device="cpu"):
    """float64 (d l_Z / d l_Z_IAF) . v of the MADE/IAF flow: P float32 numpy weights, z_iaf, v (n,100) -> (n,100)"""
    ot, Q, t, masks = _setup(P, device)
    return _jvp(lambda z: ot.full_latent(Q, z, masks), t(z_iaf), t(v))


def flow_vjp64(P, z_iaf, u, device="cpu"):
    """float64 (d l_Z / d l_Z_IAF)^T . u"""
    ot, Q, t, masks = _setup(P, device)
    return _vjp(lambda z: ot.full_latent(Q, z, masks), t(z_iaf), t(u))


def pre_jvp64(g, P, x, v, device="cpu"):
    """float64 (d mu / d x) . v of graph g's encoder (Zfn: l_Z_IAF = mu; encode itself on IAN_simple)"""
    ot, Q, t, _ = _setup(P, device)
    return _jvp(_zfn(ot, g, Q), t(x), t(v))


def pre_vjp64(g, P, x, u, device="cpu"):
    """float64 (d mu / d x)^T . u -> (n,3,64,64)"""
    ot, Q, t, _ = _setup(P, device)
    return _vjp(_zfn(ot, g, Q), t(x), t(u))


def _close(got, ref, tol):
    for k in range(len(ref)):
        err = np.abs(got[k] - ref[k]).max()
        assert err <= tol * np.abs(ref[k]).max(), (k, err, np.abs(ref[k]).max())


@pytest.mark.parametrize("g", GRAPHS)
def test_oracle_matches_executed_reference(g):
    f = fixture()[g]
    P = MAKE[g](f["seed"])
    _close(pre_jvp64(g, P, f["x"].astype(np.float64), f["vx"]), f["jv_zfn"], 1e-7)
    _close(flow_jvp64(P, f["z_zfn"], f["vz"]), f["jv_flow_zfn"], 1e-7)
    _close(flow_jvp64(P, f["z_prior"], f["vz"]), f["jv_flow_prior"], 1e-7)


@pytest.mark.parametrize("g", GRAPHS)
def test_stored_zfn_is_the_oracles(g):
    """the stored l_Z_IAF = mu(x) of the executed reference is the oracle's, so the flow is pinned at the right point"""
    import torch
    f = fixture()[g]
    P = MAKE[g](f["seed"])
    ot, Q, t, _ = _setup(P, "cpu")
    with torch.no_grad():
        mu = ot.full_encode_mu_ls(Q, t(f["x"]))[0].numpy()
    _close(mu, f["z_zfn"], 1e-9)

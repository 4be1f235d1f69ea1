"""The encoder JVP's float64 oracle -- torch forward-mode autograd on the restatements of oracle/ian_torch.py (encode /
full_encode, the MADE/IAF flow included) -- against the EXECUTED reference: every central difference
(Z(x + h v) - Z(x - h v)) / 2h of the reference's own Z_hat (and, with eps, of Z_IAF_fn of mu + exp(logsigma) eps) in
tests/golden/ref_exec_encjvp.npz (tests/golden/make_golden_encjvp.py; two golden images per graph, without and with eps)
equals the oracle's (d z / d x) . v, and so do central differences of the numpy oracle (oracle/ian_numpy.py,
oracle/ian_full_numpy.py).  <dz, oracle J v> also reproduces the directional derivatives the encoder VJP is pinned to
(tests/golden/ref_exec_encvjp.npz).  The GPU tests (tests/test_gpu_encode_jvp.py) hold ian_encode_jvp_* to this oracle."""
import os

import numpy as np
import pytest

from oracle import ian_full_numpy as fn
from oracle import ian_numpy as on
from oracle import weights as ow

from test_ref_exec_encvjp import fixture as vjp_fixture

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAKE = {"simple": ow.make_simple_weights, "full": ow.make_full_weights, "v1": ow.make_v1_weights}
GRAPHS = ["simple", "full", "v1"]


def fixture():
    """{graph: (x, weight seed, v, eps, jv)}: the stored central differences [without eps, with eps][image][100] and the
    images / directions / eps they were taken at"""
    f = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_exec_encjvp.npz")))
    rng = np.random.RandomState(int(f["seed"]))
    n = int(f["n_img"])
    draws = {g: (rng.standard_normal((n, 3, 64, 64)), rng.standard_normal((n, 100)), rng.standard_normal((n, 100)))
             for g in GRAPHS}
    out = {}
    for g in GRAPHS:
        gold = np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % g))
        x = on.to_tanh(gold["images"][:n].astype(np.float64)).astype(np.float32)   # as the generator stages them
        v, _, eps = draws[g]
        out[g] = (x, int(gold["weight_seed"]), v, eps, f["jv_" + g])
    return out


def jvp64(g, P, x, v, eps=None, device="cpu"):
    """float64 (d z / d x) . v by torch forward-mode autograd on the oracle encoder of graph g, z = mu (+ exp(logsigma)
    eps), through the MADE/IAF flow on IAN.py / IANv1.py; P: float32 numpy weights, x, v (n,3,64,64), eps (n,100) or
    None -> (n,100) float64 numpy"""
    import torch
    import torch.autograd.forward_ad as fwAD
    from oracle import ian_torch as ot
    Q = {k: t.to(device) for k, t in ot.to_torch(P, torch.float64).items()}
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64)).to(device)
    e = None if eps is None else t(eps)
    with torch.no_grad(), fwAD.dual_level():
        xd = fwAD.make_dual(t(x), t(v))
        if g == "simple":
            out = ot.encode(Q, xd, eps is None, e)
        else:
            masks = [t(m) for m in fn.made_masks(fn.made_ordering())]
            out = ot.full_encode(Q, xd, masks, eps is None, e)
        return fwAD.unpack_dual(out).tangent.cpu().numpy()


def numpy_encode(g, P, x, eps=None):
    if g == "simple":
        return on.simple_encode(P, x, eps is None, eps)
    return fn.full_encode(P, x, fn.made_masks(fn.made_ordering()), eps is None, eps)


@pytest.mark.parametrize("g", GRAPHS)
def test_oracle_jvp_matches_executed_reference(g):
    x, seed, v, eps, jv = fixture()[g]
    P = MAKE[g](seed)
    for j, e in enumerate((None, eps)):
        got = jvp64(g, P, x.astype(np.float64), v, e)
        for k in range(len(x)):
            err = np.abs(got[k] - jv[j, k]).max()
            assert err <= 1e-7 * np.abs(jv[j, k]).max(), (g, j, k, err)


@pytest.mark.parametrize("g", GRAPHS)
def test_oracle_jvp_matches_numpy_central_differences(g):
    x, seed, v, eps, _ = fixture()[g]
    P = MAKE[g](seed)
    h = 1e-7
    x = x.astype(np.float64)
    for e in (None, eps):
        fd = (numpy_encode(g, P, x + h * v, e) - numpy_encode(g, P, x - h * v, e)) / (2 * h)
        got = jvp64(g, P, x, v, e)
        for k in range(len(x)):
            err = np.abs(got[k] - fd[k]).max()
            assert err <= 1e-6 * np.abs(fd[k]).max(), (g, k, err)


@pytest.mark.parametrize("g", GRAPHS)
def test_oracle_jvp_reproduces_encoder_vjp_fixture(g):
    """<dz, J v> of the oracle equals every dz . (Z(x + h v) - Z(x - h v)) / 2h stored for the encoder VJP"""
    x, seed, (v, dz, eps), dd = vjp_fixture()[g]
    P = MAKE[g](seed)
    for j, e in enumerate((None, eps)):
        jv = jvp64(g, P, x.astype(np.float64), v, e)
        for k in range(len(x)):
            got = float((dz[k] * jv[k]).sum())
            assert abs(got - dd[j, k]) <= 1e-7 * abs(dd[j, k]), (g, j, k, got, dd[j, k])

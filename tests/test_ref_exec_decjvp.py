"""The decoder JVP's float64 oracle -- torch forward-mode autograd on the restatements of oracle/ian_torch.py -- against the
EXECUTED reference: every central difference (X(z + h v) - X(z - h v)) / 2h of the reference's own X_hat in
tests/golden/ref_exec_decjvp.npz (tests/golden/make_golden_decjvp.py; two (z, v) pairs per graph) equals the oracle's
(d x_hat / d z) . v to 1e-7 of its largest pixel, and so do central differences of the numpy oracle
(oracle/ian_numpy.py, oracle/ian_full_numpy.py).  The GPU tests (tests/test_gpu_decode_jvp.py) hold ian_decode_jvp_* to
both."""
import os

import numpy as np
import pytest

from oracle import ian_full_numpy as fn
from oracle import ian_numpy as on
from oracle import weights as ow

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAKE = {"simple": ow.make_simple_weights, "full": ow.make_full_weights, "v1": ow.make_v1_weights}


def weight_seed(g):
    return int(np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % g))["weight_seed"])


def fixture():
    """{graph: (weight seed, z, v, dx)}: the stored central differences and the (z, v) pairs they were taken at"""
    f = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_exec_decjvp.npz")))
    rng = np.random.RandomState(int(f["seed"]))
    n = int(f["n_pairs"])
    draws = {g: (rng.standard_normal((n, 100)), rng.standard_normal((n, 100))) for g in ("simple", "full", "v1")}
    return {g: (weight_seed(g),) + draws[g] + (f["dx_" + g],) for g in ("simple", "full", "v1")}


def jvp64(g, P, z, v, device="cpu"):
    """float64 (d x_hat / d z) . v by torch forward-mode autograd on the oracle decoder of graph g; P: float32 numpy
    weights, z, v (n,100) -> (n,3,64,64) float64 numpy"""
    import torch
    import torch.autograd.forward_ad as fwAD
    from oracle import ian_torch as ot
    dec = {"simple": ot.decode, "full": ot.full_decode, "v1": ot.v1_decode}[g]
    Q = {k: t.to(device) for k, t in ot.to_torch(P, torch.float64).items()}
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64)).to(device)
    with torch.no_grad(), fwAD.dual_level():
        out = dec(Q, fwAD.make_dual(t(z), t(v)))
        return fwAD.unpack_dual(out).tangent.cpu().numpy()


def numpy_decode(g, P, z):
    return {"simple": on.simple_decode, "full": fn.full_decode, "v1": fn.v1_decode}[g](P, z)


@pytest.mark.parametrize("g", ["simple", "full", "v1"])
def test_oracle_jvp_matches_executed_reference(g):
    seed, z, v, dx = fixture()[g]
    got = jvp64(g, MAKE[g](seed), z, v)
    for k in range(len(z)):
        assert np.abs(got[k] - dx[k]).max() <= 1e-7 * np.abs(dx[k]).max(), (g, k, np.abs(got[k] - dx[k]).max())


@pytest.mark.parametrize("g", ["simple", "full", "v1"])
def test_oracle_jvp_matches_numpy_central_differences(g):
    seed, z, v, _ = fixture()[g]
    P = MAKE[g](seed)
    h = 1e-7                  # the generator's step: at 1e-6 a rectifier of IAN.py's first pair crosses its kink
    fd = (numpy_decode(g, P, z + h * v) - numpy_decode(g, P, z - h * v)) / (2 * h)
    got = jvp64(g, P, z, v)
    for k in range(len(z)):
        assert np.abs(got[k] - fd[k]).max() <= 1e-6 * np.abs(fd[k]).max(), (g, k, np.abs(got[k] - fd[k]).max())

"""torch autograd of the float64 oracle's prior-space functions (oracle/ian_torch.py: full_latent = Z_IAF_fn, the mu of
full_encode_mu_ls / encode_mu_ls = Zfn), in reverse and forward mode, against numpy central differences of the independent
numpy oracle (oracle/ian_full_numpy.py, oracle/ian_numpy.py).  These are the references tests/test_gpu_flow_grad.py holds the
library's ian_flow_vjp/jvp_* and ian_encode_pre_vjp/jvp_* to."""
import numpy as np
import pytest

from oracle import ian_full_numpy as fn
from oracle import ian_numpy as on

from test_ref_exec_encjvp import MAKE
from test_ref_exec_flowjvp import flow_jvp64, flow_vjp64, pre_jvp64, pre_vjp64

H = 1e-7
SEEDS = {"simple": 11, "full": 12, "v1": 13}


def _np_flow(P, z):
    return fn.full_latent(P, z, fn.made_masks(fn.made_ordering()))


def _np_zfn(g, P, x):
    if g == "simple":
        return on.simple_encode(P, x, True, None)
    return fn.full_encode_mu_ls(P, x)[0]


def _draw(g, n=3):
    rng = np.random.default_rng(SEEDS[g])
    x = np.tanh(rng.standard_normal((n, 3, 64, 64)))
    return x, rng.standard_normal((n, 3, 64, 64)), rng.standard_normal((n, 100)), rng.standard_normal((n, 100)), \
        rng.standard_normal((n, 100))


def _check(got, fd, tol):
    for k in range(len(fd)):
        err = np.abs(got[k] - fd[k]).max()
        assert err <= tol * np.abs(fd[k]).max(), (k, err)


@pytest.mark.parametrize("g", ["full", "v1"])
def test_flow_grad_matches_numpy_central_differences(g):
    P = MAKE[g](1000 + SEEDS[g])
    x, _, z, u, v = _draw(g)
    for zi in (z, _np_zfn(g, P, x)):
        fd = (_np_flow(P, zi + H * v) - _np_flow(P, zi - H * v)) / (2 * H)
        _check(flow_jvp64(P, zi, v), fd, 1e-6)
        # reverse mode: <u, fd> = <J^T u, v>
        lhs = (u * fd).sum(1)
        rhs = (flow_vjp64(P, zi, u) * v).sum(1)
        assert np.all(np.abs(lhs - rhs) <= 1e-6 * np.abs(u * fd).sum(1)), (lhs, rhs)


@pytest.mark.parametrize("g", ["simple", "full", "v1"])
def test_zfn_grad_matches_numpy_central_differences(g):
    P = MAKE[g](1000 + SEEDS[g])
    x, vx, _, u, _ = _draw(g, 2)
    fd = (_np_zfn(g, P, x + H * vx) - _np_zfn(g, P, x - H * vx)) / (2 * H)
    _check(pre_jvp64(g, P, x, vx), fd, 1e-6)
    lhs = (u * fd).sum(1)
    rhs = (pre_vjp64(g, P, x, u) * vx).reshape(len(x), -1).sum(1)
    assert np.all(np.abs(lhs - rhs) <= 1e-6 * np.abs(u * fd).sum(1)), (lhs, rhs)

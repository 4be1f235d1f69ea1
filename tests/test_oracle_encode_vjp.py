"""CPU tests of the encoder vector-Jacobian product's oracle (tests/encode_vjp_oracle.py), dx = (d Z_hat / d X)^T dz (the
reverse mode of reference API.py:50 for any cotangent dz; include/ian_b200.h ian_encode_vjp_*):
  * the float64 numpy reverse mode and float64 torch autograd of oracle/ian_torch.py's encode / full_encode agree to 1e-10
    relative on all three graphs (IANv1's encoder and flow are IAN.py's), with and without eps;
  * conv5x5_s2_bwd_data is the adjoint of conv5x5_s2: <conv(x), y> = <x, conv^T(y)>;
  * one central-difference directional derivative per graph agrees to 1e-7 relative."""
import os

import numpy as np
import pytest
import torch

from oracle import ian_full_numpy as fn
from oracle import ian_numpy as on
from oracle import ian_torch as ot
from oracle import weights as ow

import encode_vjp_oracle as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _seed(name):
    return int(np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % name))["weight_seed"])


GRAPHS = {"simple": ow.make_simple_weights, "full": ow.make_full_weights, "v1": ow.make_v1_weights}


@pytest.fixture(scope="module")
def params():
    out = {}
    for name, make in GRAPHS.items():
        P = make(_seed(name))
        out[name] = (P, ot.to_torch(P, torch.float64))
    return out


def _masks(name):
    return fn.made_masks(fn.made_ordering()) if name != "simple" else None


def numpy_vjp(name, P, x, dz, eps):
    if name == "simple":
        return eo.simple_encode_vjp(P, x, dz, eps)
    return (eo.full_encode_vjp if name == "full" else eo.v1_encode_vjp)(P, x, _masks(name), dz, eps)


def numpy_encode(name, P, x, eps):
    if name == "simple":
        return on.simple_encode(P, x, eps is None, eps)
    return fn.full_encode(P, x, _masks(name), eps is None, eps)


def torch_vjp(name, P64, x, dz, eps):
    xt = torch.from_numpy(np.asarray(x, np.float64)).requires_grad_(True)
    e = None if eps is None else torch.from_numpy(np.asarray(eps, np.float64))
    if name == "simple":
        z = ot.encode(P64, xt, e is None, e)
    else:
        masks = [torch.from_numpy(np.asarray(m, np.float64)) for m in _masks(name)]
        z = ot.full_encode(P64, xt, masks, e is None, e)
    (g,) = torch.autograd.grad(z, xt, grad_outputs=torch.from_numpy(np.asarray(dz, np.float64)))
    return g.numpy()


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize("name", ["simple", "full", "v1"])
@pytest.mark.parametrize("with_eps", [False, True])
def test_numpy_and_torch_encoder_vjp_agree(params, name, with_eps):
    P, P64 = params[name]
    rng = np.random.default_rng(1 + with_eps)
    x = np.tanh(rng.standard_normal((2, 3, 64, 64)))
    dz = rng.standard_normal((2, 100))
    eps = rng.standard_normal((2, 100)) if with_eps else None
    a = numpy_vjp(name, P, x, dz, eps)
    b = torch_vjp(name, P64, x, dz, eps)
    assert a.shape == (2, 3, 64, 64)
    assert _rel(a, b) <= 1e-10


def test_conv_bwd_data_is_the_adjoint():
    rng = np.random.default_rng(3)
    for c, o, hw in ((3, 8, 64), (16, 8, 8)):
        x = rng.standard_normal((2, c, hw, hw))
        W = rng.standard_normal((o, c, 5, 5))
        y = rng.standard_normal((2, o, hw // 2, hw // 2))
        lhs = float((on.conv5x5_s2(x, W) * y).sum())
        rhs = float((x * eo.conv5x5_s2_bwd_data(y, W, hw)).sum())
        assert abs(lhs - rhs) <= 1e-10 * abs(lhs)


@pytest.mark.parametrize("name", ["simple", "full", "v1"])
def test_encoder_vjp_matches_central_differences(params, name):
    P, _ = params[name]
    rng = np.random.default_rng(7)
    x = np.tanh(rng.standard_normal((1, 3, 64, 64)))
    dz = rng.standard_normal((1, 100))
    v = rng.standard_normal((1, 3, 64, 64))
    eps = rng.standard_normal((1, 100)) if name != "simple" else None
    h = 1e-5
    fd = float((dz * (numpy_encode(name, P, x + h * v, eps) - numpy_encode(name, P, x - h * v, eps))).sum() / (2 * h))
    an = float((numpy_vjp(name, P, x, dz, eps) * v).sum())
    assert abs(fd - an) <= 1e-7 * abs(an)

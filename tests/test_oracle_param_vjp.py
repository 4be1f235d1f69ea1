"""CPU check of the float64 reference the GPU parameter-VJP tests compare against: torch autograd of oracle/ian_torch.decode
with respect to the 13 trainable decoder tensors of IAN_simple (train_IAN_simple.py:353, `decoder_params`) agrees with
central differences of the float64 numpy decoder oracle/ian_numpy.simple_decode along a random direction per tensor.

The two oracles share no arithmetic code, so agreement pins both the autograd graph (inference BatchNorm with mean /
inv_std constant, as X_hat_fn evaluates it, API.py:46) and the numpy restatement."""
import numpy as np
import pytest
import torch

from oracle import ian_numpy as on
from oracle import ian_torch as ot
from oracle import weights as ow

PARAM_VJP_NAMES = ["l_dec_fc2.W", "dec_conv1.W", "dec_conv2.W", "dec_conv3.W", "dec_out.W",
                   "bnorm_dec_fc2.beta", "bnorm_dec_fc2.gamma", "bnorm_dc1.beta", "bnorm_dc1.gamma",
                   "bnorm_dc2.beta", "bnorm_dc2.gamma", "bnorm_dc3.beta", "bnorm_dc3.gamma"]


def param_grads64(P, z, dx, names=PARAM_VJP_NAMES):
    """float64 (dz, {name: dL/dparam}) of L = <decode(P, z), dx> by torch autograd of oracle/ian_torch.decode."""
    T = ot.to_torch(P, torch.float64)
    for n in names:
        T[n].requires_grad_(True)
    zt = torch.from_numpy(np.asarray(z, np.float64)).requires_grad_(True)
    out = ot.decode(T, zt)
    g = torch.autograd.grad(out, [zt] + [T[n] for n in names], grad_outputs=torch.from_numpy(np.asarray(dx, np.float64)))
    return g[0].numpy(), {n: v.numpy() for n, v in zip(names, g[1:])}


@pytest.mark.parametrize("seed", [0, 1])
def test_autograd_matches_central_differences_of_numpy_oracle(seed):
    P = {k: np.asarray(v, np.float64) for k, v in ow.make_simple_weights(seed).items()}
    rng = np.random.default_rng(100 + seed)
    z = rng.standard_normal((2, 100))
    dx = rng.standard_normal((2, 3, 64, 64))
    _, grads = param_grads64(P, z, dx)
    h = 1e-8        # the smallest rectifier pre-activation of these inputs is ~3e-6: a larger step crosses kinks
    for name in PARAM_VJP_NAMES:
        V = rng.standard_normal(P[name].shape)
        Pp, Pm = dict(P), dict(P)
        Pp[name] = P[name] + h * V
        Pm[name] = P[name] - h * V
        fd = float(np.sum(dx * (on.simple_decode(Pp, z) - on.simple_decode(Pm, z)))) / (2 * h)
        ad = float(np.sum(grads[name] * V))
        assert abs(ad - fd) <= 1e-6 * max(1.0, abs(fd)), (name, ad, fd)

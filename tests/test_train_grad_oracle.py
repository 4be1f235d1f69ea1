"""CPU: the float64 autograd restatement of the training-mode ops (tests/train_grad_oracle.py) against the numpy forward
(oracle/train_numpy.py) and the executed reference's directional derivatives (tests/golden/ref_exec_train_grad.npz), and
the closed forms of DESIGN §5.6b against that autograd."""
import os

import numpy as np
import pytest
import torch

import train_grad_oracle as tg
from oracle import train_numpy as tn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = np.load(os.path.join(ROOT, "tests", "golden", "ref_exec_train_grad.npz"))
T = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)


def _directional(fn, inputs, R, keys):
    """⟨∇(Σ R·fn), v⟩ per key by autograd"""
    ts = {k: T(v).requires_grad_(True) for k, v in inputs.items()}
    (fn(**ts) * T(R)).sum().backward()
    return {k: ts[k].grad for k in keys}


@pytest.mark.parametrize("tag", ["main", "n1", "k1p1", "k13p5"])
def test_mb_restatement_matches_reference(tag):
    a = lambda k: FIX["mb_%s_%s" % (tag, k)]
    args = dict(x=a("x"), theta=a("theta"), lws=a("lws"), b=a("b"))
    out = tg.mb_layer(*[T(args[k]) for k in ("x", "theta", "lws", "b")])
    want = tn.minibatch_layer(args["x"], args["theta"], args["lws"], args["b"])
    assert np.abs(out.numpy() - want).max() <= 1e-13
    assert abs(float((out * T(a("R"))).sum()) - float(a("L"))) <= 1e-12 * (1 + abs(float(a("L"))))
    grads = _directional(lambda x, theta, lws, b: tg.mb_layer(x, theta, lws, b), args, a("R"), args)
    for k in args:
        got = float((grads[k] * T(a("v_" + k))).sum())
        want = float(a("dL_" + k))
        assert abs(got - want) <= 1e-8 * max(1.0, abs(want)), (tag, k, got, want)


@pytest.mark.parametrize("tag", ["conv", "dense", "edges"])
def test_bn_restatement_matches_reference(tag):
    a = lambda k: FIX["bn_%s_%s" % (tag, k)]
    args = dict(x=a("x"), gamma=a("gamma"), beta=a("beta"))
    y = tg.bn_train(T(args["x"]), T(args["gamma"]), T(args["beta"]))
    want = tn.batch_norm_train(args["x"], args["gamma"], args["beta"], np.zeros(len(args["gamma"])), np.ones(len(args["gamma"])))[0]
    assert np.abs(y.numpy() - want).max() <= 1e-12
    grads = _directional(tg.bn_train, args, a("R"), args)
    for k in args:
        got = float((grads[k] * T(a("v_" + k))).sum())
        want = float(a("dL_" + k))
        assert abs(got - want) <= 1e-8 * max(1.0, abs(want)), (tag, k, got, want)


@pytest.mark.parametrize("shape", [(5, 8, 6, 6), (9, 20), (1, 7), (3, 4, 11)])
@pytest.mark.parametrize("affine", [True, False])
def test_bn_closed_form_is_autograd(shape, affine):
    rng = np.random.default_rng(sum(shape))
    x = T(rng.standard_normal(shape) * 3 + 2).requires_grad_(True)
    c = shape[1]
    g = T(rng.uniform(0.5, 1.5, c)).requires_grad_(True) if affine else None
    b = T(rng.normal(0, 1, c)).requires_grad_(True) if affine else None
    if affine:
        g.data[0] = 0.0                                                  # gamma = 0: dx = 0 there, dgamma is not
    x.data[:, -1] = 4.25                                                 # a constant channel: s = 1/sqrt(eps)
    dy = T(rng.standard_normal(shape))
    y = tg.bn_train(x, g, b)
    want = torch.autograd.grad(y, [t for t in (x, g, b) if t is not None], dy)
    dx, dg, db = tg.bn_backward(x.detach(), None if g is None else g.detach(), dy)
    assert torch.allclose(dx, want[0], rtol=1e-10, atol=1e-11)
    if affine:
        assert torch.all(dx[:, 0] == 0)
        assert torch.allclose(dg, want[1], rtol=1e-10, atol=1e-11) and torch.allclose(db, want[2], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("n,d,K,P,dup", [(6, 20, 7, 5, False), (1, 9, 3, 2, False), (9, 33, 13, 5, True), (5, 4, 1, 1, True)])
def test_mb_closed_form_is_autograd(n, d, K, P, dup):
    rng = np.random.default_rng(n * 31 + d)
    x = rng.standard_normal((n, d))
    if dup:
        x[-1] = x[0]                                                     # ties A_i = A_j: sgn(0) = 0 in both
    ins = [T(x), T(rng.normal(0, 0.05, (d, K, P))), T(rng.normal(np.log(0.2 / P), 0.1, (K, P))), T(rng.normal(-1, 0.5, K))]
    ins = [t.requires_grad_(True) for t in ins]
    g = T(rng.standard_normal((n, d + K)))
    want = torch.autograd.grad(tg.mb_layer(*ins), ins, g)
    got = tg.mb_backward(*[t.detach() for t in ins], g)
    for u, v, name in zip(got, want, ("dx", "dtheta", "dlws", "db")):
        assert torch.allclose(u, v, rtol=1e-10, atol=1e-12), name

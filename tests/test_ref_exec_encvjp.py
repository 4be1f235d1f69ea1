"""The encoder VJP's float64 oracle (tests/encode_vjp_oracle.py) against the EXECUTED reference: every directional
derivative dz . (Z(x + h v) - Z(x - h v)) / 2h of the reference's own Z_hat in tests/golden/ref_exec_encvjp.npz
(tests/golden/make_golden_encvjp.py; two golden images per graph, without and with eps) equals <dx_oracle, v> to 1e-7
relative."""
import os

import numpy as np
import pytest

from oracle import ian_full_numpy as fn
from oracle import ian_numpy as on
from oracle import weights as ow

import encode_vjp_oracle as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def fixture():
    """the stored directional derivatives, and the images / directions / cotangents / eps they were taken at"""
    f = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_exec_encvjp.npz")))
    rng = np.random.RandomState(int(f["seed"]))
    n = int(f["n_img"])
    draws = {g: (rng.standard_normal((n, 3, 64, 64)), rng.standard_normal((n, 100)), rng.standard_normal((n, 100)))
             for g in ("simple", "full", "v1")}
    out = {}
    for g in ("simple", "full", "v1"):
        gold = np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % g))
        x = on.to_tanh(gold["images"][:n].astype(np.float64)).astype(np.float32)   # as the generator stages them
        out[g] = (x, int(gold["weight_seed"]), draws[g], f["dd_" + g])
    return out


def oracle_dd(g, P, x, v, dz, eps):
    if g == "simple":
        dx = eo.simple_encode_vjp(P, x, dz, eps)
    else:
        dx = eo.full_encode_vjp(P, x, fn.made_masks(fn.made_ordering()), dz, eps)
    return float((dx * v).sum())


@pytest.mark.parametrize("g", ["simple", "full", "v1"])
def test_oracle_matches_executed_reference(g):
    x, seed, (v, dz, eps), dd = fixture()[g]
    P = {"simple": ow.make_simple_weights, "full": ow.make_full_weights, "v1": ow.make_v1_weights}[g](seed)
    for k in range(len(x)):
        for j, e in enumerate((None, eps[k:k + 1])):
            got = oracle_dd(g, P, x[k:k + 1].astype(np.float64), v[k:k + 1], dz[k:k + 1], e)
            assert abs(got - dd[j, k]) <= 1e-7 * abs(dd[j, k]), (g, k, j, got, dd[j, k])

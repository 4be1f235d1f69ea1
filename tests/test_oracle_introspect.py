"""The float64 references of the introspection features and the feature fit (tests/introspect_oracle.py), on the CPU:
  * the torch restatement of l_introspect and its JVP against the EXECUTED reference (tests/golden/ref_exec_introspect.npz:
    the reference's own features and their central differences, at a channel subset and as probe projections);
  * the torch restatement of l_introspect against the independent numpy oracle's layers (oracle/ian_numpy.py) on every
    graph's golden images, and its JVP (torch.func.jvp) against central differences of the numpy features;
  * feature_loss against train_IAN.py:244's batch formula: the batch mean of the per-sample l_f is that formula;
  * jacobians64 / gram64 on a small case: e = E, and g = dE/dz / 2 against central differences of the numpy E."""
import os

import numpy as np
import pytest
import torch

import introspect_oracle as io
from oracle import ian_numpy as on
from test_ref_exec_decjvp import MAKE, weight_seed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H = 1e-6
GRAPHS = ["simple", "full", "v1"]


def features_np(P, x):
    """l_introspect from oracle/ian_numpy.py's layers, float64"""
    h1 = on.lrelu(on.conv5x5_s2(x, P["enc_conv1.W"], P["enc_conv1.b"]))
    h2 = on.lrelu(on.batchnorm_inf(on.conv5x5_s2(h1, P["enc_conv2.W"]), on._bn(P, "bnorm2")))
    h3 = on.lrelu(on.batchnorm_inf(on.conv5x5_s2(h2, P["enc_conv3.W"]), on._bn(P, "bnorm3")))
    h4 = on.lrelu(on.batchnorm_inf(on.conv5x5_s2(h3, P["enc_conv4.W"]), on._bn(P, "bnorm4")))
    return [h1, h2, h3, h4]


def _images(g):
    return np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % g))["images"].astype(np.float64)


# measured worst: features 1.8e-15 / 3.0e-15 (channels / probes), tangents 8.4e-9 / 8.3e-9 -- the error of the fixture's
# central differences (h = 1e-7) themselves
REF_BOUND = {"f": 1e-14, "p": 1e-14, "df": 2e-8, "dp": 2e-8}


@pytest.mark.parametrize("g", GRAPHS)
def test_restatement_matches_the_executed_reference(g):
    x, seed, v, probes, stored = io.fixture()[g]
    Q = io.weights64(MAKE[g](seed), "cpu")
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    f, tan = torch.func.jvp(lambda a: tuple(io.features(Q, a)), (t(x),), (t(v),))
    err = io.against_fixture([a.numpy() for a in f], [a.numpy() for a in tan], probes, stored)
    assert all(err[k] <= REF_BOUND[k] for k in err), err


@pytest.mark.parametrize("g", GRAPHS)
def test_restatement_matches_numpy_features_and_differences(g):
    P = MAKE[g](weight_seed(g))
    x = _images(g)
    Q = io.weights64(P, "cpu")
    v = np.random.default_rng(5).standard_normal(x.shape)
    f, t = torch.func.jvp(lambda a: tuple(io.features(Q, a)), (torch.from_numpy(x),), (torch.from_numpy(v),))
    ref = features_np(P, x)
    assert [tuple(a.shape[1:]) for a in f] == [(128, 32, 32), (256, 16, 16), (512, 8, 8), (1024, 4, 4)]
    for a, b in zip(f, ref):
        assert np.abs(a.numpy() - b).max() <= 1e-12 * np.abs(b).max()
    fp, fm = features_np(P, x + H * v), features_np(P, x - H * v)
    for a, p, m in zip(t, fp, fm):
        fd = (p - m) / (2 * H)
        assert np.linalg.norm(a.numpy() - fd) <= 1e-6 * np.linalg.norm(fd)


def test_feature_loss_is_the_training_formula():
    rng = np.random.default_rng(1)
    shapes = [(128, 32, 32), (256, 16, 16), (512, 8, 8), (1024, 4, 4)]
    ga = [rng.standard_normal((5,) + s) for s in shapes]
    gb = [rng.standard_normal((5,) + s) for s in shapes]
    # train_IAN.py:244: T.mean([T.mean(squared_error(g_X[i], g_X_hat[i])) for i in ...]) over the whole batch
    batch = np.mean([np.mean((a - b) ** 2) for a, b in zip(ga, gb)])
    per = io.feature_loss(ga, gb)
    assert per.shape == (5,) and np.isclose(per.mean(), batch, rtol=1e-13, atol=0)
    assert np.isclose(per[2], np.mean([np.mean((a[2] - b[2]) ** 2) for a, b in zip(ga, gb)]), rtol=1e-13, atol=0)


def test_gram_is_the_objective_and_its_gradient():
    g = "simple"
    P = MAKE[g](weight_seed(g))
    rng = np.random.default_rng(3)
    z = rng.standard_normal((1, 100))
    x = np.tanh(rng.standard_normal((1, 3, 64, 64)))
    a, b = 0.5, 2.0
    (J, Jf, r, rf), = io.jacobians64(g, P, z, x)
    A, gv, e = io.gram64(J, Jf, r, rf, a, b)

    def E(zz):
        xh = on.simple_decode(P, zz)
        lf = io.feature_loss(features_np(P, xh), features_np(P, x))
        return a * ((xh - x) ** 2).sum() + b * 12288 * lf[0]
    assert np.isclose(e, E(z), rtol=1e-12, atol=0), (e, E(z))
    assert np.abs(A - A.T).max() <= 1e-12 * np.abs(A).max()
    d = rng.standard_normal((1, 100))
    fd = (E(z + H * d) - E(z - H * d)) / (2 * H)       # at h = 1e-5 a rectifier of these weights crosses its kink
    assert np.isclose(2 * gv @ d[0], fd, rtol=1e-7), (2 * gv @ d[0], fd)

"""The float64 reference of the discriminator head (tests/discrim_oracle.py), on the CPU:
  * its logits, probabilities and probe derivatives against the EXECUTED reference (tests/golden/ref_exec_discrim.npz) on
    every graph, including a derivative that exists only through the MinibatchLayer's coupling;
  * its torch MinibatchLayer against the numpy one of oracle/train_numpy.py, and f = b exactly at n = 1;
  * the fixture's log_weight_scale: the reference's init rule puts every kernel's mean nearest-pair distance at 2 (half of
    it at 1), so the pair terms exp(-distance) of the fixture's batch do not underflow."""
import numpy as np
import pytest
import torch

import discrim_oracle as do
import introspect_oracle as io
from oracle import train_numpy as tn
from test_ref_exec_decjvp import MAKE

FIX = do.fixture()


def _t(a):
    return torch.from_numpy(np.asarray(a, np.float64))


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - b) / np.linalg.norm(b))


# measured worst over the graphs: logits 1.1e-14 (small logits, summed in another order), p 6.2e-16, probe derivatives
# 8.9e-8 -- the error of the fixture's central differences (h = 1e-7) themselves
BOUND = {"logits": 5e-14, "p": 5e-15, "dp": 3e-7}


@pytest.mark.parametrize("g", do.GRAPHS)
def test_restatement_matches_the_executed_reference(g):
    x, seed, H, stored = FIX[g]
    Q, Hd = io.weights64(MAKE[g](seed), "cpu"), do.head64(H)
    lg = do.logits(Q, Hd, _t(x))
    err = {"logits": _rel(lg.numpy(), stored["logits"]), "p": _rel(do.probs(lg).numpy(), stored["p"])}
    dp = [float((_t(stored["probe"][t]) * torch.func.jvp(lambda a: do.logits(Q, Hd, a), (_t(x),), (_t(stored["v"][t]),))[1]).sum())
          for t in range(len(stored["v"]))]
    err["dp"] = float(np.max(np.abs(np.array(dp) - stored["dp"]) / np.abs(stored["dp"])))
    assert all(err[k] <= BOUND[k] for k in err), err
    assert abs(stored["dp"][2]) > 1e-3 * np.abs(stored["dp"]).max()      # the coupled derivative is there to be matched


def test_minibatch_matches_numpy_oracle_and_is_b_at_one_sample():
    rng = np.random.RandomState(4)
    H = do.make_discriminator_weights("simple", 3)
    x = rng.standard_normal((5, 1024)) * 0.3
    H[do.NAMES[1]] = do.init_log_weight_scale(x, H[do.NAMES[0]], H[do.NAMES[1]])
    ref = tn.minibatch_layer(x, H[do.NAMES[0]], H[do.NAMES[1]], H[do.NAMES[2]])
    got = do.minibatch(do.head64(H), _t(x)).numpy()
    assert np.abs(got - ref).max() <= 1e-13 * np.abs(ref).max()
    one = do.minibatch(do.head64(H), _t(x[:1])).numpy()
    assert np.array_equal(one[0, 1024:], H[do.NAMES[2]].astype(np.float64)) and np.array_equal(one[0, :1024], x[0])


@pytest.mark.parametrize("g", do.GRAPHS)
def test_fixture_head_puts_pair_distances_near_one(g):
    x, seed, H, _ = FIX[g]
    pooled = do.pooled(io.weights64(MAKE[g](seed), "cpu"), _t(x)).numpy()
    again = do.init_log_weight_scale(pooled, H[do.NAMES[0]], H[do.NAMES[1]])
    assert np.abs(again - H[do.NAMES[1]]).max() <= 1e-5                   # a second init step is a no-op: mean min = 2
    f = do.minibatch(do.head64(H), _t(pooled)).numpy()[:, 1024:] - H[do.NAMES[2]]
    assert f.min() > 1e-3                                                 # every kernel's pair terms are alive

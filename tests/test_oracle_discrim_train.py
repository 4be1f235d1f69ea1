"""The float64 restatement of the training-mode discriminator (tests/discrim_train_oracle.py), on the CPU, against the
EXECUTED reference (tests/golden/ref_exec_discrim_train.npz) on every graph: the batch's logits and probabilities, the
logits of a one-image batch, bnorm2..4's batch statistics, and the probe derivatives -- one of them a derivative of image
0's logit along a direction on image 1 alone, which exists only through the batch's coupling."""
import numpy as np
import pytest
import torch

import discrim_oracle as do
import discrim_train_oracle as dto
import introspect_oracle as io
from test_ref_exec_decjvp import MAKE

FIX = dto.fixture()
RAW = dict(np.load(dto.os.path.join(dto.ROOT, "tests", "golden", "ref_exec_discrim_train.npz")))


def _t(a):
    return torch.from_numpy(np.asarray(a, np.float64))


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - b) / np.linalg.norm(b))


# measured worst over the graphs: logits 4.5e-15, the one-image batch 1.1e-14, p 3.7e-16, stats 1.2e-16, probe derivatives
# 1.1e-7 -- the error of the fixture's central differences (h = 1e-7) themselves
BOUND = {"logits": 5e-14, "logits1": 5e-14, "p": 5e-15, "stats": 5e-15, "dp": 3e-7}


@pytest.mark.parametrize("g", dto.GRAPHS)
def test_restatement_matches_the_executed_reference(g):
    x, seed, H, stored = FIX[g]
    Q, Hd = io.weights64(MAKE[g](seed), "cpu"), do.head64(H)
    lg = dto.logits(Q, Hd, _t(x))
    err = {"logits": _rel(lg.numpy(), stored["logits"]), "p": _rel(do.probs(lg).numpy(), stored["p"]),
           "logits1": _rel(dto.logits(Q, Hd, _t(x[:1])).numpy(), RAW["logits1_%s" % g]),
           "stats": _rel(dto.stats(Q, x), stored["stats"])}
    dp = [float((_t(stored["probe"][t]) * torch.func.jvp(lambda a: dto.logits(Q, Hd, a), (_t(x),), (_t(stored["v"][t]),))[1]).sum())
          for t in range(len(stored["v"]))]
    err["dp"] = float(np.max(np.abs(np.array(dp) - stored["dp"]) / np.abs(stored["dp"])))
    assert all(err[k] <= BOUND[k] for k in err), err
    assert abs(stored["dp"][2]) > 1e-3 * np.abs(stored["dp"]).max()      # the coupled derivative is there to be matched


@pytest.mark.parametrize("g", dto.GRAPHS)
def test_training_mode_differs_from_inference(g):
    """the fixture exercises what is new: batch statistics move the logits well away from the running-statistics ones
    (measured: by 0.65 to 2.7 in relative L2)"""
    x, seed, H, stored = FIX[g]
    Q, Hd = io.weights64(MAKE[g](seed), "cpu"), do.head64(H)
    assert _rel(do.logits(Q, Hd, _t(x)).numpy(), stored["logits"]) > 1e-3


def test_vjp_is_the_transpose_of_the_jvp():
    x, seed, H, stored = FIX["full"]
    Q, Hd = io.weights64(MAKE["full"](seed), "cpu"), do.head64(H)
    u, v = stored["probe"][0], stored["v"][0]
    jv = torch.func.jvp(lambda a: dto.logits(Q, Hd, a), (_t(x),), (_t(v),))[1].numpy()
    lhs, rhs = float(np.sum(u * jv)), float(np.sum(dto.vjp(Q, Hd, x, u) * v))
    assert abs(lhs - rhs) <= 1e-12 * abs(lhs)

"""The float64 restatement of the training-mode IAN_simple decoder (tests/decode_train_oracle.py), on the CPU, against the
EXECUTED reference (tests/golden/ref_exec_decode_train.npz): x_hat of the batch and of a one-sample batch, the four
BatchNorms' batch statistics, and the probe derivatives along z -- one of them a derivative of sample 0 along a direction
on sample 1 alone, which exists only through the batch statistics -- and along one direction of each trainable tensor."""
import numpy as np
import torch

import decode_train_oracle as dto
from oracle import ian_torch as ot

FIX = dto.fixture()


def _t(a):
    return torch.from_numpy(np.asarray(a, np.float64))


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - b) / np.linalg.norm(b))


# measured: x_hat 6.3e-16, the one-sample batch 8.0e-16, stats 1.6e-17, z probes 2.4e-8, tensor probes 9.7e-7 -- the error
# of the fixture's central differences (h = 1e-7) themselves, largest where a step meets a rectifier kink
BOUND = {"x_hat": 1e-14, "x_hat1": 1e-14, "stats": 1e-15, "dp": 1e-7, "dq": 5e-6}


def test_restatement_matches_the_executed_reference():
    P = dto.weights64(FIX["weights"])
    z = FIX["z"]
    err = {"x_hat": _rel(dto.decode(P, _t(z)).numpy(), FIX["x_hat"]),
           "x_hat1": _rel(dto.decode(P, _t(z[:1])).numpy(), FIX["x_hat1"]),
           "stats": _rel(dto.stats(FIX["weights"], z), FIX["stats"])}
    dp = [float((_t(FIX["probe"][t]) * torch.func.jvp(lambda a: dto.decode(P, a), (_t(z),), (_t(FIX["v"][t]),))[1]).sum())
          for t in range(3)]
    err["dp"] = float(np.max(np.abs(np.array(dp) - FIX["dp"]) / np.abs(FIX["dp"])))
    dq = []
    for k, name in enumerate(dto.PARAM_NAMES):
        def f(w):
            Q = dict(P)
            Q[name] = w
            return dto.decode(Q, _t(z))
        dq.append(float((_t(FIX["pprobe"][k]) * torch.func.jvp(f, (P[name],), (_t(FIX["pdir"][name]),))[1]).sum()))
    err["dq"] = float(np.max(np.abs(np.array(dq) - FIX["dq"]) / np.abs(FIX["dq"])))
    assert all(err[k] <= BOUND[k] for k in err), err
    assert abs(FIX["dp"][2]) > 1e-3 * np.abs(FIX["dp"]).max()      # the coupled derivative is there to be matched


def test_training_mode_differs_from_inference():
    """the fixture exercises what is new: batch statistics move x_hat well away from the running-statistics one (measured:
    0.79 relative L2)"""
    P = dto.weights64(FIX["weights"])
    assert _rel(ot.decode(P, _t(FIX["z"])).numpy(), FIX["x_hat"]) > 1e-2


def test_one_sample_batch_ignores_z():
    """n = 1: bnorm_dec_fc2 normalises a single sample, so x_hat = h(beta) whatever z is, and dz is exactly 0"""
    P = dto.weights64(FIX["weights"])
    a = dto.decode(P, _t(FIX["z"][:1])).numpy()
    b = dto.decode(P, _t(FIX["z"][1:2])).numpy()
    assert np.abs(a - b).max() <= 1e-15 * np.abs(a).max()
    _, dz, g = dto.vjp(FIX["weights"], FIX["z"][:1], FIX["probe"][0][:1])
    assert np.all(dz == 0) and np.all(g["l_dec_fc2.W"] == 0)


def test_vjp_is_the_transpose_of_the_jvp():
    P = dto.weights64(FIX["weights"])
    z, u, v = FIX["z"], FIX["probe"][0], FIX["v"][0]
    jv = torch.func.jvp(lambda a: dto.decode(P, a), (_t(z),), (_t(v),))[1].numpy()
    _, dz, _ = dto.vjp(FIX["weights"], z, u, names=[])
    lhs, rhs = float(np.sum(u * jv)), float(np.sum(dz * v))
    assert abs(lhs - rhs) <= 1e-12 * abs(lhs)

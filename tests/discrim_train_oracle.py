"""float64 reference of the IAN's discriminator head l_discrim in training mode (include/ian_b200.h
ian_discriminate_train_*, ian_discriminate_train_vjp_*), get_output(l_discrim, x, deterministic=False):
  enc_conv1 (bias, LeakyRectify(0.2)); enc_conv2..4: convolution, BatchNorm with the BATCH's statistics -- per channel the
  mean and the biased variance over (n, h, w), inv_std = 1/sqrt(var + 1e-4), y = (x - mean) (gamma inv_std) + beta
  (lasagne BatchNormLayer, deterministic=False) -- and LeakyRectify(0.2); then discrim_oracle's pool, MinibatchLayer and
  dense head.  The VJP is float64 autograd through the statistics, as Theano's T.grad.  The fixture
  tests/golden/ref_exec_discrim_train.npz (tests/golden/make_golden_discrim_train.py) holds the EXECUTED reference's
  logits, probabilities, batch statistics and probe derivatives."""
import os

import numpy as np
import torch
import torch.nn.functional as F

import discrim_oracle as do
from oracle import ian_torch as ot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRAPHS = do.GRAPHS
BN_EPS = 1e-4
BN_CHANNELS = (256, 512, 1024)


def _bn_train(P, name, x, stats):
    mean = x.mean(dim=(0, 2, 3))
    var = ((x - mean[None, :, None, None]) ** 2).mean(dim=(0, 2, 3))
    inv_std = 1.0 / torch.sqrt(var + BN_EPS)
    stats.append((mean, inv_std))
    g, b = P[name + ".gamma"], P[name + ".beta"]
    return (x - mean[None, :, None, None]) * (g * inv_std)[None, :, None, None] + b[None, :, None, None]


def trunk(P, x, stats=None):
    """P: torch weights (introspect_oracle.weights64), x (n,3,64,64) -> a4 (n,1024,4,4); stats (a list) receives
    (mean, inv_std) of bnorm2..4"""
    stats = [] if stats is None else stats
    h = ot._lrelu(F.conv2d(x, P["enc_conv1.W"], P["enc_conv1.b"], stride=2, padding=2))
    for k in (2, 3, 4):
        h = ot._lrelu(_bn_train(P, "bnorm%d" % k, F.conv2d(h, P["enc_conv%d.W" % k], None, stride=2, padding=2), stats))
    return h


def logits(Q, H, x, stats=None):
    """Q: the graph's weights (introspect_oracle.weights64), H: discrim_oracle.head64, x (n,3,64,64) torch -> logits (n, U)"""
    return do.minibatch(H, trunk(Q, x, stats).mean(dim=(2, 3))) @ H[do.NAMES[3]]


def stats(Q, x):
    """(2, 1792) float64 numpy: row 0 the batch means of bnorm2 | bnorm3 | bnorm4, row 1 their inv_std"""
    s = []
    with torch.no_grad():
        trunk(Q, torch.from_numpy(np.asarray(x, np.float64)), s)
    return np.stack([torch.cat([m for m, _ in s]).numpy(), torch.cat([i for _, i in s]).numpy()])


def vjp(Q, H, x, dl):
    """dx = (d logits / d x)^T dl by float64 autograd, x and dl numpy -> numpy"""
    xt = torch.from_numpy(np.asarray(x, np.float64)).requires_grad_(True)
    (dx,) = torch.autograd.grad(logits(Q, H, xt), xt, torch.from_numpy(np.asarray(dl, np.float64)))
    return dx.numpy()


def draws(seed, n=4):
    """per graph: tangents v (3,n,3,64,64) and probes (3,n,U), float64.  The third pair moves image 1 alone and reads sample
    0 alone: with the MinibatchLayer's pair terms and the trunk's batch statistics both coupling the batch, it is a
    derivative that exists only through that coupling."""
    rng = np.random.RandomState(seed)
    out = {}
    for g in GRAPHS:
        v = rng.standard_normal((3, n, 3, 64, 64))
        probe = rng.standard_normal((3, n, do.units(g)))
        v[2, [i for i in range(n) if i != 1]] = 0.0
        probe[2, 1:] = 0.0
        out[g] = (v, probe)
    return out


def fixture():
    """{graph: (x (n,3,64,64) float32, graph weight seed, head tensors (float32, lws as stored), stored)} with stored =
    {"logits", "p", "stats" (2,1792), "dp" (3,)} and draws()'s "v" and "probe": dp[t] = <probe[t], d logits . v[t]>"""
    from oracle import ian_numpy as on
    f = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_exec_discrim_train.npz")))
    n = int(f["n_img"])
    d = draws(int(f["seed"]), n)
    imgs = np.load(os.path.join(ROOT, "tests", "golden", "ian_simple_golden.npz"))["images"][:n]
    x = on.to_tanh(imgs.astype(np.float64)).astype(np.float32)
    out = {}
    for g in GRAPHS:
        gold = np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % g))
        H = do.make_discriminator_weights(g, int(f["head_seed_%s" % g]))
        for k in do.NAMES[1:]:
            H[k] = f["%s_%s" % (k, g)]
        stored = {k: f["%s_%s" % (k, g)] for k in ("logits", "p", "stats", "dp")}
        stored["v"], stored["probe"] = d[g]
        out[g] = (x, int(gold["weight_seed"]), H, stored)
    return out

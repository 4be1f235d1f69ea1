"""float64 reference of the IAN's discriminator head l_discrim (include/ian_b200.h ian_discriminate_*,
ian_discriminate_vjp_*) under deterministic=True:
  logits = [pool(g_4(x)) | f] W,  p = sigmoid (U = 1: IAN_simple, IANv1) or softmax (U = 3: IAN.py) of the logits,
with g_4 introspect_oracle's enc_conv4 features, pool the mean over the 4 x 4 pixels (GlobalPoolLayer) and f the
MinibatchLayer's features of the pooled batch (layers.py:486-524, oracle/train_numpy.minibatch_layer restated in torch so
that its VJP comes from float64 autograd).  The head's seeded tensors and the data-dependent log_weight_scale rule
(layers.py:510-513, init=True) live here too; the fixture tests/golden/ref_exec_discrim.npz
(tests/golden/make_golden_discrim.py) holds the EXECUTED reference's logits, probabilities and probe derivatives."""
import os

import numpy as np
import torch

import introspect_oracle as io

K, P, D = 500, 5, 1024
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRAPHS = ("simple", "full", "v1")
NAMES = ("minibatch_discrim.theta", "minibatch_discrim.log_weight_scale", "minibatch_discrim.b", "discrimi.W")


def units(g):
    return 3 if g == "full" else 1


def make_discriminator_weights(g, seed):
    """the head's tensors with the reference's initialisations, float32: theta N(0, 0.05) (layers.py:487), log_weight_scale
    0 and b -1 (layers.py:488), W N(0, 0.02) (the graphs' initmethod(0.02); IAN_simple's initmethod() draws at the same
    scale here)"""
    rng = np.random.RandomState(seed)
    return {NAMES[0]: (0.05 * rng.standard_normal((D, K, P))).astype(np.float32),
            NAMES[1]: np.zeros((K, P), np.float32),
            NAMES[2]: np.full((K,), -1.0, np.float32),
            NAMES[3]: (0.02 * rng.standard_normal((D + K, units(g)))).astype(np.float32)}


def init_log_weight_scale(pooled, theta, lws):
    """MinibatchLayer.get_output_for(init=True)'s update of log_weight_scale (layers.py:510-513) on the batch `pooled`
    (n, 1024): lws - log(0.5 mean_i min_{j != i} sum_p |A_ikp - A_jkp|) per kernel k, float64"""
    pooled, theta, lws = (np.asarray(a, np.float64) for a in (pooled, theta, lws))
    W = theta * (np.exp(lws) / np.sqrt(np.sum(np.square(theta), axis=0)))[None]
    act = np.tensordot(pooled, W, [[1], [0]])
    abs_dif = (np.sum(np.abs(act[:, :, :, None] - act.transpose(1, 2, 0)[None]), axis=2) + 1e6 * np.eye(len(pooled))[:, None, :])
    mean_min = 0.5 * np.mean(np.min(abs_dif, axis=2), axis=0)
    return lws - np.log(mean_min)[:, None]


def head64(H, device="cpu"):
    return {k: torch.from_numpy(np.asarray(v, np.float64)).to(device) for k, v in H.items()}


def pooled(Q, x):
    return io.features(Q, x)[3].mean(dim=(2, 3))


def minibatch(H, x):
    """layers.py:495, :503-524 (init=False) in torch: x (n, 1024) -> (n, 1524) = [x | f]"""
    theta, lws, b = H[NAMES[0]], H[NAMES[1]], H[NAMES[2]]
    W = theta * (torch.exp(lws) / torch.sqrt((theta ** 2).sum(0)))[None]
    act = torch.tensordot(x, W, dims=([1], [0]))                                          # (n, K, P)
    abs_dif = (act[:, :, :, None] - act.permute(1, 2, 0)[None]).abs().sum(2)             # (n, K, n)
    abs_dif = abs_dif + 1e6 * torch.eye(len(x), dtype=x.dtype, device=x.device)[:, None, :]
    f = torch.exp(-abs_dif).sum(2) + b[None]
    return torch.cat([x, f], 1)


def logits(Q, H, x):
    """Q: the graph's weights (introspect_oracle.weights64), H: head64, x (n,3,64,64) torch -> logits (n, U)"""
    return minibatch(H, pooled(Q, x)) @ H[NAMES[3]]


def probs(lg):
    return torch.sigmoid(lg) if lg.shape[1] == 1 else torch.softmax(lg, 1)


def vjp(Q, H, x, dl):
    """dx = (d logits / d x)^T dl by float64 autograd, x and dl numpy -> numpy"""
    xt = torch.from_numpy(np.asarray(x, np.float64)).requires_grad_(True)
    (dx,) = torch.autograd.grad(logits(Q, H, xt), xt, torch.from_numpy(np.asarray(dl, np.float64)))
    return dx.numpy()


def draws(seed, n=4):
    """per graph: tangents v (3,n,3,64,64) and probes (3,n,U), float64.  The third pair moves image n-1 alone and reads
    sample 0 alone: a derivative that exists only through the MinibatchLayer's coupling."""
    rng = np.random.RandomState(seed)
    out = {}
    for g in GRAPHS:
        v = rng.standard_normal((3, n, 3, 64, 64))
        probe = rng.standard_normal((3, n, units(g)))
        v[2, :n - 1] = 0.0
        probe[2, 1:] = 0.0
        out[g] = (v, probe)
    return out


def fixture():
    """{graph: (x (4,3,64,64) float32 -- the first 4 images of ian_simple_golden.npz on every graph --, graph weight seed, head tensors (float32, lws as stored), stored)} with stored =
    {"logits", "p", "dp" (3,)} and draws()'s "v" (3,4,3,64,64) and "probe" (3,4,U): dp[t] = <probe[t], d logits . v[t]>"""
    from oracle import ian_numpy as on
    f = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_exec_discrim.npz")))
    n = int(f["n_img"])
    d = draws(int(f["seed"]), n)
    imgs = np.load(os.path.join(ROOT, "tests", "golden", "ian_simple_golden.npz"))["images"][:n]
    x = on.to_tanh(imgs.astype(np.float64)).astype(np.float32)
    out = {}
    for g in GRAPHS:
        gold = np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % g))
        H = make_discriminator_weights(g, int(f["head_seed_%s" % g]))
        for k in (NAMES[1], NAMES[2], NAMES[3]):
            H[k] = f["%s_%s" % (k, g)]
        stored = {k: f["%s_%s" % (k, g)] for k in ("logits", "p", "dp")}
        stored["v"], stored["probe"] = d[g]
        out[g] = (x, int(gold["weight_seed"]), H, stored)
    return out

"""float64 reference of the IAN_simple decoder in training mode (include/ian_b200.h ian_decode_train_*,
ian_decode_train_vjp_*), get_output(l_out, {l_Z: z}) under deterministic=False (IAN_simple.py:129-223):
  h0 = rectify(BN_fc2(z W_fc2)), bnorm_dec_fc2 normalising each of the 16384 features over the n samples;
  h1..h3 = rectify(BN_dck(deconv(h, W_k))), bnorm_dc1..3 normalising each channel over (n, h, w);
  x_hat = tanh(deconv(h3, W_out)),
with lasagne's training-mode BatchNorm: the batch's mean and biased variance, inv_std = 1/sqrt(var + 1e-4),
y = (x - mean) (gamma inv_std) + beta.  The VJP is float64 autograd through the statistics, as Theano's T.grad.  The
fixture tests/golden/ref_exec_decode_train.npz (tests/golden/make_golden_decode_train.py) holds the EXECUTED reference's
x_hat, batch statistics and probe derivatives."""
import os

import numpy as np
import torch

from oracle import ian_torch as ot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BN_EPS = 1e-4
BNORMS = ("bnorm_dec_fc2", "bnorm_dc1", "bnorm_dc2", "bnorm_dc3")
PARAM_NAMES = ["l_dec_fc2.W", "dec_conv1.W", "dec_conv2.W", "dec_conv3.W", "dec_out.W",
               "bnorm_dec_fc2.beta", "bnorm_dec_fc2.gamma", "bnorm_dc1.beta", "bnorm_dc1.gamma",
               "bnorm_dc2.beta", "bnorm_dc2.gamma", "bnorm_dc3.beta", "bnorm_dc3.gamma"]


def _bn_train(P, name, x, stats):
    axes = (0,) if x.dim() == 2 else (0, 2, 3)
    shp = (1, -1) + (1,) * (x.dim() - 2)
    mean = x.mean(dim=axes)
    var = ((x - mean.reshape(shp)) ** 2).mean(dim=axes)
    inv_std = 1.0 / torch.sqrt(var + BN_EPS)
    stats.append((mean, inv_std))
    return (x - mean.reshape(shp)) * (P[name + ".gamma"] * inv_std).reshape(shp) + P[name + ".beta"].reshape(shp)


def decode(P, z, stats=None, return_pre=False):
    """P: torch weights, z (n,100) torch -> x_hat (n,3,64,64); stats (a list) receives (mean, inv_std) of the four
    BatchNorms; return_pre: also the four batch-normalised pre-activations"""
    stats = [] if stats is None else stats
    pre = [_bn_train(P, BNORMS[0], z @ P["l_dec_fc2.W"], stats)]
    h = ot._relu(pre[0]).reshape(-1, 1024, 4, 4)
    for k in (1, 2, 3):
        pre.append(_bn_train(P, BNORMS[k], ot.deconv(h, P["dec_conv%d.W" % k]), stats))
        h = ot._relu(pre[-1])
    x = torch.tanh(ot.deconv(h, P["dec_out.W"]))
    return (x, pre) if return_pre else x


def weights64(P):
    return ot.to_torch({k: np.asarray(v, np.float64) for k, v in P.items()}, torch.float64)


def stats(P, z):
    """(2, 17280) float64 numpy: row 0 the batch means of bnorm_dec_fc2 (reference feature order) | bnorm_dc1 | bnorm_dc2 |
    bnorm_dc3, row 1 their inv_std"""
    s = []
    with torch.no_grad():
        decode(weights64(P), torch.from_numpy(np.asarray(z, np.float64)), s)
    return np.stack([torch.cat([m for m, _ in s]).numpy(), torch.cat([i for _, i in s]).numpy()])


def vjp(P, z, dx, names=PARAM_NAMES):
    """float64 (x_hat, dz, {name: dL/dparam}) of L = <decode(P, z), dx> by autograd, numpy in and out"""
    T = weights64(P)
    for n in names:
        T[n].requires_grad_(True)
    zt = torch.from_numpy(np.asarray(z, np.float64)).requires_grad_(True)
    x = decode(T, zt)
    g = torch.autograd.grad(x, [zt] + [T[n] for n in names], torch.from_numpy(np.asarray(dx, np.float64)))
    return x.detach().numpy(), g[0].numpy(), {n: v.numpy() for n, v in zip(names, g[1:])}


def draws(seed, n=4):
    """latents z (n,100), three z-directions v (3,n,100), per-direction probes (3,n,3,64,64), and per trainable tensor a
    direction (unit L2 norm, so a central difference of the whole tensor stays clear of the rectifier kinks) and a probe,
    all float64 from one seed.  The third z-direction moves sample 1 alone and its probe reads sample
    0 alone: a derivative that exists only through the batch statistics."""
    from oracle import weights as ow
    rng = np.random.RandomState(seed)
    z = rng.standard_normal((n, 100))
    v = rng.standard_normal((3, n, 100))
    probe = rng.standard_normal((3, n, 3, 64, 64))
    v[2, [i for i in range(n) if i != 1]] = 0.0
    probe[2, 1:] = 0.0
    shapes = {k: np.shape(a) for k, a in ow.make_simple_weights(0).items()}
    pdir = {k: rng.standard_normal(shapes[k]) for k in PARAM_NAMES}
    pdir = {k: d / np.linalg.norm(d) for k, d in pdir.items()}   # unit L2: the step h moves a tensor by h, not h sqrt(size)
    pprobe = rng.standard_normal((len(PARAM_NAMES), n, 3, 64, 64))
    return z, v, probe, pdir, pprobe


def fixture():
    """the stored fixture as a dict, with weights (float32, the checkpoint's) and draws() added"""
    from oracle import weights as ow
    raw = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_exec_decode_train.npz")))
    raw["weights"] = ow.make_simple_weights(int(raw["weight_seed"]))
    raw["z"], raw["v"], raw["probe"], raw["pdir"], raw["pprobe"] = draws(int(raw["seed"]), int(raw["n_img"]))
    return raw

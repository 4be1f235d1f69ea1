"""float64 references of the IAN's introspection features and of the fit under its feature-wise loss (include/ian_b200.h
ian_introspect_*, ian_feature_gauss_newton_*, ian_fit_latent_features_*).
  features:     l_introspect = [enc_conv1, enc_conv2, enc_conv3, enc_conv4] of every graph (IAN_simple.py:73-116; IAN.py and
                IANv1.py share the layers) under deterministic=True: conv, inference BatchNorm, LeakyRectify(0.2);
  feature_loss: the per-sample form of train_IAN.py:244, (1/4) sum_i mean((g_i(a) - g_i(b))^2);
  jacobians64:  J = d decode(z) / d z and the stacked J_i = d g_i(decode(z)) / d z by torch.func.jacfwd, with r and r_i;
  fixture:      tests/golden/ref_exec_introspect.npz (tests/golden/make_golden_introspect.py): the EXECUTED reference's
                features at a channel subset and as seeded probe projections, and central differences of both along seeded
                image tangents, on the golden images and weights of every graph;
  gram64:       A = a J^T J + sum_i c_i J_i^T J_i, g = a J^T r + sum_i c_i J_i^T r_i, e = a |r|^2 + sum_i c_i |r_i|^2,
                c_i = 3072 b / M_i."""
import os

import numpy as np
import torch
import torch.nn.functional as F

from oracle import ian_torch as ot

M = (131072, 65536, 32768, 16384)
SHAPES = ((128, 32, 32), (256, 16, 16), (512, 8, 8), (1024, 4, 4))
CHANNELS = ((0, 77), (5, 200), (31, 444), (2, 1000))       # make_golden_introspect.py's channel subset
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DECODER = {"simple": ot.decode, "full": ot.full_decode, "v1": ot.v1_decode}


def features(P, x):
    """P: torch weights (ot.to_torch), x (n,3,64,64) torch -> [g1..g4] in x's dtype, NCHW"""
    h1 = ot._lrelu(F.conv2d(x, P["enc_conv1.W"], P["enc_conv1.b"], stride=2, padding=2))
    h2 = ot._lrelu(ot._bn(P, "bnorm2", F.conv2d(h1, P["enc_conv2.W"], None, stride=2, padding=2)))
    h3 = ot._lrelu(ot._bn(P, "bnorm3", F.conv2d(h2, P["enc_conv3.W"], None, stride=2, padding=2)))
    h4 = ot._lrelu(ot._bn(P, "bnorm4", F.conv2d(h3, P["enc_conv4.W"], None, stride=2, padding=2)))
    return [h1, h2, h3, h4]


def fixture():
    """{graph: (x (n,3,64,64) float32, weight seed, v (n,3,64,64), probes [(PROBES, C, H, W)] x 4, stored)} with stored =
    {"f", "df", "p", "dp"}: per layer the reference's features and central differences at CHANNELS[i], and their probe
    projections"""
    from oracle import ian_numpy as on
    f = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_exec_introspect.npz")))
    rng = np.random.RandomState(int(f["seed"]))
    n, k = int(f["n_img"]), int(f["probes"])
    draws = {g: (rng.standard_normal((n, 3, 64, 64)), [rng.standard_normal((k,) + s) for s in SHAPES])
             for g in ("simple", "full", "v1")}
    out = {}
    for g, (v, probes) in draws.items():
        gold = np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % g))
        x = on.to_tanh(gold["images"][:n].astype(np.float64)).astype(np.float32)   # as the generator stages them
        stored = {key: [f["%s_%s_%d" % (key, g, i)] for i in range(4)] for key in ("f", "df", "p", "dp")}
        out[g] = (x, int(gold["weight_seed"]), v, probes, stored)
    return out


def against_fixture(feats, tangents, probes, stored):
    """relative errors {f, df, p, dp} (max over layers, L2 per layer) of features / tangents (n, C, H, W) x 4 against a
    fixture entry"""
    err = {}
    for key, arrs in (("f", feats), ("df", tangents)):
        err[key] = max(float(np.linalg.norm(np.asarray(a, np.float64)[:, list(CHANNELS[i])] - stored[key][i]) /
                             np.linalg.norm(stored[key][i])) for i, a in enumerate(arrs))
        pk = {"f": "p", "df": "dp"}[key]
        err[pk] = max(float(np.linalg.norm(np.einsum("nchw,jchw->nj", np.asarray(a, np.float64), probes[i]) - stored[pk][i]) /
                            np.linalg.norm(stored[pk][i])) for i, a in enumerate(arrs))
    return err


def feature_loss(ga, gb):
    """per-sample (1/4) sum_i mean((ga_i - gb_i)^2) of two feature lists (numpy or torch), float64 numpy"""
    n = len(ga[0])
    return sum(((np.asarray(a, np.float64) - np.asarray(b, np.float64)).reshape(n, -1) ** 2).mean(1) for a, b in zip(ga, gb)) / 4


def weights64(P, device):
    return {k: t.to(device) for k, t in ot.to_torch(P, torch.float64).items()}


def jacobians64(g, P, z, x, device="cpu"):
    """per sample k: J (100,12288), Jf (100,245760) -- row i the derivative along z_i --, r (12288) and rf (245760), float64
    numpy; features flattened NCHW layer after layer"""
    Q = weights64(P, device)
    dec = DECODER[g]
    out = []
    for k in range(len(z)):
        zk = torch.from_numpy(np.asarray(z[k], np.float64)).to(device)
        xk = torch.from_numpy(np.asarray(x[k], np.float64)).to(device)[None]

        def both(v):
            xh = dec(Q, v[None])
            return torch.cat([xh.reshape(-1)] + [f.reshape(-1) for f in features(Q, xh)])
        jac = torch.func.jacfwd(both)(zk)                                        # (12288 + 245760, 100)
        val = both(zk)
        tgt = torch.cat([xk.reshape(-1)] + [f.reshape(-1) for f in features(Q, xk)])
        res = (val - tgt).cpu().numpy()
        J = jac.T.cpu().numpy()
        out.append((J[:, :12288], J[:, 12288:], res[:12288], res[12288:]))
        del jac
    return out


def layer_weights(b):
    """c_i per feature element, float64 (245760,)"""
    return np.concatenate([np.full(m, 3072.0 * b / m) for m in M])


def gram64(J, Jf, r, rf, a, b):
    c = layer_weights(b)
    A = a * (J @ J.T) + (Jf * c) @ Jf.T
    gv = a * (J @ r) + (Jf * c) @ rf
    e = a * (r @ r) + (c * rf) @ rf
    return A, gv, e

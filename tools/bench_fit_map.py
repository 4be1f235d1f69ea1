"""(GPU) Cost and recovery of the masked latent fit under the prior (ian_fit_latent_map_*, API.IAN.fit_latent_map) next to
the plain latent fit (ian_fit_latent_*); prints one JSON line.

    python tools/bench_fit_map.py [--rounds 3] [--min-seconds 1.0] [--out profiles/h100_fit_map.json]

Reported, with the card's name and power limit read in the same run:
  * per graph (IAN_simple, IANv1.py, IAN.py in float32 and bf16) at batches 1 and 32: the time of one Levenberg-Marquardt
    step of a 10-step fit_latent_map_dev (random weights in [0, 1], prior 1e-2) and of a 10-step fit_latent_dev on the same
    targets, CUDA events on one stream, the two alternated over `--rounds` rounds (median and range), and their ratio;
  * "map_gram" against "gn_gram" per sample, from ian_layer_time_ms (layer timing on: plain launches);
  * on the inpainting targets of tests/test_gpu_fit_map.py (margin weights, 3 certified targets, starts 5 % away, a 24 x 24
    square or the left half at weight 0 with NaN there, 10 steps, prior 0): |u - u*| / |u*| and the hole's max error,
    and the hole's max error of fit_latent on the same image with the hole filled with 0.
Synthetic and margin weights only: nothing here says how well a trained model fills a real photo's hole.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_fit import ITERS, open_model, run, step_ms  # noqa: E402

BETA = 1e-2


def fits(model, n, rng):
    """a 10-step fit_latent_map_dev (random weights in [0, 1], prior BETA) and a 10-step fit_latent_dev on its targets"""
    st = torch.cuda.current_stream().cuda_stream
    us = rng.standard_normal((n, 100)).astype(np.float32)
    x = torch.from_numpy(model.sample(us)).cuda()
    w = torch.from_numpy(rng.uniform(0, 1, (n, 3, 64, 64)).astype(np.float32)).cuda()
    u0 = torch.from_numpy((us + 0.05 * rng.standard_normal((n, 100))).astype(np.float32)).cuda()
    u, z = torch.empty_like(u0), torch.empty_like(u0)

    def fmap():
        u.copy_(u0)
        model.fit_latent_map_dev(x.data_ptr(), w.data_ptr(), BETA, n, u.data_ptr(), ITERS, z.data_ptr(), 0, st)

    def ffit():
        u.copy_(u0)
        model.fit_latent_dev(x.data_ptr(), n, u.data_ptr(), ITERS, 0, st)
    return {"map": fmap, "fit": ffit}


def gram_ms(model, n=4):
    """per-sample ms of "map_gram" and "gn_gram" over two steps of each fit"""
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(1)
    us = rng.standard_normal((n, 100)).astype(np.float32)
    x = torch.from_numpy(model.sample(us)).cuda()
    w = torch.from_numpy(rng.uniform(0, 1, (n, 3, 64, 64)).astype(np.float32)).cuda()
    u = torch.from_numpy(us).cuda()
    model.set_layer_timing(True)
    try:
        for name in ("map_gram", "gn_gram"):
            model.layer_time_ms(name, reset=True)
        model.fit_latent_map_dev(x.data_ptr(), w.data_ptr(), BETA, n, u.data_ptr(), 2, 0, 0, st)
        model.fit_latent_dev(x.data_ptr(), n, u.data_ptr(), 2, 0, st)
        torch.cuda.synchronize()
        return {name: model.layer_time_ms(name, reset=True) / (2 * n) for name in ("map_gram", "gn_gram")}
    finally:
        model.set_layer_timing(False)


def recovery(model, g, P):
    import fit_map_oracle as fo
    us = fo.recovery_targets(g, P)[0]
    d = np.random.default_rng(5).standard_normal(us.shape)
    u0 = (us + 0.05 * d * np.linalg.norm(us, axis=1, keepdims=True) / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    x = model.sample(us)
    out = {}
    for hole, w in fo.masks(len(us)).items():
        inside = w == 0
        u, _ = model.fit_latent_map(np.where(inside, np.float32(np.nan), x), w, 0.0, u0, iters=ITERS)
        zf = model.fit_latent(np.where(inside, np.float32(0), x), model.Z_IAF_fn(u0), iters=ITERS)
        miss = lambda xh: float(np.abs(xh - x)[inside].max())
        out[hole] = {"du_max": float((np.linalg.norm(u.astype(np.float64) - us, axis=1) / np.linalg.norm(us, axis=1)).max()),
                     "hole_max_err": miss(model.sample(u)), "hole_max_err_fit_latent": miss(model.sample_at(zf))}
    return out


def measure(m, prec, a):
    return {"step_ms": step_ms(m, a.rounds, a.min_seconds, fits), "gram_ms_per_sample": gram_ms(m)}


def inpainting(npe, g, prec, a):
    if prec != "fp32":
        return {}
    import margin_weights as mw
    P = mw.weights(g, device="cuda")
    mm = open_model(npe, g, prec, P)
    r = {"inpainting": recovery(mm, g, P)}
    mm.close()
    return r


if __name__ == "__main__":
    run({"iters": ITERS, "prior": BETA}, measure, inpainting)

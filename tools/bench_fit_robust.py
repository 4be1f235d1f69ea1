"""(GPU) Cost and outlier recovery of the robust latent fit (ian_fit_latent_robust_*, API.IAN.fit_latent_robust) next to
the masked fit (ian_fit_latent_map_*); prints one JSON line.

    python tools/bench_fit_robust.py [--rounds 3] [--min-seconds 1.0] [--out profiles/h100_fit_robust.json]

Reported, with the card's name and power limit read in the same run:
  * per graph (IAN_simple, IANv1.py, IAN.py in float32 and bf16) at batches 1 and 32: the time of one Levenberg-Marquardt
    step of a 10-step fit_latent_robust_dev (Cauchy, automatic scale, random weights in [0, 1], prior 1e-2) and of a 10-step
    fit_latent_map_dev on the same targets, CUDA events on one stream, the two alternated over `--rounds` rounds (median and
    range), and their ratio;
  * "robust_gram" and "map_gram" per sample and "robust_scale" per fit, from ian_layer_time_ms (layer timing on);
  * on the outlier targets of tests/test_gpu_fit_robust.py (margin weights, 3 certified targets corrupted by a 16 x 16 noise
    block and 2 % salt and pepper, starts 5 % away, 20 steps, no mask, prior 0): |u - u*| / |u*| of fit_latent_map and of
    both robust losses.
Synthetic and margin weights only: nothing here says how a trained model fits a real photo.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_fit import ITERS, open_model, run, step_ms  # noqa: E402

RECOVERY_ITERS = 20
BETA = 1e-2


def fits(model, n, rng):
    """a 10-step fit_latent_robust_dev (Cauchy, automatic scale, random weights in [0, 1], prior BETA) and a 10-step
    fit_latent_map_dev on its targets"""
    st = torch.cuda.current_stream().cuda_stream
    us = rng.standard_normal((n, 100)).astype(np.float32)
    x = torch.from_numpy(model.sample(us)).cuda()
    w = torch.from_numpy(rng.uniform(0, 1, (n, 3, 64, 64)).astype(np.float32)).cuda()
    u0 = torch.from_numpy((us + 0.05 * rng.standard_normal((n, 100))).astype(np.float32)).cuda()
    u, z = torch.empty_like(u0), torch.empty_like(u0)

    def frob():
        u.copy_(u0)
        model.fit_latent_robust_dev(x.data_ptr(), w.data_ptr(), BETA, "cauchy", 0, n, u.data_ptr(), ITERS, z.data_ptr(), stream=st)

    def fmap():
        u.copy_(u0)
        model.fit_latent_map_dev(x.data_ptr(), w.data_ptr(), BETA, n, u.data_ptr(), ITERS, z.data_ptr(), 0, st)
    return {"robust": frob, "map": fmap}


def gram_ms(model, n=4):
    """per-sample ms of "robust_gram" and "map_gram" over two steps of each fit, and "robust_scale" per fit of n samples"""
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(1)
    us = rng.standard_normal((n, 100)).astype(np.float32)
    x = torch.from_numpy(model.sample(us)).cuda()
    w = torch.from_numpy(rng.uniform(0, 1, (n, 3, 64, 64)).astype(np.float32)).cuda()
    u = torch.from_numpy(us).cuda()
    model.set_layer_timing(True)
    try:
        names = ("robust_gram", "map_gram", "robust_scale")
        for name in names:
            model.layer_time_ms(name, reset=True)
        model.fit_latent_robust_dev(x.data_ptr(), w.data_ptr(), BETA, "cauchy", 0, n, u.data_ptr(), 2, stream=st)
        model.fit_latent_map_dev(x.data_ptr(), w.data_ptr(), BETA, n, u.data_ptr(), 2, 0, 0, st)
        torch.cuda.synchronize()
        out = {name: model.layer_time_ms(name, reset=True) for name in names}
        return {"robust_gram": out["robust_gram"] / (2 * n), "map_gram": out["map_gram"] / (2 * n),
                "robust_scale_per_fit": out["robust_scale"]}
    finally:
        model.set_layer_timing(False)


def recovery(model, g, P):
    import fit_map_oracle as fo
    import fit_robust_oracle as ro
    us = fo.recovery_targets(g, P)[0]
    d = np.random.default_rng(5).standard_normal(us.shape)
    u0 = (us + 0.05 * d * np.linalg.norm(us, axis=1, keepdims=True) / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    x, _ = ro.corrupt(model.sample(us), 21)
    du = lambda u: float((np.linalg.norm(u.astype(np.float64) - us, axis=1) / np.linalg.norm(us, axis=1)).max())
    out = {"map": du(model.fit_latent_map(x, None, 0.0, u0, iters=RECOVERY_ITERS)[0])}
    for kind in ro.KINDS:
        out[kind] = du(model.fit_latent_robust(x, kind, None, None, 0.0, u0, iters=RECOVERY_ITERS)[0])
    return out


def measure(m, prec, a):
    return {"step_ms": step_ms(m, a.rounds, a.min_seconds, fits), "gram_ms_per_sample": gram_ms(m)}


def outliers(npe, g, prec, a):
    if prec != "fp32":
        return {}
    import margin_weights as mw
    P = mw.weights(g, device="cuda")
    mm = open_model(npe, g, prec, P)
    r = {"outliers_du_max": recovery(mm, g, P)}
    mm.close()
    return r


if __name__ == "__main__":
    run({"iters": ITERS, "prior": BETA}, measure, outliers)

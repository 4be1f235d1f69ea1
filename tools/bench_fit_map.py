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
import argparse
import importlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import weights as ow  # noqa: E402
from bench_vjp import gpu_info, timed  # noqa: E402

CONFIG = {"simple": "IAN_simple.py", "v1": "IANv1.py", "full": "IAN.py"}
MAKE = {"simple": ow.make_simple_weights, "v1": ow.make_v1_weights, "full": ow.make_full_weights}
ITERS = 10
BETA = 1e-2


def step_ms(model, rounds, min_s):
    """{batch: {map, fit, ratio}}: ms per step of the two 10-step fits at batches 1 and 32, alternated round by round"""
    rng = np.random.default_rng(0)
    st = torch.cuda.current_stream().cuda_stream
    fns = {}
    for n in (1, 32):
        us = rng.standard_normal((n, 100)).astype(np.float32)
        x = torch.from_numpy(model.sample(us)).cuda()
        w = torch.from_numpy(rng.uniform(0, 1, (n, 3, 64, 64)).astype(np.float32)).cuda()
        u0 = torch.from_numpy((us + 0.05 * rng.standard_normal((n, 100))).astype(np.float32)).cuda()
        u, z = torch.empty_like(u0), torch.empty_like(u0)

        def fmap(n=n, x=x, w=w, u0=u0, u=u, z=z):
            u.copy_(u0)
            model.fit_latent_map_dev(x.data_ptr(), w.data_ptr(), BETA, n, u.data_ptr(), ITERS, z.data_ptr(), 0, st)

        def ffit(n=n, x=x, u0=u0, u=u):
            u.copy_(u0)
            model.fit_latent_dev(x.data_ptr(), n, u.data_ptr(), ITERS, 0, st)
        fns[(n, "map")], fns[(n, "fit")] = fmap, ffit
    reps = {}
    for k, f in fns.items():
        f()
        reps[k] = max(2, int(np.ceil(min_s / timed(f, 1))))
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            ms[k].append(timed(f, reps[k]) / reps[k] / ITERS * 1e3)
    out = {}
    for n in (1, 32):
        r = {m: {"median": float(np.median(ms[(n, m)])), "range": [float(min(ms[(n, m)])), float(max(ms[(n, m)]))]}
             for m in ("map", "fit")}
        r["ratio"] = r["map"]["median"] / r["fit"]["median"]
        out[str(n)] = r
    return out


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fit_map.py measures the GPU path and needs a CUDA device")
    import margin_weights as mw
    npe = importlib.import_module("neural-photo-editor_b200")
    res = {"gpu": gpu_info(0), "iters": ITERS, "prior": BETA}
    # a stream of its own: the legacy default stream's handle is 0, which the C-ABI reads as "the handle's own stream"
    torch.cuda.set_stream(torch.cuda.Stream())
    for g in ("simple", "v1", "full"):
        for prec in (("fp32", "bf16") if g == "full" else ("fp32",)):
            m = npe.IAN(CONFIG[g], True, weights=MAKE[g](0))
            if prec == "bf16":
                m.set_precision("bf16")
            r = {"step_ms": step_ms(m, a.rounds, a.min_seconds), "gram_ms_per_sample": gram_ms(m)}
            m.close()
            if prec == "fp32":
                P = mw.weights(g, device="cuda")
                mm = npe.IAN(CONFIG[g], True, weights=P)
                r["inpainting"] = recovery(mm, g, P)
                mm.close()
            res["%s_%s" % (g, prec)] = r
            print(g, prec, json.dumps(r), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

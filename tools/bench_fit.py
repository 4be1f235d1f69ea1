"""(GPU) Cost and convergence of the latent fit (ian_fit_latent_*, API.IAN.fit_latent); prints one JSON line.

    python tools/bench_fit.py [--rounds 3] [--min-seconds 1.0] [--out profiles/h100_fit.json]

Reported, with the card's name and power limit read in the same run:
  * per graph (IAN_simple, IANv1.py, IAN.py in float32 and bf16) at batches 1 and 32: fits/s of a 10-step fit_latent_dev
    (CUDA events on one stream, the two batches alternated over `--rounds` rounds; median and range), and the split of one
    step: the batch-100 JVP pass that gives one sample's J (decode_jvp_dev at n = 100), "gn_gram" per sample and
    "gn_solve" per batch from ian_layer_time_ms (layer timing on: plain launches, no programmatic dependent launch), and
    the trial decode at the batch size (decode_dev);
  * on the realisable targets of tests/test_gpu_fit_latent.py's recovery test (margin weights of tests/margin_weights.py,
    8 certified pool latents z*, x = sample_at(z*), starts 5 % away), the mean MSE reached against host wall time by
    fit_latent (1 to 10 steps) and by edit_steps with a whole-frame box and the target frame at NPE's weight 0.05 (1 to 256
    steps), the two methods alternated over the rounds.
Synthetic and margin weights only: nothing here says how well a trained model reproduces a photo.
"""
import argparse
import importlib
import json
import os
import sys
import time

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


def alternated(fns, rounds, min_s):
    """{key: [seconds per call, one per round]}: every fn warmed up and given enough calls per round for min_s, then all
    of them timed in turn, round by round"""
    reps = {}
    for k, f in fns.items():
        f()
        reps[k] = max(2, int(np.ceil(min_s / timed(f, 1))))
    sec = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            sec[k].append(timed(f, reps[k]) / reps[k])
    return sec


def spread(v):
    return {"median": float(np.median(v)), "range": [float(min(v)), float(max(v))]}


def step_ms(model, rounds, min_s, fits):
    """{batch: {a, b, ratio}}: ms per step of two ITERS-step fits at batches 1 and 32, alternated round by round, and the
    ratio a / b of their medians; fits(model, n, rng) -> {a: fn, b: fn} sets up both on the same targets"""
    rng = np.random.default_rng(0)
    fns = {(n, m): f for n in (1, 32) for m, f in fits(model, n, rng).items()}
    sec = alternated(fns, rounds, min_s)
    out = {}
    for n in (1, 32):
        r = {m: spread([t / ITERS * 1e3 for t in sec[(k, m)]]) for k, m in fns if k == n}
        a, b = r
        r["ratio"] = r[a]["median"] / r[b]["median"]
        out[str(n)] = r
    return out


def open_model(npe, g, prec, weights):
    m = npe.IAN(CONFIG[g], True, weights=weights)
    if prec == "bf16":
        m.set_precision("bf16")
    return m


def run(fields, measure, extra=None, after=None):
    """the command line of every bench_fit*.py.  Per graph and precision, r = measure(model, prec, args) on a model with
    seeded synthetic weights, closed before r.update(extra(npe, g, prec, args)); res = {"gpu", **fields, "<g>_<prec>": r},
    after(res), then res as one JSON line on stdout and in --out"""
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("%s measures the GPU path and needs a CUDA device" % os.path.basename(sys.argv[0]))
    npe = importlib.import_module("neural-photo-editor_b200")
    res = dict({"gpu": gpu_info(0)}, **fields)
    # a stream of its own: the legacy default stream's handle is 0, which the C-ABI reads as "the handle's own stream",
    # and the timing events must be recorded on the stream the library calls are enqueued on
    torch.cuda.set_stream(torch.cuda.Stream())
    for g in ("simple", "v1", "full"):
        for prec in (("fp32", "bf16") if g == "full" else ("fp32",)):
            m = open_model(npe, g, prec, MAKE[g](0))
            r = measure(m, prec, a)
            m.close()
            if extra:
                r.update(extra(npe, g, prec, a))
            res["%s_%s" % (g, prec)] = r
            print(g, prec, json.dumps(r), file=sys.stderr, flush=True)
    if after:
        after(res)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


def fit_rates(model, rounds, min_s):
    """{batch: fits/s} of a 10-step fit_latent_dev at batches 1 and 32, alternated round by round"""
    rng = np.random.default_rng(0)
    st = torch.cuda.current_stream().cuda_stream
    fns = {}
    for n in (1, 32):
        zs = rng.standard_normal((n, 100)).astype(np.float32)
        x = torch.from_numpy(model.sample_at(zs)).cuda()
        z0 = torch.from_numpy((zs + 0.05 * rng.standard_normal((n, 100))).astype(np.float32)).cuda()
        z = torch.empty_like(z0)

        def f(n=n, x=x, z0=z0, z=z):
            z.copy_(z0)
            model.fit_latent_dev(x.data_ptr(), n, z.data_ptr(), ITERS, 0, st)
        fns[n] = f
    return {str(n): spread([n / t for t in v]) for n, v in alternated(fns, rounds, min_s).items()}


def step_split_ms(model, n, reps=10):
    """one step's parts in ms: the JVP pass and gn_gram per sample, gn_solve per batch, the trial decode at batch n"""
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(1)
    z100 = torch.from_numpy(np.repeat(rng.standard_normal((1, 100)).astype(np.float32), 100, 0)).cuda()
    eye = torch.eye(100, device="cuda")
    J, xh = torch.empty(100, 3, 64, 64, device="cuda"), torch.empty(100, 3, 64, 64, device="cuda")
    zn = torch.from_numpy(rng.standard_normal((n, 100)).astype(np.float32)).cuda()
    xn = torch.empty(n, 3, 64, 64, device="cuda")
    jvp = lambda: model.decode_jvp_dev(z100.data_ptr(), eye.data_ptr(), 100, J.data_ptr(), xh.data_ptr(), st)
    dec = lambda: model.decode_dev(zn.data_ptr(), n, xn.data_ptr(), st)
    for f in (jvp, dec):
        f()
    out = {"jvp_pass": timed(jvp, reps) / reps * 1e3, "trial_decode": timed(dec, reps) / reps * 1e3}
    x = torch.from_numpy(model.sample_at(zn.cpu().numpy())).cuda()
    z = zn.clone()
    model.set_layer_timing(True)
    try:
        model.layer_time_ms("gn_gram", reset=True)
        model.layer_time_ms("gn_solve", reset=True)
        model.fit_latent_dev(x.data_ptr(), n, z.data_ptr(), 2, 0, st)
        torch.cuda.synchronize()
        out["gn_gram"] = model.layer_time_ms("gn_gram", reset=True)
        out["gn_solve"] = model.layer_time_ms("gn_solve", reset=True)
    finally:
        model.set_layer_timing(False)
    out["step_estimate"] = n * (out["jvp_pass"] + out["gn_gram"]) + out["gn_solve"] + out["trial_decode"]
    return out


def convergence(model, g, rounds):
    """mean MSE against host wall time (s) for fit_latent and for edit_steps on the recovery test's targets"""
    import margin_weights as mw
    p = mw.pool()
    idx = np.linspace(0, mw.POOL - 1, 8).astype(int)
    zs = p["z"][idx]
    u = np.random.default_rng(608).standard_normal((8, 100))
    u *= 0.05 * np.linalg.norm(zs, axis=1, keepdims=True) / np.linalg.norm(u, axis=1, keepdims=True)
    z0 = (zs + u).astype(np.float32)
    x = model.sample_at(zs)
    box = np.tile(np.array([[0, 0, 64, 64]], np.int32), (8, 1))
    mse = lambda z: float(np.mean((model.sample_at(z).astype(np.float64) - x) ** 2))
    runs = {"fit_latent": [(k, lambda k=k: model.fit_latent(x, z0, iters=k)) for k in (1, 2, 3, 5, 10)],
            "edit_steps": [(k, lambda k=k: model.edit_steps(z0, box, x, n_steps=k)) for k in (1, 4, 16, 64, 256)]}
    for items in runs.values():
        for _, f in items:
            f()
    times = {m: {k: [] for k, _ in items} for m, items in runs.items()}
    res = {m: {} for m in runs}
    for _ in range(rounds):
        for m, items in runs.items():
            for k, f in items:
                t0 = time.perf_counter()
                z = f()
                times[m][k].append(time.perf_counter() - t0)
                res[m][k] = mse(z)
    out = {m: [{"steps": k, "seconds": float(np.median(times[m][k])), "mse": res[m][k]} for k, _ in items]
           for m, items in runs.items()}
    out["start_mse"] = mse(z0)
    return out


def measure(m, prec, a):
    return {"fits_per_s": fit_rates(m, a.rounds, a.min_seconds), "step_ms": {str(n): step_split_ms(m, n) for n in (1, 32)}}


def recovery(npe, g, prec, a):
    import margin_weights as mw
    mm = open_model(npe, g, prec, mw.weights(g, device="cuda"))
    r = {"mse_vs_time": convergence(mm, g, a.rounds)}
    mm.close()
    return r


if __name__ == "__main__":
    run({"iters": ITERS}, measure, recovery)

"""(GPU) Cost of the latent fit under the IAN's feature-wise loss (ian_fit_latent_features_*, API.IAN.fit_latent_features)
next to the plain latent fit (ian_fit_latent_*); prints one JSON line.

    python tools/bench_fit_features.py [--rounds 3] [--min-seconds 1.0] [--out profiles/h100_fit_features.json]

Reported, with the card's name, power limit and SM clock read in the same run:
  * per graph (IAN_simple, IANv1.py, IAN.py in float32 and bf16) at batches 1 and 32: the time of one Levenberg-Marquardt
    step of a 10-step fit_latent_features_dev (pixel_weight 1, feature_weight 1) and of a 10-step fit_latent_dev on the
    same targets, CUDA events on one stream, the two alternated over `--rounds` rounds (median and range), and their ratio;
  * the split of one step per sample: the decoder JVP pass (decode_jvp_dev at batch 100), the encoder JVP pass
    (introspect_jvp_dev at batch 100), "feat_gram" (ian_layer_time_ms, layer timing on), "gn_solve" per batch, and the
    trial decode + encoder to enc_conv4 (decode_dev + introspect_dev at the batch size);
  * "feat_gram" against data-sheet bounds (none of them measured): the tangent planes it reads at 3.35 TB/s, and its
    101 * 102 / 2 * 245760 multiply-adds at 67 TFLOP/s (FP64 tensor cores) and 34 TFLOP/s (DFMA).
Synthetic weights: nothing here says how well a trained model's latent fits a real photo.
"""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_fit import ITERS, run, step_ms  # noqa: E402
from bench_vjp import timed  # noqa: E402

FEAT = 245760
MACS = 101 * 102 // 2 * FEAT


def sm_clock():
    """the SM clock now and its maximum, MHz (nvidia-smi)"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"sm_clock_mhz": float(out[0]), "sm_clock_max_mhz": float(out[1])}
    except Exception:
        return {}


def fits(model, n, rng):
    """a 10-step fit_latent_features_dev (pixel_weight 1, feature_weight 1) and a 10-step fit_latent_dev on its targets"""
    st = torch.cuda.current_stream().cuda_stream
    zs = rng.standard_normal((n, 100)).astype(np.float32)
    x = torch.from_numpy(model.sample_at(zs)).cuda()
    z0 = torch.from_numpy((zs + 0.05 * rng.standard_normal((n, 100))).astype(np.float32)).cuda()
    z = torch.empty_like(z0)

    def ffeat():
        z.copy_(z0)
        model.fit_latent_features_dev(x.data_ptr(), n, z.data_ptr(), ITERS, 0, 1.0, 1.0, st)

    def ffit():
        z.copy_(z0)
        model.fit_latent_dev(x.data_ptr(), n, z.data_ptr(), ITERS, 0, st)
    return {"features": ffeat, "fit": ffit}


def split_ms(model, n=4, reps=20):
    """ms of each part of one step, per sample (the solve and the accept per batch of n)"""
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(1)
    zs = rng.standard_normal((n, 100)).astype(np.float32)
    z100 = torch.from_numpy(np.repeat(zs[:1], 100, 0)).cuda()
    eye = torch.eye(100, device="cuda")
    J = torch.empty(100, 3, 64, 64, device="cuda")
    xh100 = torch.empty(100, 3, 64, 64, device="cuda")
    t = [torch.empty((100,) + s, device="cuda") for s in ((128, 32, 32), (256, 16, 16), (512, 8, 8), (1024, 4, 4))]
    f = [torch.empty((n,) + s, device="cuda") for s in ((128, 32, 32), (256, 16, 16), (512, 8, 8), (1024, 4, 4))]
    zn = torch.from_numpy(zs).cuda()
    xn = torch.empty(n, 3, 64, 64, device="cuda")
    dec_jvp = lambda: model.decode_jvp_dev(z100.data_ptr(), eye.data_ptr(), 100, J.data_ptr(), xh100.data_ptr(), st)
    enc_jvp = lambda: model.introspect_jvp_dev(xh100.data_ptr(), J.data_ptr(), 100, [a.data_ptr() for a in t], stream=st)

    def trial():
        model.decode_dev(zn.data_ptr(), n, xn.data_ptr(), st)
        model.introspect_dev(xn.data_ptr(), n, [a.data_ptr() for a in f], st)
    out = {}
    for name, fn, per in (("decoder_jvp_pass", dec_jvp, 1), ("encoder_jvp_pass", enc_jvp, 1), ("trial_decode_encode", trial, n)):
        fn()
        out[name] = timed(fn, reps) / reps * 1e3 / per
    x = torch.from_numpy(model.sample_at(zs)).cuda()
    model.set_layer_timing(True)
    try:
        for name in ("feat_gram", "gn_solve", "feat_accept"):
            model.layer_time_ms(name, reset=True)
        model.fit_latent_features_dev(x.data_ptr(), n, zn.data_ptr(), 2, 0, 1.0, 1.0, st)
        torch.cuda.synchronize()
        for name in ("feat_gram", "gn_solve", "feat_accept"):
            model.layer_time_ms(name, reset=True)
        model.fit_latent_features_dev(x.data_ptr(), n, zn.data_ptr(), 2, 0, 1.0, 1.0, st)
        torch.cuda.synchronize()
        # ian_layer_time_ms: the mean over the timed launches -- feat_gram once per sample, the others once per batch
        out["feat_gram"] = model.layer_time_ms("feat_gram", reset=True)
        out["gn_solve_per_batch"] = model.layer_time_ms("gn_solve", reset=True)
        out["feat_accept_per_batch"] = model.layer_time_ms("feat_accept", reset=True)
    finally:
        model.set_layer_timing(False)
    return out


def measure(m, prec, a):
    r = {"step_ms": step_ms(m, a.rounds, a.min_seconds, fits), "split_ms": split_ms(m)}
    planes = 2 if prec == "fp32" else 1
    r["feat_gram_bounds_ms"] = {"hbm_3.35TBps": 100 * FEAT * 2 * planes / 3.35e12 * 1e3,
                                "fp64_tensor_67TFLOPs": 2 * MACS / 67e12 * 1e3, "dfma_34TFLOPs": 2 * MACS / 34e12 * 1e3}
    r["feat_gram_fp64_tflops"] = 2 * MACS / (r["split_ms"]["feat_gram"] * 1e-3) / 1e12
    return r


if __name__ == "__main__":
    # the SM clock is sampled right after the timed work
    run({"iters": ITERS, "pixel_weight": 1.0, "feature_weight": 1.0}, measure, after=lambda res: res["gpu"].update(sm_clock()))

"""(GPU) Cost of the encoder vector-Jacobian product against a reconstruct at the same batch; prints one JSON line.

    python tools/bench_encode_vjp.py [--batch 256] [--flow-batch 128] [--rounds 3] [--min-seconds 1.0] [--out FILE]

An encoder VJP runs the encoder forward and then its adjoint: five backward tap-GEMMs whose shapes are the decoder's
(conv4^T like dec_conv1, conv3^T like dec_conv2, conv2^T like dec_conv3), plus enc_conv1's adjoint with dec_out's geometry.
A reconstruct runs the encoder forward and the decoder, so the two calls do about the same work.  Each comparison
alternates the two calls over `--rounds` rounds of at least `--min-seconds` each (device-pointer entry points, CUDA
events on one stream) and reports the median and min-max range of samples/s.  Also: per-layer times of the backward
GEMMs next to their decoder twins in the same run (layer timing on), IAN.py in float32 and bf16, the batch-1 host latency
of encode_vjp against encode, and the card's name and power limit.
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

from oracle import weights as ow  # noqa: E402
from bench_vjp import alternate, gpu_info  # noqa: E402

BWD_LAYERS = ["bwd_enc_head", "bwd_enc_fc1", "bwd_enc_conv4", "bwd_enc_conv3", "bwd_enc_conv2", "enc_conv1_bwd"]
TWINS = {"bwd_enc_conv4": "dec_conv1", "bwd_enc_conv3": "dec_conv2", "bwd_enc_conv2": "dec_conv3"}


def layer_times(model, fns, names, reps=20):
    out = {}
    model.set_layer_timing(True)
    try:
        for f in fns:
            for nm in names:
                model.layer_time_ms(nm, reset=True)
            for _ in range(reps):
                f()
            torch.cuda.synchronize()
            for nm in names:
                t = model.layer_time_ms(nm, reset=True)
                if t >= 0:
                    out[nm] = t
    finally:
        model.set_layer_timing(False)
    return out


def vjp_vs_reconstruct(model, n, rounds, min_s, twins=True):
    rng = np.random.default_rng(0)
    x = torch.from_numpy(np.tanh(rng.standard_normal((n, 3, 64, 64))).astype(np.float32)).cuda()
    dz = torch.from_numpy(rng.standard_normal((n, 100)).astype(np.float32)).cuda()
    dx, xh = torch.empty_like(x), torch.empty_like(x)
    st = torch.cuda.current_stream().cuda_stream
    fns = {"encode_vjp": lambda: model.encode_vjp_dev(x.data_ptr(), dz.data_ptr(), n, dx.data_ptr(), 0, st),
           "reconstruct": lambda: model.reconstruct_dev(x.data_ptr(), n, 0, xh.data_ptr(), st)}
    r = alternate(fns, n, rounds, min_s)
    out = {"batch": n, "samples_per_s": r, "time_ratio_vjp_over_reconstruct": r["reconstruct"]["median"] / r["encode_vjp"]["median"]}
    names = BWD_LAYERS + ["enc_conv1", "enc_conv2", "enc_conv3", "enc_conv4", "enc_fc1", "enc_head"]
    if twins:
        names += list(TWINS.values())
    lt = layer_times(model, list(fns.values()), names)
    out["layer_ms"] = lt
    if twins:
        out["bwd_over_twin"] = {k: lt[k] / lt[v] for k, v in TWINS.items() if k in lt and v in lt}
    return out


def host_latency_ms(model, reps=200):
    rng = np.random.default_rng(1)
    x = np.tanh(rng.standard_normal((1, 3, 64, 64))).astype(np.float32)
    dz = rng.standard_normal((1, 100)).astype(np.float32)
    fns = {"encode_vjp": lambda: model.encode_vjp(x, dz), "encode": lambda: model.encode(x)}
    out = {}
    for k, f in fns.items():
        for _ in range(10):
            f()
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            for _ in range(reps):
                f()
            ts.append((time.perf_counter() - t0) / reps * 1e3)
        out[k] = float(np.median(ts))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--flow-batch", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_encode_vjp.py measures the GPU path and needs a CUDA device")
    npe = importlib.import_module("neural-photo-editor_b200")
    res = {"gpu": gpu_info(0)}
    # a stream of its own: handle 0 means "the handle's own stream" to the C-ABI, and the events must share the stream
    torch.cuda.set_stream(torch.cuda.Stream())
    simple = npe.IAN("IAN_simple.py", True, weights=ow.make_simple_weights(0))
    res["ian_simple"] = vjp_vs_reconstruct(simple, a.batch, a.rounds, a.min_seconds)
    print("ian_simple", json.dumps(res["ian_simple"]), file=sys.stderr, flush=True)
    res["ian_simple"]["batch1_host_latency_ms"] = host_latency_ms(simple)
    simple.close()
    full = npe.IAN("IAN.py", True, weights=ow.make_full_weights(0))
    res["ian_full"] = {}
    for prec in ("fp32", "bf16"):
        full.set_precision(prec)
        res["ian_full"][prec] = vjp_vs_reconstruct(full, a.flow_batch, a.rounds, a.min_seconds, twins=False)
        print("ian_full", prec, json.dumps(res["ian_full"][prec]), file=sys.stderr, flush=True)
    full.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

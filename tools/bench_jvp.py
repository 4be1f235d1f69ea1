"""(GPU) Cost of the decoder Jacobian-vector product against a decode and a decoder VJP; prints one JSON line.

    python tools/bench_jvp.py [--rounds 3] [--min-seconds 1.0] [--out FILE]

Method of tools/bench_vjp.py: device-pointer entry points on one stream, CUDA events, the calls compared alternated over
`--rounds` rounds of at least `--min-seconds` each, median and min-max range of samples/s.  Reported:
  * decode_jvp_dev against decode_dev and decode_vjp_dev, IAN_simple at batches 128 and 256, IAN.py at 128 in float32 and
    bf16 precision;
  * per layer, the tangent tap-GEMM ("jvp_<layer>") against its forward twin, from ian_layer_time_ms in the same calls
    (layer timing on: plain launches, no programmatic dependent launch), and the JVP's edge kernels;
  * the host latency of decoder_jacobian for one z (one batch-100 JVP).
The card's name and power limit are read in the same run.
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

FWD = {"simple": ["l_dec_fc2", "dec_conv1", "dec_conv2", "dec_conv3"],
       "full": ["full_dec_fc2", "full_dec_conv1", "dec_conv2a", "dec_conv2a2", "full_dec_conv2", "dec_conv3a", "dec_conv3a2",
                "full_dec_conv3", "dec_conv4a", "dec_conv4a2", "full_dec_conv4"]}
EDGE = {"simple": [("dec_out", "dec_out_jvp")], "full": [("rgb_head", "rgb_head_jvp")]}


def three_calls(model, n, rounds, min_s):
    rng = np.random.default_rng(0)
    z = torch.from_numpy(rng.standard_normal((n, 100)).astype(np.float32)).cuda()
    v = torch.from_numpy(rng.standard_normal((n, 100)).astype(np.float32)).cuda()
    u = torch.from_numpy(rng.standard_normal((n, 3, 64, 64)).astype(np.float32)).cuda()
    x, dx, dz = (torch.empty(n, 3, 64, 64, device="cuda"), torch.empty(n, 3, 64, 64, device="cuda"),
                 torch.empty(n, 100, device="cuda"))
    st = torch.cuda.current_stream().cuda_stream
    fns = {"decode": lambda: model.decode_dev(z.data_ptr(), n, x.data_ptr(), st),
           "decode_jvp": lambda: model.decode_jvp_dev(z.data_ptr(), v.data_ptr(), n, dx.data_ptr(), 0, st),
           "decode_vjp": lambda: model.decode_vjp_dev(z.data_ptr(), u.data_ptr(), n, dz.data_ptr(), st)}
    r = alternate(fns, n, rounds, min_s)
    return fns, {"batch": n, "samples_per_s": r,
                 "time_ratio_jvp_over_decode": r["decode"]["median"] / r["decode_jvp"]["median"],
                 "time_ratio_jvp_over_vjp": r["decode_vjp"]["median"] / r["decode_jvp"]["median"]}


def layer_ms(model, fn, graph, reps=20):
    """{layer: [forward ms, tangent ms, tangent / forward]} from the same decode_jvp calls"""
    names = [(f, "jvp_" + f) for f in FWD[graph]] + EDGE[graph]
    model.set_layer_timing(True)
    try:
        for f, t in names:
            model.layer_time_ms(f, reset=True)
            model.layer_time_ms(t, reset=True)
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        out = {}
        for f, t in names:
            a, b = model.layer_time_ms(f, reset=True), model.layer_time_ms(t, reset=True)
            out[f] = [a, b, b / a if a > 0 else None]
        return out
    finally:
        model.set_layer_timing(False)


def jacobian_latency_ms(model, reps=20):
    z = np.random.default_rng(1).standard_normal((1, 100)).astype(np.float32)
    for _ in range(3):
        model.decoder_jacobian(z)
    ts = []
    for _ in range(3):
        t0 = time.perf_counter()
        for _ in range(reps):
            model.decoder_jacobian(z)
        ts.append((time.perf_counter() - t0) / reps * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jvp.py measures the GPU path and needs a CUDA device")
    npe = importlib.import_module("neural-photo-editor_b200")
    res = {"gpu": gpu_info(0)}
    # a stream of its own: the legacy default stream's handle is 0, which the C-ABI reads as "the handle's own stream",
    # and the timing events must be recorded on the stream the library calls are enqueued on
    torch.cuda.set_stream(torch.cuda.Stream())
    simple = npe.IAN("IAN_simple.py", True, weights=ow.make_simple_weights(0))
    res["ian_simple"] = {}
    for n in (128, 256):
        fns, r = three_calls(simple, n, a.rounds, a.min_seconds)
        r["layer_ms"] = layer_ms(simple, fns["decode_jvp"], "simple")
        res["ian_simple"][str(n)] = r
        print("ian_simple", n, json.dumps(r), file=sys.stderr, flush=True)
    res["ian_simple"]["decoder_jacobian_latency_ms"] = jacobian_latency_ms(simple)
    simple.close()
    full = npe.IAN("IAN.py", True, weights=ow.make_full_weights(0))
    res["ian_full"] = {}
    for prec in ("fp32", "bf16"):
        full.set_precision(prec)
        fns, r = three_calls(full, 128, a.rounds, a.min_seconds)
        r["layer_ms"] = layer_ms(full, fns["decode_jvp"], "full")
        res["ian_full"][prec] = r
        print("ian_full", prec, json.dumps(r), file=sys.stderr, flush=True)
    full.set_precision("fp32")
    res["ian_full"]["decoder_jacobian_latency_ms"] = jacobian_latency_ms(full)
    full.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

"""(GPU) Cost of the encoder Jacobian-vector product against an encode and an encoder VJP; prints one JSON line.

    python tools/bench_encode_jvp.py [--rounds 3] [--min-seconds 1.0] [--out FILE]

Method of tools/bench_jvp.py: device-pointer entry points on one stream, CUDA events, the calls compared alternated over
`--rounds` rounds of at least `--min-seconds` each, median and min-max range of samples/s.  Reported:
  * encode_jvp_dev against encode_dev and encode_vjp_dev at batches 1 and 128, on IAN_simple, IANv1.py, and IAN.py in
    float32 and bf16 precision;
  * per layer at batch 128, the tangent ("jvp_<layer>", "jvp_enc_conv1") against its forward twin, from
    ian_layer_time_ms in the same calls (layer timing on: plain launches, no programmatic dependent launch).
The card's name and power limit are read in the same run.
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

from oracle import weights as ow  # noqa: E402
from bench_vjp import alternate, gpu_info  # noqa: E402

LAYERS = ["enc_conv1", "enc_conv2", "enc_conv3", "enc_conv4", "enc_fc1", "enc_head"]


def three_calls(model, n, rounds, min_s):
    rng = np.random.default_rng(0)
    x = torch.from_numpy(np.tanh(rng.standard_normal((n, 3, 64, 64))).astype(np.float32)).cuda()
    v = torch.from_numpy(rng.standard_normal((n, 3, 64, 64)).astype(np.float32)).cuda()
    u = torch.from_numpy(rng.standard_normal((n, 100)).astype(np.float32)).cuda()
    z, dz, dx = torch.empty(n, 100, device="cuda"), torch.empty(n, 100, device="cuda"), torch.empty(n, 3, 64, 64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    fns = {"encode": lambda: model.encode_dev(x.data_ptr(), n, z.data_ptr(), 0, st),
           "encode_jvp": lambda: model.encode_jvp_dev(x.data_ptr(), v.data_ptr(), n, dz.data_ptr(), 0, 0, st),
           "encode_vjp": lambda: model.encode_vjp_dev(x.data_ptr(), u.data_ptr(), n, dx.data_ptr(), 0, st)}
    r = alternate(fns, n, rounds, min_s)
    return fns, {"batch": n, "samples_per_s": r,
                 "time_ratio_jvp_over_encode": r["encode"]["median"] / r["encode_jvp"]["median"],
                 "time_ratio_jvp_over_vjp": r["encode_vjp"]["median"] / r["encode_jvp"]["median"]}


def layer_ms(model, fn, reps=20):
    """{layer: [forward ms, tangent ms, tangent / forward]} from the same encode_jvp calls"""
    names = [(f, "jvp_" + f) for f in LAYERS]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_encode_jvp.py measures the GPU path and needs a CUDA device")
    npe = importlib.import_module("neural-photo-editor_b200")
    res = {"gpu": gpu_info(0)}
    # a stream of its own: the legacy default stream's handle is 0, which the C-ABI reads as "the handle's own stream",
    # and the timing events must be recorded on the stream the library calls are enqueued on
    torch.cuda.set_stream(torch.cuda.Stream())
    cases = [("ian_simple", "IAN_simple.py", ow.make_simple_weights, ["fp32"]),
             ("ian_v1", "IANv1.py", ow.make_v1_weights, ["fp32"]),
             ("ian_full", "IAN.py", ow.make_full_weights, ["fp32", "bf16"])]
    for key, config, make, precs in cases:
        m = npe.IAN(config, True, weights=make(0))
        res[key] = {}
        for prec in precs:
            if prec != "fp32":
                m.set_precision(prec)
            for n in (1, 128):
                fns, r = three_calls(m, n, a.rounds, a.min_seconds)
                if n == 128:
                    r["layer_ms"] = layer_ms(m, fns["encode_jvp"])
                res[key]["%s_%d" % (prec, n)] = r
                print(key, prec, n, json.dumps(r), file=sys.stderr, flush=True)
        m.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

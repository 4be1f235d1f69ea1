"""(GPU) Cost of the IAN_simple decoder's parameter VJP against the decoder VJP and the decoder forward; prints one JSON line.

    python tools/bench_param_vjp.py [--batches 128,256] [--rounds 3] [--min-seconds 1.0] [--out FILE]

Per batch size, decode_param_vjp_dev (all 13 gradients), decode_vjp_dev and decode_dev are alternated over `--rounds`
rounds of at least `--min-seconds` each (device pointers, CUDA events on one stream); the median and min-max range of
samples/s are reported.  With layer timing on, each weight-gradient kernel (ian_layer_time_ms("wgrad_*")) is set against
its forward twin in the same call, with its achieved rate: the algorithmic MACs equal the forward layer's, over the
data-sheet dense bf16 rate / 3 (three bf16 products per float32 MAC).  Then the same for the SIMT path's wgrad kernels.
The card's name and power limit are read in the same run.
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import weights as ow  # noqa: E402

BF16_DENSE_TFLOPS = 989.0                      # H100 SXM data sheet, dense, at a 700 W limit
# per image: (wgrad slot, forward twin, MACs)
LAYERS = [("wgrad_l_dec_fc2", "l_dec_fc2", 100 * 16384), ("wgrad_dec_conv1", "dec_conv1", 1024 * 512 * 25 * 16),
          ("wgrad_dec_conv2", "dec_conv2", 512 * 256 * 25 * 64), ("wgrad_dec_conv3", "dec_conv3", 256 * 128 * 25 * 256),
          ("wgrad_dec_out", "dec_out", 128 * 3 * 25 * 1024)]


def gpu_info(index=0):
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out)
    except Exception:
        pass
    return info


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / 1e3


def alternate(fns, n, rounds, min_s):
    reps = {}
    for k, f in fns.items():
        for _ in range(3):
            f()
        reps[k] = min(10000, max(3, int(np.ceil(min_s / (timed(f, 3) / 3)))))
    rates = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            rates[k].append(n * reps[k] / timed(f, reps[k]))
    return {k: {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))} for k, v in rates.items()}


def layer_times(m, call, names, reps=5):
    m.set_layer_timing(True)
    for nm in names:
        m.layer_time_ms(nm, reset=True)
    for _ in range(reps):
        call()
    torch.cuda.synchronize()
    out = {nm: m.layer_time_ms(nm, reset=True) for nm in names}
    m.set_layer_timing(False)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="128,256")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--out")
    a = ap.parse_args()
    npe = importlib.import_module("neural-photo-editor_b200")
    m = npe.IAN("IAN_simple.py", True, weights=ow.make_simple_weights(0))
    names = m.param_vjp_names()
    side = torch.cuda.Stream()                 # a real stream handle: 0 would select the library's own stream
    torch.cuda.set_stream(side)
    st = side.cuda_stream
    res = {"gpu": gpu_info(), "batches": {}}
    for n in [int(b) for b in a.batches.split(",")]:
        g = torch.Generator(device="cuda").manual_seed(n)
        z = torch.randn((n, 100), device="cuda", generator=g)
        dx = torch.randn((n, 3, 64, 64), device="cuda", generator=g)
        dz = torch.empty((n, 100), device="cuda")
        xh = torch.empty((n, 3, 64, 64), device="cuda")
        from_api = importlib.import_module("neural-photo-editor_b200.API").model_param_specs(m.kind)
        grads = {k: torch.empty(shape, device="cuda") for k, shape in from_api if k in names}
        ptrs = {k: v.data_ptr() for k, v in grads.items()}
        fns = {"decode_param_vjp": lambda: m.decode_param_vjp_dev(z.data_ptr(), dx.data_ptr(), n, dz.data_ptr(), ptrs, st),
               "decode_vjp": lambda: m.decode_vjp_dev(z.data_ptr(), dx.data_ptr(), n, dz.data_ptr(), st),
               "decode": lambda: m.decode_dev(z.data_ptr(), n, xh.data_ptr(), st)}
        r = {"samples_per_s": alternate(fns, n, a.rounds, a.min_seconds)}
        r["param_vjp_over_vjp"] = r["samples_per_s"]["decode_vjp"]["median"] / r["samples_per_s"]["decode_param_vjp"]["median"]
        for path in ("tc", "simt"):
            m.set_path(path)
            t = layer_times(m, fns["decode_param_vjp"], [x for l in LAYERS for x in l[:2]])
            r["layers_" + path] = {
                w: {"ms": t[w], "forward_ms": t[f], "over_forward": t[w] / t[f] if t[f] > 0 else None,
                    "tflops": 2 * macs * n / (t[w] * 1e-3) / 1e12,
                    "of_bf16_over_3": 2 * macs * n / (t[w] * 1e-3) / 1e12 / (BF16_DENSE_TFLOPS / 3)}
                for w, f, macs in LAYERS}
        m.set_path("tc")
        res["batches"][str(n)] = r
    m.close()
    line = json.dumps(res, sort_keys=True)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

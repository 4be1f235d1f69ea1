"""(GPU) Cost of the prior-space derivatives; prints one JSON line.

    python tools/bench_flow_grad.py [--rounds 3] [--min-seconds 0.5] [--out FILE]

Method of tools/bench_jvp.py: device-pointer entry points on one stream, CUDA events, the calls compared alternated over
`--rounds` rounds of at least `--min-seconds` each, median and min-max range of samples/s.  Reported at batches 1, 32, 128
and 512, on IAN.py and IANv1.py, in float32 and bf16 precision:
  * flow_vjp_dev and flow_jvp_dev against flow_dev (Z_IAF_fn);
  * encode_pre_vjp_dev / encode_pre_jvp_dev against encode_vjp_dev / encode_jvp_dev.
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

BATCHES = (1, 32, 128, 512)


def calls(model, n, rounds, min_s):
    rng = np.random.default_rng(0)
    t = lambda a: torch.from_numpy(a.astype(np.float32)).cuda()
    x = t(np.tanh(rng.standard_normal((n, 3, 64, 64))))
    v = t(rng.standard_normal((n, 3, 64, 64)))
    zi, u, vz = (t(rng.standard_normal((n, 100))) for _ in range(3))
    z, dz, dx = torch.empty(n, 100, device="cuda"), torch.empty(n, 100, device="cuda"), torch.empty(n, 3, 64, 64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    flow = {"flow": lambda: model.flow_dev(zi.data_ptr(), n, z.data_ptr(), 0, st),
            "flow_vjp": lambda: model.flow_vjp_dev(zi.data_ptr(), u.data_ptr(), n, dz.data_ptr(), st),
            "flow_jvp": lambda: model.flow_jvp_dev(zi.data_ptr(), vz.data_ptr(), n, dz.data_ptr(), 0, st)}
    enc = {"encode_vjp": lambda: model.encode_vjp_dev(x.data_ptr(), u.data_ptr(), n, dx.data_ptr(), 0, st),
           "encode_pre_vjp": lambda: model.encode_pre_vjp_dev(x.data_ptr(), u.data_ptr(), n, dx.data_ptr(), st),
           "encode_jvp": lambda: model.encode_jvp_dev(x.data_ptr(), v.data_ptr(), n, dz.data_ptr(), 0, 0, st),
           "encode_pre_jvp": lambda: model.encode_pre_jvp_dev(x.data_ptr(), v.data_ptr(), n, dz.data_ptr(), 0, st)}
    rf = alternate(flow, n, rounds, min_s)
    re = alternate(enc, n, rounds, min_s)
    med = lambda r, k: r[k]["median"]
    return {"batch": n, "samples_per_s": dict(rf, **re),
            "time_ratio_flow_vjp_over_flow": med(rf, "flow") / med(rf, "flow_vjp"),
            "time_ratio_flow_jvp_over_flow": med(rf, "flow") / med(rf, "flow_jvp"),
            "time_ratio_pre_vjp_over_encode_vjp": med(re, "encode_vjp") / med(re, "encode_pre_vjp"),
            "time_ratio_pre_jvp_over_encode_jvp": med(re, "encode_jvp") / med(re, "encode_pre_jvp")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_flow_grad.py measures the GPU path and needs a CUDA device")
    npe = importlib.import_module("neural-photo-editor_b200")
    res = {"gpu": gpu_info(0)}
    # a stream of its own: the legacy default stream's handle is 0, which the C-ABI reads as "the handle's own stream"
    torch.cuda.set_stream(torch.cuda.Stream())
    for key, config, make in (("ian_full", "IAN.py", ow.make_full_weights), ("ian_v1", "IANv1.py", ow.make_v1_weights)):
        m = npe.IAN(config, True, weights=make(0))
        res[key] = {}
        for prec in ("fp32", "bf16"):
            m.set_precision(prec)
            for n in BATCHES:
                r = calls(m, n, a.rounds, a.min_seconds)
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

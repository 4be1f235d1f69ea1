"""(GPU) Cost of the IAN_simple decoder in training mode: ian_decode_train_dev and ian_decode_train_vjp_dev (all 13
gradients and dz) next to the inference decoder ian_decode_dev and its parameter VJP ian_decode_param_vjp_dev, in one run;
prints one JSON line.

    python tools/bench_decode_train.py [--rounds 3] [--min-seconds 1.0] [--out profiles/h100_decode_train.json]

Reported, with the card's name, power limit and SM clock read in the same run:
  * at batches 16, 128 and 256: samples/s of the four calls, alternated over `--rounds` rounds (median and range);
  * the device memory the first training-mode forward and VJP allocate at n = 256, on top of what decode and
    decode_param_vjp allocated at that batch before them (cudaMemGetInfo deltas), per image.
Synthetic weights: the cost does not depend on the weights' values.
"""
import argparse
import importlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from oracle import weights as ow  # noqa: E402
from bench_fit_features import sm_clock  # noqa: E402
from bench_vjp import alternate, gpu_info  # noqa: E402

BATCHES = (16, 128, 256)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    npe = importlib.import_module("neural-photo-editor_b200")
    P = ow.make_simple_weights(0)
    m = npe.IAN("IAN_simple.py", True, weights=P)
    names = m.param_vjp_names()
    rng = np.random.default_rng(0)
    res = {"gpu": gpu_info(), "batches": {}}
    try:
        for n in BATCHES:
            z = torch.from_numpy(rng.standard_normal((n, 100)).astype(np.float32)).cuda()
            dx = torch.from_numpy(rng.standard_normal((n, 3, 64, 64)).astype(np.float32)).cuda()
            x = torch.empty((n, 3, 64, 64), device="cuda")
            dz = torch.empty((n, 100), device="cuda")
            grads = {k: torch.empty(tuple(s), device="cuda") for k, s in ow_shapes(P, names).items()}
            ptrs = {k: v.data_ptr() for k, v in grads.items()}
            st = torch.cuda.current_stream().cuda_stream
            fns = {"decode": lambda: m.decode_dev(z.data_ptr(), n, x.data_ptr(), st),
                   "decode_param_vjp": lambda: m.decode_param_vjp_dev(z.data_ptr(), dx.data_ptr(), n, dz.data_ptr(), ptrs, st),
                   "decode_train": lambda: m.decode_train_dev(z.data_ptr(), n, x.data_ptr(), 0, st),
                   "decode_train_vjp": lambda: m.decode_train_vjp_dev(z.data_ptr(), dx.data_ptr(), n, dz.data_ptr(), ptrs, st)}
            if n == BATCHES[-1]:
                mem = {}
                for k, f in fns.items():
                    torch.cuda.synchronize()
                    free0 = torch.cuda.mem_get_info()[0]
                    f()
                    torch.cuda.synchronize()
                    mem[k] = (free0 - torch.cuda.mem_get_info()[0]) / n / 2**20
                res["first_call_alloc_mb_per_image_n256"] = mem
            res["batches"][str(n)] = alternate(fns, n, a.rounds, a.min_seconds)
        res["sm_clock_mhz"] = sm_clock()
    finally:
        m.close()
    line = json.dumps(res, sort_keys=True)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


def ow_shapes(P, names):
    return {k: np.shape(P[k]) for k in names}


if __name__ == "__main__":
    main()

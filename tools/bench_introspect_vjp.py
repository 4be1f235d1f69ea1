"""(GPU) Cost of the introspection features' vector-Jacobian product (ian_introspect_vjp_dev, API.IAN.introspect_vjp_dev)
next to the encoder VJP (ian_encode_vjp_dev); prints one JSON line.

    python tools/bench_introspect_vjp.py [--rounds 3] [--min-seconds 1.0] [--out profiles/h100_introspect_vjp.json]

Reported, with the card's name, power limit and SM clock read in the same run:
  * per graph (IAN_simple, IANv1.py, IAN.py in float32 and bf16) at batches 1, 32 and 256: samples/s of introspect_vjp with
    all four cotangents, with c1 alone (the forward stops after enc_conv1 and no backward GEMM runs) and of encode_vjp,
    the three alternated over `--rounds` rounds (median and range);
  * at batch 256, ian_layer_time_ms of every kernel of the all-four chain, and "feat_cotangent" against its HBM bound at
    3.35 TB/s (data sheet, not measured): the float32 cotangents it reads, the bf16 split planes it writes and the a4 mask
    it reads, bytes computed from the shapes below;
  * one torch step of feature_loss(decode(z), x).sum().backward() at batch 128 (forward and backward, CUDA events).
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
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from oracle import weights as ow  # noqa: E402
from bench_fit_features import sm_clock  # noqa: E402
from bench_vjp import alternate, gpu_info, timed  # noqa: E402

CONFIG = {"simple": "IAN_simple.py", "v1": "IANv1.py", "full": "IAN.py"}
MAKE = {"simple": ow.make_simple_weights, "v1": ow.make_v1_weights, "full": ow.make_full_weights}
SHAPES = ((128, 32, 32), (256, 16, 16), (512, 8, 8), (1024, 4, 4))
ELEMS = [c * h * w for c, h, w in SHAPES]
CHAIN = ("enc_conv1", "enc_conv2", "enc_conv3", "enc_conv4", "feat_cotangent", "introspect_bwd_enc_conv4",
         "introspect_bwd_enc_conv3", "introspect_bwd_enc_conv2", "enc_conv1_bwd")


def cotangent_bytes():
    """per image: the four float32 cotangents read, both bf16 planes of their split written, and a4's hi plane read as the
    deepest layer's mask.  In bf16 mode the deepest layer's lo plane is written only where its GEMM's split-K finalize
    would write it, so there this is an upper bound"""
    return sum(ELEMS) * 4 + sum(ELEMS) * 2 * 2 + ELEMS[3] * 2


def rates(model, rounds, min_s):
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(0)
    out = {}
    for n in (1, 32, 256):
        x = torch.from_numpy(rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)).cuda()
        c = [torch.from_numpy(rng.standard_normal((n,) + s).astype(np.float32)).cuda() for s in SHAPES]
        dz = torch.from_numpy(rng.standard_normal((n, 100)).astype(np.float32)).cuda()
        dx = torch.empty_like(x)
        fns = {
            "introspect_vjp": lambda n=n, x=x, c=c, dx=dx: model.introspect_vjp_dev(x.data_ptr(), n, [a.data_ptr() for a in c],
                                                                                    dx.data_ptr(), st),
            "introspect_vjp_c1": lambda n=n, x=x, c=c, dx=dx: model.introspect_vjp_dev(x.data_ptr(), n, [c[0].data_ptr(), 0, 0, 0],
                                                                                       dx.data_ptr(), st),
            "encode_vjp": lambda n=n, x=x, dz=dz, dx=dx: model.encode_vjp_dev(x.data_ptr(), dz.data_ptr(), n, dx.data_ptr(), 0, st),
        }
        r = alternate(fns, n, rounds, min_s)
        r["ratio_introspect_vjp_to_encode_vjp"] = r["introspect_vjp"]["median"] / r["encode_vjp"]["median"]
        out[str(n)] = r
    return out


def layers(model, n=256, reps=20):
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(1)
    x = torch.from_numpy(rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)).cuda()
    c = [torch.from_numpy(rng.standard_normal((n,) + s).astype(np.float32)).cuda() for s in SHAPES]
    dx = torch.empty_like(x)
    call = lambda: model.introspect_vjp_dev(x.data_ptr(), n, [a.data_ptr() for a in c], dx.data_ptr(), st)
    call()
    model.set_layer_timing(True)
    try:
        for name in CHAIN:
            model.layer_time_ms(name, reset=True)
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
        ms = {name: model.layer_time_ms(name, reset=True) for name in CHAIN}
    finally:
        model.set_layer_timing(False)
    bound = n * cotangent_bytes() / 3.35e12 * 1e3
    return {"batch": n, "layer_ms": ms, "feat_cotangent_bytes": n * cotangent_bytes(),
            "feat_cotangent_hbm_bound_ms": bound, "feat_cotangent_share_of_hbm_bound": bound / ms["feat_cotangent"]}


def torch_step(model, n=128, reps=10):
    ops = importlib.import_module("neural-photo-editor_b200.torch_ops")
    rng = np.random.default_rng(2)
    z = torch.from_numpy(rng.standard_normal((n, 100)).astype(np.float32)).cuda().requires_grad_(True)
    x = torch.from_numpy(rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)).cuda()

    def step():
        z.grad = None
        ops.feature_loss(model, ops.decode(model, z), x).sum().backward()
    step()
    torch.cuda.synchronize()
    return {"batch": n, "ms": timed(step, reps) / reps * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_introspect_vjp.py measures the GPU path and needs a CUDA device")
    npe = importlib.import_module("neural-photo-editor_b200")
    res = {"gpu": gpu_info(0)}
    # a stream of its own: the legacy default stream's handle is 0, which the C-ABI reads as "the handle's own stream"
    torch.cuda.set_stream(torch.cuda.Stream())
    for g in ("simple", "v1", "full"):
        for prec in (("fp32", "bf16") if g == "full" else ("fp32",)):
            m = npe.IAN(CONFIG[g], True, weights=MAKE[g](0))
            if prec == "bf16":
                m.set_precision("bf16")
            r = {"samples_per_s": rates(m, a.rounds, a.min_seconds), "layers": layers(m),
                 "torch_feature_loss_step": torch_step(m)}
            m.close()
            res["%s_%s" % (g, prec)] = r
            print(g, prec, json.dumps(r), file=sys.stderr, flush=True)
    res["gpu"].update(sm_clock())                          # sampled right after the timed work
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

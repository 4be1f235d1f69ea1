"""(GPU) Cost of the discriminator head l_discrim: ian_discriminate_dev and ian_discriminate_vjp_dev next to the
introspection features (ian_introspect_dev, the same trunk); prints one JSON line.

    python tools/bench_discriminate.py [--rounds 3] [--min-seconds 1.0] [--out profiles/h100_discriminate.json]
    python tools/bench_discriminate.py --training [--out profiles/h100_discriminate_train.json]

Reported, with the card's name, power limit and SM clock read in the same run:
  * per graph (IAN_simple, IANv1.py, IAN.py in float32 and bf16) at batches 16, 128 and 256: samples/s of discriminate, of
    discriminate_vjp and of introspect (the trunk alone), the three alternated over `--rounds` rounds (median and range);
  * at each batch, ian_layer_time_ms of the head's kernels (disc_pool, disc_mb, disc_head; disc_head_bwd, disc_mb_bwd,
    disc_cotangent in the VJP) and of the trunk's, and the head's share of the summed kernel time: the MinibatchLayer's
    pair terms grow as n^2, the trunk as n.
With --training, the training-mode entries (ian_discriminate_train_dev, ian_discriminate_train_vjp_dev) are alternated
with the inference ones at batches 16 and 256, and each phase's device time per call is reported: the trunk's layers with
their raw-sum twins, the batch statistics, the normalisation, the head, and in the VJP the BatchNorm backward and the
backward twins.
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

from oracle import weights as ow  # noqa: E402
from bench_fit_features import sm_clock  # noqa: E402
from bench_vjp import alternate, gpu_info  # noqa: E402
import discrim_oracle as do  # noqa: E402

CONFIG = {"simple": "IAN_simple.py", "v1": "IANv1.py", "full": "IAN.py"}
MAKE = {"simple": ow.make_simple_weights, "v1": ow.make_v1_weights, "full": ow.make_full_weights}
TRUNK = ("enc_conv1", "enc_conv2", "enc_conv3", "enc_conv4")
TRUNK_BWD = ("feat_cotangent", "bwd_enc_conv4", "bwd_enc_conv3", "bwd_enc_conv2", "enc_conv1_bwd")
HEAD = ("disc_pool", "disc_mb", "disc_head")
HEAD_BWD = ("disc_head_bwd", "disc_mb_bwd", "disc_cotangent")
# the training-mode phases and how many timed launches each makes per single-chunk call (forward, VJP)
TRAIN_FWD = {"enc_conv1": 1, "disc_train_enc_conv2": 1, "disc_train_enc_conv3": 1, "disc_train_enc_conv4": 1,
             "disc_train_stats": 3, "disc_train_norm": 3, "disc_pool": 1, "disc_mb": 1, "disc_head": 1}
TRAIN_VJP = dict(TRAIN_FWD, enc_conv1=2, disc_train_norm=5, disc_head=0, disc_head_bwd=1, disc_mb_bwd=1,
                 disc_train_cotangent=1, disc_train_bn_bwd=3, disc_train_bn_dx=3, disc_train_bwd_enc_conv4=1,
                 disc_train_bwd_enc_conv3=1, bwd_enc_conv2=1, enc_conv1_bwd=1)


def calls(model, g, n, rng):
    st = torch.cuda.current_stream().cuda_stream
    U = do.units(g)
    x = torch.from_numpy(rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)).cuda()
    dl = torch.from_numpy(rng.standard_normal((n, U)).astype(np.float32)).cuda()
    lg, dx = torch.empty(n, U, device="cuda"), torch.empty_like(x)
    f4 = torch.empty(n, 1024, 4, 4, device="cuda")
    return {"discriminate": lambda: model.discriminate_dev(x.data_ptr(), n, lg.data_ptr(), 0, st),
            "discriminate_vjp": lambda: model.discriminate_vjp_dev(x.data_ptr(), dl.data_ptr(), n, dx.data_ptr(), st),
            "introspect": lambda: model.introspect_dev(x.data_ptr(), n, [0, 0, 0, f4.data_ptr()], st),
            "discriminate_train": lambda: model.discriminate_train_dev(x.data_ptr(), n, lg.data_ptr(), 0, 0, st),
            "discriminate_train_vjp": lambda: model.discriminate_train_vjp_dev(x.data_ptr(), dl.data_ptr(), n, dx.data_ptr(), st)}


def phase_ms(model, fn, counts, reps=10):
    """the per-call device time of each named phase: its mean launch time times its launches per call"""
    ms = layer_ms(model, fn, tuple(counts), reps=reps)
    return {k: ms[k] * c for k, c in counts.items()}


def train_main(a, npe, res, rng):
    for g in ("simple", "v1", "full"):
        for prec in (("fp32", "bf16") if g == "full" else ("fp32",)):
            m = npe.IAN(CONFIG[g], True, weights=MAKE[g](0))
            m.load_discriminator(do.make_discriminator_weights(g, 1))
            if prec == "bf16":
                m.set_precision("bf16")
            r = {}
            for n in (16, 256):
                fns = calls(m, g, n, rng)
                fns = {k: fns[k] for k in ("discriminate", "discriminate_train", "discriminate_vjp", "discriminate_train_vjp")}
                rates = alternate(fns, n, a.rounds, a.min_seconds)
                pf = phase_ms(m, fns["discriminate_train"], TRAIN_FWD)
                pb = phase_ms(m, fns["discriminate_train_vjp"], TRAIN_VJP)
                r[str(n)] = {"samples_per_s": rates, "train_forward_phase_ms": pf, "train_vjp_phase_ms": pb,
                             "train_forward_ms": sum(pf.values()), "train_vjp_ms": sum(pb.values())}
            m.close()
            res["%s_%s" % (g, prec)] = r
            print(g, prec, json.dumps(r), file=sys.stderr, flush=True)


def layer_ms(model, fn, names, twice=(), reps=10):
    """the per-call device time of each named kernel; those in `twice` run twice per call"""
    fn()
    model.set_layer_timing(True)
    try:
        for k in names:
            model.layer_time_ms(k, reset=True)
        out = {k: 0.0 for k in names}
        for _ in range(reps):
            fn()
            torch.cuda.synchronize()
            for k in names:
                out[k] += max(model.layer_time_ms(k, reset=True), 0.0) * (2 if k in twice else 1)
        return {k: v / reps for k, v in out.items()}
    finally:
        model.set_layer_timing(False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    ap.add_argument("--training", action="store_true", help="the training-mode entries next to the inference ones")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_discriminate.py measures the GPU path and needs a CUDA device")
    npe = importlib.import_module("neural-photo-editor_b200")
    res = {"gpu": gpu_info(0)}
    torch.cuda.set_stream(torch.cuda.Stream())             # the C-ABI reads stream 0 as the handle's own stream
    rng = np.random.default_rng(0)
    for g in (() if a.training else ("simple", "v1", "full")):
        for prec in (("fp32", "bf16") if g == "full" else ("fp32",)):
            m = npe.IAN(CONFIG[g], True, weights=MAKE[g](0))
            m.load_discriminator(do.make_discriminator_weights(g, 1))
            if prec == "bf16":
                m.set_precision("bf16")
            r = {}
            for n in (16, 128, 256):
                fns = calls(m, g, n, rng)
                rates = alternate(fns, n, a.rounds, a.min_seconds)
                lf = layer_ms(m, fns["discriminate"], TRUNK + HEAD)
                lb = layer_ms(m, fns["discriminate_vjp"], TRUNK + TRUNK_BWD + HEAD + HEAD_BWD, twice=TRUNK)
                head_f, head_b = sum(lf[k] for k in HEAD), sum(lb[k] for k in HEAD + HEAD_BWD)
                r[str(n)] = {"samples_per_s": rates, "forward_layer_ms": lf, "vjp_layer_ms": lb,
                             "forward_head_share": head_f / sum(lf.values()), "vjp_head_share": head_b / sum(lb.values())}
            m.close()
            res["%s_%s" % (g, prec)] = r
            print(g, prec, json.dumps(r), file=sys.stderr, flush=True)
    if a.training:
        train_main(a, npe, res, rng)
    res["gpu"].update(sm_clock())                          # sampled right after the timed work
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

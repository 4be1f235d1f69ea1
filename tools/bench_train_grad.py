"""(GPU) Time of the training-mode backward calls (ian_bn_backward_sums_dev + ian_bn_backward_dx_dev, and
ian_minibatch_discrim_bwd_dev) next to torch's own float32 backward of the same ops; prints one JSON line.

    python tools/bench_train_grad.py [--rounds 5] [--min-seconds 0.5] [--out profiles/h100_train_grad.json]

Reported, with the card's name and power limit read in the same run, as ms per call (median and range over `--rounds`
rounds, ours and torch's alternated round by round, CUDA events on one stream):
  * BatchNorm at IAN_simple.py's BN shapes at its batch of 128 (cfg['batch_size']): enc_conv2..4, enc_fc1, dec_fc2 and
    dec_conv1..3.  Ours: both backward calls, with dgamma and dbeta.  torch: autograd.grad of F.batch_norm(training=True)
    in float32 (cuDNN or torch's native kernel, whichever torch picks) for dx, dgamma, dbeta.
  * MinibatchLayer at the discriminator shape d = 1024 (after GlobalPoolLayer(enc_conv4)), K = 500, P = 5, n = 64 and 128.
    Ours: dx, dtheta, dlog_weight_scale and db in one call.  torch: autograd.grad of the layers.py:486-524 formula written
    in float32 torch ops, same four gradients.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_vjp import gpu_info, timed  # noqa: E402
import train_grad_oracle as tg  # noqa: E402

BN_SHAPES = {"enc_conv2": (128, 256, 16, 16), "enc_conv3": (128, 512, 8, 8), "enc_conv4": (128, 1024, 4, 4), "enc_fc1": (128, 1000),
             "dec_fc2": (128, 16384), "dec_conv1": (128, 512, 8, 8), "dec_conv2": (128, 256, 16, 16), "dec_conv3": (128, 128, 32, 32)}
EPS = 1e-4


def alternate(fns, rounds, min_s):
    """{name: {median, min, max}} ms per call, the calls alternated round by round"""
    reps = {}
    for k, f in fns.items():
        for _ in range(3):
            f()
        t = timed(f, 5) / 5
        reps[k] = max(5, int(np.ceil(min_s / t)))
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            ms[k].append(1e3 * timed(f, reps[k]) / reps[k])
    return {k: {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))} for k, v in ms.items()}


def bn_case(model, shape, rng, rounds, min_s):
    st = torch.cuda.current_stream().cuda_stream
    x = torch.from_numpy(rng.standard_normal(shape).astype(np.float32) * 2 + 0.5).cuda()
    dy = torch.from_numpy(rng.standard_normal(shape).astype(np.float32)).cuda()
    n, c = shape[:2]
    hw = int(np.prod(shape[2:], dtype=np.int64))
    g = torch.from_numpy(rng.uniform(0.5, 1.5, c).astype(np.float32)).cuda()
    b = torch.zeros(c, device="cuda")
    sums, bs = torch.empty(2, c, dtype=torch.float64, device="cuda"), torch.empty(2, c, dtype=torch.float64, device="cuda")
    dx, dg, db = torch.empty_like(x), torch.empty_like(g), torch.empty_like(g)
    model._check(model._lib.ian_bn_batch_stats_dev(model._h, x.data_ptr(), n, c, hw, sums[0].data_ptr(), sums[1].data_ptr(), st))
    count = float(n * hw)

    def ours():
        model._lib.ian_bn_backward_sums_dev(model._h, x.data_ptr(), dy.data_ptr(), n, c, hw, sums[0].data_ptr(), sums[1].data_ptr(),
                                            count, EPS, bs[0].data_ptr(), bs[1].data_ptr(), dg.data_ptr(), db.data_ptr(), st)
        model._lib.ian_bn_backward_dx_dev(model._h, x.data_ptr(), dy.data_ptr(), n, c, hw, sums[0].data_ptr(), sums[1].data_ptr(),
                                          count, bs[0].data_ptr(), bs[1].data_ptr(), g.data_ptr(), EPS, dx.data_ptr(), st)

    xr, gr, br = x.clone().requires_grad_(True), g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    y = torch.nn.functional.batch_norm(xr, None, None, gr, br, training=True, eps=EPS)

    def theirs():
        torch.autograd.grad(y, (xr, gr, br), dy, retain_graph=True)

    r = alternate({"ours": ours, "torch": theirs}, rounds, min_s)
    ours()
    want = torch.autograd.grad(y, (xr, gr, br), dy, retain_graph=True)
    r["max_abs_diff_dx_vs_torch"] = float((dx - want[0]).abs().max())
    return r


def mb_case(model, n, rng, rounds, min_s):
    d, K, P = 1024, 500, 5
    st = torch.cuda.current_stream().cuda_stream
    x = torch.from_numpy(rng.standard_normal((n, d)).astype(np.float32)).cuda()
    th = torch.from_numpy(rng.normal(0, 0.05, (d, K, P)).astype(np.float32)).cuda()
    lw = torch.from_numpy(rng.normal(np.log(0.04), 0.1, (K, P)).astype(np.float32)).cuda()
    b = torch.from_numpy(rng.normal(-1, 0.5, K).astype(np.float32)).cuda()
    g = torch.from_numpy(rng.standard_normal((n, d + K)).astype(np.float32)).cuda()
    outs = [torch.empty_like(t) for t in (x, th, lw, b)]

    def ours():
        model._lib.ian_minibatch_discrim_bwd_dev(model._h, x.data_ptr(), n, d, th.data_ptr(), lw.data_ptr(), b.data_ptr(), K, P,
                                                 g.data_ptr(), *[t.data_ptr() for t in outs], st)

    ins = [t.clone().requires_grad_(True) for t in (x, th, lw, b)]
    out = tg.mb_layer(*ins)                               # the formula in float32 torch ops

    def theirs():
        torch.autograd.grad(out, ins, g, retain_graph=True)

    r = alternate({"ours": ours, "torch": theirs}, rounds, min_s)
    ours()
    want = torch.autograd.grad(out, ins, g, retain_graph=True)
    r["max_abs_diff_dx_vs_torch"] = float((outs[0] - want[0]).abs().max())
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_train_grad.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_grad.py measures the GPU path and needs a CUDA device")
    from oracle import weights as ow
    npe = importlib.import_module("neural-photo-editor_b200")
    # a stream of its own: the legacy default stream's handle is 0, which the C-ABI reads as "the handle's own stream"
    torch.cuda.set_stream(torch.cuda.Stream())
    model = npe.IAN("IAN_simple.py", True, weights=ow.make_simple_weights(0))
    rng = np.random.default_rng(0)
    res = {"gpu": gpu_info(0), "unit": "ms per call", "bn": {}, "minibatch": {}}
    for name, shape in BN_SHAPES.items():
        res["bn"][name] = dict(shape=list(shape), **bn_case(model, shape, rng, a.rounds, a.min_seconds))
        print(name, json.dumps(res["bn"][name]), file=sys.stderr, flush=True)
    for n in (64, 128):
        res["minibatch"]["n%d" % n] = dict(shape=[n, 1024, 500, 5], **mb_case(model, n, rng, a.rounds, a.min_seconds))
        print("minibatch", n, json.dumps(res["minibatch"]["n%d" % n]), file=sys.stderr, flush=True)
    model.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

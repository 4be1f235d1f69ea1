"""(GPU) Cost of the decoder vector-Jacobian product against the brush gradient it generalises; prints one JSON line.

    python tools/bench_vjp.py [--batch 128] [--rounds 3] [--min-seconds 1.0] [--out FILE]

decode_vjp and grad run the same kernels except the loss seed (a dense cotangent over the whole frame against a box), so
at one batch size on one handle their time ratio is the price of the dense seed.  Each comparison alternates the two
calls over `--rounds` rounds of at least `--min-seconds` each (device-pointer entry points, CUDA events on one stream) and
reports the median and the min-max range of sample-steps/s.  Also: the seed kernel's own time in both modes
(ian_layer_time_ms("brush_seed"), layer timing on), batch-1 host latency of decode_vjp against imgradRGB (IAN_simple), the
same throughput comparison on IAN.py in float32 and bf16 precision, and the steps/s of a torch autograd SGD loop through
torch_ops.decode.  The card's name and power limit are read in the same run.
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import weights as ow  # noqa: E402


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
    """device time of `reps` calls of fn enqueued back to back on the current stream, in seconds"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / 1e3


def alternate(fns, n, rounds, min_s):
    """{name: (median, min, max) sample-steps/s}, the calls alternated round by round; reps sized for >= min_s per round"""
    reps = {}
    for k, f in fns.items():
        for _ in range(3):
            f()
        t = timed(f, 5) / 5
        reps[k] = max(5, int(np.ceil(min_s / t)))
    rates = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            rates[k].append(n * reps[k] / timed(f, reps[k]))
    return {k: {"median": float(np.median(v)), "range": [float(min(v)), float(max(v))]} for k, v in rates.items()}


def seed_kernel_ms(model, fns, reps=20):
    out = {}
    model.set_layer_timing(True)
    try:
        for k, f in fns.items():
            model.layer_time_ms("brush_seed", reset=True)
            for _ in range(reps):
                f()
            torch.cuda.synchronize()
            out[k] = model.layer_time_ms("brush_seed", reset=True)
    finally:
        model.set_layer_timing(False)
    return out


def vjp_vs_grad(model, n, rounds, min_s, with_seed_time=False):
    rng = np.random.default_rng(0)
    z0, boxes, rgb = ow.config4_inputs(n)
    z = torch.from_numpy(z0).cuda()
    dx = torch.from_numpy(rng.standard_normal((n, 3, 64, 64)).astype(np.float32)).cuda()
    bx = torch.from_numpy(np.ascontiguousarray(boxes, np.int32)).cuda()
    tg = torch.from_numpy(np.ascontiguousarray(rgb, np.float32)).cuda()
    dz, g = torch.empty(n, 100, device="cuda"), torch.empty(n, 100, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    fns = {"decode_vjp": lambda: model.decode_vjp_dev(z.data_ptr(), dx.data_ptr(), n, dz.data_ptr(), st),
           "grad": lambda: model.grad_dev(z.data_ptr(), bx.data_ptr(), tg.data_ptr(), 0, n, g.data_ptr(), st)}
    r = alternate(fns, n, rounds, min_s)
    out = {"batch": n, "sample_steps_per_s": r,
           "time_ratio_vjp_over_grad": r["grad"]["median"] / r["decode_vjp"]["median"]}
    if with_seed_time:
        out["seed_kernel_ms"] = seed_kernel_ms(model, fns)
    return out


def host_latency_ms(model, reps=200):
    rng = np.random.default_rng(1)
    z = rng.standard_normal((1, 100)).astype(np.float32)
    dx = rng.standard_normal((1, 3, 64, 64)).astype(np.float32)
    frame = rng.uniform(-1, 1, (1, 3, 64, 64)).astype(np.float32)
    fns = {"decode_vjp": lambda: model.decode_vjp(z, dx), "imgradRGB": lambda: model.imgradRGB(20, 20, 36, 36, frame, z)}
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


def torch_sgd_steps_per_s(model, n, min_s):
    ops = importlib.import_module("neural-photo-editor_b200.torch_ops")
    rng = np.random.default_rng(2)
    z = torch.from_numpy(rng.standard_normal((n, 100)).astype(np.float32)).cuda()
    t = torch.from_numpy(rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)).cuda()
    yy, xx = torch.meshgrid(torch.arange(64.0, device="cuda"), torch.arange(64.0, device="cuda"), indexing="ij")
    mask = torch.exp(-((yy - 32) ** 2 + (xx - 32) ** 2) / (2 * 8.0 ** 2))[None, None]

    def step():
        nonlocal z
        zz = z.detach().requires_grad_(True)
        loss = ((mask * (ops.decode(model, zz) - t).abs()).sum(dim=(1, 2, 3)) / (3 * mask.sum())).sum()
        (g,) = torch.autograd.grad(loss, zz)
        z = zz.detach() - 20.0 * g
    for _ in range(3):
        step()
    reps = max(5, int(np.ceil(min_s / (timed(step, 5) / 5))))
    return {"batch": n, "steps_per_s": reps / timed(step, reps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vjp.py measures the GPU path and needs a CUDA device")
    npe = importlib.import_module("neural-photo-editor_b200")
    res = {"gpu": gpu_info(0)}
    # a stream of its own: the legacy default stream's handle is 0, which the C-ABI reads as "the handle's own stream",
    # and the timing events must be recorded on the stream the library calls are enqueued on
    torch.cuda.set_stream(torch.cuda.Stream())
    simple = npe.IAN("IAN_simple.py", True, weights=ow.make_simple_weights(0))
    res["ian_simple"] = vjp_vs_grad(simple, a.batch, a.rounds, a.min_seconds, with_seed_time=True)
    print("ian_simple", json.dumps(res["ian_simple"]), file=sys.stderr, flush=True)
    res["ian_simple"]["batch1_host_latency_ms"] = host_latency_ms(simple)
    res["torch_sgd"] = torch_sgd_steps_per_s(simple, a.batch, a.min_seconds)
    print("torch_sgd", json.dumps(res["torch_sgd"]), file=sys.stderr, flush=True)
    simple.close()
    full = npe.IAN("IAN.py", True, weights=ow.make_full_weights(0))
    res["ian_full"] = {}
    for prec in ("fp32", "bf16"):
        full.set_precision(prec)
        res["ian_full"][prec] = vjp_vs_grad(full, a.batch, a.rounds, a.min_seconds, with_seed_time=True)
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

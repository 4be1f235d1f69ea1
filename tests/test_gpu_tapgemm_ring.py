"""The float32-mode tap-GEMM's operand ring at its edges: every batch entry point with an executed-reference fixture, on
all three graphs, at batches 1, 2, 37, 256 and 513 under whole tiles, automatic and forced stream-K (IAN_STREAMK=0/1/2),
each with and without split-K (IAN_SPLITK=0/1).

Those batches give work items of every length the ring meets: stream-K segments one K step long, tiles that begin at
any position of the ring (a CTA's earlier tiles leave the stage counter wherever their K steps ended), split-K ranges
at small batch, and a partial last m-tile.  Each batch repeats the fixture cases sample by sample, so every sample is
held to the reference at the tolerances of tests/test_gpu_reference_exec.py and tests/test_gpu_full.py, and a second
run of the same handle must give the same bits.  Copies of one brush case at different rows of a batch are cut at
different K steps by stream-K, so their sums round differently; on the flow graphs that can put one rectifier unit in
the brush footprint on the other side of zero for some copies (measured 1.5e-3 on IAN.py, batch 37), so those are held
to test_gpu_full's batched bound for such flips: every copy <= 2e-2 and the closest <= 1e-3."""
import os

import numpy as np
import pytest

from oracle import ian_numpy as on
from oracle import weights as ow

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = {"simple": "IAN_simple.py", "full": "IAN.py", "v1": "IANv1.py"}
ENV = ("IAN_STREAMK", "IAN_SPLITK", "IAN_GRAPHS", "IAN_PDL", "IAN_FINALIZE8", "IAN_CHUNK", "IAN_PATH", "IAN_EPI_TMA")
BATCHES = (1, 2, 37, 256, 513)
SCHED = [(sk, sp) for sk in (0, 1, 2) for sp in (0, 1)]


def _load(name):
    return np.load(os.path.join(ROOT, "tests", "golden", name))


def _tile(a, n):
    return np.ascontiguousarray(a[np.arange(n) % len(a)])


def _frame(rgb):
    return np.broadcast_to(np.asarray(rgb, np.float32).reshape(1, 3, 1, 1), (1, 3, 64, 64))


def _cases(graph):
    """(images, image refs, latents, decode refs, brush cases, checks) of one graph's fixtures.  A brush case is
    (z, box, rgb or None, reference gradient)."""
    gold = _load("ian_%s_golden.npz" % graph)
    x = on.to_tanh(gold["images"].astype(np.float64)).astype(np.float32)
    if graph == "simple":
        ref = _load("ref_exec_simple.npz")
        z0, b0 = gold["z_rand"][0], gold["boxes"][0]
        brush = [(z0, b0, gold["rgb"][0], ref["g0_rgb"][0]), (gold["z_rand"][5], ref["g5_box"], gold["rgb"][5], ref["g5_rgb"][0]),
                 (z0, b0, None, ref["g0_light"][0])]
        kx = ref["xhat_dnn"].shape[0]
        zs = np.concatenate([ref["mu_dnn"][:kx], gold["z_rand"][:kx]]).astype(np.float32)
        xs = np.concatenate([ref["xhat_dnn"], ref["xhat_rand_dnn"]])
        return x[:len(ref["mu_dnn"])], {"encode": (ref["mu_dnn"], 2e-4, False)}, zs, xs, brush, 1e-4
    ref = _load("ref_exec_%s.npz" % graph)
    k = len(ref["z"])
    z0 = gold["z_rand"][0]
    brush = [(z0, ref["grad_box"], ref["grad_rgb_target"], ref["g_rgb"][0]), (z0, ref["grad_box"], None, ref["g_light"][0])]
    zs = np.concatenate([ref["z"], gold["z_rand"][:k]]).astype(np.float32)
    xs = np.concatenate([ref["xhat"], ref["xhat_rand"]])
    return x[:k], {"encode": (ref["z"], 3e-4, True), "Zfn": (ref["mu"], 2e-4, False)}, zs, xs, brush, 2e-4


def _run(m, graph, n):
    """every result of batch n, with its per-sample reference and tolerance check"""
    x, enc_refs, zs, xs, brush, dec_tol = _cases(graph)
    out = []
    xn = _tile(x, n)
    for name, (refs, tol, relative) in enc_refs.items():
        got = m.encode_images(xn) if name == "encode" else m.Zfn(xn)
        out.append((name, got, _tile(refs, n), tol, relative))
    out.append(("decode", m.sample_at(_tile(zs, n)), _tile(xs, n), dec_tol, False))
    for light in (False, True):
        cs = [c for c in brush if (c[2] is None) == light]
        pick = np.arange(n) % len(cs)
        z = np.stack([cs[i][0] for i in pick]).astype(np.float32)
        boxes = np.stack([np.asarray(cs[i][1], np.int32) for i in pick])
        rgb = None if light else np.stack([np.asarray(cs[i][2], np.float32) for i in pick])
        out.append(("grad_light" if light else "grad_rgb", m.grad(z, boxes, rgb), np.stack([cs[i][3] for i in pick]), None, None))
    return out


@pytest.mark.parametrize("streamk,splitk", SCHED, ids=["sk%d-split%d" % s for s in SCHED])
@pytest.mark.parametrize("graph", ["simple", "full", "v1"])
def test_float32_tapgemm_ring_edges(npe, monkeypatch, graph, streamk, splitk):
    gold = _load("ian_%s_golden.npz" % graph)
    make = {"simple": ow.make_simple_weights, "full": ow.make_full_weights, "v1": ow.make_v1_weights}[graph]
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("IAN_STREAMK", str(streamk))
    monkeypatch.setenv("IAN_SPLITK", str(splitk))
    m = npe.IAN(CONFIG[graph], True, weights=make(int(gold["weight_seed"])), path="tc")
    try:
        for n in BATCHES:
            first = _run(m, graph, n)
            for name, got, ref, tol, relative in first:
                assert got.shape[0] == n and np.isfinite(got).all(), (name, n)
                if tol is None:               # brush gradients: relative to the reference's largest component
                    err = np.abs(got - ref).max(axis=1) / np.abs(ref).max(axis=1)
                    if graph == "simple":
                        assert err.max() <= 1e-3, (name, n, err.max())
                    else:                     # a rectifier unit may flip per sample (the batched bound of test_gpu_full)
                        assert err.max() <= 2e-2 and err.min() <= 1e-3, (name, n, err.max(), err.min())
                elif relative:
                    assert (np.abs(got - ref) <= tol * (1.0 + np.abs(ref))).all(), (name, n, np.abs(got - ref).max())
                else:
                    assert np.abs(got - ref).max() <= tol, (name, n, np.abs(got - ref).max())
            for (name, a, _, _, _), (_, b, _, _, _) in zip(first, _run(m, graph, n)):
                assert np.array_equal(a, b), ("rerun", name, n)
    finally:
        m.close()

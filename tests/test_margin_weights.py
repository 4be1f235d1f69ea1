"""CPU checks of the premise of tests/test_gpu_well_conditioned.py: on the weights of tests/margin_weights.py no rectifier
of the test pool is near its kink, so every gradient path is well-conditioned, and the per-sample bounds BOUNDS are
tight enough to see a single-pass bf16 slip in one backward layer.

  certificate     float64 on the whole pool: min s_c * pre >= delta for every rectifier element (both MADE applications
                  included), both signs in every layer, every head sigmoid argument in [-2, 2], x_hat finite and not
                  saturated; the two edit-loop steps stay off every kink; the walk is oracle/ian_torch.py's graph.
  conditioning    scaling x, and separately z, by 1 + 1e-5 N(0,1) moves every sample of SAMPLES on every path by < a
                  tenth of the bounds: decoder VJP, brush gradients with each target kind, encoder VJP with and without eps.
  discrimination  rounding one backward operand to bf16 (round to nearest even, in numpy) moves every sample of the
                  pool by >= 3x the bounds: the head's backward GEMM, one MDC block's (a deconv's on IANv1 / IAN_simple), enc_conv3's adjoint."""
import numpy as np
import pytest
import torch

import margin_weights as mw
from oracle import ian_torch as ot

GRAPHS = ["simple", "full", "v1"]
# one of each box kind of the pool (fixed, 1x1, full width, random), samples between the GPU test's probes (5, 25, 106)
# and its probes at batch 130 (both sides of the head's CTA rounds, the middle, the last)
SAMPLES = [0, 1, 2, 3, 5, 25, 43, 44, 65, 87, 88, 106, 129]


def _sub(inp, idx):
    return {k: v[idx] for k, v in inp.items()}


@pytest.mark.parametrize("graph", GRAPHS)
def test_certificate(graph):
    P, inp = mw.weights(graph), mw.pool()
    c = mw.certificate(graph, P, inp)
    rect = {k: v for k, v in c.items() if isinstance(v, dict)}
    assert len(rect) == {"simple": 8, "full": 18, "v1": 11}[graph], sorted(rect)
    for knob, r in rect.items():
        assert r["min_margin"] >= mw.DELTA, (knob, r)
        assert r["pos"] > 0 and r["neg"] > 0, (knob, r)
    if graph != "simple":
        assert c["head_max_arg"] <= 2.0, c["head_max_arg"]
    assert c["x_hat_finite"] and c["saturated_fraction"] <= 0.05, c          # IAN_simple 1.8 %, the Beta head 0


@pytest.mark.parametrize("graph", GRAPHS)
def test_walk_is_the_oracle_graph_and_edits_stay_off_kinks(graph):
    """the walk computes oracle/ian_torch.py's forward; two edit steps of the pool's first samples keep the margin"""
    P, inp = mw.weights(graph), _sub(mw.pool(), SAMPLES)
    o = mw.Oracle(graph, P)
    P64 = ot.to_torch(P, torch.float64)
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    with torch.no_grad():
        xh = mw.DECODER[graph](P64, t(inp["z"])).numpy()
        if graph == "simple":
            z = ot.encode(P64, t(inp["x"]), False, t(inp["eps"])).numpy()
        else:
            z = ot.full_encode(P64, t(inp["x"]), o.masks, False, t(inp["eps"])).numpy()
    assert np.abs(o.decode(inp["z"]) - xh).max() <= 1e-12
    assert np.abs(o.encode(inp["x"], inp["eps"]) - z).max() <= 1e-12 * (1 + np.abs(z).max())
    z2 = o.edit(inp["z"], inp["boxes"], inp["rgb"], 2)
    margin, head = mw.decoder_margin(graph, P, z2)
    assert margin >= mw.DELTA * 0.9 and head <= 2.0, (margin, head)


def _paths(o, inp, x, z):
    """every gradient path on the samples, as {name: result}"""
    ct = mw.cotangents(len(z), 3)
    dz = np.random.default_rng(4).standard_normal(z.shape)
    out = {"decode_vjp": o.decode_vjp(z, ct["gauss"])}
    g = o.grads(z, inp["boxes"], {"light": None, "colour": inp["rgb"], "frame": inp["frame"]})
    out.update({"grad_" + k: v for k, v in g.items()})
    out["encode_vjp"] = o.encode_vjp(x, dz)
    out["encode_vjp_eps"] = o.encode_vjp(x, dz, inp["eps"])
    return out


@pytest.mark.parametrize("graph", GRAPHS)
def test_conditioning(graph):
    P, inp = mw.weights(graph), _sub(mw.pool(), SAMPLES)
    o = mw.Oracle(graph, P)
    x, z = inp["x"], inp["z"]
    rng = np.random.default_rng(5)
    base = _paths(o, inp, x, z)
    for what, xs, zs in (("x", x * (1 + 1e-5 * rng.standard_normal(x.shape)), z),
                         ("z", x, z * (1 + 1e-5 * rng.standard_normal(z.shape)))):
        moved = _paths(o, inp, xs, zs)
        for k in base:
            l2, mx = mw.rel_l2(moved[k], base[k]), mw.rel_max(moved[k], base[k])
            b_l2, b_max = mw.BOUNDS["encoder" if k.startswith("encode") else "decoder"]
            assert (l2 < b_l2 / 10).all() and (mx < b_max / 10).all(), (what, k, l2, mx)


@pytest.mark.parametrize("graph", GRAPHS)
def test_discrimination(graph):
    """every sample of the pool, in chunks of 26"""
    P, pool = mw.weights(graph), mw.pool()
    o = mw.Oracle(graph, P)
    dx_all = mw.cotangents(mw.POOL, 3)["gauss"]
    dz_all = np.random.default_rng(4).standard_normal((mw.POOL, 100))
    moves = {}
    for c0 in range(0, mw.POOL, 26):
        idx = list(range(c0, min(c0 + 26, mw.POOL)))
        x, z, dx, dz = pool["x"][idx], pool["z"][idx], dx_all[idx], dz_all[idx]
        base_d, base_e = o.decode_vjp(z, dx), o.encode_vjp(x, dz)
        for slip, got, ref, kind in (("head", o.decode_vjp(z, dx, "head"), base_d, "decoder"),
                                     ("block", o.decode_vjp(z, dx, "block"), base_d, "decoder"),
                                     ("enc", o.encode_vjp(x, dz, slip="enc"), base_e, "encoder")):
            m = moves.setdefault(slip, (kind, [], []))
            m[1].extend(mw.rel_l2(got, ref))
            m[2].extend(mw.rel_max(got, ref))
    for slip, (kind, l2, mx) in moves.items():
        b_l2, b_max = mw.BOUNDS[kind]
        assert min(l2) >= 3 * b_l2 and min(mx) >= 3 * b_max, (slip, min(l2), int(np.argmin(l2)), min(mx), int(np.argmin(mx)))


def test_bf16_round():
    """ties to even, above the tie rounds up, the sign is kept"""
    a = np.array([1.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -1.0 - 2 ** -9, 1.0 + 2 ** -8 + 2 ** -20], np.float32)
    want = np.array([1.0, 1.0, 1.0 + 2 ** -6, -1.0, 1.0 + 2 ** -7], np.float32)
    got = mw.bf16_round(a)
    assert np.array_equal(got, want), got
    assert np.array_equal(mw.bf16_round(got), got)

"""GPU tests of the introspection features' vector-Jacobian product (include/ian_b200.h ian_introspect_vjp_*;
API.IAN.introspect_vjp; torch_ops.introspect / feature_loss) on all three graphs, on the tensor-core and SIMT paths and,
on IAN.py, in bf16 mode.

  1. against the executed reference: <introspect_vjp(x, c_i = probe_j), v> against the stored central difference of the
     reference's own l_introspect along v (tests/golden/ref_exec_introspect.npz), every graph, layer and probe.
  2. against float64 autograd of sum_i <c_i, g_i(x)> through tests/introspect_oracle.py, seeded cotangents on the
     margin-weight pool's images, every sample, under every tap-GEMM schedule; the float32 bound is at most a third of the
     floor that rounding the cotangents to bf16 moves the float64 gradient by.
  3. adjointness: <c, introspect_jvp(x, v)> = <introspect_vjp(x, c), v> per sample.
  4. NULL cotangents: a NULL c_i and an all-zero c_i give the same dx; all four NULL give dx = 0; c1 alone runs no
     enc_conv2..4 (layer timing).
  5. the feature-loss gradient by two routes: torch.autograd through torch_ops.decode and torch_ops.introspect against
     2 g of ian_feature_gauss_newton_* (forward-mode Jacobian columns).
  6. decoder fine-tuning under the feature loss (IAN_simple): the 13 decoder parameters' gradients against float64
     autograd of the oracle decoder composed with the oracle features.
  7. the torch op's bits: forward = introspect, backward = introspect_vjp, a forward-mode dual = introspect_jvp, an unused
     output passes NULL; wrong dtype, device or shape are refused.
  8. bits: reruns, device form = host form, IAN_PDL=0, IAN_CHUNK=16, and one sample's inputs never change another's bits.
  9. errors.
Measured values go to introspect_vjp.json when IAN_TEST_RECORD names a directory."""
import ctypes as C
import importlib
import json
import os

import numpy as np
import pytest

import introspect_oracle as io
import margin_weights as mw
from oracle import ian_torch as ot
from test_gpu_fit_features import CONFIG, GRAPHS, MODES, _margin, _rel, handles, io_shapes, synth  # noqa: F401
from test_ref_exec_decjvp import MAKE

pytestmark = pytest.mark.gpu
# Bounds set from one run on an H100 80GB HBM3 at 700 W (the results are the same bits on every rerun).
# 1. against the executed reference, relative L2 of the (images x probes) projections per layer: float32 mode worst 1.4e-4
#    (IAN_simple on the SIMT path: on the synthetic golden weights some rectifier sits near its kink; 1.2e-5 or better
#    elsewhere); bf16 mode on IAN.py worst 5.6e-2.  Bounds >= 2x over the worst.
REF_BOUND, REF_BF16 = 3e-4, 0.11
# 2. against float64, per-sample relative L2 of dx on the margin weights: worst 8.0e-6 (tensor cores with IAN_SPLITK=0;
#    7.2e-6 under the other schedules, 5.3e-6 on the SIMT path), 3.1e-3 in bf16 mode on IAN.py.  Rounding the cotangents
#    to bf16 moves the float64 dx by at least 1.6e-3, so the float32 bound is 1/80 of that floor (the rule: at most a third).
DX_BOUND, DX_BF16 = 2e-5, 8e-3
# 3. adjointness, |<c, Jv> - <J^T c, v>| / (|c| |Jv|) per sample: worst 2.6e-8 (float32), 1.7e-5 (bf16 mode on IAN.py).
ADJ_BOUND, ADJ_BF16 = 1e-7, 5e-5
# 5. the two routes to the feature-loss gradient, per-sample relative L2: worst 2.9e-5 (IAN.py on the tensor cores), 6.6e-3
#    in bf16 mode on IAN.py.
ROUTES_BOUND, ROUTES_BF16 = 6e-5, 1.5e-2
# 6. decoder parameter gradients under the feature loss, per-tensor relative L2 against float64: worst 3.2e-5
#    (bnorm_dec_fc2.gamma and l_dec_fc2.W).
PARAMS_BOUND = 7e-5
SCHEDS = [{}, {"IAN_STREAMK": 0}, {"IAN_STREAMK": 2}, {"IAN_SPLITK": 0}]
RECORD = {}


def _record(key, value):
    RECORD[key] = value
    if os.environ.get("IAN_TEST_RECORD"):
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "introspect_vjp.json"), "w") as f:
            json.dump(RECORD, f, indent=1, sort_keys=True)


def _ops():
    return importlib.import_module("neural-photo-editor_b200.torch_ops")


def _cotangents(n, seed):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal((n,) + s).astype(np.float32) for s in io_shapes()]


def _dx64(Q, x, c):
    """float64 d/dx sum_i <c_i, g_i(x)> through the oracle features, on the GPU"""
    import torch
    xt = torch.from_numpy(np.asarray(x, np.float64)).cuda().requires_grad_(True)
    f = io.features(Q, xt)
    s = sum((fi * torch.from_numpy(np.asarray(ci, np.float64)).cuda()).sum() for fi, ci in zip(f, c) if ci is not None)
    (dx,) = torch.autograd.grad(s, xt)
    return dx.cpu().numpy()


# ---- 1. against the executed reference -----------------------------------------------------------------------------------
@pytest.mark.parametrize("g,mode", MODES)
def test_against_the_executed_reference(handles, g, mode):
    x, seed, v, probes, stored = io.fixture()[g]
    m = handles(g, MAKE[g](seed), mode)
    n, k = len(x), len(probes[0])
    xr = np.repeat(x, k, axis=0)                                 # sample (a, j): image a, probe j
    err = []
    for i in range(4):
        c = [None] * 4
        c[i] = np.ascontiguousarray(np.tile(probes[i], (n, 1, 1, 1)).astype(np.float32))
        dx = m.introspect_vjp(xr, c).astype(np.float64).reshape(n, k, -1)
        got = np.einsum("ajp,ap->aj", dx, v.reshape(n, -1))
        ref = stored["dp"][i]
        err.append(float(np.linalg.norm(got - ref) / np.linalg.norm(ref)))
    _record("1_ref_%s_%s" % (g, mode), err)
    assert max(err) <= (REF_BF16 if mode == "bf16" else REF_BOUND), err


# ---- 2. against float64 -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g,mode", MODES)
def test_against_float64(handles, g, mode):
    P = _margin(g)
    Q = io.weights64(P, "cuda")
    x = mw.pool()["x"][:6]
    c = _cotangents(6, 11)
    ref = _dx64(Q, x, c)
    floor = float(_rel(_dx64(Q, x, [mw.bf16_round(a) for a in c]), ref).min())
    rec = {"bf16_c_floor": floor}
    for sched in (SCHEDS if mode == "tc" else SCHEDS[:1]):
        m = handles(g, P, mode, **sched)
        e = _rel(m.introspect_vjp(x, c), ref)
        rec[json.dumps(sched)] = float(e.max())
        _record("2_%s_%s" % (g, mode), rec)
        assert e.max() <= (DX_BF16 if mode == "bf16" else DX_BOUND), (sched, e)
    assert DX_BOUND <= floor / 3, (DX_BOUND, floor)


# ---- 3. adjointness ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g,mode", MODES)
def test_adjoint_of_introspect_jvp(handles, g, mode):
    m = handles(g, _margin(g), mode)
    x = mw.pool()["x"][:5]
    v = np.random.default_rng(5).standard_normal(x.shape).astype(np.float32)
    c = _cotangents(5, 12)
    t = m.introspect_jvp(x, v)
    dx = m.introspect_vjp(x, c)
    n = len(x)
    lhs = sum((a.astype(np.float64).reshape(n, -1) * b.reshape(n, -1)).sum(1) for a, b in zip(c, t))
    rhs = (dx.astype(np.float64).reshape(n, -1) * v.reshape(n, -1)).sum(1)
    scale = np.sqrt(sum((a.astype(np.float64).reshape(n, -1) ** 2).sum(1) for a in c) *
                    sum((b.astype(np.float64).reshape(n, -1) ** 2).sum(1) for b in t))
    e = np.abs(lhs - rhs) / scale
    _record("3_%s_%s" % (g, mode), float(e.max()))
    assert e.max() <= (ADJ_BF16 if mode == "bf16" else ADJ_BOUND), e


# ---- 4. NULL cotangents ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g,mode", MODES)
def test_null_cotangents(handles, g, mode):
    m = handles(g, _margin(g), mode)
    x = mw.pool()["x"][:3]
    c = _cotangents(3, 13)
    for drop in range(4):
        cn, cz = list(c), list(c)
        cn[drop] = None
        cz[drop] = np.zeros_like(c[drop])
        assert np.array_equal(m.introspect_vjp(x, cn), m.introspect_vjp(x, cz)), drop
    assert np.array_equal(m.introspect_vjp(x, [None] * 4), np.zeros_like(x))
    # c1 alone: the forward stops after enc_conv1 and no backward GEMM runs
    mt = handles(g, _margin(g), mode)
    mt.set_layer_timing(True)
    dx1 = mt.introspect_vjp(x, [c[0], None, None, None])
    for name in ("enc_conv2", "enc_conv3", "enc_conv4", "bwd_enc_conv2", "introspect_bwd_enc_conv2"):
        assert mt.layer_time_ms(name) < 0, name
    assert mt.layer_time_ms("feat_cotangent") > 0 and mt.layer_time_ms("enc_conv1_bwd") > 0
    assert np.array_equal(dx1, m.introspect_vjp(x, [c[0], None, None, None]))
    # c4 and c2: enc_conv2..4 run, the GEMM landing on a2 joins c2, the one landing on a3 runs without res
    mt.introspect_vjp(x, [None, c[1], None, c[3]])
    assert mt.layer_time_ms("introspect_bwd_enc_conv3") > 0 and mt.layer_time_ms("bwd_enc_conv4") > 0
    assert mt.layer_time_ms("introspect_bwd_enc_conv4") < 0 and mt.layer_time_ms("introspect_bwd_enc_conv2") < 0


# ---- 5. the feature-loss gradient by two routes -----------------------------------------------------------------------
@pytest.mark.parametrize("g,mode", MODES)
def test_feature_loss_gradient_matches_gauss_newton(handles, g, mode):
    import torch
    ops = _ops()
    m = handles(g, _margin(g), mode)
    p = mw.pool()
    z, x = p["z"][:3], p["x"][3:6].copy()
    a, b = 0.5, 2.0
    zt = torch.from_numpy(z).cuda().requires_grad_(True)
    xt = torch.from_numpy(x).cuda()
    xh = ops.decode(m, zt)
    E = a * ((xh - xt) ** 2).reshape(3, -1).sum(1) + 12288 * b * ops.feature_loss(m, xh, xt)
    E.sum().backward()
    _, gv, e = m.gauss_newton_features(z, x, a, b)
    err = _rel(zt.grad.cpu().numpy(), 2 * gv)
    eE = float(np.abs(E.detach().cpu().numpy() / e - 1).max())
    _record("5_%s_%s" % (g, mode), {"grad": float(err.max()), "E": eE})
    bound = ROUTES_BF16 if mode == "bf16" else ROUTES_BOUND
    assert err.max() <= bound, err


# ---- 6. decoder fine-tuning under the feature loss ------------------------------------------------------------------------
def test_decoder_parameter_gradients_under_the_feature_loss(handles):
    import torch
    ops = _ops()
    P = _margin("simple")
    m = handles("simple", P)
    p = mw.pool()
    z, x = p["z"][:4], p["x"][10:14].copy()
    params = ops.decoder_parameters(m, P)
    zt, xt = torch.from_numpy(z).cuda(), torch.from_numpy(x).cuda()
    ops.feature_loss(m, ops.decode(m, zt, params), xt).sum().backward()
    Q = io.weights64(P, "cuda")
    for k in params:
        Q[k].requires_grad_(True)
    z64, x64 = zt.double(), xt.double()
    xh = ot.decode(Q, z64)
    l64 = sum(((u - w) ** 2).reshape(4, -1).mean(1) for u, w in zip(io.features(Q, xh), io.features(Q, x64))).sum() / 4
    ref = torch.autograd.grad(l64, [Q[k] for k in params])
    err = {k: float((params[k].grad.double() - r).norm() / r.norm()) for k, r in zip(params, ref)}
    _record("6_params", err)
    assert len(err) == 13 and max(err.values()) <= PARAMS_BOUND, err


# ---- 7. the torch op --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_torch_op_bits(handles, g):
    import torch
    import torch.autograd.forward_ad as fwAD
    ops = _ops()
    m = handles(g, _margin(g))
    x = mw.pool()["x"][:3]
    c = _cotangents(3, 14)
    xt = torch.from_numpy(x).cuda().requires_grad_(True)
    f = ops.introspect(m, xt)
    assert all(np.array_equal(a.detach().cpu().numpy(), b) for a, b in zip(f, m.introspect(x)))
    torch.autograd.backward(f, [torch.from_numpy(a).cuda() for a in c])
    assert np.array_equal(xt.grad.cpu().numpy(), m.introspect_vjp(x, c))
    # an unused output passes NULL, so the chain starts at f2: on a fresh handle, timed from the backward on, enc_conv3 and
    # enc_conv4 never run (a zero cotangent for f3 / f4 would give the same dx, but would run them)
    mt = handles(g, _margin(g))
    xt = torch.from_numpy(x).cuda().requires_grad_(True)
    f = ops.introspect(mt, xt)
    torch.cuda.synchronize()
    mt.set_layer_timing(True)
    (f[0] * torch.from_numpy(c[0]).cuda()).sum().add((f[1] * torch.from_numpy(c[1]).cuda()).sum()).backward()
    torch.cuda.synchronize()
    assert mt.layer_time_ms("enc_conv3") < 0 and mt.layer_time_ms("enc_conv4") < 0
    assert mt.layer_time_ms("enc_conv2") > 0 and mt.layer_time_ms("introspect_bwd_enc_conv2") > 0
    mt.set_layer_timing(False)
    assert np.array_equal(xt.grad.cpu().numpy(), m.introspect_vjp(x, [c[0], c[1], None, None]))
    # forward mode
    v = np.random.default_rng(6).standard_normal(x.shape).astype(np.float32)
    with fwAD.dual_level():
        out = ops.introspect(m, fwAD.make_dual(torch.from_numpy(x).cuda(), torch.from_numpy(v).cuda()))
        t = [fwAD.unpack_dual(o).tangent.cpu().numpy() for o in out]
    assert all(np.array_equal(a, b) for a, b in zip(t, m.introspect_jvp(x, v)))
    # feature_loss is API.IAN.feature_loss's formula on the same features
    xh = torch.from_numpy(x[::-1].copy()).cuda()
    lf = ops.feature_loss(m, xh, torch.from_numpy(x).cuda()).cpu().numpy()
    assert lf.dtype == np.float32 and lf.shape == (3,)
    assert np.allclose(lf, m.feature_loss(x[::-1].copy(), x), rtol=1e-5, atol=0)
    # refusals
    with pytest.raises(TypeError):
        ops.introspect(m, torch.from_numpy(x).cuda().double())
    with pytest.raises(TypeError):
        ops.introspect(m, torch.from_numpy(x))
    with pytest.raises(ValueError):
        ops.introspect(m, torch.zeros(3, 3, 32, 32, device="cuda"))


# ---- 8. bits ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("n", [3, 12])
def test_a_seeded_chain_leaves_the_encoder_vjp_as_it_was(handles, path, n):
    """bf16 mode on IAN.py: a c1-only call seeds e1, the encoder VJP's own planes, which enc_conv1's adjoint reads as hi + lo.
    Afterwards encode_vjp (host form: its captured graph) and an all-four introspect_vjp give the bits they gave before, on
    the tensor cores with (n = 3) and without (n = 12) a split-K finalize on the GEMM landing on a1, and on the SIMT path."""
    m = handles("full", _margin("full"), path)
    m.set_precision("bf16")
    x = mw.pool()["x"][:n]
    dz = np.random.default_rng(18).standard_normal((n, 100)).astype(np.float32)
    c = _cotangents(n, 17)
    e0, a0 = m.encode_vjp(x, dz), m.introspect_vjp(x, c)
    d1 = m.introspect_vjp(x, [c[0], None, None, None])
    assert np.array_equal(m.encode_vjp(x, dz), e0)
    assert np.array_equal(m.introspect_vjp(x, c), a0)
    z = [np.zeros_like(a) for a in c]
    assert np.array_equal(m.introspect_vjp(x, [c[0], z[1], None, None]), d1)
    assert np.array_equal(m.introspect_vjp(x, [c[0], None, None, z[3]]), d1)
    assert np.array_equal(m.introspect_vjp(x, [c[0], None, None, None]), d1)


@pytest.mark.parametrize("g", GRAPHS)
def test_bits(handles, g):
    import torch
    m = handles(g, _margin(g))
    x = mw.pool()["x"][:20]
    c = _cotangents(20, 15)
    dx = m.introspect_vjp(x, c)
    assert np.array_equal(dx, m.introspect_vjp(x, c))
    xd = torch.from_numpy(x).cuda()
    cd = [torch.from_numpy(a).cuda() for a in c]
    dd = torch.empty_like(xd)
    m.introspect_vjp_dev(xd.data_ptr(), 20, [a.data_ptr() for a in cd], dd.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(dd.cpu().numpy(), dx)
    assert np.array_equal(handles(g, _margin(g), IAN_PDL=0).introspect_vjp(x, c), dx)
    # chunked: samples 0..15 at batch 16, 16..19 at batch 4
    got = handles(g, _margin(g), IAN_CHUNK=16).introspect_vjp(x, c)
    parts = [m.introspect_vjp(x[s], [a[s] for a in c]) for s in (slice(0, 16), slice(16, 20))]
    assert np.array_equal(got, np.concatenate(parts))


@pytest.mark.parametrize("g", GRAPHS)
def test_samples_stay_apart(handles, g):
    m = handles(g, synth(g))
    rng = np.random.default_rng(78)
    x = rng.uniform(-1, 1, (4, 3, 64, 64)).astype(np.float32)
    c = _cotangents(4, 16)
    base = m.introspect_vjp(x, c)
    keep = [0, 2, 3]
    cases = []
    x1 = x.copy()
    x1[1] = rng.uniform(-1, 1, (3, 64, 64))
    cases.append((x1, c))
    x2 = x.copy()
    x2[1, 0, 5, 7] = np.nan
    cases.append((x2, c))
    for i, bad in ((0, np.inf), (2, np.nan), (3, -np.inf)):
        ci = [a.copy() for a in c]
        ci[i][1].flat[17] = bad
        cases.append((x, ci))
    for xx, cc in cases:
        assert np.array_equal(m.introspect_vjp(xx, cc)[keep], base[keep])


# ---- 9. errors --------------------------------------------------------------------------------------------------------
def test_errors(npe, model):
    lib, h = model._lib, model._h
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    x = np.zeros((2, 3, 64, 64), np.float32)
    dx = np.full((2, 3, 64, 64), 7, np.float32)
    c = [np.zeros((2,) + s, np.float32) for s in io_shapes()]
    assert lib.ian_introspect_vjp_host(h, fp(x), -1, *[fp(a) for a in c], fp(dx)) == -1
    assert lib.ian_introspect_vjp_host(h, None, 2, *[fp(a) for a in c], fp(dx)) == -1
    assert lib.ian_introspect_vjp_host(h, fp(x), 2, *[fp(a) for a in c], None) == -1
    assert lib.ian_introspect_vjp_host(h, fp(x), 0, *[fp(a) for a in c], fp(dx)) == 0 and np.all(dx == 7)
    assert lib.ian_introspect_vjp_host(h, None, 0, None, None, None, None, None) == 0
    assert model.introspect_vjp(np.zeros((0, 3, 64, 64), np.float32), [None] * 4).shape == (0, 3, 64, 64)
    with pytest.raises(ValueError):
        model.introspect_vjp(x, c[:3])
    with pytest.raises(ValueError):
        model.introspect_vjp(x, [c[1], None, None, None])
    raw = C.c_void_p()
    assert lib.ian_create(0, 0, C.byref(raw)) == 0
    try:
        assert lib.ian_introspect_vjp_host(raw, fp(x), 2, *[fp(a) for a in c], fp(dx)) == -3
    finally:
        lib.ian_destroy(raw)

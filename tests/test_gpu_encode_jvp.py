"""GPU tests of the encoder Jacobian-vector product dz = (d z / d x) . v (include/ian_b200.h ian_encode_jvp_*,
API.IAN.encode_jvp, torch_ops.encode under torch.autograd.forward_ad) on all three graphs and both CUDA paths.

  1. against the executed reference (tests/golden/ref_exec_encjvp.npz) and the float64 oracle (torch forward mode on
     oracle/ian_torch.py, tests/test_ref_exec_encjvp.py), eps absent and present, at batches 3 and 130.  The synthetic
     weights put rectifiers within float32 reach of their kinks (see tests/test_gpu_encode_vjp.py), so these use a median
     rule and a per-sample cap (_kink_rule).
  2. duality with the encoder VJP, per sample: <u, JVP(v)> against <encode_vjp(u), v>, dot products in float64 on the
     host, on the synthetic and the margin weights.  Both sides use the same forward bits and masks, so this holds at
     kinks too.  Bound: DUALITY of sum|u * Jv|.
  3. fidelity on the well-conditioned weights of tests/margin_weights.py (130-input pool): every sample against the
     float64 oracle, eps absent and present, under three schedules, the SIMT path and chunking at IAN_CHUNK=16.  The bound
     is checked against the floor a single bf16-rounded tangent operand (v itself) moves the float64 JVP by: a third of it
     in relative L2, below it in max-abs (see BOUND).  bf16 mode on IAN.py against float32 is recorded and bounded.
  4. bit-level properties: z equals ian_encode_*'s bits, v = 0 gives 0, JVP(2v) = 2 JVP(v), reruns, graph replay against
     IAN_GRAPHS=0, IAN_PDL=0, and every other entry point's bits before and after a JVP call.
  5. the device form equals the host form at batches 3 and 47 and chunked (n = 40, IAN_CHUNK=16), eps present and absent,
     bf16 on IAN.py.
  6. torch forward mode: make_dual through ops.encode equals encode_jvp_dev bit for bit on the default and a side stream;
     forward mode through ops.decode(ops.encode(x)) equals decode_jvp(encode(x), encode_jvp(x, v)) bit for bit and
     matches the float64 oracle; a dual eps is refused; reverse mode is unchanged.
  7. errors: n < 0, NULL pointers, an unfinalized handle; n = 0 is a no-op.
Measured values go to encode_jvp.json when IAN_TEST_RECORD names a directory."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import margin_weights as mw
from test_ref_exec_encjvp import MAKE, fixture, jvp64

pytestmark = pytest.mark.gpu
CONFIG = {"simple": "IAN_simple.py", "full": "IAN.py", "v1": "IANv1.py"}
GRAPHS = ["simple", "full", "v1"]
ENV = ("IAN_STREAMK", "IAN_SPLITK", "IAN_GRAPHS", "IAN_PDL", "IAN_FINALIZE8", "IAN_CHUNK", "IAN_PATH")
# <u, Jv> - <J^T u, v> relative to sum|u * Jv|, float32 mode, every graph and path, eps absent and present: measured worst
# 6.3e-6 (IAN_simple, tensor cores, with eps) on an H100 80GB HBM3 at 700 W; the SIMT path reaches 4.4e-6.  This misses the
# decoder's 1e-6.  Both chains store every intermediate as a bf16 hi|lo pair (16 significand bits, relative rounding up to
# 2^-17 = 7.6e-6 per element), so a gap of this size needs no convention mismatch; a mismatched derivative rule would
# show at the size of the derivative, orders of magnitude larger.
DUALITY = 1e-5
# well-conditioned weights: per-sample relative L2 / max-abs over max|ref| against the float64 oracle.  Measured on an H100
# 80GB HBM3 at 700 W, worst of every run: 2.6e-4 / 4.0e-4 (IAN_simple, whole tiles).  The bf16-tangent floor (v rounded
# to bf16, float64) is 1.08e-3 / 6.1e-4 at its smallest (IAN.py).  The relative L2 bound is a third of that floor; the
# max-abs bound cannot be, because the worst sample already sits at two thirds of the floor.  That is the encoder chain's
# own precision, not the tangent's: the encoder VJP reaches 2.1e-4 / 3.0e-4 on the same weights (margin_weights.BOUNDS),
# and whole tiles are the worst schedule for both.  So max-abs is held below the floor, not below a third of it.
BOUND = (3.5e-4, 5.0e-4)
FLOOR_FACTOR = (3.0, 1.2)
BF16_L2 = 5e-2
RECORD = {}


def _record(key, value):
    RECORD[key] = value
    if os.environ.get("IAN_TEST_RECORD"):
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "encode_jvp.json"), "w") as f:
            json.dump(RECORD, f, indent=1, sort_keys=True)
    return value


def _seed(g):
    return int(np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                                    "ian_%s_golden.npz" % g))["weight_seed"])


_SYNTH = {}


def synth(g):
    if g not in _SYNTH:
        _SYNTH[g] = MAKE[g](_seed(g))
    return _SYNTH[g]


@pytest.fixture
def handles(npe, monkeypatch):
    """make(graph, weights, **env): a handle with exactly `env` among the schedule variables, closed at test end"""
    made = []

    def make(graph, weights, **env):
        for k in ENV:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, str(v))
        try:
            m = npe.IAN(CONFIG[graph], True, weights=weights)
        finally:
            for k in env:
                monkeypatch.delenv(k, raising=False)
        made.append(m)
        return m
    try:
        yield make
    finally:
        for m in made:
            m.close()


def _xv(n, seed, with_eps=False):
    rng = np.random.default_rng(seed)
    x = np.tanh(rng.standard_normal((n, 3, 64, 64))).astype(np.float32)
    v = rng.standard_normal((n, 3, 64, 64)).astype(np.float32)
    eps = rng.standard_normal((n, 100)).astype(np.float32) if with_eps else None
    return x, v, eps


def _per_sample_rel(got, ref):
    n = len(ref)
    return np.abs(got - ref).reshape(n, -1).max(axis=1) / np.abs(ref).reshape(n, -1).max(axis=1)


def _kink_rule(rel):
    """per-sample max-abs / max|ref| on the synthetic weights: a LeakyRectify of the encoder within float32 reach of its
    kink flips a mask in the GPU forward against float64 and moves that sample's JVP at full size (the encoder VJP's
    tests measure the same conditioning).  The fidelity check is test_fidelity_on_margin_weights."""
    return np.median(rel) <= 1e-3 and rel.max() <= 0.2


_REF = {}


def _ref64(g, key, P, x, v, eps):
    k = (g, key, x.tobytes(), v.tobytes(), None if eps is None else eps.tobytes())
    if k not in _REF:
        _REF[k] = jvp64(g, P, x, v, eps, device="cuda")
    return _REF[k]


# ---- 1. against the executed reference and the float64 oracle ------------------------------------------------------
@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("g", GRAPHS)
def test_against_executed_reference_and_oracle(handles, g, path):
    m = handles(g, synth(g))
    m.set_path(path)
    x, _, v, eps, jv = fixture()[g]
    rec = {}
    for j, e in enumerate((None, eps.astype(np.float32))):
        got = m.encode_jvp(x, v.astype(np.float32), e)
        ref = jvp64(g, synth(g), x, v.astype(np.float32), e, device="cuda")
        rec["exec_%d" % j] = _per_sample_rel(got, jv[j]).tolist()
        # the stored pairs are float64; the float32 rounding of v and eps moves the oracle by far less than the rule
        assert _per_sample_rel(ref, jv[j]).max() <= 1e-4
        assert max(rec["exec_%d" % j]) <= 0.2, rec
    for n in (3, 130):
        for with_eps in (False, True):
            x, v, e = _xv(n, 100 + n, with_eps)
            r = _per_sample_rel(m.encode_jvp(x, v, e), _ref64(g, "synth", synth(g), x, v, e))
            rec["n%d_%d" % (n, with_eps)] = {"median": float(np.median(r)), "max": float(r.max())}
            _record("1_%s_%s" % (g, path), rec)
            assert _kink_rule(r), (n, with_eps, r)


# ---- 2. duality with the encoder VJP ---------------------------------------------------------------------------------
@pytest.mark.parametrize("weights", ["synth", "margin"])
@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("g", GRAPHS)
def test_duality_with_encoder_vjp(handles, g, path, weights):
    m = handles(g, synth(g) if weights == "synth" else mw.weights(g))
    m.set_path(path)
    n = 6
    rec = {}
    for with_eps in (False, True):
        x, v, e = _xv(n, 300, with_eps)
        u = np.random.default_rng(301).standard_normal((n, 100)).astype(np.float32)
        jv = m.encode_jvp(x, v, e).astype(np.float64)
        jtu = m.encode_vjp(x, u, e).astype(np.float64)
        lhs = (u.astype(np.float64) * jv).sum(axis=1)
        rhs = (jtu * v.astype(np.float64)).reshape(n, -1).sum(axis=1)
        scale = np.abs(u.astype(np.float64) * jv).sum(axis=1)
        err = np.abs(lhs - rhs) / scale
        rec[str(with_eps)] = err.tolist()
        _record("2_%s_%s_%s" % (g, path, weights), rec)
        assert err.max() <= DUALITY, (with_eps, err)


# ---- 3. fidelity on the well-conditioned weights --------------------------------------------------------------------
def _pool_xv(n):
    p = mw.pool()
    v = np.random.default_rng(401).standard_normal((n, 3, 64, 64)).astype(np.float32)
    return p["x"][:n].astype(np.float32), v, p["eps"][:n].astype(np.float32)


def test_bound_is_below_the_bf16_tangent_floor():
    """the float64 JVP moves, on every sample of the pool, by at least FLOOR_FACTOR x BOUND when v is rounded to bf16 (one
    tangent operand in single-pass precision): 3x for relative L2, 1.2x for max-abs"""
    x, v, eps = _pool_xv(mw.POOL)
    vb = mw.bf16_round(v)
    rec = {}
    for g in GRAPHS:
        P = mw.weights(g)
        for e in (None, eps):
            ref = _ref64(g, "margin", P, x, v, e)
            slip = jvp64(g, P, x, vb, e, device="cuda")
            l2, mx = mw.rel_l2(slip, ref), mw.rel_max(slip, ref)
            rec["%s_%d" % (g, e is not None)] = (float(l2.min()), float(mx.min()))
            _record("3_floor", rec)
            assert FLOOR_FACTOR[0] * BOUND[0] <= l2.min() and FLOOR_FACTOR[1] * BOUND[1] <= mx.min(), (g, rec)


RUNS = [("default", "tc", {}), ("whole", "tc", {"IAN_SPLITK": 0, "IAN_STREAMK": 0}),
        ("sk", "tc", {"IAN_SPLITK": 0, "IAN_STREAMK": 2}), ("default", "simt", {}), ("chunk", "tc", {"IAN_CHUNK": 16})]


@pytest.mark.parametrize("g", GRAPHS)
def test_fidelity_on_margin_weights(handles, g):
    x, v, eps = _pool_xv(mw.POOL)
    P = mw.weights(g)
    rec = {}
    for name, path, env in RUNS:
        m = handles(g, P, **env)
        m.set_path(path)
        for e in (None, eps):
            ref = _ref64(g, "margin", P, x, v, e)
            got = m.encode_jvp(x, v, e)
            l2, mx = mw.rel_l2(got, ref), mw.rel_max(got, ref)
            rec["%s_%s_%d" % (name, path, e is not None)] = (float(l2.max()), float(mx.max()))
            _record("3_%s" % g, rec)
            assert l2.max() <= BOUND[0] and mx.max() <= BOUND[1], (name, path, rec)
    if g != "simple":
        m = handles(g, P)
        m.set_precision("bf16")
        ref = _ref64(g, "margin", P, x, v, None)
        l2 = mw.rel_l2(m.encode_jvp(x, v), ref)
        rec["bf16"] = float(l2.max())
        _record("3_%s" % g, rec)
        assert l2.max() <= BF16_L2, rec


# ---- 4. bit-level properties ------------------------------------------------------------------------------------------
def _others(m, z, x):
    """every other entry point's outputs on one handle"""
    rng = np.random.default_rng(501)
    dz = rng.standard_normal((len(x), 100)).astype(np.float32)
    return {"decode": m.sample_at(z), "encode": m.encode_images(x), "recon": m.reconstruct(x),
            "enc_vjp": m.encode_vjp(x, dz)}


@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("g", GRAPHS)
def test_bit_properties(handles, g, path):
    m = handles(g, synth(g))
    m.set_path(path)
    n = 5
    x, v, eps = _xv(n, 600, True)
    z_ref = m.encode_images(x)
    before = _others(m, z_ref, x)
    z, a = m.encode_jvp(x, v, return_z=True)
    assert np.array_equal(z, z_ref)
    ze, ae = m.encode_jvp(x, v, eps, return_z=True)
    assert np.array_equal(ze, m.encode(x, eps))
    assert np.all(m.encode_jvp(x, np.zeros_like(v)) == 0)
    assert np.array_equal(m.encode_jvp(x, 2 * v), 2 * a)
    for _ in range(2):
        assert np.array_equal(m.encode_jvp(x, v), a)
        assert np.array_equal(m.encode_jvp(x, v, eps), ae)
    after = _others(m, z_ref, x)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    for env in ({"IAN_GRAPHS": 0}, {"IAN_PDL": 0}):
        o = handles(g, synth(g), **env)
        o.set_path(path)
        assert np.array_equal(o.encode_jvp(x, v), a), env
        assert np.array_equal(o.encode_jvp(x, v, eps), ae), env


# ---- 5. launch forms ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [(3, {}, "fp32"), (47, {}, "fp32"), (40, {"IAN_CHUNK": 16}, "fp32"), (47, {}, "bf16")])
@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("g", GRAPHS)
def test_device_form_equals_host_form(handles, g, path, case):
    import torch
    n, env, prec = case
    if prec == "bf16" and g != "full":
        pytest.skip("bf16 mode is checked on IAN.py")
    m = handles(g, synth(g), **env)
    m.set_path(path)
    if prec == "bf16":
        m.set_precision("bf16")
    for with_eps in (False, True):
        x, v, eps = _xv(n, 700 + n, with_eps)
        z, dz = m.encode_jvp(x, v, eps, return_z=True)
        xd, vd = torch.from_numpy(x).cuda(), torch.from_numpy(v).cuda()
        ed = torch.from_numpy(eps).cuda() if with_eps else None
        zd, dd = torch.empty(n, 100, device="cuda"), torch.empty(n, 100, device="cuda")
        m.encode_jvp_dev(xd.data_ptr(), vd.data_ptr(), n, dd.data_ptr(), zd.data_ptr(), ed.data_ptr() if with_eps else 0)
        torch.cuda.synchronize()
        assert np.array_equal(dd.cpu().numpy(), dz) and np.array_equal(zd.cpu().numpy(), z), with_eps
        dd.zero_()
        m.encode_jvp_dev(xd.data_ptr(), vd.data_ptr(), n, dd.data_ptr(), 0, ed.data_ptr() if with_eps else 0)   # z left out
        torch.cuda.synchronize()
        assert np.array_equal(dd.cpu().numpy(), dz), with_eps


# ---- 6. torch --------------------------------------------------------------------------------------------------------
def _ops():
    import importlib
    return importlib.import_module("neural-photo-editor_b200.torch_ops")


@pytest.mark.parametrize("g", GRAPHS)
def test_torch_forward_mode(handles, npe, g):
    import torch
    import torch.autograd.forward_ad as fwAD
    ops = _ops()
    m = handles(g, synth(g))
    x, v, eps = _xv(4, 800, True)
    xd, vd, ed = torch.from_numpy(x).cuda(), torch.from_numpy(v).cuda(), torch.from_numpy(eps).cuda()
    ref = torch.empty(4, 100, device="cuda")
    m.encode_jvp_dev(xd.data_ptr(), vd.data_ptr(), 4, ref.data_ptr())
    refe = torch.empty(4, 100, device="cuda")
    m.encode_jvp_dev(xd.data_ptr(), vd.data_ptr(), 4, refe.data_ptr(), 0, ed.data_ptr())
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for stream in (None, side):
        with torch.cuda.stream(stream):
            with fwAD.dual_level():
                primal, tangent = fwAD.unpack_dual(ops.encode(m, fwAD.make_dual(xd, vd)))
                pe, te = fwAD.unpack_dual(ops.encode(m, fwAD.make_dual(xd, vd), ed))
                primal, tangent, pe, te = [t.clone() for t in (primal, tangent, pe, te)]
        torch.cuda.synchronize()
        assert torch.equal(tangent, ref) and torch.equal(te, refe), stream
        assert np.array_equal(primal.cpu().numpy(), m.encode_images(x))
        assert np.array_equal(pe.cpu().numpy(), m.encode(x, eps))
    # reverse mode is unchanged
    xr = xd.clone().requires_grad_(True)
    u = torch.randn(4, 100, device="cuda", generator=torch.Generator("cuda").manual_seed(801))
    (ops.encode(m, xr) * u).sum().backward()
    assert np.array_equal(xr.grad.cpu().numpy(), m.encode_vjp(x, u.cpu().numpy()))


@pytest.mark.parametrize("g", GRAPHS)
def test_torch_forward_mode_through_decode_of_encode(handles, npe, g):
    import torch
    import torch.autograd.forward_ad as fwAD
    from oracle import ian_torch as ot
    ops = _ops()
    P = mw.weights(g)
    m = handles(g, P)
    x, v, _ = _pool_xv(4)
    xd, vd = torch.from_numpy(x).cuda(), torch.from_numpy(v).cuda()
    with fwAD.dual_level():
        out = ops.decode(m, ops.encode(m, fwAD.make_dual(xd, vd)))
        tangent = fwAD.unpack_dual(out).tangent.cpu().numpy()
    z, dz = m.encode_jvp(x, v, return_z=True)
    assert np.array_equal(tangent, m.decode_jvp(z, dz))
    # float64 forward mode through the oracle's decoder of the oracle's encoder
    Q = {k: t.cuda() for k, t in ot.to_torch(P, torch.float64).items()}
    t64 = lambda a: torch.from_numpy(np.asarray(a, np.float64)).cuda()
    with torch.no_grad(), fwAD.dual_level():
        xx = fwAD.make_dual(t64(x), t64(v))
        if g == "simple":
            zz = ot.encode(Q, xx)
        else:
            zz = ot.full_encode(Q, xx, mw.made_masks("cuda"))
        dec = {"simple": ot.decode, "full": ot.full_decode, "v1": ot.v1_decode}[g]
        ref = fwAD.unpack_dual(dec(Q, zz)).tangent.cpu().numpy()
    # the margin weights certify the decoder at the pool's latents, not at encode(x): a decoder rectifier may sit near its
    # kink there (measured on an H100: <= 7.6e-5 on three samples of each graph, 7.7e-3 on one IANv1 sample), so this is
    # held to the composite rule of the encoder VJP's decode(encode(x)) test
    l2 = mw.rel_l2(tangent, ref)
    _record("6_composite_%s" % g, l2.tolist())
    assert np.median(l2) <= 1e-4 and l2.max() <= 1e-2, l2


def test_torch_dual_eps_refused(npe, model):
    import torch
    import torch.autograd.forward_ad as fwAD
    ops = _ops()
    x = torch.zeros(2, 3, 64, 64, device="cuda")
    eps = torch.zeros(2, 100, device="cuda")
    with fwAD.dual_level():
        with pytest.raises(ValueError):
            ops.encode(model, fwAD.make_dual(x, torch.ones_like(x)), fwAD.make_dual(eps, torch.ones_like(eps)))
        with pytest.raises(ValueError):
            ops.encode(model, x, fwAD.make_dual(eps, torch.ones_like(eps)))
        z = ops.encode(model, fwAD.make_dual(x, torch.ones_like(x)), eps)     # a plain eps is accepted
        assert fwAD.unpack_dual(z).tangent is not None


# ---- 7. errors -------------------------------------------------------------------------------------------------------
def test_errors(npe, model):
    import torch
    lib, h = model._lib, model._h
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    x = np.zeros((2, 3, 64, 64), np.float32)
    dz = np.full((2, 100), 7, np.float32)
    xd, dd = torch.zeros(2, 3, 64, 64, device="cuda"), torch.zeros(2, 100, device="cuda")
    assert lib.ian_encode_jvp_host(h, fp(x), fp(x), -1, None, None, fp(dz)) == -1
    assert lib.ian_encode_jvp_dev(h, xd.data_ptr(), xd.data_ptr(), -1, None, None, dd.data_ptr(), None) == -1
    assert lib.ian_encode_jvp_host(h, None, fp(x), 2, None, None, fp(dz)) == -1
    assert lib.ian_encode_jvp_host(h, fp(x), None, 2, None, None, fp(dz)) == -1
    assert lib.ian_encode_jvp_host(h, fp(x), fp(x), 2, None, None, None) == -1
    assert lib.ian_encode_jvp_dev(h, xd.data_ptr(), None, 2, None, None, dd.data_ptr(), None) == -1
    assert lib.ian_encode_jvp_host(h, None, None, 0, None, None, None) == 0
    assert lib.ian_encode_jvp_host(h, fp(x), fp(x), 0, None, None, fp(dz)) == 0 and np.all(dz == 7)
    assert model.encode_jvp(np.zeros((0, 3, 64, 64), np.float32), np.zeros((0, 3, 64, 64), np.float32)).shape == (0, 100)
    with pytest.raises(ValueError):
        model.encode_jvp(x, x[:1])
    with pytest.raises(TypeError):
        model.encode_jvp(x, x.astype(np.float64))
    raw = C.c_void_p()
    assert lib.ian_create(0, 0, C.byref(raw)) == 0
    try:
        assert lib.ian_encode_jvp_host(raw, fp(x), fp(x), 2, None, None, fp(dz)) == -3
    finally:
        lib.ian_destroy(raw)

"""GPU tests of the decoder Jacobian-vector product dx_hat = (d x_hat / d z) . v (include/ian_b200.h ian_decode_jvp_*,
API.IAN.decode_jvp / decoder_jacobian, torch_ops.decode under torch.autograd.forward_ad) on all three graphs and both
CUDA paths.

  1. against the executed reference (tests/golden/ref_exec_decjvp.npz) and the float64 oracle (torch forward mode on
     oracle/ian_torch.py, tests/test_ref_exec_decjvp.py) at batches 1, 3, SMs/3 + 3 and 130, under IAN_STREAMK=0/1/2 with
     IAN_SPLITK=0, and chunked (IAN_CHUNK=16 at n = 40).  The synthetic weights have rectifier kinks near the inputs, so
     these use a median rule in the style of the decoder VJP's (DESIGN section 5.6c), per-sample max-abs / max|ref|:
     median <= 1e-4 on IAN_simple and <= 5e-2 on the flow graphs, every sample <= 0.5 (_kink_rule).
  2. duality with the decoder VJP, per sample: <u, JVP(v)> against <decode_vjp(u), v>, dot products in float64 on the host.
     Both sides use the same forward bits and masks, so this holds at kinks too.  Bound: DUALITY of sum|u * Jv|.
  3. fidelity on the well-conditioned weights of tests/margin_weights.py (130-input pool): every sample against the float64
     oracle at margin_weights.BOUNDS["decoder"], under three schedules, the SIMT path and chunking; the bound is checked to
     be at most a third of the floor a single bf16-rounded tangent operand (v itself) moves the float64 JVP by.  bf16 mode
     on IAN.py against float32.
  4. bit-level properties: x_hat equals ian_decode_*'s bits, v = 0 gives 0, JVP(2v) = 2 JVP(v), reruns, graph replay
     against IAN_GRAPHS=0, IAN_PDL=0, and every other entry point's bits before and after a JVP call.
  5. the device form equals the host form at batches 3 and 47 and chunked.
  6. decoder_jacobian: equal to decode_jvp with one-hot tangents, against float64 torch.func.jacfwd on the margin weights,
     and its rows against decode_vjp with one-hot cotangents.
  7. torch forward mode: the tangent equals the C-ABI's bits, the primal equals ops.decode's; reverse mode is unchanged.
  8. errors: n < 0, NULL pointers, an unfinalized handle; n = 0 is a no-op.
Measured values go to decode_jvp.json when IAN_TEST_RECORD names a directory."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import margin_weights as mw
from test_ref_exec_decjvp import MAKE, fixture, jvp64, weight_seed

pytestmark = pytest.mark.gpu
CONFIG = {"simple": "IAN_simple.py", "full": "IAN.py", "v1": "IANv1.py"}
GRAPHS = ["simple", "full", "v1"]
ENV = ("IAN_STREAMK", "IAN_SPLITK", "IAN_GRAPHS", "IAN_PDL", "IAN_FINALIZE8", "IAN_CHUNK", "IAN_PATH")
# <u, Jv> - <J^T u, v> relative to sum|u * Jv|, float32 mode, every graph and path: measured worst 4.2e-7 (IAN.py, tensor
# cores) on an H100 80GB HBM3 at 700 W
DUALITY = 1e-6
BF16_L2 = 3e-2
RECORD = {}


def _record(key, value):
    RECORD[key] = value
    if os.environ.get("IAN_TEST_RECORD"):
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "decode_jvp.json"), "w") as f:
            json.dump(RECORD, f, indent=1, sort_keys=True)


_SYNTH = {}


def synth(g):
    if g not in _SYNTH:
        _SYNTH[g] = MAKE[g](weight_seed(g))
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


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _zv(n, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, 100)).astype(np.float32), rng.standard_normal((n, 100)).astype(np.float32)


def _per_sample_rel(got, ref):
    n = len(ref)
    return np.abs(got - ref).reshape(n, -1).max(axis=1) / np.abs(ref).reshape(n, -1).max(axis=1)


def _kink_rule(g, rel):
    """per-sample max-abs / max|ref| on the synthetic weights.  A rectifier within float32 reach of its kink flips a mask
    in the GPU forward against float64; the JVP carries that flip into a patch of pixels at full size, so its max-abs error
    is larger than the VJP's on the same samples (measured on an H100: medians <= 1.6e-5 on IAN_simple and <= 1.3e-2 on the
    flow graphs, single samples up to 0.23).  The fidelity check is test_fidelity_on_margin_weights."""
    return np.median(rel) <= (1e-4 if g == "simple" else 5e-2) and rel.max() <= 0.5


_REF = {}


def _ref64(g, P_key, P, z, v):
    key = (g, P_key, z.tobytes(), v.tobytes())
    if key not in _REF:
        _REF[key] = jvp64(g, P, z, v, device="cuda")
    return _REF[key]


# ---- 1. against the executed reference and the float64 oracle ------------------------------------------------------
@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("g", GRAPHS)
def test_against_executed_reference_and_oracle(handles, sms, g, path):
    m = handles(g, synth(g))
    m.set_path(path)
    _, z, v, dx = fixture()[g]
    got = m.decode_jvp(z.astype(np.float32), v.astype(np.float32))
    ref = jvp64(g, synth(g), z.astype(np.float32), v.astype(np.float32), device="cuda")
    rel_exec = _per_sample_rel(got, dx)
    rel = {"exec": rel_exec.tolist()}
    _record("1_%s_%s" % (g, path), rel)
    assert rel_exec.max() <= 0.5, rel_exec                # two pairs cannot carry a median
    # the stored pairs are float64; the float32 rounding of z and v moves the oracle by far less than the rule
    assert _per_sample_rel(ref, dx).max() <= 1e-4
    for n in (1, 3, sms // 3 + 3, 130):
        z, v = _zv(n, 100 + n)
        r = _per_sample_rel(m.decode_jvp(z, v), _ref64(g, "synth", synth(g), z, v))
        rel["n%d" % n] = r.tolist()
        _record("1_%s_%s" % (g, path), rel)
        assert _kink_rule(g, r), (n, r)


SCHED = {"sk0": {"IAN_SPLITK": 0, "IAN_STREAMK": 0}, "sk1": {"IAN_SPLITK": 0, "IAN_STREAMK": 1},
         "sk2": {"IAN_SPLITK": 0, "IAN_STREAMK": 2}, "chunk": {"IAN_CHUNK": 16}}


@pytest.mark.parametrize("sched", list(SCHED))
@pytest.mark.parametrize("g", GRAPHS)
def test_schedules_and_chunking(handles, g, sched):
    n = 40 if sched == "chunk" else 130
    z, v = _zv(n, 200 + n)
    ref = _ref64(g, "synth", synth(g), z, v)
    base = handles(g, synth(g)).decode_jvp(z, v)
    got = handles(g, synth(g), **SCHED[sched]).decode_jvp(z, v)
    r = _per_sample_rel(got, ref)
    _record("1s_%s_%s" % (g, sched), r.tolist())
    assert _kink_rule(g, r), r
    assert _kink_rule(g, _per_sample_rel(base, ref))


# ---- 2. duality with the decoder VJP ---------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("g", GRAPHS)
def test_duality_with_decoder_vjp(handles, g, path):
    m = handles(g, synth(g))
    m.set_path(path)
    n = 6
    z, v = _zv(n, 300)
    u = np.random.default_rng(301).standard_normal((n, 3, 64, 64)).astype(np.float32)
    jv = m.decode_jvp(z, v).astype(np.float64)
    jtu = m.decode_vjp(z, u).astype(np.float64)
    lhs = (u.astype(np.float64) * jv).reshape(n, -1).sum(axis=1)
    rhs = (jtu * v.astype(np.float64)).sum(axis=1)
    scale = np.abs(u.astype(np.float64) * jv).reshape(n, -1).sum(axis=1)
    err = np.abs(lhs - rhs) / scale
    _record("2_%s_%s" % (g, path), err.tolist())
    assert err.max() <= DUALITY, err


# ---- 3. fidelity on the well-conditioned weights --------------------------------------------------------------------
def _margin(g):
    return mw.weights(g, device="cuda")


def _pool_zv(n):
    z = mw.pool()["z"][:n]
    v = np.random.default_rng(401).standard_normal((n, 100)).astype(np.float32)
    return z, v


def test_bound_is_a_third_of_the_bf16_tangent_floor():
    """the float64 JVP moves, on every sample of the pool, by at least 3x margin_weights.BOUNDS["decoder"] when v is rounded
    to bf16 (one tangent operand in single-pass precision)"""
    z, v = _pool_zv(mw.POOL)
    vb = mw.bf16_round(v)
    rec = {}
    for g in GRAPHS:
        P = _margin(g)
        ref = _ref64(g, "margin", P, z, v)
        slip = jvp64(g, P, z, vb, device="cuda")
        l2, mx = mw.rel_l2(slip, ref), mw.rel_max(slip, ref)
        rec[g] = (float(l2.min()), float(mx.min()))
        b_l2, b_max = mw.BOUNDS["decoder"]
        assert 3 * b_l2 <= l2.min() and 3 * b_max <= mx.min(), (g, rec[g])
    _record("3_floor", rec)


RUNS = [("default", "tc", {}), ("whole", "tc", {"IAN_SPLITK": 0, "IAN_STREAMK": 0}),
        ("sk", "tc", {"IAN_SPLITK": 0, "IAN_STREAMK": 2}), ("default", "simt", {}), ("chunk", "tc", {"IAN_CHUNK": 48})]


@pytest.mark.parametrize("g", GRAPHS)
def test_fidelity_on_margin_weights(handles, g):
    z, v = _pool_zv(mw.POOL)
    ref = _ref64(g, "margin", _margin(g), z, v)
    b_l2, b_max = mw.BOUNDS["decoder"]
    rec = {}
    for name, path, env in RUNS:
        m = handles(g, _margin(g), **env)
        m.set_path(path)
        n = 100 if name == "chunk" else mw.POOL
        got = m.decode_jvp(z[:n], v[:n])
        l2, mx = mw.rel_l2(got, ref[:n]), mw.rel_max(got, ref[:n])
        rec["%s_%s" % (name, path)] = (float(l2.max()), float(mx.max()))
        assert l2.max() <= b_l2 and mx.max() <= b_max, (name, path, rec)
    if g != "simple":
        m = handles(g, _margin(g))
        m.set_precision("bf16")
        l2 = mw.rel_l2(m.decode_jvp(z, v), ref)
        rec["bf16"] = float(l2.max())
        assert l2.max() <= BF16_L2, rec
    _record("3_%s" % g, rec)


# ---- 4. bit-level properties ------------------------------------------------------------------------------------------
def _others(m, z, x):
    """every other entry point's outputs on one handle"""
    rng = np.random.default_rng(501)
    dx = rng.standard_normal((len(z), 3, 64, 64)).astype(np.float32)
    boxes = np.array([[3, 5, 20, 17]] * len(z), np.int32)
    return {"decode": m.sample_at(z), "vjp": m.decode_vjp(z, dx), "grad": m.grad(z, boxes, None),
            "encode": m.encode_images(x), "recon": m.reconstruct(x)}


@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("g", GRAPHS)
def test_bit_properties(handles, g, path):
    m = handles(g, synth(g))
    m.set_path(path)
    n = 5
    z, v = _zv(n, 600)
    x = np.random.default_rng(601).uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)
    before = _others(m, z, x)
    xh, a = m.decode_jvp(z, v, return_x_hat=True)
    assert np.array_equal(xh, before["decode"])
    assert np.all(m.decode_jvp(z, np.zeros_like(v)) == 0)
    assert np.array_equal(m.decode_jvp(z, 2 * v), 2 * a)
    for _ in range(2):
        assert np.array_equal(m.decode_jvp(z, v), a)
    after = _others(m, z, x)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    for env in ({"IAN_GRAPHS": 0}, {"IAN_PDL": 0}):
        o = handles(g, synth(g), **env)
        o.set_path(path)
        assert np.array_equal(o.decode_jvp(z, v), a), env


# ---- 5. launch forms ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [(3, {}), (47, {}), (40, {"IAN_CHUNK": 16})])
@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("g", GRAPHS)
def test_device_form_equals_host_form(handles, g, path, case):
    import torch
    n, env = case
    m = handles(g, synth(g), **env)
    m.set_path(path)
    z, v = _zv(n, 700 + n)
    xh, dx = m.decode_jvp(z, v, return_x_hat=True)
    zd, vd = torch.from_numpy(z).cuda(), torch.from_numpy(v).cuda()
    xd, dd = torch.empty(n, 3, 64, 64, device="cuda"), torch.empty(n, 3, 64, 64, device="cuda")
    m.decode_jvp_dev(zd.data_ptr(), vd.data_ptr(), n, dd.data_ptr(), xd.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(dd.cpu().numpy(), dx) and np.array_equal(xd.cpu().numpy(), xh)
    dd.zero_()
    m.decode_jvp_dev(zd.data_ptr(), vd.data_ptr(), n, dd.data_ptr())      # x_hat left out
    torch.cuda.synchronize()
    assert np.array_equal(dd.cpu().numpy(), dx)


# ---- 6. the Jacobian ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_decoder_jacobian(handles, g):
    import torch
    from oracle import ian_torch as ot
    m = handles(g, _margin(g))
    z = mw.pool()["z"][:2]
    J = m.decoder_jacobian(z)
    assert J.shape == (2, 100, 3, 64, 64)
    eye = np.eye(100, dtype=np.float32)
    for k in range(2):
        assert np.array_equal(J[k], m.decode_jvp(np.repeat(z[k:k + 1], 100, 0), eye))
    dec = {"simple": ot.decode, "full": ot.full_decode, "v1": ot.v1_decode}[g]
    Q = {k: t.cuda() for k, t in ot.to_torch(_margin(g), torch.float64).items()}
    rec = {}
    for k in range(2):
        jac = torch.func.jacfwd(lambda zz: dec(Q, zz[None])[0])(torch.from_numpy(z[k].astype(np.float64)).cuda())
        ref = jac.permute(3, 0, 1, 2).cpu().numpy()                         # (100, 3, 64, 64): column i = d x_hat / d z_i
        l2 = float(np.linalg.norm(J[k] - ref) / np.linalg.norm(ref))
        rec["jacfwd_%d" % k] = l2
        _record("6_%s" % g, rec)
        assert l2 <= mw.BOUNDS["decoder"][0], (k, l2)
    # rows: a few pixels' cotangents through decode_vjp
    pix = [(0, 0, 0), (1, 31, 17), (2, 63, 63), (0, 12, 50)]
    u = np.zeros((len(pix), 3, 64, 64), np.float32)
    for i, (c, r, q) in enumerate(pix):
        u[i, c, r, q] = 1
    rows = m.decode_vjp(np.repeat(z[:1], len(pix), 0), u).astype(np.float64)
    for i, (c, r, q) in enumerate(pix):
        col = J[0, :, c, r, q].astype(np.float64)
        err = np.abs(col - rows[i]).max() / np.abs(col).max()
        rec["row_%d" % i] = float(err)
        _record("6_%s" % g, rec)
        assert err <= 5e-5, (i, err)                       # measured worst 2.2e-5


# ---- 7. torch --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_torch_forward_mode(handles, npe, g):
    import torch
    import torch.autograd.forward_ad as fwAD
    import importlib
    ops = importlib.import_module("neural-photo-editor_b200.torch_ops")
    m = handles(g, synth(g))
    z, v = _zv(4, 800)
    zd, vd = torch.from_numpy(z).cuda(), torch.from_numpy(v).cuda()
    with fwAD.dual_level():
        out = ops.decode(m, fwAD.make_dual(zd, vd))
        primal, tangent = fwAD.unpack_dual(out)
        primal, tangent = primal.cpu().numpy(), tangent.cpu().numpy()
    assert np.array_equal(tangent, m.decode_jvp(z, v))
    assert np.array_equal(primal, ops.decode(m, zd).detach().cpu().numpy())
    zr = zd.clone().requires_grad_(True)
    u = torch.randn(4, 3, 64, 64, device="cuda", generator=torch.Generator("cuda").manual_seed(801))
    (ops.decode(m, zr) * u).sum().backward()
    assert np.array_equal(zr.grad.cpu().numpy(), m.decode_vjp(z, u.cpu().numpy()))


# ---- 8. errors -------------------------------------------------------------------------------------------------------
def test_errors(npe, model):
    import torch
    lib, h = model._lib, model._h
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    z = np.zeros((2, 100), np.float32)
    x = np.full((2, 3, 64, 64), 7, np.float32)
    zd, xd = torch.zeros(2, 100, device="cuda"), torch.zeros(2, 3, 64, 64, device="cuda")
    assert lib.ian_decode_jvp_host(h, fp(z), fp(z), -1, None, fp(x)) == -1
    assert lib.ian_decode_jvp_dev(h, zd.data_ptr(), zd.data_ptr(), -1, None, xd.data_ptr(), None) == -1
    assert lib.ian_decode_jvp_host(h, None, fp(z), 2, None, fp(x)) == -1
    assert lib.ian_decode_jvp_host(h, fp(z), None, 2, None, fp(x)) == -1
    assert lib.ian_decode_jvp_host(h, fp(z), fp(z), 2, None, None) == -1
    assert lib.ian_decode_jvp_dev(h, zd.data_ptr(), None, 2, None, xd.data_ptr(), None) == -1
    assert lib.ian_decode_jvp_host(h, None, None, 0, None, None) == 0
    assert lib.ian_decode_jvp_host(h, fp(z), fp(z), 0, None, fp(x)) == 0 and np.all(x == 7)
    assert model.decode_jvp(np.zeros((0, 100), np.float32), np.zeros((0, 100), np.float32)).shape == (0, 3, 64, 64)
    with pytest.raises(ValueError):
        model.decode_jvp(z, z[:1])
    with pytest.raises(TypeError):
        model.decode_jvp(z, z.astype(np.float64))
    raw = C.c_void_p()
    assert lib.ian_create(0, 0, C.byref(raw)) == 0
    try:
        assert lib.ian_decode_jvp_host(raw, fp(z), fp(z), 2, None, fp(x)) == -3
    finally:
        lib.ian_destroy(raw)

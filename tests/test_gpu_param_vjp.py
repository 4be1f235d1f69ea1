"""GPU tests of the IAN_simple decoder's parameter vector-Jacobian product (include/ian_b200.h ian_decode_param_vjp_*,
API.IAN.decode_param_vjp / decode_param_vjp_dev): dL/dtheta for the 13 trainable decoder tensors of
train_IAN_simple.py:353 on X_hat_fn's deterministic graph, on both CUDA paths.

  A. against float64 torch autograd (tests/test_oracle_param_vjp.py pins it to the numpy oracle) at batches 1, 3,
     SMs/3 + 3 and 128 with the default schedule, at SMs/3 + 3 under IAN_STREAMK=0, IAN_STREAMK=2 and IAN_SPLITK=0, and
     across batch chunks (IAN_CHUNK=16).  Per tensor relative L2 error; bounds in DESIGN.md section 5.6e.
  B. well-conditioned cases (every rectifier pre-activation >= 0.5): every tensor and dz to 3e-4 relative L2 on both paths
     under three schedules, which a single-pass bf16 slip in a weight-gradient kernel (~2e-3) would fail; and a channel
     with gamma = 0 in each decoder BatchNorm gets its (nonzero) beta / gamma gradients.
  C. dz is decode_vjp's bit for bit; repeated calls, graph replay against plain launches, IAN_PDL=0 and IAN_FINALIZE8=0 do
     not change a bit; the device-pointer form equals the host form; batch additivity.
  D. errors: IAN.py / IANv1.py are unsupported, a gradient pointer for a parameter without a gradient is invalid, n = 0
     does nothing.
Measured errors go to param_vjp_parity.json when IAN_TEST_RECORD names a directory."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import weights as ow

from test_oracle_param_vjp import PARAM_VJP_NAMES, param_grads64

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENV = ("IAN_STREAMK", "IAN_SPLITK", "IAN_GRAPHS", "IAN_PDL", "IAN_FINALIZE8", "IAN_CHUNK", "IAN_PATH")
RECORD = {}
# Rectifier kinks make these sums ill-conditioned at float32 scale: with these inputs the smallest rectifier pre-activation
# is ~3e-6, and in float64 itself a relative move of 1e-5 of z (the size of the float32 forward's error) changes the
# gradients by up to 1.9e-2 relative L2 (median 1.5e-3), while dec_out.W, which sees no rectifier after h3, moves by 7e-6.
# So every tensor is held to 5e-2, the median to 1e-2, and the best tensor to 1e-4 (measured on an H100: 1.9e-2, 5.2e-3 and
# 1.1e-5; a case without a flipped rectifier, B on the SIMT path, measured a median of 7.6e-6).
BOUND_MAX, BOUND_MEDIAN, BOUND_MIN = 5e-2, 1e-2, 1e-4


def _record(key, value):
    RECORD[key] = value
    if os.environ.get("IAN_TEST_RECORD"):
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "param_vjp_parity.json"), "w") as f:
            json.dump(RECORD, f, indent=1, sort_keys=True)


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture
def handles(npe, weights, monkeypatch):
    """make(P=None, **env): an IAN_simple handle built with exactly `env` among the schedule variables, closed at test end"""
    made = []

    def make(P=None, **env):
        for k in ENV:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, str(v))
        try:
            m = npe.IAN("IAN_simple.py", True, weights=weights if P is None else P)
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


@pytest.fixture(params=["tc", "simt"])
def path(request):
    return request.param


_ORACLE = {}


def _inputs(n, seed=0):
    rng = np.random.default_rng(1000 + n + seed)
    return rng.standard_normal((n, 100)).astype(np.float32), rng.standard_normal((n, 3, 64, 64)).astype(np.float32)


def _oracle(P, n):
    if n not in _ORACLE:
        z, dx = _inputs(n)
        _ORACLE[n] = (z, dx) + param_grads64({k: np.asarray(v, np.float64) for k, v in P.items()}, z, dx)
    return _ORACLE[n]


def _rel(got, ref):
    return {k: float(np.linalg.norm(got[k].astype(np.float64) - ref[k]) / np.linalg.norm(ref[k])) for k in ref}


def _check(rel, key):
    _record(key, rel)
    v = np.array(list(rel.values()))
    assert v.max() <= BOUND_MAX and np.median(v) <= BOUND_MEDIAN and v.min() <= BOUND_MIN, (key, rel)


def test_names_and_shapes(model):
    assert model.param_vjp_names() == PARAM_VJP_NAMES
    z, dx = _inputs(2)
    dz, g = model.decode_param_vjp(z, dx)
    shapes = dict(model_param_specs(model))
    assert sorted(g) == sorted(PARAM_VJP_NAMES)
    for k, v in g.items():
        assert v.shape == shapes[k] and v.dtype == np.float32 and np.all(np.isfinite(v)), k


def model_param_specs(model):
    import importlib
    return importlib.import_module("neural-photo-editor_b200.API").model_param_specs(model.kind)


@pytest.mark.parametrize("batch", ["1", "3", "sms3", "128"])
def test_against_float64_oracle(handles, weights, path, batch):
    n = _sms() // 3 + 3 if batch == "sms3" else int(batch)
    m = handles(IAN_PATH=path)
    z, dx, dz64, g64 = _oracle(weights, n)
    dz, g = m.decode_param_vjp(z, dx)
    _check(_rel(g, g64), "A_%s_n%d" % (path, n))
    assert np.linalg.norm(dz - dz64) / np.linalg.norm(dz64) <= BOUND_MAX


@pytest.mark.parametrize("sched", [{"IAN_STREAMK": "0"}, {"IAN_STREAMK": "2"}, {"IAN_SPLITK": "0"}, {"IAN_CHUNK": "16"}],
                         ids=["streamk0", "streamk2", "splitk0", "chunk16"])
def test_schedules_against_float64_oracle(handles, weights, path, sched):
    n = _sms() // 3 + 3
    m = handles(IAN_PATH=path, **sched)
    z, dx, _, g64 = _oracle(weights, n)
    _, g = m.decode_param_vjp(z, dx)
    _check(_rel(g, g64), "A_%s_%s" % (path, "_".join("%s%s" % kv for kv in sched.items())))


GAMMA_ZERO = (("bnorm_dec_fc2", 7), ("bnorm_dc1", 3), ("bnorm_dc2", 11), ("bnorm_dc3", 5))
# Measured on an H100: 3e-5 to 1.3e-4, uniform across tensors and dz (dec_out.W included), i.e. the float32 forward and the
# tanh seed of these weights rather than the contraction; a single-pass bf16 weight gradient would sit near 2e-3.
WELL_BOUND = 3e-4


def margin_weights(P, z, zero_gamma=()):
    """P with each decoder BatchNorm's beta raised, layer by layer, until every rectifier pre-activation of the batch z is
    >= 0.5.  With no rectifier near its kink the parameter gradients are well-conditioned, so the float32 fidelity of the
    kernels shows: in float64, dropping the lo cross terms of the weight-gradient contraction (single-pass bf16 operands)
    moves dec_conv1-3.W by ~2e-3 relative L2, the hi|lo scheme by ~5e-6.  Channels in zero_gamma get gamma = 0 first."""
    from oracle import ian_numpy as on
    Q = {k: np.array(v, np.float64) for k, v in P.items()}
    for name, ch in zero_gamma:
        Q[name + ".gamma"][ch] = 0.0
    for k, name in enumerate(("bnorm_dec_fc2", "bnorm_dc1", "bnorm_dc2", "bnorm_dc3")):
        u = on.simple_decode(Q, z, return_cache=True)[1][k]
        lo = u.min(axis=0) if u.ndim == 2 else u.min(axis=(0, 2, 3))
        Q[name + ".beta"] = Q[name + ".beta"] + np.maximum(0.0, 0.5 - lo)
    return {k: v.astype(np.float32) for k, v in Q.items()}


@pytest.mark.parametrize("sched", [{}, {"IAN_SPLITK": "0"}, {"IAN_STREAMK": "2"}], ids=["default", "splitk0", "streamk2"])
@pytest.mark.parametrize("batch", ["3", "sms3"])
def test_well_conditioned_against_float64_oracle(handles, weights, path, batch, sched):
    """every tensor and dz to WELL_BOUND relative L2 when no rectifier is near its kink"""
    n = _sms() // 3 + 3 if batch == "sms3" else int(batch)
    z, dx = _inputs(n, seed=11)
    P = margin_weights(weights, z)
    m = handles(P, IAN_PATH=path, **sched)
    dz64, g64 = param_grads64({k: np.asarray(v, np.float64) for k, v in P.items()}, z, dx)
    dz, g = m.decode_param_vjp(z, dx)
    rel = _rel(g, g64)
    rel["dz"] = float(np.linalg.norm(dz - dz64) / np.linalg.norm(dz64))
    _record("W_%s_n%d_%s" % (path, n, "_".join("%s%s" % kv for kv in sched.items()) or "default"), rel)
    assert max(rel.values()) <= WELL_BOUND, rel


def test_gamma_zero_channel(handles, weights, path):
    """gamma = 0 on one channel of every decoder BatchNorm (beta raised so the channel is active): its beta / gamma
    gradients, nonzero, and every tensor match the oracle to WELL_BOUND"""
    z, dx = _inputs(3, seed=5)
    P = margin_weights(weights, z, GAMMA_ZERO)
    m = handles(P, IAN_PATH=path)
    _, g64 = param_grads64({k: np.asarray(v, np.float64) for k, v in P.items()}, z, dx)
    _, g = m.decode_param_vjp(z, dx)
    rel = _rel(g, g64)
    _record("B_%s" % path, rel)
    assert max(rel.values()) <= WELL_BOUND, rel
    for name, ch in GAMMA_ZERO:
        for f in ("beta", "gamma"):
            ref = g64["%s.%s" % (name, f)][ch]
            assert abs(ref) > 1e-6, (name, f, ref)
            # one channel's sum, not a tensor's L2: measured up to 4.2e-4 of |ref|; a division by gamma would give inf / NaN
            assert abs(g["%s.%s" % (name, f)][ch] - ref) <= 2e-3 * abs(ref), (name, f, ref)


def test_bit_identities(handles, model, path):
    z, dx = _inputs(5, seed=7)
    model.set_path(path)
    try:
        dz, g = model.decode_param_vjp(z, dx)
        assert np.array_equal(dz, model.decode_vjp(z, dx))
        dz2, g2 = model.decode_param_vjp(z, dx)
        assert np.array_equal(dz, dz2) and all(np.array_equal(g[k], g2[k]) for k in g)
    finally:
        model.set_path("tc")
    for env in ({"IAN_GRAPHS": "0"}, {"IAN_PDL": "0"}, {"IAN_FINALIZE8": "0"}):
        m = handles(IAN_PATH=path, **env)
        dz3, g3 = m.decode_param_vjp(z, dx)
        assert np.array_equal(dz, dz3), env
        assert all(np.array_equal(g[k], g3[k]) for k in g), (env, [k for k in g if not np.array_equal(g[k], g3[k])])


def test_device_pointer_form_and_additivity(handles, path):
    """whole tiles and no split-K: a sample's forward is then the same bits at every batch size, so batch additivity is
    only a matter of the order of the weight-gradient sums"""
    import torch
    model = handles(IAN_PATH=path, IAN_SPLITK="0", IAN_STREAMK="0")
    n = 40
    z, dx = _inputs(n, seed=9)
    dz_h, g_h = model.decode_param_vjp(z, dx)
    zt, dxt = torch.from_numpy(z).cuda(), torch.from_numpy(dx).cuda()
    want = ["dec_conv2.W", "bnorm_dc1.gamma", "dec_out.W"]
    out = {k: torch.full(g_h[k].shape, float("nan"), device="cuda") for k in want}
    dzt = torch.empty((n, 100), device="cuda")
    torch.cuda.synchronize()
    model.decode_param_vjp_dev(zt.data_ptr(), dxt.data_ptr(), n, dzt.data_ptr(), {k: v.data_ptr() for k, v in out.items()})
    torch.cuda.synchronize()
    assert np.array_equal(dzt.cpu().numpy(), dz_h)
    for k in want:
        assert np.array_equal(out[k].cpu().numpy(), g_h[k]), k
    _, ga = model.decode_param_vjp(z[:17], dx[:17])
    _, gb = model.decode_param_vjp(z[17:], dx[17:])
    rel = {k: float(np.linalg.norm(ga[k] + gb[k] - g_h[k]) / np.linalg.norm(g_h[k])) for k in g_h}
    _record("C_additivity_%s" % path, rel)
    assert max(rel.values()) <= 1e-5, rel


def test_errors_and_empty_batch(npe, model):
    lib = model._lib
    specs = model_param_specs(model)
    z, dx = _inputs(2)
    buf = np.zeros(1 << 20, np.float32)
    ptrs = (C.c_void_p * len(specs))()
    ptrs[[n for n, _ in specs].index("enc_conv1.W")] = buf.ctypes.data
    f = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    assert lib.ian_decode_param_vjp_host(model._h, f(z), f(dx), 2, None, ptrs) == -1          # IAN_ERR_INVALID
    assert lib.ian_param_vjp_supported(0, [n for n, _ in specs].index("dec_conv1.W")) == 1
    assert lib.ian_param_vjp_supported(0, [n for n, _ in specs].index("bnorm_dc1.mean")) == 0
    assert lib.ian_param_vjp_supported(1, 0) == 0 and lib.ian_param_vjp_supported(2, 0) == 0
    dz, g = model.decode_param_vjp(np.zeros((0, 100), np.float32), np.zeros((0, 3, 64, 64), np.float32))
    assert dz.shape == (0, 100) and all(np.all(v == 0) for v in g.values())
    v1 = npe.IAN("IANv1.py", True, weights=ow.make_v1_weights(int(np.load(os.path.join(ROOT, "tests", "golden", "ian_v1_golden.npz"))["weight_seed"])))
    try:
        assert v1.param_vjp_names() == []
        assert lib.ian_decode_param_vjp_host(v1._h, f(z), f(dx), 2, None, None) == -4   # IAN_ERR_UNSUPPORTED
    finally:
        v1.close()

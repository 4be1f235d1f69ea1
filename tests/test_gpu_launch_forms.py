"""The two forms of every batch entry point compute the same bits.

Each of encode, decode, reconstruct, grad, decode_vjp, decode_param_vjp, encode_vjp and edit_loop has a device form
(ian_*_dev: the caller's device pointers, the caller's stream) and a host form (ian_*_host: the inputs staged into plan
buffers, the kernel chain replayed as a CUDA graph on plans of <= 32 images, the outputs copied back).  Both run one body
per batch chunk; this module holds every pair equal bit for bit:
  - on IAN_simple, IAN.py and IANv1.py, on the tensor-core and the SIMT path, and in bf16 mode on IAN.py;
  - at batch 3 (the host form captures and replays a graph) and 47 (plain launches in both forms), and with IAN_CHUNK=16
    at n = 40 (three chunks of 16, 16 and 8);
  - encode and encode_vjp with and without eps; grad and edit_loop with no target, a per-sample RGB and a frame target;
    reconstruct with and without z_out.
The parameter VJP exists on IAN_simple only; on the flow graphs both forms refuse it with the same error."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import weights as ow

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = {"simple": "IAN_simple.py", "full": "IAN.py", "v1": "IANv1.py"}
ENV = ("IAN_STREAMK", "IAN_SPLITK", "IAN_GRAPHS", "IAN_PDL", "IAN_FINALIZE8", "IAN_CHUNK", "IAN_PATH")
_WEIGHTS = {}


def _weights(graph):
    if graph not in _WEIGHTS:
        seed = int(np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % graph))["weight_seed"])
        make = {"simple": ow.make_simple_weights, "full": ow.make_full_weights, "v1": ow.make_v1_weights}[graph]
        _WEIGHTS[graph] = make(seed)
    return _WEIGHTS[graph]


def _inputs(n, seed):
    rng = np.random.default_rng(seed)
    c1, r1 = rng.integers(0, 48, n), rng.integers(0, 48, n)
    boxes = np.stack([c1, r1, c1 + rng.integers(1, 17, n), r1 + rng.integers(1, 17, n)], 1).astype(np.int32)
    f = lambda *s: rng.standard_normal(s).astype(np.float32)
    return {"x": rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32), "z": f(n, 100), "eps": f(n, 100),
            "rgb": rng.uniform(-1, 1, (n, 3)).astype(np.float32), "frame": rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32),
            "boxes": boxes, "dx": f(n, 3, 64, 64), "dz": f(n, 100)}


@pytest.fixture
def handle(npe, monkeypatch):
    """make(graph, path, precision, **env): a handle built with exactly `env` among the library's variables, closed when
    the test ends"""
    made = []

    def make(graph, path, precision, **env):
        for k in ENV:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, str(v))
        try:
            m = npe.IAN(CONFIG[graph], True, weights=_weights(graph), path=path)
        finally:
            for k in env:
                monkeypatch.delenv(k, raising=False)
        made.append(m)
        m.set_precision(precision)
        return m
    try:
        yield make
    finally:
        for m in made:
            m.close()


class _Dev:
    """device copies of numpy arrays and result tensors; every call through it is followed by a device synchronise (the
    library's default stream does not order against torch's)"""

    def __init__(self):
        import torch
        self.torch = torch
        self.keep = []

    def put(self, a):
        if a is None:
            return 0
        t = self.torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.keep.append(t)
        return t.data_ptr()

    def empty(self, shape, like=None):
        t = self.torch.zeros(shape, dtype=self.torch.float32, device="cuda") if like is None else \
            self.torch.from_numpy(np.ascontiguousarray(like)).cuda()
        self.keep.append(t)
        return t

    def run(self, call):
        self.torch.cuda.synchronize()
        call()
        self.torch.cuda.synchronize()


def _pairs(m, npe, inp):
    """(name, host-form result, device-form result) of every entry point on `inp`"""
    d = _Dev()
    n = len(inp["z"])
    x, z, eps, boxes, dx, dz = inp["x"], inp["z"], inp["eps"], inp["boxes"], inp["dx"], inp["dz"]
    xp, zp, ep, bp, dxp, dzp = d.put(x), d.put(z), d.put(eps), d.put(boxes), d.put(dx), d.put(dz)
    np_ = lambda t: t.cpu().numpy()
    out = []

    for tag, e, eptr in (("", None, 0), ("_eps", eps, ep)):
        zt = d.empty((n, 100))
        d.run(lambda: m.encode_dev(xp, n, zt.data_ptr(), eptr))
        out.append(("encode" + tag, m.encode(x, e), np_(zt)))
        dxt = d.empty((n, 3, 64, 64))
        d.run(lambda: m.encode_vjp_dev(xp, dzp, n, dxt.data_ptr(), eptr))
        out.append(("encode_vjp" + tag, m.encode_vjp(x, dz, e), np_(dxt)))

    xt = d.empty((n, 3, 64, 64))
    d.run(lambda: m.decode_dev(zp, n, xt.data_ptr()))
    out.append(("decode", m.sample_at(z), np_(xt)))

    xh, zh = m.reconstruct(x, return_z=True)
    xt, zt = d.empty((n, 3, 64, 64)), d.empty((n, 100))
    d.run(lambda: m.reconstruct_dev(xp, n, zt.data_ptr(), xt.data_ptr()))
    out += [("reconstruct_x", xh, np_(xt)), ("reconstruct_z", zh, np_(zt))]
    xh = np.empty_like(x)                                    # host form without z_out (the API always passes one)
    m._check(m._lib.ian_reconstruct_host(m._h, x.ctypes.data_as(C.POINTER(C.c_float)), n, None,
                                         xh.ctypes.data_as(C.POINTER(C.c_float))))
    xt = d.empty((n, 3, 64, 64))
    d.run(lambda: m.reconstruct_dev(xp, n, 0, xt.data_ptr()))
    out.append(("reconstruct_no_z", xh, np_(xt)))

    for tag, t in (("light", None), ("rgb", inp["rgb"]), ("frame", inp["frame"])):
        tp, frame = d.put(t), int(t is not None and t.ndim == 4)
        gt = d.empty((n, 100))
        d.run(lambda: m.grad_dev(zp, bp, tp, frame, n, gt.data_ptr()))
        out.append(("grad_" + tag, m.grad(z, boxes, t), np_(gt)))
        zt = d.empty((n, 100), like=z)
        d.run(lambda: m.edit_loop_dev(zt.data_ptr(), bp, tp, frame, n, 2, 0.05))
        out.append(("edit_loop_" + tag, m.edit_steps(z, boxes, t, n_steps=2, weight=0.05), np_(zt)))

    dzt = d.empty((n, 100))
    d.run(lambda: m.decode_vjp_dev(zp, dxp, n, dzt.data_ptr()))
    out.append(("decode_vjp", m.decode_vjp(z, dx), np_(dzt)))

    if m.kind == npe._lib.IAN_MODEL_SIMPLE:
        dzh, gh = m.decode_param_vjp(z, dx)
        dzt = d.empty((n, 100))
        gt = {k: d.empty(v.shape) for k, v in gh.items()}
        d.run(lambda: m.decode_param_vjp_dev(zp, dxp, n, dzt.data_ptr(), {k: t.data_ptr() for k, t in gt.items()}))
        out.append(("param_vjp_dz", dzh, np_(dzt)))
        out += [("param_vjp_" + k, gh[k], np_(gt[k])) for k in gh]
    else:
        errs = []
        for call in (lambda: m.decode_param_vjp(z, dx), lambda: m.decode_param_vjp_dev(zp, dxp, n, d.empty((n, 100)).data_ptr(), {})):
            with pytest.raises(npe._lib.IanError) as e:
                call()
            errs.append(str(e.value))
        assert errs[0] == errs[1], errs
    return out


CASES = [(g, p, "fp32", {}, (3, 47)) for g in ("simple", "full", "v1") for p in ("tc", "simt")]
CASES += [("full", "tc", "bf16", {}, (3, 47))]
CASES += [(g, "tc", "fp32", {"IAN_CHUNK": 16}, (40,)) for g in ("simple", "full", "v1")]


@pytest.mark.parametrize("graph,path,precision,env,sizes", CASES,
                         ids=["%s-%s-%s%s" % (c[0], c[1], c[2], "-chunk16" if c[3] else "") for c in CASES])
def test_device_form_equals_host_form(handle, npe, graph, path, precision, env, sizes):
    m = handle(graph, path, precision, **env)
    for n in sizes:
        for name, host, dev in _pairs(m, npe, _inputs(n, 7000 + n)):
            assert host.shape == dev.shape and host.dtype == dev.dtype, (name, n, host.shape, dev.shape)
            assert np.isfinite(host).all(), (name, n)
            assert np.array_equal(host, dev), (name, n, float(np.abs(host.astype(np.float64) - dev).max()))

"""GPU tests of the encoder vector-Jacobian product dx = (d z / d x)^T . dz (include/ian_b200.h ian_encode_vjp_*,
API.IAN.encode_vjp, torch_ops.encode) on all three graphs and both CUDA paths.

  A. against the float64 reverse mode of tests/encode_vjp_oracle.py (itself pinned to float64 torch autograd by
     tests/test_oracle_encode_vjp.py), eps absent and present, at batches 1, 3, SMs/3 + 3 and 130, on probe samples (first,
     middle, last).  Three cotangents, one per sample in turn: a dense Gaussian dz, a one-hot dz (the saliency of one
     latent) and the dz of the latent-consistency loss |E(x) - E(x')|^2.  Metric: per-sample max-abs error / max|ref|.
     Every graph: median <= 1e-4 (the brush-gradient rule) and every sample <= 1e-1 rather than 1e-2.  The encoder VJP
     is ill-conditioned at the scale of a float32 forward: dx changes by 0.8 W wherever a LeakyRectify pre-activation
     changes sign.  In float64 alone, scaling the input of a sample by 1 + s N(0,1) (three draws) moves its VJP, as a
     fraction of max|dx|, by:
        IAN_simple, with eps (seed 1001):  s = 1e-5: up to 3.0e-2;  s = 1e-4: up to 3.9e-2
        IAN_simple, no eps (seed 1):       s = 1e-5: 3.6e-6;         s = 1e-4: up to 2.0e-2
        IAN.py, with eps (seed 1001):      s = 1e-5: up to 3.0e-2;  s = 1e-4: up to 5.6e-2
        IAN.py, no eps (seed 1):           s = 1e-5: 2.5e-7;         s = 1e-4: up to 2.8e-2
     (IANv1's encoder and flow are IAN.py's, with the same weights here), and the GPU forward is only held to 2e-4.
     Measured on an H100, tensor-core path (enc_conv1's adjoint on conv1_bwd_tc_kernel): IAN_simple median 3.8e-5,
     worst 5.0e-2; IAN.py / IANv1 median 2.9e-5, worst 3.9e-2 (SIMT path: 1.1e-5 / 6.5e-3 and 9.2e-6 / 1.7e-3).  The schedule and chunk tests check 3-4 probes, whose
     median is a single sample: they are held to median <= 1e-3 (measured worst 2.6e-4).
     bf16 against float32 on IAN.py: relative L2 <= 0.1 (measured 0.075).
  B. schedules: whole tiles (IAN_SPLITK=0 IAN_STREAMK=0) and forced stream-K (IAN_SPLITK=0 IAN_STREAMK=2) stay within A's
     bounds, on IAN.py and IAN_simple at batch 130.
  C. properties: dz = 0 gives dx = 0 exactly; reruns, graph replay (IAN_GRAPHS=0), programmatic dependent launch
     (IAN_PDL=0) and the first call (which builds the lazy state) are bit-identical; a chunked batch of 520 on both
     sides of the chunk boundary; bf16 against float32 on IAN.py; encode / decode / grad on a plan give the same bits
     before and after an encoder VJP on it.
  D. the torch autograd binding: bit-identical to encode_vjp_dev on the default and a side stream, decode(encode(x))
     against float64 autograd of the composite, once-differentiable, eps.requires_grad refused.
These bounds are set by rectifier kinks of the synthetic weights.  The fidelity check is tests/test_gpu_well_conditioned.py:
on weights with no rectifier near its kink, every sample on every graph, with and without eps, to 5.2e-4 relative L2 and
3.65e-4 max-abs / max|ref| (measured on an H100 80GB HBM3 at 700 W: worst 2.1e-4 / 3.0e-4 on IAN_simple, 1.0e-4 / 1.2e-4 on the
flow graphs).
Measured values go to encvjp_parity.json when IAN_TEST_RECORD names a directory."""
import json
import os

import numpy as np
import pytest

from oracle import ian_full_numpy as fn
from oracle import weights as ow

import encode_vjp_oracle as eo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RECORD = {}


def _record(key, value):
    RECORD[key] = value
    if os.environ.get("IAN_TEST_RECORD"):
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "encvjp_parity.json"), "w") as f:
            json.dump(RECORD, f, indent=1, sort_keys=True)
    return value


def _seed(name):
    return int(np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % name))["weight_seed"])


MAKE = {"simple": ow.make_simple_weights, "full": ow.make_full_weights, "v1": ow.make_v1_weights}
CONFIG = {"simple": "IAN_simple.py", "full": "IAN.py", "v1": "IANv1.py"}


class Graph:
    def __init__(self, name, P, model):
        self.name, self.P, self.m = name, P, model
        self.masks = fn.made_masks(model.made_ordering.astype(np.float32)) if name != "simple" else None
        self.cache = {}

    def oracle(self, x, dz, eps, idx):
        out = []
        for k in idx:
            key = (x[k].tobytes(), dz[k].tobytes(), None if eps is None else eps[k].tobytes())
            if key not in self.cache:
                e = None if eps is None else eps[k:k + 1]
                if self.name == "simple":
                    self.cache[key] = eo.simple_encode_vjp(self.P, x[k:k + 1], dz[k:k + 1], e)[0]
                else:
                    self.cache[key] = eo.full_encode_vjp(self.P, x[k:k + 1], self.masks, dz[k:k + 1], e)[0]
            out.append(self.cache[key])
        return np.stack(out)


@pytest.fixture(scope="module")
def graphs(npe, model, weights):
    full = npe.IAN("IAN.py", True, weights=MAKE["full"](_seed("full")))
    v1 = npe.IAN("IANv1.py", True, weights=MAKE["v1"](_seed("v1")))
    out = {"simple": Graph("simple", weights, model), "full": Graph("full", MAKE["full"](_seed("full")), full),
           "v1": Graph("v1", MAKE["v1"](_seed("v1")), v1)}
    yield out
    full.close()
    v1.close()


def _inputs(m, n, with_eps, seed):
    """images, cotangents (Gaussian / one-hot / latent-consistency, one per sample in turn) and eps"""
    rng = np.random.default_rng(seed)
    x = np.tanh(rng.standard_normal((n, 3, 64, 64))).astype(np.float32)
    eps = rng.standard_normal((n, 100)).astype(np.float32) if with_eps else None
    dz = rng.standard_normal((n, 100)).astype(np.float32)
    z = m.encode(x, eps)
    for k in range(n):
        if k % 3 == 1:
            dz[k] = 0.0
            dz[k, (7 * k) % 100] = 1.0
        elif k % 3 == 2:
            dz[k] = 2.0 * (z[k] - z[(k + 1) % n])
    return x, dz, eps


def _probes(n):
    return sorted({0, n // 2, n - 1})


def _per_sample_rel(dx, ref):
    n = len(ref)
    return np.abs(dx - ref).reshape(n, -1).max(axis=1) / np.abs(ref).reshape(n, -1).max(axis=1)


def _check(rel, tag, name, few=False):
    """few: 3-4 probe samples, whose median is one sample's value -- held to the flow graphs' 1e-3"""
    _record(tag, {"median": float(np.median(rel)), "max": float(rel.max())})
    assert np.median(rel) <= (1e-3 if few else 1e-4) and rel.max() <= 1e-1, (tag, rel)


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("name", ["simple", "full", "v1"])
def test_against_float64_oracle(graphs, name, path):
    g = graphs[name]
    g.m.set_path(path)
    try:
        rels = []
        for n in (1, 3, _sms() // 3 + 3, 130):
            for with_eps in (False, True):
                x, dz, eps = _inputs(g.m, n, with_eps, seed=n + 1000 * with_eps)
                dx = g.m.encode_vjp(x, dz, eps)
                assert dx.shape == x.shape and np.isfinite(dx).all()
                idx = _probes(n)
                rels.append(_per_sample_rel(dx[idx], g.oracle(x, dz, eps, idx)))
        _check(np.concatenate(rels), "oracle_%s_%s" % (name, path), name)
    finally:
        g.m.set_path("tc")


@pytest.mark.parametrize("sched", [{"IAN_SPLITK": "0", "IAN_STREAMK": "0"}, {"IAN_SPLITK": "0", "IAN_STREAMK": "2"},
                                   {"IAN_SPLITK": "0"}], ids=["whole", "streamk", "nosplitk"])
@pytest.mark.parametrize("name", ["simple", "full"])
def test_schedules(npe, graphs, monkeypatch, name, sched):
    g = graphs[name]
    for k, v in sched.items():
        monkeypatch.setenv(k, v)
    m = npe.IAN(CONFIG[name], True, weights=g.P)
    try:
        x, dz, eps = _inputs(m, 130, True, seed=5)
        dx = m.encode_vjp(x, dz, eps)
        idx = _probes(130)
        _check(_per_sample_rel(dx[idx], g.oracle(x, dz, eps, idx)), "sched_%s_%s" % (name, "_".join(sorted(sched.values()))), name, few=True)
    finally:
        m.close()


@pytest.mark.parametrize("name", ["simple", "full", "v1"])
def test_zero_rerun_first_call(npe, graphs, name):
    """dz = 0 -> dx = 0 exactly; the first call on a fresh handle (lazy weights, plan buffers, graph capture) equals the
    later ones bit for bit, through the host API (graph replay) and the device-pointer API."""
    import torch
    g = graphs[name]
    m = npe.IAN(CONFIG[name], True, weights=g.P)
    try:
        x, dz, eps = _inputs(g.m, 4, True, seed=11)
        first = m.encode_vjp(x, dz, eps)
        assert np.array_equal(first, m.encode_vjp(x, dz, eps))
        assert np.array_equal(first, m.encode_vjp(x, dz, eps))
        assert not m.encode_vjp(x, np.zeros_like(dz), eps).any()
        xd, dzd, ed = (torch.from_numpy(a).cuda() for a in (x, dz, eps))
        dxd = torch.empty_like(xd)
        m.encode_vjp_dev(xd.data_ptr(), dzd.data_ptr(), 4, dxd.data_ptr(), ed.data_ptr())
        torch.cuda.synchronize()
        assert np.array_equal(first, dxd.cpu().numpy())
    finally:
        m.close()


@pytest.mark.parametrize("name", ["simple", "full"])
def test_graph_replay_and_pdl(npe, graphs, monkeypatch, name):
    g = graphs[name]
    for with_eps in (False, True):
        x, dz, eps = _inputs(g.m, 3, with_eps, seed=21 + with_eps)
        ref = g.m.encode_vjp(x, dz, eps)
        assert np.array_equal(ref, g.m.encode_vjp(x, dz, eps))             # replay of the captured graph
        for env in ({"IAN_GRAPHS": "0"}, {"IAN_PDL": "0", "IAN_GRAPHS": "0"}):
            for k, v in env.items():
                monkeypatch.setenv(k, v)
            m = npe.IAN(CONFIG[name], True, weights=g.P)
            for k in env:
                monkeypatch.delenv(k)
            try:
                assert np.array_equal(ref, m.encode_vjp(x, dz, eps)), env
            finally:
                m.close()


def test_chunked_batch(graphs):
    """520 samples run as chunks of 512 + 8: probes on both sides of the boundary against the oracle"""
    g = graphs["full"]
    x, dz, eps = _inputs(g.m, 520, True, seed=31)
    dx = g.m.encode_vjp(x, dz, eps)
    idx = [0, 511, 512, 519]
    _check(_per_sample_rel(dx[idx], g.oracle(x, dz, eps, idx)), "chunk_520", "full", few=True)


def test_bf16_against_fp32(graphs):
    g = graphs["full"]
    x, dz, eps = _inputs(g.m, 64, False, seed=41)
    ref = g.m.encode_vjp(x, dz)
    g.m.set_precision("bf16")
    try:
        dx = g.m.encode_vjp(x, dz)
    finally:
        g.m.set_precision("fp32")
    rel = float(np.linalg.norm(dx - ref) / np.linalg.norm(ref))
    _record("bf16_rel_l2", rel)
    assert rel <= 0.1, rel


@pytest.mark.parametrize("name", ["simple", "full", "v1"])
def test_existing_entry_points_unchanged(npe, graphs, name):
    """encode, decode and grad on a plan give the same bits before and after an encoder VJP on the same plan"""
    g = graphs[name]
    m = npe.IAN(CONFIG[name], True, weights=g.P)
    try:
        x, dz, eps = _inputs(g.m, 5, True, seed=51)
        boxes = np.array([[10, 12, 30, 40]] * 5, np.int32)

        def run():
            z = m.encode(x, eps)
            return z, m.sample_at(z), m.grad(z, boxes), m.reconstruct(x)

        before = run()
        m.encode_vjp(x, dz, eps)
        after = run()
        for a, b in zip(before, after):
            assert np.array_equal(a, b)
    finally:
        m.close()


# ---- D. torch binding ---------------------------------------------------------------------------------------------
def _torch_ops():
    import importlib
    return importlib.import_module("neural-photo-editor_b200.torch_ops")


def test_torch_binding_bits_and_streams(npe, graphs):
    import torch
    ops = _torch_ops()
    for name in ("simple", "full"):
        m = graphs[name].m
        x, dz, eps = _inputs(m, 6, True, seed=61)
        xd, dzd, ed = (torch.from_numpy(a).cuda() for a in (x, dz, eps))
        ref = torch.empty_like(xd)
        m.encode_vjp_dev(xd.data_ptr(), dzd.data_ptr(), 6, ref.data_ptr(), ed.data_ptr())
        torch.cuda.synchronize()
        for side in (False, True):
            s = torch.cuda.Stream() if side else torch.cuda.current_stream()
            with torch.cuda.stream(s):
                xr = xd.clone().requires_grad_(True)
                z = ops.encode(m, xr, ed)
                (gx,) = torch.autograd.grad(z, xr, grad_outputs=dzd)
            torch.cuda.synchronize()
            assert torch.equal(gx, ref), (name, side)


def test_torch_decode_of_encode(npe, graphs):
    """decode(encode(x)) backpropagates to x and matches float64 autograd of the composite (IAN_simple)"""
    import torch
    from oracle import ian_torch as ot
    g = graphs["simple"]
    ops = _torch_ops()
    rng = np.random.default_rng(71)
    x = np.tanh(rng.standard_normal((2, 3, 64, 64))).astype(np.float32)
    w = rng.standard_normal((2, 3, 64, 64)).astype(np.float32)
    xr = torch.from_numpy(x).cuda().requires_grad_(True)
    loss = (ops.decode(g.m, ops.encode(g.m, xr)) * torch.from_numpy(w).cuda()).sum()
    loss.backward()
    P64 = ot.to_torch(g.P, torch.float64)
    x64 = torch.from_numpy(x.astype(np.float64)).requires_grad_(True)
    (ot.decode(P64, ot.encode(P64, x64)) * torch.from_numpy(w.astype(np.float64))).sum().backward()
    rel = _per_sample_rel(xr.grad.cpu().numpy(), x64.grad.numpy())
    _record("torch_composite", float(rel.max()))
    assert rel.max() <= 1e-2, rel


def test_torch_once_differentiable_and_eps_refused(npe, graphs):
    import torch
    m = graphs["simple"].m
    ops = _torch_ops()
    x = torch.zeros(1, 3, 64, 64, device="cuda", requires_grad=True)
    z = ops.encode(m, x)
    (gx,) = torch.autograd.grad(z.sum(), x, create_graph=True)
    with pytest.raises(RuntimeError):
        gx.sum().backward()
    with pytest.raises(ValueError, match="eps"):
        ops.encode(m, x, torch.zeros(1, 100, device="cuda", requires_grad=True))


def test_invalid_arguments(graphs):
    m = graphs["simple"].m
    lib = m._lib
    assert lib.ian_encode_vjp_host(m._h, None, 1, None, None, None) != 0
    x = np.zeros((1, 3, 64, 64), np.float32)
    with pytest.raises(Exception):
        m.encode_vjp(x, np.zeros((2, 100), np.float32))

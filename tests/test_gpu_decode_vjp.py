"""GPU tests of the decoder vector-Jacobian product dz = (d x_hat / d z)^T . dx_hat (include/ian_b200.h
ian_decode_vjp_*, API.IAN.decode_vjp, torch_ops.decode) on all three graphs and both CUDA paths.

  A. against float64 autograd / the float64 numpy decoder backward, with three cotangents: a dense Gaussian, NPE's
     per-pixel weighted brush (a soft round mask times (x_hat - target)) and an L1 box loss.  Per-sample max-abs error /
     max|ref|, with the brush-gradient convention of tests/test_gpu_parity.py and test_flow_model_brush_gradients:
     IAN_simple median <= 1e-4 and every sample <= 1e-2.  The flow graphs (IAN.py, IANv1.py): every sample <= 5e-2 (the
     outlier cap of assert_grad_close in tests/test_gpu_parity.py) and one <= 1e-4, because over the whole frame their VJP
     is ill-conditioned at the scale of a float32 forward.  In float64 itself, moving z so that x_hat moves by 2.3e-5 (the
     GPU forward is held to 2e-4) changes the VJP of these inputs by 5e-4 to 1.1e-2 on IAN.py and 9e-4 to 2.8e-2 on IANv1
     -- the steep Beta ratio 2a/(a+b+1e-8) where both sigmoids are small, and rectifier kinks (DESIGN section 3).  Measured
     on an H100: IAN.py <= 9.0e-3, IANv1 <= 2.9e-2 (the dense cotangent of the sample whose float64 VJP moved 2.8e-2), and
     samples without such pixels at 5e-6 to 4e-5.
  B. a box-loss cotangent formed in float32 with the kernels' own expression reproduces grad() bit for bit: the dense
     seed shares every instruction after the seed value with the box seed.
  C. properties: zero in -> zero out, reruns, graph replay and programmatic dependent launch bit-identical, chunked
     batches, bf16 against float32.
  D. the torch autograd binding: bit-identical to decode_vjp on the default and a side stream, a torch-driven SGD loop
     against the float64 oracle, once-differentiable.
These bounds are set by rectifier kinks of the synthetic weights.  The fidelity check is tests/test_gpu_well_conditioned.py:
on weights with no rectifier near its kink, every sample on every graph to 1.7e-4 relative L2 and 1.1e-4 max-abs / max|ref|
(measured on an H100 80GB HBM3 at 700 W: worst 8.1e-5 / 7.4e-5).
Measured values go to vjp_parity.json when IAN_TEST_RECORD names a directory."""
import json
import os

import numpy as np
import pytest

from oracle import ian_numpy as on
from oracle import weights as ow

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RECORD = {}


def _record(key, value):
    RECORD[key] = value
    if os.environ.get("IAN_TEST_RECORD"):
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "vjp_parity.json"), "w") as f:
            json.dump(RECORD, f, indent=1, sort_keys=True)


def simple_decode_vjp(P, z, dx):
    """float64 numpy oracle: the IAN_simple decoder backward of oracle/ian_numpy.py seeded with dx * (1 - x_hat^2)."""
    xh, cache = on.simple_decode(P, z, return_cache=True)
    return on._decoder_backward(P, cache, np.asarray(dx, np.float64) * (1 - xh ** 2))


def torch_decode_vjp(P, z, dx, decode_fn):
    """float64 torch oracle: autograd of the restatement with grad_outputs=dx."""
    import torch
    z = z.clone().requires_grad_(True)
    (g,) = torch.autograd.grad(decode_fn(P, z), z, grad_outputs=dx)
    return g


def _seed(name):
    return int(np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % name))["weight_seed"])


class Graph:
    def __init__(self, name, P, model):
        import torch
        from oracle import ian_torch as ot
        self.name, self.P, self.m = name, P, model
        self.P64 = ot.to_torch(P, torch.float64)
        self.dec = {"simple": ot.decode, "full": ot.full_decode, "v1": ot.v1_decode}[name]

    def xhat64(self, z):
        import torch
        return self.dec(self.P64, torch.from_numpy(np.asarray(z, np.float64))).numpy()

    def vjp64(self, z, dx):
        import torch
        if self.name == "simple":
            return simple_decode_vjp(self.P, z, dx)
        return torch_decode_vjp(self.P64, torch.from_numpy(np.asarray(z, np.float64)), torch.from_numpy(np.asarray(dx, np.float64)),
                                self.dec).numpy()


@pytest.fixture(scope="module")
def graphs(npe, model, weights):
    full = npe.IAN("IAN.py", True, weights=ow.make_full_weights(_seed("full")))
    v1 = npe.IAN("IANv1.py", True, weights=ow.make_v1_weights(_seed("v1")))
    out = {"simple": Graph("simple", weights, model), "full": Graph("full", ow.make_full_weights(_seed("full")), full),
           "v1": Graph("v1", ow.make_v1_weights(_seed("v1")), v1)}
    yield out
    full.close()
    v1.close()


@pytest.fixture(params=["tc", "simt"])
def path(graphs, request):
    for g in graphs.values():
        g.m.set_path(request.param)
    yield request.param
    for g in graphs.values():
        g.m.set_path("tc")
        if g.name != "simple":
            g.m.set_precision("fp32")


def _per_sample_rel(dz, ref):
    n = len(ref)
    return np.abs(dz - ref).reshape(n, -1).max(axis=1) / np.abs(ref).reshape(n, -1).max(axis=1)


def soft_round_mask(n, rng):
    """per-sample gaussian brush footprint (1,64,64) at a random centre: NPE's "user mask" as a soft round brush"""
    yy, xx = np.mgrid[0:64, 0:64]
    cy, cx = rng.uniform(12, 52, n), rng.uniform(12, 52, n)
    r = rng.uniform(4, 10, n)
    m = np.exp(-((yy[None] - cy[:, None, None]) ** 2 + (xx[None] - cx[:, None, None]) ** 2) / (2 * r[:, None, None] ** 2))
    return m[:, None]


def _cotangents(xh, rng):
    n = len(xh)
    dense = rng.standard_normal(xh.shape)
    target = rng.uniform(-1, 1, xh.shape)
    brush = soft_round_mask(n, rng) * (xh - target)
    l1 = np.zeros_like(xh)
    for k in range(n):
        c1, r1 = rng.integers(0, 48, 2)
        c2, r2 = c1 + rng.integers(4, 17), r1 + rng.integers(4, 17)
        l1[k, :, r1:r2, c1:c2] = np.sign(xh[k, :, r1:r2, c1:c2] - target[k, :, r1:r2, c1:c2]) / (3 * (r2 - r1) * (c2 - c1))
    return {"dense": dense, "brush": brush, "l1": l1}


_ORACLE = {}


@pytest.mark.parametrize("graph", ["simple", "full", "v1"])
def test_vjp_against_float64_oracle(graphs, path, graph):
    g = graphs[graph]
    if graph not in _ORACLE:                     # the oracle is path-independent: compute it once per graph
        rng = np.random.default_rng(10)
        z = rng.standard_normal((4, 100)).astype(np.float32)
        cts = {k: v.astype(np.float32) for k, v in _cotangents(g.xhat64(z), rng).items()}
        _ORACLE[graph] = (z, cts, {k: g.vjp64(z, v) for k, v in cts.items()})
    z, cts, refs = _ORACLE[graph]
    rel = {k: _per_sample_rel(g.m.decode_vjp(z, cts[k]), refs[k]) for k in cts}
    allr = np.concatenate(list(rel.values()))
    _record("A_%s_%s" % (graph, path), {k: v.tolist() for k, v in rel.items()})
    if graph != "simple":
        assert allr.max() <= 5e-2 and allr.min() <= 1e-4, rel
    else:
        assert np.median(allr) <= 1e-4 and allr.max() <= 1e-2, rel


def _box_cotangent(xh, boxes, target):
    """the box loss's dL/dx_hat in float32, formed exactly as the seed kernels form it"""
    dx = np.zeros_like(xh)
    for k, (c1, r1, c2, r2) in enumerate(boxes):
        inv = np.float32(1) / np.float32(3 * (r2 - r1) * (c2 - c1))
        if target is None:
            dx[k, :, r1:r2, c1:c2] = inv
        else:
            t = target[k].reshape(3, 1, 1) if target.ndim == 2 else target[k, :, r1:r2, c1:c2]
            dx[k, :, r1:r2, c1:c2] = (np.float32(2) * inv) * (xh[k, :, r1:r2, c1:c2] - t)
    return dx


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("graph", ["simple", "full", "v1"])
def test_box_loss_cotangent_reproduces_grad_bit_for_bit(graphs, path, graph, precision):
    g = graphs[graph]
    if precision == "bf16":
        if graph == "simple":
            pytest.skip("IAN_simple runs in float32 only")
        g.m.set_precision("bf16")
    rng = np.random.default_rng(20)
    z = rng.standard_normal((3, 100)).astype(np.float32)
    boxes = np.array([[3, 5, 20, 17], [40, 30, 41, 31], [0, 47, 64, 64]], np.int32)
    colour = rng.uniform(-1, 1, (3, 3)).astype(np.float32)
    frame = rng.uniform(-1, 1, (3, 3, 64, 64)).astype(np.float32)
    xh = g.m.sample_at(z)
    for target in (None, colour, frame):
        dz = g.m.decode_vjp(z, _box_cotangent(xh, boxes, target))
        assert np.array_equal(dz, g.m.grad(z, boxes, target)), (graph, path, precision, None if target is None else target.shape)


def test_vjp_properties(graphs, path):
    g = graphs["simple"]
    rng = np.random.default_rng(30)
    z = rng.standard_normal((5, 100)).astype(np.float32)
    dx = rng.standard_normal((5, 3, 64, 64)).astype(np.float32)
    assert np.all(g.m.decode_vjp(z, np.zeros_like(dx)) == 0)
    a = g.m.decode_vjp(z, dx)
    for _ in range(2):
        assert np.array_equal(a, g.m.decode_vjp(z, dx))
    assert g.m.decode_vjp(np.zeros((0, 100), np.float32), np.zeros((0, 3, 64, 64), np.float32)).shape == (0, 100)
    with pytest.raises(TypeError):
        g.m.decode_vjp(z, dx.astype(np.float64))
    with pytest.raises(ValueError):
        g.m.decode_vjp(z, dx[:4])
    for name in ("full", "v1"):                 # the flow graphs: zero cotangent and reruns
        f = graphs[name].m
        assert np.all(f.decode_vjp(z[:2], np.zeros_like(dx[:2])) == 0)
        b = f.decode_vjp(z[:2], dx[:2])
        assert np.array_equal(b, f.decode_vjp(z[:2], dx[:2]))


def test_graph_replay_and_pdl_are_bit_identical(npe, model, weights, monkeypatch):
    """host calls of <= 32 samples replay a captured CUDA graph (slot G_VJP): equal to a handle with IAN_GRAPHS=0 on
    the capture call and the replays; programmatic dependent launch equal to IAN_PDL=0 (plain launches, graphs off)."""
    monkeypatch.setenv("IAN_GRAPHS", "0")
    plain = npe.IAN("IAN_simple.py", True, weights=weights)
    monkeypatch.setenv("IAN_PDL", "0")
    nopdl = npe.IAN("IAN_simple.py", True, weights=weights)
    monkeypatch.delenv("IAN_PDL")
    monkeypatch.delenv("IAN_GRAPHS")
    rng = np.random.default_rng(31)
    try:
        for n in (1, 6):
            z = rng.standard_normal((n, 100)).astype(np.float32)
            dx = rng.standard_normal((n, 3, 64, 64)).astype(np.float32)
            for _ in range(3):
                assert np.array_equal(model.decode_vjp(z, dx), plain.decode_vjp(z, dx)), n
        for n in (5, 128):
            z = rng.standard_normal((n, 100)).astype(np.float32)
            dx = rng.standard_normal((n, 3, 64, 64)).astype(np.float32)
            want = nopdl.decode_vjp(z, dx)
            for _ in range(2):
                assert np.array_equal(want, plain.decode_vjp(z, dx)), n
    finally:
        plain.close()
        nopdl.close()


def test_chunked_batch_matches_oracle(model, weights):
    rng = np.random.default_rng(32)
    z = rng.standard_normal((520, 100)).astype(np.float32)     # > 512-sample plan chunk
    dx = rng.standard_normal((520, 3, 64, 64)).astype(np.float32)
    dz = model.decode_vjp(z, dx)
    pick = [0, 511, 512, 519]
    rel = _per_sample_rel(dz[pick], simple_decode_vjp(weights, z[pick], dx[pick]))
    _record("C_chunked_520", rel.tolist())
    assert np.median(rel) <= 1e-4 and rel.max() <= 1e-2, rel


def test_bf16_vjp_against_float32(graphs):
    """relative L2 of the bf16-mode VJP against float32 mode on IAN.py.  bf16 operands carry 8 significand bits (x_hat
    moves by up to 0.06, tests/test_gpu_full.py) and this VJP moves by 1e-2 for an x_hat change of 2e-5 (module
    docstring): measured 0.115 on an H100, bound 0.2."""
    m = graphs["full"].m
    rng = np.random.default_rng(33)
    z = rng.standard_normal((4, 100)).astype(np.float32)
    dx = rng.standard_normal((4, 3, 64, 64)).astype(np.float32)
    ref = m.decode_vjp(z, dx)
    try:
        m.set_precision("bf16")
        got = m.decode_vjp(z, dx)
    finally:
        m.set_precision("fp32")
    rel = float(np.linalg.norm(got - ref) / np.linalg.norm(ref))
    _record("C_bf16_vs_fp32_rel_l2_full", rel)
    assert np.isfinite(got).all() and rel <= 0.2, rel


# ---- D: torch autograd binding --------------------------------------------------------------------------------------------
def _torch_ops():
    import importlib
    return importlib.import_module("neural-photo-editor_b200.torch_ops")


def test_torch_decode_backward_is_decode_vjp(model):
    import torch
    ops = _torch_ops()
    rng = np.random.default_rng(40)
    n = 40                                       # above the graph-replay size: host and device calls run the same launches
    z_np = rng.standard_normal((n, 100)).astype(np.float32)
    g_np = rng.standard_normal((n, 3, 64, 64)).astype(np.float32)
    want = model.decode_vjp(z_np, g_np)
    assert np.array_equal(ops.decode(model, torch.from_numpy(z_np).cuda()).cpu().numpy(), model.sample_at(z_np))
    for side in (False, True):
        with torch.cuda.stream(torch.cuda.Stream()) if side else torch.cuda.stream(torch.cuda.current_stream()):
            z = torch.from_numpy(z_np).cuda().requires_grad_(True)
            g = torch.from_numpy(g_np).cuda()
            (dz,) = torch.autograd.grad(ops.decode(model, z), z, g)
            got = dz.cpu().numpy()
        assert np.array_equal(got, want), side
    # a non-contiguous incoming gradient is made contiguous
    z = torch.from_numpy(z_np[:2]).cuda().requires_grad_(True)
    gt = torch.from_numpy(np.ascontiguousarray(g_np[:2].transpose(0, 1, 3, 2))).cuda().transpose(2, 3)
    (dz,) = torch.autograd.grad(ops.decode(model, z), z, gt)
    assert np.array_equal(dz.cpu().numpy(), model.decode_vjp(z_np[:2], g_np[:2]))


def _sgd_loss(x, mask, t):
    """soft-mask L1: per sample the mask-weighted mean of |x_hat - t|, summed over the batch"""
    return ((mask * (x - t).abs()).sum(dim=(1, 2, 3)) / (3 * mask.sum(dim=(1, 2, 3)))).sum()


def test_torch_sgd_loop_matches_float64_oracle(model, weights):
    """five plain-SGD steps on a soft-mask L1 loss through torch autograd, against the same loop on the float64 torch
    oracle; edit-loop bounds relative to the move: max-abs <= 2e-2 * move, median <= 1e-4 * move."""
    import torch
    from oracle import ian_torch as ot
    ops = _torch_ops()
    rng = np.random.default_rng(41)
    n, lr, steps = 4, 20.0, 5
    z0 = rng.standard_normal((n, 100)).astype(np.float32)
    mask = soft_round_mask(n, rng)
    t = rng.uniform(-1, 1, (n, 3, 64, 64))
    z = torch.from_numpy(z0).cuda()
    mg, tg = torch.from_numpy(mask.astype(np.float32)).cuda(), torch.from_numpy(t.astype(np.float32)).cuda()
    for _ in range(steps):
        z = z.detach().requires_grad_(True)
        (g,) = torch.autograd.grad(_sgd_loss(ops.decode(model, z), mg, tg), z)
        z = z - lr * g
    z_gpu = z.detach().cpu().numpy()
    P = ot.to_torch(weights, torch.float64)
    zr = torch.from_numpy(z0.astype(np.float64))
    m64, t64 = torch.from_numpy(mask), torch.from_numpy(t)
    for _ in range(steps):
        zr = zr.detach().requires_grad_(True)
        (g,) = torch.autograd.grad(_sgd_loss(ot.decode(P, zr), m64, t64), zr)
        zr = zr - lr * g
    z_ref = zr.detach().numpy()
    move = float(np.abs(z_ref - z0).max())
    err = np.abs(z_gpu - z_ref)
    _record("D_sgd", {"move": move, "max_abs": float(err.max()), "median_abs": float(np.median(err))})
    assert move > 1e-2
    assert err.max() <= 2e-2 * move and np.median(err) <= 1e-4 * move, (move, err.max(), np.median(err))


def test_torch_decode_is_once_differentiable(model):
    import torch
    ops = _torch_ops()
    z = torch.randn(2, 100, device="cuda", requires_grad=True)
    x = ops.decode(model, z)
    x.sum().backward()
    with pytest.raises(RuntimeError):
        x.sum().backward()                        # saved tensors are freed after the first backward
    x = ops.decode(model, z)
    (g,) = torch.autograd.grad(x.sum(), z, create_graph=True)
    with pytest.raises(RuntimeError):
        g.sum().backward()                        # no double backward
    with pytest.raises(TypeError):
        ops.decode(model, z.double())

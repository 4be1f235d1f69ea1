"""GPU tests of the discriminator in training mode (include/ian_b200.h ian_discriminate_train_*,
ian_discriminate_train_vjp_*; API.IAN.discriminate_train / discriminate_train_vjp; torch_ops.discriminate(...,
training=True)) on all three graphs, on the tensor-core and SIMT paths and, on IAN.py, in bf16 mode.

  1. against the executed reference (tests/golden/ref_exec_discrim_train.npz): the logits, p, the batch statistics, a
     one-image batch, and <probe, J v> through the VJP against the reference's central differences -- one of them a
     derivative that exists only through the batch's coupling.
  2. against float64 (tests/discrim_train_oracle.py) at n = 1, 3, 47 and 128: logits, dx and the statistics.
  3. the statistics are the whole call's: IAN_CHUNK=16 at n = 40 against an unchunked handle, bit for bit under
     IAN_SPLITK=0 IAN_STREAMK=0.
  4. coupling: changing one image moves every logit; a cotangent on sample 0 alone moves every image.
  5. duality: <u, J v> by the VJP against central differences of the library's own logits.
  6. errors and bits: argument checks, no head, n == 0; reruns, and the device form = the host form.
  7. torch: training=True is the C-ABI's bits both ways.
  8. consistency: a handle whose bnorm2..4 running statistics are the returned stats gives inference logits close to the
     training-mode ones.
  9. the user story: a few Adam steps on the IAN_simple decoder's parameters under BCE(p, real) through the training-mode
     discriminator lower that loss.
Measured values go to discriminate_train.json when IAN_TEST_RECORD names a directory."""
import ctypes as C
import importlib
import json
import os

import numpy as np
import pytest

import discrim_oracle as do
import discrim_train_oracle as dto
import introspect_oracle as io
from test_gpu_fit_features import GRAPHS, MODES, _rel, handles, synth  # noqa: F401

pytestmark = pytest.mark.gpu
# Bounds set from one run on an H100 80GB HBM3 at 700 W (the results are the same bits on every rerun), >= 2x over the
# worst measured value.  As in inference mode, the MinibatchLayer's pair terms compare nearly equal pooled features, so dx at
# n >= 3 is far less accurate than the logits; a batch of one has no pair terms and is as accurate as the trunk.
# 1. against the executed reference, float32 mode: logits 3.3e-5, p 1.9e-6, the one-image batch 1.2e-5 (IAN_simple, tensor
#    cores), stats 2.0e-6, probe derivatives 1.1e-2 (IAN_simple; 1.5e-3 or better elsewhere).  bf16 mode on IAN.py: 3.8e-3,
#    6.7e-4, 1.1e-3, 8.1e-4 and 0.15.
REF_BOUND = {"logits": 1e-4, "p": 1e-5, "logits1": 5e-5, "stats": 1e-5, "dp": 2.5e-2}
REF_BF16 = {"logits": 1e-2, "p": 2e-3, "logits1": 3e-3, "stats": 2e-3, "dp": 0.35}
# 2. against float64 at n = 1, 3, 47, 128, float32 mode: per-sample relative L2 of the logits 2.1e-3 (IANv1, SIMT, n = 47:
#    a logit near 0; 1.4e-4 or better on the other graphs); relative L2 of dx 2.1e-5 at n = 1, worst 8.8e-3 (IAN_simple,
#    SIMT, n = 3); the statistics 3.3e-6.  bf16 mode on IAN.py: 5.5e-3, 0.16 (n = 3) and 3.4e-4.
LOGIT_BOUND, LOGIT_BF16 = 5e-3, 1.5e-2
DX_BOUND, DX_BF16 = 2e-2, 0.35
STATS_BOUND, STATS_BF16 = 1e-5, 1e-3
# 4. a cotangent on sample 0 alone, dx of the other images against float64: worst 6.6e-4 (IAN.py).
COUPLING_BOUND = 1.5e-3
# 5. <u, J v> (n = 5, h = 1e-3): the library's central-difference gap against float64's at the same points, and the VJP's
#    <u, J v> against float64's: worst 4.0e-3 (IAN_simple) and 1.6e-3 (IANv1); float64's own gap is 2.0e-2 to 0.14.
DUAL_BOUND = 1e-2
# 8. inference logits with the returned stats as running statistics against the training-mode logits: worst 3.4e-6.
CONSIST_BOUND = 1e-5
RECORD = {}


def _record(key, value):
    RECORD[key] = value
    if os.environ.get("IAN_TEST_RECORD"):
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "discriminate_train.json"), "w") as f:
            json.dump(RECORD, f, indent=1, sort_keys=True)


FIX = dto.fixture()
RAW = dict(np.load(os.path.join(dto.ROOT, "tests", "golden", "ref_exec_discrim_train.npz")))


def _head(g):
    return FIX[g][2]


def _model(handles, g, mode="tc", weights=None, **env):
    m = handles(g, synth(g) if weights is None else weights, mode, **env)
    m.load_discriminator(_head(g))
    return m


def _bounds(mode):
    return (REF_BF16, LOGIT_BF16, DX_BF16, STATS_BF16) if mode == "bf16" else (REF_BOUND, LOGIT_BOUND, DX_BOUND, STATS_BOUND)


def _rel_all(got, ref):
    ref = np.asarray(ref, np.float64)
    return float(np.linalg.norm(np.asarray(got, np.float64) - ref) / np.linalg.norm(ref))


def _oracle(g):
    import torch
    return io.weights64(synth(g), "cuda"), do.head64(_head(g), "cuda"), torch


def _logits64(g, x):
    Q, H, torch = _oracle(g)
    with torch.no_grad():
        return dto.logits(Q, H, torch.from_numpy(np.asarray(x, np.float64)).cuda()).cpu().numpy()


def _stats64(g, x):
    Q, _, torch = _oracle(g)
    s = []
    with torch.no_grad():
        dto.trunk(Q, torch.from_numpy(np.asarray(x, np.float64)).cuda(), s)
    return np.stack([torch.cat([a for a, _ in s]).cpu().numpy(), torch.cat([b for _, b in s]).cpu().numpy()])


def _vjp64(g, x, dl):
    Q, H, torch = _oracle(g)
    xt = torch.from_numpy(np.asarray(x, np.float64)).cuda().requires_grad_(True)
    (dx,) = torch.autograd.grad(dto.logits(Q, H, xt), xt, torch.from_numpy(np.asarray(dl, np.float64)).cuda())
    return dx.cpu().numpy()


def _images(n, seed):
    return np.random.default_rng(seed).uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)


# ---- 1. against the executed reference ---------------------------------------------------------------------------------
@pytest.mark.parametrize("g,mode", MODES)
def test_against_executed_reference(handles, g, mode):
    m = _model(handles, g, mode)
    x, _, _, stored = FIX[g]
    p, lg, st = m.discriminate_train(x, return_logits=True, return_stats=True)
    lg1 = m.discriminate_train(x[:1], return_logits=True)[1]
    dp = np.array([np.sum(m.discriminate_train_vjp(x, stored["probe"][t].astype(np.float32)).astype(np.float64) * stored["v"][t])
                   for t in range(len(stored["v"]))])
    err = {"logits": _rel_all(lg, stored["logits"]), "p": _rel_all(p, stored["p"]), "stats": _rel_all(st, stored["stats"]),
           "logits1": _rel_all(lg1, RAW["logits1_%s" % g]), "dp": float(np.max(np.abs(dp - stored["dp"]) / np.abs(stored["dp"])))}
    _record("ref_%s_%s" % (g, mode), err)
    bound = _bounds(mode)[0]
    assert all(err[k] <= bound[k] for k in err), err


# ---- 2. against float64 ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g,mode", MODES)
def test_against_float64(handles, g, mode):
    m = _model(handles, g, mode)
    _, lb, db, sb = _bounds(mode)
    errs = {}
    for n in (1, 3, 47, 128):
        x = _images(n, n)
        dl = np.random.default_rng(n + 1).standard_normal((n, do.units(g))).astype(np.float32)
        _, lg, st = m.discriminate_train(x, return_logits=True, return_stats=True)
        dx = m.discriminate_train_vjp(x, dl)
        errs[n] = (float(_rel(lg, _logits64(g, x)).max()), _rel_all(dx, _vjp64(g, x, dl)), _rel_all(st, _stats64(g, x)))
        _record("f64_%s_%s_%d" % (g, mode, n), {"logits": errs[n][0], "dx": errs[n][1], "stats": errs[n][2]})
    assert all(el <= lb and ed <= db and es <= sb for el, ed, es in errs.values()), errs


# ---- 3. the statistics are the whole call's ----------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_chunked_call_is_one_batch(handles, g):
    env = {"IAN_SPLITK": 0, "IAN_STREAMK": 0}
    a, b = _model(handles, g, **env), _model(handles, g, IAN_CHUNK=16, **env)
    x = _images(40, 40)
    dl = np.random.default_rng(41).standard_normal((40, do.units(g))).astype(np.float32)
    ra = a.discriminate_train(x, return_logits=True, return_stats=True)
    rb = b.discriminate_train(x, return_logits=True, return_stats=True)
    da, db = a.discriminate_train_vjp(x, dl), b.discriminate_train_vjp(x, dl)
    same = {"stats": bool(np.array_equal(ra[2], rb[2])), "logits": bool(np.array_equal(ra[1], rb[1])),
            "dx": bool(np.array_equal(da, db))}
    _record("chunk_%s" % g, same)
    assert all(same.values()), same


# ---- 4. coupling -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_coupling(handles, g):
    m = _model(handles, g)
    n = 6
    x = _images(n, 6)
    lg = m.discriminate_train(x, return_logits=True)[1]
    x2 = x.copy()
    x2[5] = _images(1, 99)[0]
    lg2 = m.discriminate_train(x2, return_logits=True)[1]
    assert (lg2[:5] != lg[:5]).all(axis=1).all()                    # every other sample's logits moved
    dl = np.zeros((n, do.units(g)), np.float32)
    dl[0] = 1.0
    dx = m.discriminate_train_vjp(x, dl)
    ref = _vjp64(g, x, dl)
    err = _rel_all(dx[1:], ref[1:])
    _record("coupling_%s" % g, {"others_min": min(float(np.abs(dx[i]).max()) for i in range(1, n)), "dx_others": err})
    assert min(float(np.abs(dx[i]).max()) for i in range(1, n)) > 0 and err <= COUPLING_BOUND


# ---- 5. duality --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_vjp_duality(handles, g):
    """<u, J v> by the VJP against central differences of the library's logits.  Along a random direction in image space
    the logits cross many LeakyReLU and |.| kinks, so even in float64 the central difference at h = 1e-3 is 1-14 % away
    from the exact <u, J v>: the test holds the library's gap (central difference - VJP) to the float64 restatement's gap
    at the same float32 points, and the VJP's <u, J v> to float64's."""
    import torch
    m = _model(handles, g)
    n, h = 5, 1e-3
    x = _images(n, 12).astype(np.float64)
    rng = np.random.default_rng(13)
    u = rng.standard_normal((n, do.units(g))).astype(np.float32)
    v = rng.standard_normal(x.shape)
    xp, xm, x0 = (x + h * v).astype(np.float32), (x - h * v).astype(np.float32), x.astype(np.float32)
    lib = lambda a: m.discriminate_train(a, return_logits=True)[1].astype(np.float64)
    cd = float(np.sum(u * (lib(xp) - lib(xm)) / (2 * h)))
    vj = float(np.sum(m.discriminate_train_vjp(x0, u).astype(np.float64) * v))
    Q, H, _ = _oracle(g)
    t64 = lambda a: torch.from_numpy(np.asarray(a, np.float64)).cuda()
    with torch.no_grad():
        cd64 = float(np.sum(u * (dto.logits(Q, H, t64(xp)) - dto.logits(Q, H, t64(xm))).cpu().numpy() / (2 * h)))
    jv64 = float((t64(u) * torch.func.jvp(lambda a: dto.logits(Q, H, a), (t64(x0),), (t64(v),))[1]).sum())
    err = {"gap": abs((cd - vj) - (cd64 - jv64)) / abs(jv64), "vjp": abs(vj - jv64) / abs(jv64),
           "gap64": abs(cd64 - jv64) / abs(jv64)}
    _record("dual_%s" % g, err)
    assert err["gap"] <= DUAL_BOUND and err["vjp"] <= DUAL_BOUND, err


# ---- 6. errors and bits ------------------------------------------------------------------------------------------------
def test_errors(npe, handles):
    m = handles("simple", synth("simple"))
    x = _images(2, 1)
    with pytest.raises(npe.IanError, match="-3"):                    # IAN_ERR_STATE: no head
        m.discriminate_train(x)
    with pytest.raises(npe.IanError, match="-3"):
        m.discriminate_train_vjp(x, np.zeros((2, 1), np.float32))
    m.load_discriminator(_head("simple"))
    lib, h = m._lib, m._h
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    out = np.zeros((2, 1), np.float32)
    assert lib.ian_discriminate_train_host(h, fp(x), -1, fp(out), None, None) == -1
    assert lib.ian_discriminate_train_host(h, None, 2, fp(out), None, None) == -1
    assert lib.ian_discriminate_train_host(h, fp(x), 2, None, None, None) == -1
    assert lib.ian_discriminate_train_vjp_host(h, fp(x), 2, None, fp(x)) == -1
    assert lib.ian_discriminate_train_vjp_host(h, fp(x), 2, fp(out), None) == -1
    assert lib.ian_discriminate_train_vjp_host(h, fp(x), -1, fp(out), fp(x)) == -1
    assert lib.ian_discriminate_train_host(h, None, 0, None, None, None) == 0
    assert lib.ian_discriminate_train_vjp_host(h, None, 0, None, None) == 0
    assert m.discriminate_train(np.zeros((0, 3, 64, 64), np.float32)).shape == (0, 1)
    assert lib.ian_discriminate_train_host(None, fp(x), 2, fp(out), None, None) == -1


@pytest.mark.parametrize("g,mode", MODES)
def test_bits(handles, g, mode):
    import torch
    m = _model(handles, g, mode)
    n, U = 37, do.units(g)
    x = _images(n, 9)
    dl = np.random.default_rng(10).standard_normal((n, U)).astype(np.float32)
    p, lg, st = m.discriminate_train(x, return_logits=True, return_stats=True)
    dx = m.discriminate_train_vjp(x, dl)
    p2, lg2, st2 = m.discriminate_train(x, return_logits=True, return_stats=True)
    assert np.array_equal(lg, lg2) and np.array_equal(p, p2) and np.array_equal(st, st2)
    assert np.array_equal(dx, m.discriminate_train_vjp(x, dl))
    xt, dlt = torch.from_numpy(x).cuda(), torch.from_numpy(dl).cuda()
    lt, pt, dxt = torch.empty(n, U, device="cuda"), torch.empty(n, U, device="cuda"), torch.empty_like(xt)
    stt = torch.empty(2, 1792, device="cuda")
    torch.cuda.synchronize()                                         # the library runs on its own stream
    m.discriminate_train_dev(xt.data_ptr(), n, lt.data_ptr(), pt.data_ptr(), stt.data_ptr())
    m.discriminate_train_vjp_dev(xt.data_ptr(), dlt.data_ptr(), n, dxt.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(lt.cpu().numpy(), lg) and np.array_equal(pt.cpu().numpy(), p) and np.array_equal(stt.cpu().numpy(), st)
    assert np.array_equal(dxt.cpu().numpy(), dx)
    # inference mode is untouched by a training-mode call: the running statistics are not used or changed
    a = m.discriminate(x, return_logits=True)[1]
    m.discriminate_train(x)
    assert np.array_equal(a, m.discriminate(x, return_logits=True)[1]) and not np.array_equal(a, lg)


# ---- 7. torch ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_torch_op(handles, g):
    import torch
    ops = importlib.import_module("neural-photo-editor_b200.torch_ops")
    m = _model(handles, g)
    n = 5
    x = torch.from_numpy(_images(n, 11)).cuda().requires_grad_(True)
    lg = ops.discriminate(m, x, training=True)
    assert np.array_equal(lg.detach().cpu().numpy(), m.discriminate_train(x.detach().cpu().numpy(), return_logits=True)[1])
    dl = torch.randn(n, do.units(g), device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    (dx,) = torch.autograd.grad(lg, x, dl)
    assert np.array_equal(dx.cpu().numpy(), m.discriminate_train_vjp(x.detach().cpu().numpy(), dl.cpu().numpy()))
    li = ops.discriminate(m, x)                                      # the default stays inference mode
    assert np.array_equal(li.detach().cpu().numpy(), m.discriminate(x.detach().cpu().numpy(), return_logits=True)[1])
    import torch.autograd.forward_ad as fwAD
    with fwAD.dual_level(), pytest.raises(NotImplementedError):
        ops.discriminate(m, fwAD.make_dual(x.detach(), torch.ones_like(x)), training=True)


# ---- 8. consistency with inference under the batch's statistics ---------------------------------------------------------
@pytest.mark.parametrize("g", GRAPHS)
def test_stats_as_running_statistics(handles, g):
    m = _model(handles, g)
    x = _images(24, 24)
    lg, st = m.discriminate_train(x, return_logits=True, return_stats=True)[1:]
    W = dict(synth(g))
    off = 0
    for k, c in zip((2, 3, 4), dto.BN_CHANNELS):
        W["bnorm%d.mean" % k] = st[0, off:off + c].copy()
        W["bnorm%d.inv_std" % k] = st[1, off:off + c].copy()
        off += c
    m2 = _model(handles, g, weights=W)
    li = m2.discriminate(x, return_logits=True)[1]
    err = _rel_all(li, lg)
    _record("consistency_%s" % g, err)
    assert err <= CONSIST_BOUND


# ---- 9. fine-tuning the IAN_simple decoder against the training-mode discriminator --------------------------------------
def test_decoder_adam_lowers_the_adversarial_loss(handles):
    import torch
    import torch.nn.functional as F
    ops = importlib.import_module("neural-photo-editor_b200.torch_ops")
    P = synth("simple")
    m = _model(handles, "simple")
    params = ops.decoder_parameters(m, P)
    z = torch.randn(16, 100, device="cuda", generator=torch.Generator("cuda").manual_seed(5))
    opt = torch.optim.Adam(params.values(), lr=2e-4)

    def loss():       # train_IAN_simple.py's generator term: BCE of p(X_gen) against "real"
        lg = ops.discriminate(m, ops.decode(m, z, params), training=True)
        return F.binary_cross_entropy_with_logits(lg, torch.ones_like(lg))

    losses = []
    for _ in range(6):
        opt.zero_grad()
        lv = loss()
        lv.backward()
        opt.step()
        losses.append(float(lv.detach()))
    with torch.no_grad():
        losses.append(float(loss()))
    _record("adam_simple", losses)
    assert losses[-1] < losses[0], losses          # measured: 1.20 -> 0.0057 after six steps

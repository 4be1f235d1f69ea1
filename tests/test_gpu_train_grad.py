"""Reverse mode of the training-mode ops (csrc/train_kernels.cu, DESIGN §5.6b) against the float64 autograd restatement
tests/train_grad_oracle.py (pinned on the CPU to the executed reference's central differences by
tests/test_train_grad_oracle.py).  The restatement runs in float64 on the GPU.

Shapes: every BatchNorm split, tail and tile case of tests/test_gpu_train_ops.py, and MinibatchLayer's tiles plus the
reference discriminator (d = 1024 after GlobalPoolLayer(enc_conv4), K = 500, P = 5, n = 64 and 128).
Data: offset channels (|mean|/std up to 1e4), constant channels (s = 1/sqrt(eps)), gamma = 0 channels, and duplicated
samples whose A rows tie exactly, where sgn(0) = 0 matters.

Bounds (no flat tolerance): first order in the roundings of the operations the kernels perform, doubled to cover the
float64 restatement's own roundings (the same operations, in float64).
  BatchNorm: the float64 sums are chains of at most bn_chain(n, hw) additions (the forward's split structure), so
  |δΣdy| <= L u64 Σ|dy| and |δΣdy·x| <= L u64 Σ|dy x|; mean and the one-pass variance as in the forward module; the per
  element float64 expression; one float32 rounding of dx, dgamma, dbeta.
  MinibatchLayer: A = fl(Σ_d x theta) colscale, |δA| <= (d + 3) u32 |x||theta| colscale; e_ijk through Σ_p |δA| and expf;
  a pair whose oracle difference is inside the A error may take the other sign (2 |c_ij|), except exact ties, whose rows
  the kernels compute to the same bits; the n-term float32 sums over j; the FFMA contractions over kp (dx) and n (dW);
  the float64 column sums of the theta chain.
Measured on an H100 80GB HBM3 (700 W power limit), worst error / bound: BatchNorm 0.999 (conv (100, 130, 5, 51)), the
final float32 rounding of dx realised in full; MinibatchLayer 0.997 (n = 2, d = 200, K = 300, P = 1), 0.985 at the
discriminator shape n = 128.  The data are seeded and the kernels bit-reproducible, so these ratios do not drift.

Each of these one-line mutations of csrc/train_kernels.cu fails this module (and which test catches it):
  * dropping the mean(dy) term (coef[c + ch] in bn_bwd_apply_kernel)       -> every BN shape, edge, shard and gamma test
  * accumulating Σdy·x in float32 (`q = (float)(q + g * x)`)             -> test_bn_grad_conv_shapes (all 20), the offset and
    constant channels, the shards, test_bn_grad_without_gamma_and_torch_reference
  * sgn(0) = 1 (`df >= 0.f ? cij : ...` in mb_pair_bwd_kernel)             -> test_mb_grad_ties
  * dropping the g_f[j,k] half of the pair term                            -> test_mb_grad_shapes
  * omitting the column-norm chain in dtheta (dtheta = cs dW)              -> test_mb_grad_shapes
"""
import importlib

import numpy as np
import pytest

import train_grad_oracle as tg
from test_gpu_train_ops import CONV, bn_chain, bn_data, bn_params, edge_channels, mb_data

pytestmark = pytest.mark.gpu

U32, U64 = 2.0 ** -24, 2.0 ** -53
HEAD = 2.0
EPS = 1e-4


def _ops():
    return importlib.import_module("neural-photo-editor_b200.train_ops")


def _t(a, dtype=None):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0", dtype or torch.float32)


def _d(t):
    import torch
    return t.to(torch.float64)


def _check(name, got, want, bound):
    """asserts |got - want| <= bound elementwise; returns the worst ratio"""
    import torch
    err = (_d(got) - want).abs()
    ok = err <= bound
    if not bool(ok.all()):
        r = torch.where(ok, torch.zeros_like(err), err / bound.clamp_min(1e-300))
        i = int(torch.argmax(r.flatten()))
        raise AssertionError("%s: |err| %.3g > bound %.3g at %d (got %r, want %r)" % (
            name, float(err.flatten()[i]), float(bound.flatten()[i]), i, float(got.flatten()[i]), float(want.flatten()[i])))
    return float((err / bound.clamp_min(1e-300)).max())


# ---- BatchNorm -------------------------------------------------------------------------------------------------------
def bn_grad_call(model, x, dy, gamma, beta, count=None, sums=None):
    """the two C-ABI calls on one shard: (sums, bsums, dgamma, dbeta, dx)"""
    import torch
    ops = _ops()
    n, c = int(x.shape[0]), int(x.shape[1])
    hw = int(x[0, 0].numel()) if x.dim() > 2 else 1
    if sums is None:
        sums = torch.empty(2, c, dtype=torch.float64, device="cuda:0")
        with ops._lib_stream(model, x) as st:
            model._check(model._lib.ian_bn_batch_stats_dev(model._h, x.data_ptr(), n, c, hw, sums[0].data_ptr(), sums[1].data_ptr(), st))
    count = float(n * hw) if count is None else count
    bs = torch.empty(2, c, dtype=torch.float64, device="cuda:0")
    dg, db, dx = torch.empty(c, device="cuda:0"), torch.empty(c, device="cuda:0"), torch.empty_like(x)
    p = lambda t: None if t is None else t.data_ptr()
    with ops._lib_stream(model, x) as st:
        model._check(model._lib.ian_bn_backward_sums_dev(model._h, x.data_ptr(), dy.data_ptr(), n, c, hw, sums[0].data_ptr(),
                                                         sums[1].data_ptr(), count, EPS, bs[0].data_ptr(), bs[1].data_ptr(),
                                                         dg.data_ptr(), db.data_ptr(), st))
        model._check(model._lib.ian_bn_backward_dx_dev(model._h, x.data_ptr(), dy.data_ptr(), n, c, hw, sums[0].data_ptr(),
                                                       sums[1].data_ptr(), count, bs[0].data_ptr(), bs[1].data_ptr(), p(gamma),
                                                       EPS, dx.data_ptr(), st))
    torch.cuda.synchronize()
    return sums, bs, dg, db, dx


class BnGradExpect:
    """oracle dx, dgamma, dbeta of one training-mode BatchNorm and their bounds (whole batch; chain = longest sum chain)"""

    def __init__(self, x, dy, gamma, chain):
        import torch
        x64, dy64 = _d(x), _d(dy)
        g64 = None if gamma is None else _d(gamma)
        self.dx, self.dg, self.db = tg.bn_backward(x64, g64, dy64, EPS)
        axes, shp = (0,) + tuple(range(2, x.dim())), [1, -1] + [1] * (x.dim() - 2)
        N = x64[:, 0].numel()
        mean, s = tg.bn_stats(x64, EPS)
        var = x64.var(axes, unbiased=False)
        L = chain
        e_s1 = L * U64 * dy64.abs().sum(axes)
        e_s2 = L * U64 * (dy64 * x64).abs().sum(axes)
        e_m = (L + 1) * U64 * x64.abs().mean(axes)
        e_var = (3 * L + 4) * U64 * (x64 * x64).mean(axes)
        d_s = 0.5 * (e_var + abs(float(np.float32(EPS)) - EPS)) / (var + EPS) + 4 * U64
        sdy, sdyx = dy64.sum(axes), (dy64 * x64).sum(axes)
        num = sdyx - mean * sdy
        e_num = e_s2 + mean.abs() * e_s1 + e_m * sdy.abs() + 4 * U64 * ((dy64 * x64).abs().sum(axes))
        k = s * s * num / N
        e_k = s * s * e_num / N + 2 * d_s * k.abs()
        g = torch.ones_like(mean) if g64 is None else g64
        a = (g * s).abs()
        xm = (x64 - mean.reshape(shp)).abs()
        t = self.dx.abs() / a.clamp_min(1e-300).reshape(shp)
        e_t = (e_s1 / N).reshape(shp) + xm * e_k.reshape(shp) + (e_m * k.abs()).reshape(shp) \
            + 4 * U64 * (dy64.abs() + (sdy.abs() / N).reshape(shp) + xm * k.abs().reshape(shp))
        self.dx_bound = HEAD * (a.reshape(shp) * e_t + t * (a * d_s).reshape(shp)) + U32 * self.dx.abs()
        self.dg_bound = HEAD * (s * e_num + d_s * self.dg.abs()) + U32 * self.dg.abs()
        self.db_bound = HEAD * e_s1 + U32 * self.db.abs()

    def check(self, dx, dg=None, db=None, what=""):
        worst = _check(what + " dx", dx, self.dx, self.dx_bound)
        if dg is not None:
            worst = max(worst, _check(what + " dgamma", dg, self.dg, self.dg_bound),
                        _check(what + " dbeta", db, self.db, self.db_bound))
        return worst


def bn_grad_case(model, rng, x, gamma_zero=()):
    g, _, _, _ = bn_params(rng, x.shape[1])
    g[list(gamma_zero)] = 0.0
    dy = rng.standard_normal(x.shape).astype(np.float32)
    xt, dyt, gt = _t(x), _t(dy), _t(g)
    _, _, dg, db, dx = bn_grad_call(model, xt, dyt, gt, None)
    e = BnGradExpect(xt, dyt, gt, bn_chain(x.shape[0], int(np.prod(x.shape[2:], dtype=np.int64))))
    worst = e.check(dx, dg, db, str(x.shape))
    for k in gamma_zero:
        assert bool((dx[:, k] == 0).all()), k
    return worst


@pytest.mark.parametrize("n,c,hw", CONV)
def test_bn_grad_conv_shapes(model, n, c, hw):
    rng = np.random.default_rng(n * 100003 + c * 101 + hw + 7)
    shape = (n, c, hw) if hw % 5 else (n, c, 5, hw // 5)
    bn_grad_case(model, rng, bn_data(rng, shape))


@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 257])
def test_bn_grad_dense_shapes(model, n):
    for c in (1, 255, 256, 257, 1000):
        rng = np.random.default_rng(n * 7919 + c + 7)
        bn_grad_case(model, rng, bn_data(rng, (n, c)))


@pytest.mark.parametrize("n,hw", [(32, 4096), (64, 256), (3, 1000), (257, 1), (64, 1), (5, 1)])
def test_bn_grad_offset_and_constant_channels(model, n, hw):
    """|mean|/std up to 1e4, constant channels (s = 1/sqrt(eps), x̂ = 0), and gamma = 0 on two channels (dx = 0 there)"""
    rng = np.random.default_rng(n + hw + 7)
    x = edge_channels(rng, n, hw)
    if hw == 1:
        x = x[:, :, 0].copy()
    bn_grad_case(model, rng, x, gamma_zero=(1, 6))


def test_bn_grad_without_gamma_and_torch_reference(model):
    """gamma NULL is gamma = 1; and torch's own float32 batch-norm backward lands within its float32 error of ours"""
    import torch
    rng = np.random.default_rng(3)
    x = bn_data(rng, (17, 5, 9, 11))
    dy = rng.standard_normal(x.shape).astype(np.float32)
    xt, dyt = _t(x), _t(dy)
    _, _, _, _, dx = bn_grad_call(model, xt, dyt, None, None)
    BnGradExpect(xt, dyt, None, bn_chain(17, 99)).check(dx, what="gamma=None")
    _, _, _, _, dx1 = bn_grad_call(model, xt, dyt, _t(np.ones(5, np.float32)), None)
    assert torch.equal(dx, dx1)


def test_bn_grad_synchronised_shards(model):
    """2 and 3 uneven shards: local sums added in rank order give the whole batch's dx within the bound, and the local
    dgamma / dbeta add up to the whole batch's"""
    import torch
    rng = np.random.default_rng(9)
    for shape in ((37, 5, 15, 17), (97, 260)):
        n, c = shape[:2]
        hw = int(np.prod(shape[2:], dtype=np.int64))
        x = bn_data(rng, shape)
        g = _t(bn_params(rng, c)[0])
        dy = rng.standard_normal(shape).astype(np.float32)
        xt, dyt = _t(x), _t(dy)
        for cuts in ((0, n // 3, n), (0, 5, n - n // 3, n)):
            pieces = list(zip(cuts[:-1], cuts[1:]))
            L = max(bn_chain(hi - lo, hw) for lo, hi in pieces) + len(pieces)
            e = BnGradExpect(xt, dyt, g, L)
            fsum = torch.zeros(2, c, dtype=torch.float64, device="cuda:0")
            for lo, hi in pieces:
                fsum += bn_grad_call(model, xt[lo:hi].contiguous(), dyt[lo:hi].contiguous(), g, None)[0]
            bsum, dgs, dbs = torch.zeros_like(fsum), [], []
            for lo, hi in pieces:
                _, bs, dg, db, _ = bn_grad_call(model, xt[lo:hi].contiguous(), dyt[lo:hi].contiguous(), g, None,
                                                count=float(n * hw), sums=fsum)
                bsum += bs
                dgs.append(_d(dg))
                dbs.append(_d(db))
            dxs = []
            ops = _ops()
            for lo, hi in pieces:
                xs, dys = xt[lo:hi].contiguous(), dyt[lo:hi].contiguous()
                dx = torch.empty_like(xs)
                with ops._lib_stream(model, xs) as st:
                    model._check(model._lib.ian_bn_backward_dx_dev(model._h, xs.data_ptr(), dys.data_ptr(), hi - lo, c, hw,
                                                                   fsum[0].data_ptr(), fsum[1].data_ptr(), float(n * hw),
                                                                   bsum[0].data_ptr(), bsum[1].data_ptr(), g.data_ptr(), EPS,
                                                                   dx.data_ptr(), st))
                dxs.append(dx)
            torch.cuda.synchronize()
            e.check(torch.cat(dxs), what="shards %s" % (cuts,))
            _check("sum of local dgamma", sum(dgs), e.dg, e.dg_bound + len(pieces) * U32 * sum(d.abs() for d in dgs))
            _check("sum of local dbeta", sum(dbs), e.db, e.db_bound + len(pieces) * U32 * sum(d.abs() for d in dbs))


def test_bn_grad_group_path_world_size_one(model, tmp_path):
    """batch_norm_train(group=True): the backward all-reduces its sums over the default group (NCCL, one rank)"""
    import torch
    import torch.distributed as dist
    ops = _ops()
    rng = np.random.default_rng(10)
    x = _t(bn_data(rng, (19, 6, 7, 9)))
    g0, b0, _, _ = bn_params(rng, 6)
    dy = _t(rng.standard_normal((19, 6, 7, 9)))

    def grads(**kw):
        xs, gs, bs = x.clone().requires_grad_(True), _t(g0).requires_grad_(True), _t(b0).requires_grad_(True)
        return torch.autograd.grad(ops.batch_norm_train(model, xs, gs, bs, **kw), (xs, gs, bs), dy)

    want = grads()
    assert not dist.is_initialized()
    dist.init_process_group("nccl", init_method="file://" + str(tmp_path / "store"), rank=0, world_size=1)
    try:
        got = grads(group=True)
    finally:
        dist.destroy_process_group()
    assert all(torch.equal(u, v) for u, v in zip(got, want))


@pytest.mark.parametrize("shape", [(33, 6, 17, 15), (65, 257)])
def test_bn_grad_channel_isolation(model, shape):
    """a NaN or ±Inf in one channel's x or dy leaves every other channel's dx, dgamma, dbeta bit-unchanged"""
    import torch
    rng = np.random.default_rng(shape[0] + 1)
    c = shape[1]
    x = bn_data(rng, shape)
    g = _t(bn_params(rng, c)[0])
    dy = rng.standard_normal(shape).astype(np.float32)
    clean = bn_grad_call(model, _t(x), _t(dy), g, None)
    for where, kind, k in (("x", np.nan, c // 2), ("x", np.inf, c - 1), ("dy", -np.inf, 1), ("dy", np.nan, 0)):
        xt, dyt = x.copy(), dy.copy()
        (xt if where == "x" else dyt)[(shape[0] // 2, k) + (0,) * (len(shape) - 2)] = kind
        got = bn_grad_call(model, _t(xt), _t(dyt), g, None)
        other = torch.arange(c, device="cuda:0") != k
        for u, v in zip(got[1:], clean[1:]):
            if u.dim() == 1:
                assert torch.equal(u[other], v[other]), (where, kind)
            elif u.shape[0] == 2:
                assert torch.equal(u[:, other], v[:, other]), (where, kind)
            else:
                assert torch.equal(u[:, other], v[:, other]), (where, kind)
        assert bool(torch.isnan(got[4][:, k]).any()), (where, kind)


# ---- MinibatchLayer --------------------------------------------------------------------------------------------------
def mb_grad_call(model, x, theta, lws, b, g, want=(True, True, True, True)):
    import torch
    ops = _ops()
    n, d = x.shape
    K, P = theta.shape[1:]
    outs = [torch.empty_like(t) if w else None for t, w in zip((x, theta, lws, b), want)]
    with ops._lib_stream(model, x) as st:
        model._check(model._lib.ian_minibatch_discrim_bwd_dev(model._h, x.data_ptr(), n, d, theta.data_ptr(), lws.data_ptr(),
                                                              b.data_ptr(), K, P, g.data_ptr(),
                                                              *[None if t is None else t.data_ptr() for t in outs], st))
    torch.cuda.synchronize()
    return outs


def mb_expect(x, theta, lws, b, g):
    """oracle (dx, dtheta, dlws, db) and bounds"""
    import torch
    x64, th, lw, g64 = _d(x), _d(theta), _d(lws), _d(g)
    n, d = x64.shape
    K, P = th.shape[1:]
    kp = K * P
    want = tg.mb_backward(x64, th, lw, _d(b), g64)
    r2 = (th * th).sum(0)
    cs = torch.exp(lw) / torch.sqrt(r2)
    W = th * cs[None]
    A = torch.tensordot(x64, W, dims=([1], [0]))                                      # (n, K, P)
    eA = (d + 3) * U32 * torch.tensordot(x64.abs(), th.abs(), dims=([1], [0])) * cs[None]
    diff = A[:, None] - A[None]
    adiff = diff.abs()
    off = (1 - torch.eye(n, dtype=torch.float64, device=x64.device))[:, :, None]
    e = torch.exp(-adiff.sum(-1)) * off
    e_ad = (eA[:, None] + eA[None]).sum(-1) + P * U32 * adiff.sum(-1)
    gf = g64[:, d:]
    cg = (gf[:, None] + gf[None]).abs()
    c = cg * e
    e_c = cg * e * (e_ad + 4 * U32)
    flip = ((adiff <= eA[:, None] + eA[None]) & (diff != 0)).to(torch.float64)
    e_dA = (e_c[..., None] + 2 * c[..., None] * flip).sum(1) + n * U32 * c.sum(1)[..., None]
    dA = -(((gf[:, None] + gf[None]) * e)[..., None] * torch.sign(diff)).sum(1)
    Wf, e_dAf, dAf = W.reshape(d, kp), e_dA.reshape(n, kp), dA.reshape(n, kp)
    e_dx = e_dAf @ Wf.abs().T + (kp + 5) * U32 * (dAf.abs() @ Wf.abs().T)
    e_dW = x64.abs().T @ e_dAf + (n + 1) * U32 * (x64.abs().T @ dAf.abs())                # (d, kp)
    thf = th.reshape(d, kp)
    e_S = (thf.abs() * e_dW).sum(0)
    csf, r2f = cs.reshape(kp), r2.reshape(kp)
    dWf = x64.T @ dAf
    S = (thf * dWf).sum(0)
    bounds = (HEAD * e_dx + U32 * want[0].abs(),
              (HEAD * csf * (e_dW + thf.abs() * e_S / r2f) + 4 * U32 * csf * (dWf.abs() + thf.abs() * S.abs() / r2f)).reshape(d, K, P)
              + U32 * want[1].abs(),
              (HEAD * csf * e_S + 4 * U32 * (csf * S).abs()).reshape(K, P) + U32 * want[2].abs(),
              n * U64 * gf.abs().sum(0) + U32 * want[3].abs())
    return want, bounds


def mb_grad_case(model, x, theta, lws, b, g, what=""):
    xt, tht, lwt, bt, gt = _t(x), _t(theta), _t(lws), _t(b), _t(g)
    got = mb_grad_call(model, xt, tht, lwt, bt, gt)
    want, bounds = mb_expect(xt, tht, lwt, bt, gt)
    worst = 0.0
    for name, u, v, bd in zip(("dx", "dtheta", "dlws", "db"), got, want, bounds):
        worst = max(worst, _check("%s %s" % (what, name), u, v, bd))
    return worst, got


KP = [(1, 1), (7, 5), (63, 1), (64, 1), (13, 5), (300, 1), (100, 5)]


@pytest.mark.parametrize("i", range(30))
def test_mb_grad_shapes(model, i):
    """the forward module's (n, d) x (K, P) grid: 16 x 64 activation tiles, 32-wide d chunks, the 64 x 64 gradient tiles"""
    n, d = (1, 2, 15, 16, 17, 33)[i % 6], (1, 31, 32, 33, 200)[i % 5]
    K, P = KP[i % 7]
    rng = np.random.default_rng(2000 + i)
    x, theta, lws, b = mb_data(rng, n, d, K, P)
    g = rng.standard_normal((n, d + K)).astype(np.float32)
    mb_grad_case(model, x, theta, lws, b, g, "n=%d d=%d K=%d P=%d" % (n, d, K, P))


@pytest.mark.parametrize("n", [64, 128])
def test_mb_grad_discriminator_shape(model, n):
    """GlobalPoolLayer(enc_conv4) -> MinibatchLayer(500 x 5): d = 1024"""
    rng = np.random.default_rng(n + 1)
    x, theta, lws, b = mb_data(rng, n, 1024, 500, 5)
    g = rng.standard_normal((n, 1024 + 500)).astype(np.float32)
    mb_grad_case(model, x, theta, lws, b, g, "discriminator n=%d" % n)


def test_mb_grad_ties(model):
    """duplicated samples: A rows tie exactly, sgn(0) = 0 drops the pair from dA (it still counts in f)"""
    rng = np.random.default_rng(77)
    x, theta, lws, b = mb_data(rng, 24, 200, 13, 5)
    x[5] = x[0]
    x[17] = x[0]
    x[9] = x[3]
    g = rng.standard_normal((24, 213)).astype(np.float32)
    mb_grad_case(model, x, theta, lws, b, g, "ties")


def test_mb_grad_permutation_and_outputs(model):
    """a permutation of the batch permutes dx and leaves the parameter gradients within the bound; a NULL output changes
    no other output's bits"""
    import torch
    rng = np.random.default_rng(4)
    x, theta, lws, b = mb_data(rng, 33, 200, 13, 5)
    g = rng.standard_normal((33, 213)).astype(np.float32)
    perm = rng.permutation(33)
    _, got = mb_grad_case(model, x, theta, lws, b, g)
    _, gotp = mb_grad_case(model, x[perm], theta, lws, b, g[perm])
    want, bounds = mb_expect(_t(x), _t(theta), _t(lws), _t(b), _t(g))
    _check("permuted dx", gotp[0], want[0][torch.as_tensor(perm, device="cuda:0")], 2 * bounds[0][torch.as_tensor(perm, device="cuda:0")])
    args = [_t(a) for a in (x, theta, lws, b, g)]
    for mask in ((True, False, False, False), (False, True, False, False), (False, False, True, True)):
        part = mb_grad_call(model, *args, want=mask)
        for u, v in zip(part, got):
            assert u is None or torch.equal(u, v), mask


# ---- determinism, workspace, streams, arguments ----------------------------------------------------------------------
def test_grad_reruns_workspace_history_and_streams(model):
    """bit-identical reruns; nothing depends on what the shared workspace held before; a non-default stream gives the
    same bits"""
    import torch
    rng = np.random.default_rng(12)
    xb = _t(bn_data(rng, (33, 130, 257)))
    dyb = _t(rng.standard_normal((33, 130, 257)))
    gb = _t(bn_params(rng, 130)[0])
    mb = [_t(a) for a in mb_data(rng, 17, 33, 13, 5)] + [_t(rng.standard_normal((17, 46)))]
    big = [_t(a) for a in mb_data(rng, 128, 1024, 500, 5)] + [_t(rng.standard_normal((128, 1524)))]
    first = (bn_grad_call(model, xb, dyb, gb, None), mb_grad_call(model, *mb))

    def same(got):
        assert all(torch.equal(u, v) for u, v in zip(got[0], first[0]))
        assert all(torch.equal(u, v) for u, v in zip(got[1], first[1]))

    same((bn_grad_call(model, xb, dyb, gb, None), mb_grad_call(model, *mb)))
    mb_grad_call(model, *big)
    same((bn_grad_call(model, xb, dyb, gb, None), mb_grad_call(model, *mb)))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = (bn_grad_call(model, xb, dyb, gb, None), mb_grad_call(model, *mb))
    s.synchronize()
    same(got)


def test_grad_argument_errors(model):
    import torch
    lib, h = model._lib, model._h
    x = torch.zeros(4, 3, device="cuda:0")
    s = torch.zeros(2, 3, dtype=torch.float64, device="cuda:0")
    p = x.data_ptr()
    q = s.data_ptr()
    assert lib.ian_bn_backward_sums_dev(h, p, p, -1, 3, 1, q, q, 4.0, EPS, q, q, None, None, None) != 0
    assert lib.ian_bn_backward_sums_dev(h, None, p, 4, 3, 1, q, q, 4.0, EPS, q, q, None, None, None) != 0
    assert lib.ian_bn_backward_sums_dev(h, p, p, 4, 0, 1, q, q, 4.0, EPS, q, q, None, None, None) != 0
    assert lib.ian_bn_backward_dx_dev(h, p, p, 4, 3, 1, q, q, 0.0, q, q, None, EPS, p, None) != 0
    assert lib.ian_bn_backward_dx_dev(h, p, p, 4, 3, 1, q, q, 4.0, q, q, None, EPS, None, None) != 0
    assert lib.ian_minibatch_discrim_bwd_dev(h, p, 4, 3, p, p, p, 0, 1, p, None, None, None, None, None) != 0
    assert lib.ian_minibatch_discrim_bwd_dev(h, p, 4, 3, p, p, None, 1, 1, p, None, None, None, None, None) != 0
    before = s.clone()                                   # n == 0 does nothing
    assert lib.ian_bn_backward_sums_dev(h, p, p, 0, 3, 1, q, q, 4.0, EPS, q, q, None, None, None) == 0
    assert lib.ian_minibatch_discrim_bwd_dev(h, p, 0, 3, p, p, p, 1, 1, p, p, None, None, None, None) == 0
    torch.cuda.synchronize()
    assert torch.equal(s, before)


# ---- torch -----------------------------------------------------------------------------------------------------------
def test_torch_autograd_is_the_c_abi(model):
    """autograd.grad through the wrappers gives the C-ABI's bits; inputs that do not require grad give the old forward
    bit for bit, running statistics included"""
    import torch
    ops = _ops()
    rng = np.random.default_rng(31)
    x = bn_data(rng, (21, 6, 5, 7))
    g, b, rm0, ris0 = bn_params(rng, 6)
    dy = _t(rng.standard_normal(x.shape))
    xt, gt, bt = _t(x).requires_grad_(True), _t(g).requires_grad_(True), _t(b).requires_grad_(True)
    rm, ris = _t(rm0), _t(ris0)
    y = ops.batch_norm_train(model, xt, gt, bt, rm, ris)
    rm_plain, ris_plain = _t(rm0), _t(ris0)
    y_plain = ops.batch_norm_train(model, _t(x), _t(g), _t(b), rm_plain, ris_plain)
    assert y_plain.grad_fn is None and torch.equal(y.detach(), y_plain)
    assert torch.equal(rm, rm_plain) and torch.equal(ris, ris_plain)
    grads = torch.autograd.grad(y, (xt, gt, bt), dy)
    _, _, dg, db, dx = bn_grad_call(model, xt.detach(), dy, gt.detach(), None)
    assert torch.equal(grads[0], dx) and torch.equal(grads[1], dg) and torch.equal(grads[2], db)

    xm, th, lw, bm = mb_data(rng, 19, 4 * 4 * 4, 7, 5)
    gm = _t(rng.standard_normal((19, 64 + 7)))
    ins = [_t(xm.reshape(19, 4, 4, 4)), _t(th), _t(lw), _t(bm)]
    out_plain = ops.minibatch_layer(model, *ins)
    ins = [t.requires_grad_(True) for t in ins]
    out = ops.minibatch_layer(model, *ins)
    assert out_plain.grad_fn is None and torch.equal(out.detach(), out_plain)
    grads = torch.autograd.grad(out, ins, gm)
    ref = mb_grad_call(model, ins[0].detach().reshape(19, 64), *[t.detach() for t in ins[1:]], gm)
    assert torch.equal(grads[0], ref[0].reshape(19, 4, 4, 4))
    assert all(torch.equal(u, v) for u, v in zip(grads[1:], ref[1:]))


def test_torch_adam_lowers_a_discriminator_loss(model):
    """BN + MinibatchLayer + a dense head, trained by torch.optim.Adam on a fixed batch for 30 steps"""
    import torch
    ops = _ops()
    rng = np.random.default_rng(5)
    n, d, K, P = 32, 64, 10, 3
    x = _t(bn_data(rng, (n, d, 2, 2)))
    labels = _t((rng.uniform(size=n) > 0.5).astype(np.float32))
    gamma = _t(np.ones(d, np.float32)).requires_grad_(True)
    beta = _t(np.zeros(d, np.float32)).requires_grad_(True)
    theta = _t(rng.normal(0, 0.05, (4 * d, K, P)).astype(np.float32)).requires_grad_(True)
    lws = _t(np.full((K, P), np.log(0.1), np.float32)).requires_grad_(True)
    b = _t(np.full(K, -1.0, np.float32)).requires_grad_(True)
    w = _t(rng.normal(0, 0.05, (4 * d + K,)).astype(np.float32)).requires_grad_(True)
    opt = torch.optim.Adam([gamma, beta, theta, lws, b, w], lr=1e-2)
    losses = []
    for _ in range(30):
        h = torch.relu(ops.batch_norm_train(model, x, gamma, beta))
        feats = ops.minibatch_layer(model, h, theta, lws, b)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(feats @ w, labels)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert all(np.isfinite(losses)) and losses[-1] < 0.8 * losses[0], losses

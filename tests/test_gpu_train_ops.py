"""Training-mode BatchNorm and MinibatchLayer (csrc/train_kernels.cu) at the edges of their index math and arithmetic,
against the float64 oracle oracle/train_numpy.py (pinned to the executed reference by tests/test_train_ops.py).

These are the only kernels of the library whose shapes are all arguments, so their splits, tails and tiles are held
here shape by shape:
  BatchNorm, conv path (hw > 1): S = min(n, 32) CTAs per channel with uneven image ranges, 256-thread sweeps over hw
  (hw under, at and over one sweep), c up to 130 CTAs; dense path (hw == 1): S = 1 below n = 64 and 8 from there, and
  the 256-channel grid tails.  3-D / 5-D inputs and (n, c, 1, 1) against their flat forms bit for bit.
  MinibatchLayer: the 16-sample x 64-column tiles of mb_activation_kernel and its 32-wide d chunks, K*P at 63/64/65
  columns, K > 128 for the second pass of mb_features_kernel's thread loop, and the discriminator's 16384 -> 100 x 5.

BatchNorm bound: no flat tolerance.  Per element, from the operations the kernels perform: the float64 sums' roundings
(a chain of at most `bn_chain(n, hw)` additions, which the one-pass variance Sum x^2/N - mean^2 amplifies by
mean(x^2) / (var + eps)), the rounding of mean to float32 (every float32 the double mean may round to), x - mean_f, the
float32 inv_std and gamma * inv_std, the product and + beta; running statistics likewise.  25 % headroom over that
first-order bound.  Measured on an H100 80GB HBM3 (700 W power limit): worst error 0.80 of the bound, the float32
rounding of mean realised in full.  The bound is tight enough that float32 per-thread partial sums fail it on offset
channels and on constant ones, which must give y = beta exactly.

MinibatchLayer bound: |f - f_ref| <= MB_TOL * (sum_j exp(-sum_p |act_i - act_j|) + |b|), i.e. relative to the terms the
kernel adds.  Measured worst on the same H100: 1.09e-6 (16384 -> 100 x 5 at n = 128; 3.5e-7 at the small shapes), so
MB_TOL = 4e-6.  The data keep every pair's term above 0.1 (exp(log_weight_scale) ~ 0.2 / P), so a dropped or added pair (the self-pair counted, the last sample skipped) moves f by far more
than the bound, and nothing hides under exp underflow or b.
"""
import importlib
import os

import numpy as np
import pytest

from oracle import train_numpy as tn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EDGES = np.load(os.path.join(ROOT, "tests", "golden", "ref_exec_train_edges.npz"))
U32, U64 = 2.0 ** -24, 2.0 ** -53
MB_TOL = 4e-6
INV_SQRT_EPS = 1 / np.sqrt(1e-4)                  # inv_std of a constant channel at lasagne's eps
MB_MIN_TERM = 0.1


def _ops():
    return importlib.import_module("neural-photo-editor_b200.train_ops")


def dev(a):
    import torch
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to("cuda:0")


def host(t):
    import torch
    torch.cuda.synchronize()
    return None if t is None else t.cpu().numpy()


# ---- BatchNorm -------------------------------------------------------------------------------------------------------
def bn_chain(n, hw):
    """the longest float64 addition chain behind one channel's sums: a thread's terms, the block tree, the split reduce"""
    if hw == 1:
        S = 8 if n >= 64 else 1
        return -(-n // S) + S + 1
    S = min(n, 32)
    return -(-n // S) * -(-hw // 256) + 10 + S + 1


class BnExpect:
    """oracle outputs and per-element bounds for one training-mode BatchNorm call (alpha as the float32 the kernel gets)"""

    def __init__(self, x, gamma, beta, rm0, ris0, eps=1e-4, alpha=0.1, chain=None):
        c = x.shape[1]
        alpha = float(np.float32(alpha))
        g = np.ones(c) if gamma is None else gamma.astype(np.float64)
        b = np.zeros(c) if beta is None else beta.astype(np.float64)
        rm0 = np.zeros(c) if rm0 is None else rm0.astype(np.float64)
        ris0 = np.ones(c) if ris0 is None else ris0.astype(np.float64)
        self.y, self.rm, self.ris, m, inv_std = tn.batch_norm_train(x, g, b, rm0, ris0, eps, alpha)
        x64 = x.astype(np.float64)
        axes = (0,) + tuple(range(2, x.ndim))
        shp = [1, -1] + [1] * (x.ndim - 2)
        L = chain or bn_chain(x.shape[0], int(np.prod(x.shape[2:], dtype=np.int64)))
        e_m = (L + 1) * U64 * np.abs(x64).mean(axes)                 # float64 error of sum / count
        term_m = np.maximum(np.abs(m - (m - e_m).astype(np.float32)), np.abs(m - (m + e_m).astype(np.float32)))
        e_var = (3 * L + 4) * U64 * np.square(x64).mean(axes)        # Sum x^2/N - mean^2 in float64
        d_eps = abs(float(np.float32(eps)) - eps)                    # the kernel takes eps as a float32
        d_i = U32 + 0.5 * (e_var + d_eps) / (x64.var(axes) + eps) + 4 * U64    # relative, float32 inv_std
        s = np.abs(g * inv_std)
        self.y_bound = 1.25 * ((s * term_m * (1 + 2 * U32)).reshape(shp)
                               + np.abs(x64 - m.reshape(shp)) * (s * (3 * U32 + d_i)).reshape(shp) + U32 * np.abs(self.y))
        self.rm_bound = 1.25 * ((1 - alpha) * np.abs(rm0) * 3 * U32 + alpha * (term_m + 2 * U32 * np.abs(m)) + U32 * np.abs(self.rm))
        self.ris_bound = 1.25 * ((1 - alpha) * np.abs(ris0) * 3 * U32 + alpha * inv_std * (d_i + 2 * U32) + U32 * np.abs(self.ris))
        self.mean, self.inv_std = m, inv_std

    def check(self, y, rm=None, ris=None, what=""):
        """asserts; returns the worst error / bound ratio over y and the running statistics given"""
        worst = 0.0
        for name, got, want, bound in (("y", y, self.y, self.y_bound), ("running_mean", rm, self.rm, self.rm_bound),
                                       ("running_inv_std", ris, self.ris, self.ris_bound)):
            if got is None:
                continue
            err = np.abs(got.astype(np.float64) - want)
            ok = err <= bound
            if not ok.all():
                bad = np.unravel_index(np.argmin(np.where(ok, np.inf, -err / np.maximum(bound, 1e-300))), err.shape)
                raise AssertionError("%s %s: |err| %.3g > bound %.3g at %s (got %r, want %r)"
                                     % (what, name, err[bad], bound[bad], bad, got[bad], want[bad]))
            worst = max(worst, float((err / np.maximum(bound, 1e-300)).max()))
        return worst


def run_bn(model, x, gamma=None, beta=None, rm0=None, ris0=None, **kw):
    rm, ris = dev(rm0), dev(ris0)
    y = _ops().batch_norm_train(model, dev(x), dev(gamma), dev(beta), rm, ris, **kw)
    return host(y), host(rm), host(ris)


def bn_params(rng, c):
    return (rng.uniform(0.5, 1.5, c).astype(np.float32), rng.normal(0, 0.5, c).astype(np.float32),
            rng.normal(0, 2, c).astype(np.float32), rng.uniform(0.5, 2, c).astype(np.float32))


def bn_data(rng, shape):
    """per channel: std from 1e-2 to 1e1, |mean| / std from 1e-1 to 1e3, either sign"""
    c, shp = shape[1], [1, -1] + [1] * (len(shape) - 2)
    std = 10.0 ** rng.uniform(-2, 1, c)
    mean = std * 10.0 ** rng.uniform(-1, 3, c) * rng.choice([-1.0, 1.0], c)
    return (rng.standard_normal(shape) * std.reshape(shp) + mean.reshape(shp)).astype(np.float32)


def bn_case(model, rng, shape, what):
    x = bn_data(rng, shape)
    g, b, rm0, ris0 = bn_params(rng, shape[1])
    y, rm, ris = run_bn(model, x, g, b, rm0, ris0)
    return BnExpect(x, g, b, rm0, ris0).check(y, rm, ris, what)


def test_executed_reference_edges(model):
    """the fixture's cases first: the stand-in BatchNormLayer on an offset and a constant channel, the reference's own
    MinibatchLayer at n = 1, K = P = 1 and K = 13, P = 5 with d = 33"""
    x, g, b = EDGES["bn_x"], EDGES["bn_gamma"], EDGES["bn_beta"]
    rm0, ris0 = np.array([0.5, -1.0], np.float32), np.array([1.5, 0.7], np.float32)
    y, rm, ris = run_bn(model, x, g, b, rm0, ris0)
    e = BnExpect(x, g, b, rm0, ris0)
    assert np.abs(e.y - EDGES["bn_y"]).max() <= 1e-12
    e.check(y, rm, ris, "fixture bn")
    assert np.all(y[:, 1] == b[1]) and e.inv_std[1] == INV_SQRT_EPS
    for tag in ("n1", "k1p1", "k13p5"):
        a = lambda k: EDGES["mb_%s_%s" % (tag, k)]
        mb_check(model, a("x"), a("theta"), a("lws"), a("b"), ref=a("out"), what=tag)


CONV = [(1, 3, 2), (1, 1, 4096), (1, 130, 257), (2, 1, 35), (2, 130, 256), (2, 3, 1024), (31, 3, 255), (31, 1, 4096),
        (31, 130, 2), (32, 130, 35), (32, 3, 256), (32, 1, 4096), (33, 1, 257), (33, 3, 1024), (33, 130, 2),
        (100, 3, 35), (100, 1, 4096), (100, 130, 2), (100, 3, 257), (100, 130, 255)]


@pytest.mark.parametrize("n,c,hw", CONV)
def test_bn_conv_shapes(model, n, c, hw):
    rng = np.random.default_rng(n * 100003 + c * 101 + hw)
    shape = (n, c, hw) if hw % 5 else (n, c, 5, hw // 5)
    bn_case(model, rng, shape, "conv %s" % (shape,))


@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 257])
def test_bn_dense_shapes(model, n):
    for c in (1, 255, 256, 257, 1000):
        bn_case(model, np.random.default_rng(n * 7919 + c), (n, c), "dense (%d, %d)" % (n, c))


def test_bn_layouts_agree_bit_for_bit(model):
    rng = np.random.default_rng(5)
    g, b, rm0, ris0 = bn_params(rng, 7)
    x = bn_data(rng, (33, 7, 4, 6, 11))
    want = run_bn(model, x.reshape(33, 7, 264), g, b, rm0, ris0)
    for shape in ((33, 7, 264), (33, 7, 24, 11), (33, 7, 4, 6, 11)):
        got = run_bn(model, x.reshape(shape), g, b, rm0, ris0)
        assert all(np.array_equal(u.reshape(v.shape), v) for u, v in zip(got, want)), shape
    xd = bn_data(rng, (65, 7))
    want = run_bn(model, xd, g, b, rm0, ris0)
    got = run_bn(model, xd.reshape(65, 7, 1, 1), g, b, rm0, ris0)
    assert all(np.array_equal(u.reshape(v.shape), v) for u, v in zip(got, want))
    BnExpect(xd, g, b, rm0, ris0).check(*want, what="dense")


def edge_channels(rng, n, hw):
    """(n, 11, hw): |mean|/std of 1e1 .. 1e4, constants 0 / 3.7 / 1000.1 / -1e4, std 1e-3 next to std 30 / mean -5e3,
    and a channel of 2.5 everywhere but one 7.0"""
    x = np.empty((n, 11, hw), np.float32)
    for k, (m, s) in enumerate(((10.0, 1.0), (-100.0, 1.0), (1000.0, 1.0), (1e4, 1.0))):
        x[:, k] = m + s * rng.standard_normal((n, hw))
    for k, v in enumerate((0.0, 3.7, 1000.1, -1e4)):
        x[:, 4 + k] = np.float32(v)
    x[:, 8] = 0.5 + 1e-3 * rng.standard_normal((n, hw))
    x[:, 9] = -5e3 + 30 * rng.standard_normal((n, hw))
    x[:, 10] = 2.5
    x[n // 2, 10, hw // 3] = 7.0
    return x


@pytest.mark.parametrize("n,hw", [(32, 4096), (64, 256), (3, 1000), (257, 1), (64, 1), (5, 1)])
def test_bn_offset_and_constant_channels(model, n, hw):
    rng = np.random.default_rng(n + hw)
    x = edge_channels(rng, n, hw)
    if hw == 1:
        x = x[:, :, 0].copy()
    g, b, rm0, ris0 = bn_params(rng, 11)
    y, rm, ris = run_bn(model, x, g, b, rm0, ris0)
    e = BnExpect(x, g, b, rm0, ris0)
    e.check(y, rm, ris, "edges n=%d hw=%d" % (n, hw))
    for k in range(4, 8):                                 # constant channels: y = beta exactly (oracle inv_std 1/sqrt(eps))
        assert np.all(y[:, k] == b[k]), k
        assert e.inv_std[k] == INV_SQRT_EPS, k


def test_bn_dense_single_sample_is_beta(model):
    rng = np.random.default_rng(8)
    x = (rng.standard_normal((1, 300)) * 10.0 ** rng.uniform(-3, 4, 300)).astype(np.float32)
    g, b, rm0, ris0 = bn_params(rng, 300)
    y, rm, ris = run_bn(model, x, g, b, rm0, ris0)
    assert np.array_equal(y[0], b)
    BnExpect(x, g, b, rm0, ris0).check(y, rm, ris, "dense n=1")


@pytest.mark.parametrize("shape", [(17, 5, 9, 11), (70, 300)])
def test_bn_options(model, shape):
    rng = np.random.default_rng(shape[0])
    x = bn_data(rng, shape)
    g, b, rm0, ris0 = bn_params(rng, shape[1])
    y, rm, ris = run_bn(model, x, g, b, rm0, ris0)
    BnExpect(x, g, b, rm0, ris0).check(y, rm, ris, "defaults")
    y0, _, _ = run_bn(model, x, g, b)                                       # no running statistics: the same y
    assert np.array_equal(y0, y)
    y1, rm1, _ = run_bn(model, x, g, b, rm0=rm0)                           # running_mean only
    assert np.array_equal(y1, y) and np.array_equal(rm1, rm)
    yn, rmn, risn = run_bn(model, x, None, None, rm0, ris0)                # no gamma / beta: 1 and 0
    BnExpect(x, None, None, rm0, ris0).check(yn, rmn, risn, "gamma=beta=None")
    ye, rme, rise = run_bn(model, x, g, b, rm0, ris0, eps=2.5e-3, alpha=0.35)
    BnExpect(x, g, b, rm0, ris0, eps=2.5e-3, alpha=0.35).check(ye, rme, rise, "eps, alpha")


def test_bn_synchronised_shards(model):
    """cross-GPU synchronised BN simulated on one GPU: per-shard sums, added in rank order, normalised with the global
    count, match the whole batch; every shard ends with the same running statistics"""
    import torch
    ops = _ops()
    rng = np.random.default_rng(9)
    for shape in ((37, 5, 15, 17), (97, 260)):
        n, c = shape[:2]
        hw = int(np.prod(shape[2:], dtype=np.int64))
        x = bn_data(rng, shape)
        g, b, rm0, ris0 = bn_params(rng, c)
        yw, rmw, risw = run_bn(model, x, g, b, rm0, ris0)
        BnExpect(x, g, b, rm0, ris0).check(yw, rmw, risw, "whole batch")
        for cuts in ((0, n // 3, n), (0, 5, n - n // 3, n)):
            e = BnExpect(x, g, b, rm0, ris0, chain=max(bn_chain(hi - lo, hw) for lo, hi in zip(cuts[:-1], cuts[1:])) + len(cuts))
            shards = [dev(x[lo:hi]) for lo, hi in zip(cuts[:-1], cuts[1:])]
            total = torch.zeros(2, c, dtype=torch.float64, device="cuda:0")
            for sh in shards:
                sums = torch.empty(2, c, dtype=torch.float64, device="cuda:0")
                with ops._lib_stream(model, sh) as st:
                    model._check(model._lib.ian_bn_batch_stats_dev(model._h, sh.data_ptr(), int(sh.shape[0]), c, hw,
                                                                   sums[0].data_ptr(), sums[1].data_ptr(), st))
                total += sums
            ys, stats, gd, bd = [], [], dev(g), dev(b)
            for sh in shards:
                y, rm, ris = torch.empty_like(sh), dev(rm0), dev(ris0)
                with ops._lib_stream(model, sh) as st:
                    model._check(model._lib.ian_bn_train_normalize_dev(
                        model._h, sh.data_ptr(), int(sh.shape[0]), c, hw, total[0].data_ptr(), total[1].data_ptr(),
                        float(n * hw), gd.data_ptr(), bd.data_ptr(), 1e-4, 0.1, rm.data_ptr(), ris.data_ptr(),
                        y.data_ptr(), st))
                ys.append(host(y))
                stats.append((host(rm), host(ris)))
            for rm, ris in stats[1:]:                       # every rank holds the same running statistics
                assert np.array_equal(rm, stats[0][0]) and np.array_equal(ris, stats[0][1])
            e.check(np.concatenate(ys), *stats[0], what="shards %s" % (cuts,))
            assert np.all(np.abs(np.concatenate(ys) - yw) <= 2 * e.y_bound)


def test_bn_group_path_world_size_one(model, tmp_path):
    """batch_norm_train(group=True): sums all-reduced over the default group (NCCL, one rank), count times world size"""
    import torch.distributed as dist
    rng = np.random.default_rng(10)
    x = bn_data(rng, (19, 6, 7, 9))
    g, b, rm0, ris0 = bn_params(rng, 6)
    want = run_bn(model, x, g, b, rm0, ris0)
    assert not dist.is_initialized()
    dist.init_process_group("nccl", init_method="file://" + str(tmp_path / "store"), rank=0, world_size=1)
    try:
        got = run_bn(model, x, g, b, rm0, ris0, group=True)
    finally:
        dist.destroy_process_group()
    assert all(np.array_equal(u, v) for u, v in zip(got, want))
    BnExpect(x, g, b, rm0, ris0).check(*got, what="group=True")


# ---- MinibatchLayer --------------------------------------------------------------------------------------------------
def mb_data(rng, n, d, K, P, x_scale=1.0):
    x = (x_scale * rng.standard_normal((n, d))).astype(np.float32)
    theta = rng.normal(0, 0.05, (d, K, P)).astype(np.float32)
    lws = rng.normal(np.log(0.2 / P / x_scale), 0.1, (K, P)).astype(np.float32)
    b = rng.normal(-1, 0.5, K).astype(np.float32)
    return x, theta, lws, b


def mb_min_term(x, theta, lws):
    """the smallest exp(-sum_p |act_i - act_j|) over pairs i != j (1 for n = 1)"""
    x = x.reshape(len(x), -1).astype(np.float64)
    th = theta.astype(np.float64)
    act = np.tensordot(x, th * (np.exp(lws.astype(np.float64)) / np.sqrt(np.square(th).sum(0)))[None], [[1], [0]])
    ad = np.abs(act[:, None] - act[None]).sum(-1).max(-1)                   # (n, n): the farthest kernel of each pair
    np.fill_diagonal(ad, 0.0)
    return float(np.exp(-ad.max()))


def mb_check(model, x, theta, lws, b, ref=None, what=""):
    """asserts [x | f] against the oracle (or a fixture); returns the worst |f - f_ref| / (sum of terms + |b|)"""
    out = host(_ops().minibatch_layer(model, dev(x), dev(theta), dev(lws), dev(b)))
    ref = tn.minibatch_layer(x, theta, lws, b) if ref is None else ref
    n = len(x)
    x2 = x.reshape(n, -1)
    d = x2.shape[1]
    assert out.shape == ref.shape == (n, d + len(b)), what
    assert np.array_equal(out[:, :d], x2), what                                  # the concatenated x: copied bits
    if n == 1:
        assert np.array_equal(out[0, d:], b), what                               # the self-pair only: exp(-1e6) = 0
    scale = (ref[:, d:] - b.astype(np.float64)) + np.abs(b.astype(np.float64))
    err = np.abs(out[:, d:] - ref[:, d:]) / scale
    assert err.max() <= MB_TOL, (what, float(err.max()), np.unravel_index(np.argmax(err), err.shape))
    return float(err.max()), out


KP = [(1, 1), (7, 5), (63, 1), (64, 1), (13, 5), (300, 1), (100, 5)]


@pytest.mark.parametrize("i", range(30))
def test_mb_shapes(model, i):
    """every (n, d) of {1, 2, 15, 16, 17, 33} x {1, 31, 32, 33, 200} once, (K, P) cycling through KP"""
    n, d = (1, 2, 15, 16, 17, 33)[i % 6], (1, 31, 32, 33, 200)[i % 5]
    K, P = KP[i % 7]
    rng = np.random.default_rng(1000 + i)
    x, theta, lws, b = mb_data(rng, n, d, K, P)
    assert mb_min_term(x, theta, lws) > MB_MIN_TERM
    mb_check(model, x, theta, lws, b, what="n=%d d=%d K=%d P=%d" % (n, d, K, P))


@pytest.mark.parametrize("n", [64, 128])
def test_mb_discriminator_shape(model, n):
    """IAN_simple.py:225-231: a (n, 1024, 4, 4) feature map -> 100 kernels x 5"""
    rng = np.random.default_rng(n)
    x, theta, lws, b = mb_data(rng, n, 16384, 100, 5, x_scale=0.5)
    x = x.reshape(n, 1024, 4, 4)
    assert mb_min_term(x, theta, lws) > MB_MIN_TERM
    mb_check(model, x, theta, lws, b, what="16384 -> 100x5, n=%d" % n)


def test_mb_batch_permutation(model):
    rng = np.random.default_rng(4)
    x, theta, lws, b = mb_data(rng, 33, 200, 13, 5)
    perm = rng.permutation(33)
    _, out = mb_check(model, x, theta, lws, b)
    _, outp = mb_check(model, x[perm], theta, lws, b)
    ref = tn.minibatch_layer(x, theta, lws, b)[perm, 200:]
    scale = ref - b + np.abs(b)
    assert np.all(np.abs(outp[:, 200:] - out[perm, 200:]) <= 2 * MB_TOL * scale)
    assert np.array_equal(outp[:, :200], out[perm, :200])


# ---- determinism and isolation ---------------------------------------------------------------------------------------
def test_reruns_workspace_history_and_streams(model):
    """bit-identical reruns; nothing depends on what the shared workspace held before (a larger MinibatchLayer call in
    between, c growing and shrinking); a non-default torch stream gives the default stream's bits"""
    import torch
    ops = _ops()
    rng = np.random.default_rng(12)
    bn_inputs = []
    for shape in ((33, 130, 257), (5, 3, 40), (65, 1000)):
        bn_inputs.append((bn_data(rng, shape),) + bn_params(rng, shape[1]))
    mb_small = mb_data(rng, 17, 33, 13, 5)
    mb_big = mb_data(rng, 128, 2048, 100, 5)
    first = [run_bn(model, *a) for a in bn_inputs] + [mb_check(model, *mb_small)[1]]

    def same(got):
        for u, v in zip(got[:-1], first[:-1]):
            assert all(np.array_equal(p, q) for p, q in zip(u, v))
        assert np.array_equal(got[-1], first[-1])

    same([run_bn(model, *a) for a in bn_inputs] + [mb_check(model, *mb_small)[1]])
    mb_check(model, *mb_big)                                       # grows the workspace past every BN need
    same([run_bn(model, *a) for a in reversed(bn_inputs)][::-1] + [mb_check(model, *mb_small)[1]])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = []
        for x, g, b, rm0, ris0 in bn_inputs:
            rm, ris = dev(rm0), dev(ris0)
            got.append((ops.batch_norm_train(model, dev(x), dev(g), dev(b), rm, ris), rm, ris))
        mb = ops.minibatch_layer(model, *[dev(a) for a in mb_small])
    s.synchronize()
    same([tuple(host(t) for t in r) for r in got] + [host(mb)])


@pytest.mark.parametrize("shape", [(33, 6, 17, 15), (65, 257)])
def test_bn_channel_isolation(model, shape):
    """one channel's data replaced -- by other data, a NaN, an Inf -- leaves every other channel's y and running
    statistics bit-unchanged; a non-finite channel comes back NaN in every sample, as the reference's does"""
    rng = np.random.default_rng(shape[0])
    c = shape[1]
    x = bn_data(rng, shape)
    g, b, rm0, ris0 = bn_params(rng, c)
    clean = run_bn(model, x, g, b, rm0, ris0)
    for kind, k in (("new", 0), ("nan", c // 2), ("inf", c - 1), ("-inf", 1)):
        xt = x.copy()
        if kind == "new":
            xt[:, k] = bn_data(rng, (shape[0], 1) + shape[2:])[:, 0]
        else:
            xt[(shape[0] // 2, k) + (0,) * (len(shape) - 2)] = {"nan": np.nan, "inf": np.inf, "-inf": -np.inf}[kind]
        got = run_bn(model, xt, g, b, rm0, ris0)
        other = np.arange(c) != k
        for u, v in zip(got, clean):
            assert np.array_equal(u[:, other] if u.ndim > 1 else u[other], v[:, other] if v.ndim > 1 else v[other]), kind
        if kind == "new":
            BnExpect(xt, g, b, rm0, ris0).check(*got, what="new channel")
            continue
        with np.errstate(invalid="ignore"):
            want = tn.batch_norm_train(xt[:, k:k + 1], g[k:k + 1], b[k:k + 1], rm0[k:k + 1], ris0[k:k + 1])
        assert np.isnan(want[0]).all() and np.isnan(got[0][:, k]).all(), kind
        for u, v in zip(got[1:], want[1:3]):
            assert np.array_equal(u[k:k + 1], v.astype(np.float32), equal_nan=True), (kind, u[k], v)

"""CPU ORACLE (test infrastructure, NOT product code) -- float64 definitional restatement.

PARITY: PINNED TO THE EXECUTED REFERENCE, with one stated limit.  Theano 0.9 / Lasagne 0.2.dev1 (and Python 2)
are absent and the trained weights are git-LFS pointers, so the reference cannot run as shipped and has no golden
vectors (SURVEY.md F2/F3/F5).  Instead the reference's OWN files -- API.py, IAN_simple.py, IANv1.py, IAN.py,
layers.py, mask_generator.py, GANcheckpoints.py -- are executed unmodified from the original project on numpy stand-ins
for those two third-party packages (oracle/refshim/), with the synthetic seeded checkpoint loaded by the reference's
own loader; the outputs are committed as tests/golden/ref_exec_*.npz (tests/golden/make_golden_ref.py) and this
file agrees with them to 1e-12 (forward) / 1e-8 (gradients, vs numeric differentiation of the reference forward):
tests/test_reference_exec.py.  So graph wiring, hyper-parameters, parameter names and the loading path are pinned
to the reference's code; what remains restated (not pinned) is the semantics of the third-party layers underneath
(Lasagne's documented behaviour, cuDNN's convolution definition; SURVEY.md Appendix C) and Theano's float32
rounding.  Executing the reference already corrected one reading error (MADE wiring, see ian_full_numpy.made_forward).
It is also cross-checked against an independent float32 torch restatement (oracle/ian_torch.py) and against
self-consistency KATs in tests/.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this package.  The product (neural-photo-editor_b200/) never does.

Every function cites the reference file:line it follows (paths relative to the reference root).
All arrays are NCHW float64 unless stated.
"""
from __future__ import annotations

import numpy as np

F64 = np.float64

# ----------------------------------------------------------------------------------------------
# nonlinearities -- lasagne.nonlinearities as used at IAN_simple.py:17-19,80,121,132,179
# (assumption C.5: rectify = 0.5*(x+|x|); LeakyRectify(a) = f1*x + f2*|x| with
#  f1=0.5*(1+a), f2=0.5*(1-a); elu = x>0 ? x : exp(x)-1)
# ----------------------------------------------------------------------------------------------

def rectify(x):
    return 0.5 * (x + np.abs(x))


def lrelu(x, alpha=0.2):
    f1, f2 = 0.5 * (1 + alpha), 0.5 * (1 - alpha)
    return f1 * x + f2 * np.abs(x)


def elu(x):
    return np.where(x > 0, x, np.expm1(np.minimum(x, 0)))


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


ACT = {"lrelu": lrelu, "relu": rectify, "elu": elu, "tanh": np.tanh, "sigmoid": sigmoid,
       "identity": lambda x: x}


# ----------------------------------------------------------------------------------------------
# layers
# ----------------------------------------------------------------------------------------------

def conv5x5_s2(x, W, b=None):
    """Conv2DLayer/Conv2DDNNLayer(filter 5x5, stride 2, pad 2, flip_filters=False)
    (IAN_simple.py:73-116; assumption C.2): cross-correlation,
    y[n,o,p,q] = sum_{c,i,j} x[n,c,2p+i-2,2q+j-2] * W[o,c,i,j] (+ b[o])."""
    x = np.asarray(x, F64)
    W = np.asarray(W, F64)
    n, c, h, w = x.shape
    ho, wo = (h + 4 - 5) // 2 + 1, (w + 4 - 5) // 2 + 1
    xp = np.zeros((n, c, h + 4, w + 4), F64)
    xp[:, :, 2:2 + h, 2:2 + w] = x
    y = np.zeros((n, W.shape[0], ho, wo), F64)
    for i in range(5):
        for j in range(5):
            patch = xp[:, :, i:i + 2 * ho:2, j:j + 2 * wo:2]
            y += np.einsum("nchw,oc->nohw", patch, W[:, :, i, j], optimize=True)
    if b is not None:
        y += np.asarray(b, F64)[None, :, None, None]
    return y


def batchnorm_inf(x, p):
    """lasagne.layers.batch_norm, deterministic=True (IAN_simple.py:84-135,141-170; assumption C.1):
    y = (x - mean) * (gamma * inv_std) + beta, per channel (axis 1); inv_std is stored directly."""
    shp = (1, -1) + (1,) * (x.ndim - 2)
    g = np.asarray(p["gamma"], F64).reshape(shp)
    be = np.asarray(p["beta"], F64).reshape(shp)
    m = np.asarray(p["mean"], F64).reshape(shp)
    s = np.asarray(p["inv_std"], F64).reshape(shp)
    return (x - m) * (g * s) + be


def dense(x, W, b=None):
    """DenseLayer (IAN_simple.py:117-135; assumption C.3): flatten(2) @ W (+ b), W is (in,out)."""
    x = np.asarray(x, F64).reshape(x.shape[0], -1)
    y = x @ np.asarray(W, F64)
    if b is not None:
        y = y + np.asarray(b, F64)[None, :]
    return y


def deconv5x5_s2(x, W):
    """DeconvLayer (layers.py:436-483) == GpuDnnConvGradI with conv_mode='conv', border 2, stride 2,
    output forced to 2H x 2W (layers.py:460,479-481; assumption C.4): input-gradient of a true
    convolution.  W is (Cin, Cout, 5, 5) (layers.py:449-452).
        y[n,co,u,v] = sum_{ci,a,b} x[n,ci,a,b] * W[ci,co, 2+2a-u, 2+2b-v]   (kernel idx in [0,4])."""
    x = np.asarray(x, F64)
    W = np.asarray(W, F64)
    n, ci, h, w = x.shape
    co = W.shape[1]
    y = np.zeros((n, co, 2 * h, 2 * w), F64)
    for ki in range(5):
        for kj in range(5):
            # u = 2 + 2a - ki  -> for each a, u fixed parity
            contrib = np.einsum("nchw,co->nohw", x, W[:, :, ki, kj], optimize=True)
            a = np.arange(h)
            u = 2 + 2 * a - ki
            va = (u >= 0) & (u < 2 * h)
            b_ = np.arange(w)
            v = 2 + 2 * b_ - kj
            vb = (v >= 0) & (v < 2 * w)
            y[:, :, u[va][:, None], v[vb][None, :]] += contrib[:, :, a[va][:, None], b_[vb][None, :]]
    return y


def deconv5x5_s2_bwd_data(dy, W):
    """Adjoint of deconv5x5_s2 w.r.t. x (what T.grad derives at API.py:59,64 for each DeconvLayer):
    dx[n,ci,a,b] = sum_{co,ki,kj} dy[n,co,2+2a-ki,2+2b-kj] * W[ci,co,ki,kj]."""
    dy = np.asarray(dy, F64)
    W = np.asarray(W, F64)
    n, co, H, Wd = dy.shape
    h, w = H // 2, Wd // 2
    dx = np.zeros((n, W.shape[0], h, w), F64)
    for ki in range(5):
        for kj in range(5):
            a = np.arange(h)
            u = 2 + 2 * a - ki
            va = (u >= 0) & (u < H)
            b_ = np.arange(w)
            v = 2 + 2 * b_ - kj
            vb = (v >= 0) & (v < Wd)
            sl = dy[:, :, u[va][:, None], v[vb][None, :]]
            dx[:, :, a[va][:, None], b_[vb][None, :]] += np.einsum("nohw,co->nchw", sl, W[:, :, ki, kj],
                                                                  optimize=True)
    return dx


def gaussian_sample(mu, logsigma, eps=None, deterministic=True):
    """GaussianSampleLayer (layers.py:419-433): deterministic -> mu; else mu + exp(logsigma)*eps.
    eps is INJECTED (the MRG31k3p stream of layers.py:421 is not reproducible here; C.9)."""
    if deterministic:
        return mu
    return mu + np.exp(logsigma) * np.asarray(eps, F64)


# ----------------------------------------------------------------------------------------------
# IAN_simple graph (IAN_simple.py:56-241; SURVEY Appendix A)
# ----------------------------------------------------------------------------------------------

def _bn(P, name):
    return {k: P[name + "." + k] for k in ("beta", "gamma", "mean", "inv_std")}


def simple_encode_mu_ls(P, x):
    """l_in -> (mu, logsigma)  (IAN_simple.py:72-126)."""
    h = lrelu(conv5x5_s2(x, P["enc_conv1.W"], P["enc_conv1.b"]))
    h = lrelu(batchnorm_inf(conv5x5_s2(h, P["enc_conv2.W"]), _bn(P, "bnorm2")))
    h = lrelu(batchnorm_inf(conv5x5_s2(h, P["enc_conv3.W"]), _bn(P, "bnorm3")))
    h = lrelu(batchnorm_inf(conv5x5_s2(h, P["enc_conv4.W"]), _bn(P, "bnorm4")))
    h = elu(batchnorm_inf(dense(h, P["enc_fc1.W"]), _bn(P, "bnorm_enc_fc1")))
    mu = batchnorm_inf(dense(h, P["enc_mu.W"]), _bn(P, "mu_bnorm"))
    ls = batchnorm_inf(dense(h, P["enc_logsigma.W"]), _bn(P, "ls_bnorm"))
    return mu, ls


def simple_encode(P, x, deterministic=True, eps=None):
    """API.IAN.encode_images -> Z_hat_fn (API.py:50-51,78-90): deterministic=True returns mu."""
    mu, ls = simple_encode_mu_ls(P, x)
    return gaussian_sample(mu, ls, eps, deterministic)


def simple_decode(P, z, return_cache=False):
    """API.IAN.sample_at -> X_hat_fn (API.py:46-47,98-110; IAN_simple.py:129-181)."""
    z = np.asarray(z, F64)
    u0 = batchnorm_inf(dense(z, P["l_dec_fc2.W"]), _bn(P, "bnorm_dec_fc2"))
    h0 = rectify(u0).reshape(-1, 1024, 4, 4)
    u1 = batchnorm_inf(deconv5x5_s2(h0, P["dec_conv1.W"]), _bn(P, "bnorm_dc1"))
    h1 = rectify(u1)
    u2 = batchnorm_inf(deconv5x5_s2(h1, P["dec_conv2.W"]), _bn(P, "bnorm_dc2"))
    h2 = rectify(u2)
    u3 = batchnorm_inf(deconv5x5_s2(h2, P["dec_conv3.W"]), _bn(P, "bnorm_dc3"))
    h3 = rectify(u3)
    xh = np.tanh(deconv5x5_s2(h3, P["dec_out.W"]))
    if return_cache:
        return xh, (u0, u1, u2, u3)
    return xh


def _box(c1, r1, c2, r2):
    """theano int32 scalars with lossless float coercion (API.py:54-55; assumption C.8)."""
    out = []
    for v in (c1, r1, c2, r2):
        iv = int(v)
        if iv != v:
            raise TypeError("box coordinate %r is not integral" % (v,))
        out.append(iv)
    return out


def _decoder_backward(P, cache, dxh_pre):
    """reverse-mode through the IAN_simple decoder; dxh_pre = dL/d(pre-tanh output)."""
    u0, u1, u2, u3 = cache

    def bn_scale(name, nd):
        p = _bn(P, name)
        s = np.asarray(p["gamma"], F64) * np.asarray(p["inv_std"], F64)
        return s.reshape((1, -1) + (1,) * (nd - 2))

    d = deconv5x5_s2_bwd_data(dxh_pre, P["dec_out.W"])
    d = d * (u3 > 0) * bn_scale("bnorm_dc3", 4)
    d = deconv5x5_s2_bwd_data(d, P["dec_conv3.W"])
    d = d * (u2 > 0) * bn_scale("bnorm_dc2", 4)
    d = deconv5x5_s2_bwd_data(d, P["dec_conv2.W"])
    d = d * (u1 > 0) * bn_scale("bnorm_dc1", 4)
    d = deconv5x5_s2_bwd_data(d, P["dec_conv1.W"])
    d = d.reshape(d.shape[0], -1) * (u0 > 0) * bn_scale("bnorm_dec_fc2", 2)
    return d @ np.asarray(P["l_dec_fc2.W"], F64).T


def simple_imgrad(P, c1, r1, c2, r2, z):
    """API.IAN.imgrad -> calculate_lighten_gradient (API.py:59,66-70):
    d/dZ mean(X_hat[0,:,r1:r2,c1:c2]); only row 0 of the result is non-zero (SURVEY F8)."""
    c1, r1, c2, r2 = _box(c1, r1, c2, r2)
    xh, cache = simple_decode(P, z, return_cache=True)
    cnt = 3 * len(range(*slice(r1, r2).indices(64))) * len(range(*slice(c1, c2).indices(64)))
    seed = np.zeros_like(xh)
    seed[0, :, r1:r2, c1:c2] = 1.0 / cnt
    return _decoder_backward(P, cache, seed * (1 - xh ** 2))


def simple_imgradRGB(P, c1, r1, c2, r2, RGB, z):
    """API.IAN.imgradRGB -> calculate_RGB_gradient (API.py:64,72-76):
    d/dZ mean((RGB[0,:,r1:r2,c1:c2] - X_hat[0,:,r1:r2,c1:c2])**2)."""
    c1, r1, c2, r2 = _box(c1, r1, c2, r2)
    RGB = np.asarray(RGB, F64)
    xh, cache = simple_decode(P, z, return_cache=True)
    cnt = 3 * len(range(*slice(r1, r2).indices(64))) * len(range(*slice(c1, c2).indices(64)))
    seed = np.zeros_like(xh)
    seed[0, :, r1:r2, c1:c2] = 2.0 * (xh[0, :, r1:r2, c1:c2] - RGB[0, :, r1:r2, c1:c2]) / cnt
    return _decoder_backward(P, cache, seed * (1 - xh ** 2))


def simple_grad_batched(P, z, boxes, rgb=None):
    """Batched generalisation of imgrad / imgradRGB (SURVEY F8, section 8b 'edit_steps'):
    sample k uses its own box boxes[k]=[c1,r1,c2,r2] and target rgb[k] ((3,) colour broadcast over the
    frame, or a (3,64,64) frame); exact vmap of the single-sample function because inference BN
    keeps samples independent.  rgb=None -> lighten gradient."""
    z = np.asarray(z, F64)
    xh, cache = simple_decode(P, z, return_cache=True)
    seed = np.zeros_like(xh)
    for k in range(z.shape[0]):
        c1, r1, c2, r2 = _box(*boxes[k])
        cnt = 3 * (r2 - r1) * (c2 - c1)
        if rgb is None:
            seed[k, :, r1:r2, c1:c2] = 1.0 / cnt
        else:
            t = np.asarray(rgb[k], F64)
            t = t.reshape(3, 1, 1) if t.ndim == 1 else t[:, r1:r2, c1:c2]
            seed[k, :, r1:r2, c1:c2] = 2.0 * (xh[k, :, r1:r2, c1:c2] - t) / cnt
    return _decoder_backward(P, cache, seed * (1 - xh ** 2))


def simple_edit_loop(P, z, boxes, rgb, n_steps=32, weight=0.05, f32_state=True):
    """NPE paint step rule (NPE.py:199-209) applied per sample for n_steps:
        g = imgradRGB(box, RGB, Z);  Z <- Z - weight * g * (1 + (x2 - x1)).
    BASELINE config 4 defines the state in float32 (SURVEY 8a note on a19): z, g and the update are
    rounded to float32 each step when f32_state is set (the per-step math stays float64)."""
    z = np.asarray(z, np.float32 if f32_state else F64).copy()
    boxes = np.asarray(boxes)
    fac = (1.0 + (boxes[:, 2] - boxes[:, 0])).astype(z.dtype)[:, None]
    for _ in range(n_steps):
        g = simple_grad_batched(P, z, boxes, rgb)
        if f32_state:
            g = g.astype(np.float32)
            z = (z - np.float32(weight) * g * fac).astype(np.float32)
        else:
            z = z - weight * g * fac
    return z


# ----------------------------------------------------------------------------------------------
# NPE caller-side helpers that define the inputs of the path (NPE.py:37-41,143-156,202)
# ----------------------------------------------------------------------------------------------

def to_tanh(x):
    """NPE.py:37-38."""
    return 2.0 * (x / 255.0) - 1.0


def from_tanh(x):
    """NPE.py:40-41."""
    return 255.0 * (x + 1) / 2.0


def npe_paint_blend(xhat, recon_u8, error):
    """The photo-mode blend of NPE.paint (NPE.py:218-231) for one decoded image xhat (3,64,64):
    returns IM uint8 (3,64,64).  Uses scipy's gaussian_filter exactly as the reference does."""
    import scipy.ndimage
    recon_t = to_tanh(np.float32(recon_u8))                                   # NPE.py:218 to_tanh(np.float32(RECON))
    DELTA = np.asarray(xhat, np.float32) - recon_t
    MASK = scipy.ndimage.gaussian_filter(np.min([np.mean(np.abs(DELTA), axis=0), np.ones((64, 64))], axis=0), 0.7)
    D = MASK * DELTA + (1 - MASK) * np.asarray(error)
    return np.uint8(from_tanh(to_tanh(recon_u8) + D))                         # NPE.py:231


def npe_display(im_u8):
    """update_photo's 4x nearest upsample + HWC interleave (NPE.py:107-118)."""
    data = np.repeat(np.repeat(np.uint8(im_u8), 4, 1), 4, 2)
    return np.concatenate([data[c].reshape(256, 256, 1) for c in range(3)], axis=2)

"""Plat-style model API of the Neural Photo Editor, backed by libian_b200.so (sm_90a CUDA).

Drop-in for the reference `API.py` (reference API.py:11-110): same class name, constructor signature
and method surface (`encode_images`, `sample_at`, `get_zdim`, `imgrad`, `imgradRGB`, attributes `cfg`,
`weights_fname`, `model`), so `NPE.py:18  model = IAN(config_path='IAN_simple.py', dnn=True)` and every
later call in NPE.py work unchanged.  All numerics run in the CUDA library through its C-ABI
(include/ian_b200.h); this file only marshals numpy arrays.  There is no Theano/Lasagne dependency and
no CPU fallback.

Extensions beyond the reference surface (SURVEY.md section 8b): `reconstruct`, `encode(..., eps)`,
batched `grad` / `edit_steps`, the decoder VJP `decode_vjp` for any pixel-space loss (torch autograd binding:
`torch_ops.decode`), the decoder JVP `decode_jvp` and the Jacobian `decoder_jacobian` (torch forward-mode binding:
`torch_ops.decode` under `torch.autograd.forward_ad`), the encoder VJP `encode_vjp` for any loss on the latent (torch autograd binding:
`torch_ops.encode`), the encoder JVP `encode_jvp` (torch forward-mode binding: `torch_ops.encode` under
`torch.autograd.forward_ad`), the encoder Jacobian `encoder_jacobian`, the derivatives of the sampling script's
functions in the prior space l_Z_IAF -- `flow_vjp` / `flow_jvp` (Z_IAF_fn) and `encode_pre_vjp` / `encode_pre_jvp` (Zfn),
torch bindings `torch_ops.flow` / `torch_ops.encode_pre` --, the decoder's Gauss-Newton normal equations `gauss_newton` and
the batched Levenberg-Marquardt latent fit `fit_latent`, their pixel-weighted forms under the N(0, I) prior in the sampling
space `gauss_newton_map` / `fit_latent_map` (masked fits and inpainting), the IAN's introspection features `introspect` /
`introspect_jvp` / `introspect_vjp` / `feature_loss` (torch binding: `torch_ops.introspect` / `torch_ops.feature_loss`) and
the fit under its feature-wise loss `gauss_newton_features` / `fit_latent_features`, the discriminator head l_discrim
`load_discriminator` / `discriminate` / `discriminate_vjp` and their training-mode forms `discriminate_train` /
`discriminate_train_vjp` (torch binding: `torch_ops.discriminate`), the IAN_simple decoder in training mode
`decode_train` / `decode_train_vjp` (torch binding: `torch_ops.decode(..., training=True)`), and `*_dev` variants taking
device pointers.
"""
from __future__ import annotations

import ctypes as C
import os
import warnings

import numpy as np

from . import _lib

# cfg of reference IAN_simple.py:33-51 (the config module itself imports lasagne/theano and cannot
# be executed here; the hot path only reads cfg['num_latents'], API.py:96)
_SIMPLE_CFG = {
    'batch_size': 128, 'learning_rate': {0: 0.0002}, 'optimizer': 'Adam', 'beta1': 0.5, 'update_ratio': 1,
    'decay_rate': 0, 'reg': 1e-5, 'momentum': 0.9, 'shuffle': True, 'dims': (64, 64), 'n_channels': 3,
    'n_classes': 10, 'batches_per_chunk': 64, 'max_epochs': 250, 'checkpoint_every_nth': 1, 'num_latents': 100,
    'recon_weight': 3.0, 'feature_weight': 1.0,
}
_SIMPLE_MODEL_KEYS = ('l_in', 'l_out', 'l_mu', 'l_ls', 'l_Z', 'l_introspect', 'l_discrim')
# cfg of reference IAN.py:39-62
_FULL_CFG = {
    'batch_size': 16, 'learning_rate': {0: 0.0002, 25: 0.0001, 50: 0.00005, 75: 0.00001}, 'optimizer': 'Adam',
    'beta1': 0.5, 'update_ratio': 1, 'decay_rate': 0, 'reg': 1e-5, 'momentum': 0.9, 'shuffle': True, 'dims': (64, 64),
    'n_channels': 3, 'batches_per_chunk': 64, 'max_epochs': 80, 'checkpoint_every_nth': 1, 'num_latents': 100,
    'recon_weight': 3.0, 'feature_weight': 1.0, 'dg_weight': 1.0, 'dd_weight': 1.0, 'agr_weight': 1.0,
    'ags_weight': 1.0, 'n_shuffles': 1, 'ortho': 1e-3,
}
_FULL_MODEL_KEYS = _SIMPLE_MODEL_KEYS + ('l_IAF_mu', 'l_IAF_ls', 'l_Z_IAF')
# l_introspect = [enc_conv1, enc_conv2, enc_conv3, enc_conv4] (IAN_simple.py:240): per-image shapes
FEATURE_SHAPES = ((128, 32, 32), (256, 16, 16), (512, 8, 8), (1024, 4, 4))
# the discriminator head's checkpoint tensors (IAN_simple.py:225-231, IAN.py:210-216, IANv1.py:203-209)
DISCRIMINATOR_KEYS = ('minibatch_discrim.theta', 'minibatch_discrim.log_weight_scale', 'minibatch_discrim.b', 'discrimi.W')
# the robust fit's losses (include/ian_b200.h IAN_ROBUST_*)
ROBUST_KINDS = {"huber": 1, "cauchy": 2}


def _robust_kind(kind):
    if kind not in ROBUST_KINDS:
        raise ValueError("kind must be one of %s (got %r)" % (sorted(ROBUST_KINDS), kind))
    return ROBUST_KINDS[kind]


def made_ordering(seed=1234, n=100):
    """MADE input ordering after `reset("Once")` (reference API.py:33-36 -> layers.py:845-853 ->
    mask_generator.py:35-38,55-73): one shuffle_row_elements draw of theano RandomStreams(seed).  Recalled theano
    seeding (SURVEY Appendix D, unverifiable offline): the stream's generator is
    RandomState(RandomState(seed).randint(2**30)) and a 1-D shuffle is one permutation(n).  Pass
    `made_ordering=` to IAN(...) to override."""
    stream = np.random.RandomState(int(np.random.RandomState(seed).randint(2 ** 30)))
    return np.arange(n, dtype=np.int32)[stream.permutation(n)]


def _f32(a, ndim, what):
    """theano.function input filtering for a float32 TensorType: wrong dtype / ndim -> TypeError."""
    a = np.asarray(a)
    if a.dtype != np.float32:
        raise TypeError("%s must be float32 (got %s); the reference's theano function rejects it too" % (what, a.dtype))
    if a.ndim != ndim:
        raise TypeError("%s must have %d dimensions (got %d)" % (what, ndim, a.ndim))
    return np.ascontiguousarray(a)


def _int_scalar(v, what):
    """int32 scalar input: non-integral values are rejected, integral floats accepted (NPE.py:202 passes
    `coords//4` floats); assumption C.8 in SURVEY.md."""
    iv = int(v)
    if iv != v:
        raise TypeError("%s=%r is not an integral value" % (what, v))
    return iv


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double)) if a is not None else None


def _z(a, what='z'):
    """latents: float32 (n,100).  The C side assumes the trailing dimension; theano would raise a shape error."""
    a = _f32(a, 2, what)
    if a.shape[1] != 100:
        raise ValueError("%s must be (n,100), got %r" % (what, a.shape))
    return a


def _img(a, what='images'):
    """images: float32 (n,3,64,64) NCHW."""
    a = _f32(a, 4, what)
    if a.shape[1:] != (3, 64, 64):
        raise ValueError("%s must be (n,3,64,64), got %r" % (what, a.shape))
    return a


def model_param_specs(kind):
    """[(name, shape)] of the graph's own parameters, in the reference's checkpoint naming -- the list API.py:23-28
    builds with lasagne.layers.get_all_params and hands to GANcheckpoints.load_weights."""
    lib = _lib.load()
    n = lib.ian_model_param_count(int(kind))
    if n < 0:
        raise ValueError("unknown model kind %r" % (kind,))
    out = []
    for i in range(n):
        name, shape, nd = C.c_char_p(), (C.c_int64 * 4)(), C.c_int()
        if lib.ian_model_param_spec(int(kind), i, C.byref(name), shape, C.byref(nd)) != _lib.IAN_OK:
            raise RuntimeError("ian_model_param_spec(%d, %d) failed" % (kind, i))
        out.append((name.value.decode(), tuple(int(shape[k]) for k in range(nd.value))))
    return out


class IAN:
    """Generic class for using IAN style models with the NPE (reference API.py:11)."""

    def __init__(self, config_path, dnn=True, weights=None, device=0, path=None, made_ordering=None):
        """config_path: path of the reference-style config module ('IAN_simple.py'); the weights are read
        from config_path[:-3]+'.npz' in GANcheckpoints format (reference API.py:18-30) unless a
        {name: ndarray} dict is given in `weights`.  `dnn` is accepted for signature compatibility (both
        reference variants of the graph are numerically the same function, IAN_simple.py:141-223)."""
        base = os.path.basename(str(config_path))
        if base == 'IAN_simple.py':
            kind, self.cfg, keys = _lib.IAN_MODEL_SIMPLE, dict(_SIMPLE_CFG), _SIMPLE_MODEL_KEYS
        elif base == 'IAN.py':
            # the reference's own API.IAN cannot construct this config (get_model(interp=...) vs dnn=..., SURVEY F6)
            kind, self.cfg, keys = _lib.IAN_MODEL_FULL, dict(_FULL_CFG), _FULL_MODEL_KEYS
        elif base == 'IANv1.py':
            kind, self.cfg, keys = _lib.IAN_MODEL_V1, dict(_FULL_CFG, max_epochs=150), _FULL_MODEL_KEYS
            self.cfg.pop('ortho', None)                     # IANv1.py:39-61 has no 'ortho' entry
        else:
            raise NotImplementedError("config %r: known graphs are IAN_simple.py, IAN.py and IANv1.py" % base)
        self.kind = kind
        self.device = int(device)                           # the CUDA device the handle is bound to
        self.weights_fname = str(config_path)[:-3] + '.npz'
        self.model = {k: base[:-3] + '.' + k for k in keys}
        self.dnn = dnn
        self._lib = _lib.load()
        self._stream_outs = {}                              # reconstruct_stream's rotating pinned result buffers
        self._h = C.c_void_p()
        rc = self._lib.ian_create(kind, int(device), C.byref(self._h))
        if rc != _lib.IAN_OK:
            msg = self._lib.ian_last_error(None)
            self._h = None
            raise _lib.IanError("ian_create failed (%d): %s" % (rc, msg.decode() if msg else "?"))
        print('Loading weights')
        if weights is None:
            weights = np.load(self.weights_fname, allow_pickle=False)
        # GANcheckpoints.load_weights (reference GANcheckpoints.py:33-57): iterate the MODEL's parameters and look each
        # one up by name; keys of the file the graph does not own (the trainer's log_sigma_theta,
        # train_IAN_simple.py:300,564; discriminator weights; the pickled 'metadata') are ignored.  Where the reference
        # only warns -- a parameter missing from the file, a shape mismatch -- this loader raises (ian_set_param /
        # ian_finalize), because a silently half-loaded model is never what a caller wants.
        have = set(weights.keys() if hasattr(weights, 'keys') else weights)
        own = model_param_specs(kind)
        for name, _shape in own:
            if name not in have:
                continue                                    # reported by ian_finalize as "missing parameter"
            arr = np.ascontiguousarray(np.asarray(weights[name], dtype=np.float32))
            shape = (C.c_int64 * max(arr.ndim, 1))(*arr.shape)
            self._check(self._lib.ian_set_param(self._h, name.encode(), _fp(arr), shape, arr.ndim))
        self.ignored_keys = sorted(have - {n for n, _ in own})
        if kind != _lib.IAN_MODEL_SIMPLE:
            print('Shuffling MADE masks')                   # reference API.py:33-36
            o = np.ascontiguousarray(globals()['made_ordering']() if made_ordering is None else made_ordering, np.int32)
            self.made_ordering = o
            self._check(self._lib.ian_set_made_ordering(self._h, o.ctypes.data_as(C.POINTER(C.c_int32)), int(o.size)))
        self._check(self._lib.ian_finalize(self._h))
        if path is not None:
            self.set_path(path)

    # ---- plumbing ---------------------------------------------------------------------------
    def _check(self, rc):
        _lib.check(self._lib, self._h, rc)

    def close(self):
        if getattr(self, '_h', None):
            self._lib.ian_destroy(self._h)
            self._h = None
            self._stream_outs = {}                          # the pinned memory went with the handle

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_path(self, path):
        """'tc' (wgmma tensor cores, default) or 'simt' (fp32 FFMA verification path); both are CUDA."""
        self._check(self._lib.ian_set_path(self._h, {'tc': _lib.IAN_PATH_TC, 'simt': _lib.IAN_PATH_SIMT}[path]))

    def set_precision(self, precision):
        """'fp32' (default: float32 semantics via the 3-pass bf16 split) or 'bf16' (full IAN only, single pass)."""
        self._check(self._lib.ian_set_precision(self._h, {'fp32': 0, 'bf16': 1}[precision]))

    def launch_count(self):
        return int(self._lib.ian_launch_count(self._h))

    def set_layer_timing(self, enable):
        self._check(self._lib.ian_set_layer_timing(self._h, int(bool(enable))))

    def layer_time_ms(self, layer, reset=True):
        return float(self._lib.ian_layer_time_ms(self._h, layer.encode(), int(reset)))

    # ---- reference surface ------------------------------------------------------------------------
    def imgrad(self, c1, r1, c2, r2, z):
        """Change in latents which would lighten the local image patch (reference API.py:66-70)."""
        return self._imgrad(c1, r1, c2, r2, None, z)

    def imgradRGB(self, c1, r1, c2, r2, RGB, z):
        """Change in latents which would move the local patch towards RGB (reference API.py:72-76)."""
        return self._imgrad(c1, r1, c2, r2, RGB, z)

    def _imgrad(self, c1, r1, c2, r2, RGB, z):
        c1, r1, c2, r2 = (_int_scalar(v, n) for v, n in zip((c1, r1, c2, r2), ('c1', 'r1', 'c2', 'r2')))
        z = _z(z)
        out = np.zeros_like(z)        # only sample 0 is differentiated (API.py:59,64)
        if z.shape[0] == 0:
            return out
        # numpy/theano slice semantics of X_hat[0,:,r1:r2,c1:c2]
        ra, rb, _ = slice(r1, r2).indices(64)
        ca, cb, _ = slice(c1, c2).indices(64)
        if rb <= ra or cb <= ca:
            out[0] = np.nan           # mean over an empty slice (cannot occur from NPE.py:149)
            return out
        boxes = np.array([[ca, ra, cb, rb]], dtype=np.int32)
        tgt = None
        if RGB is not None:
            RGB = _f32(RGB, 4, 'RGB')
            tgt = np.ascontiguousarray(RGB[0:1])
            if tgt.shape != (1, 3, 64, 64):
                raise TypeError("RGB must be (>=1,3,64,64), got %r" % (RGB.shape,))
        g = np.empty((1, z.shape[1]), np.float32)
        self._check(self._lib.ian_grad_host(self._h, _fp(np.ascontiguousarray(z[0:1])),
                                            boxes.ctypes.data_as(C.POINTER(C.c_int32)),
                                            _fp(tgt) if tgt is not None else None, 1, 1, _fp(g)))
        out[0] = g[0]
        return out

    def encode_images(self, images):
        """Encode images x => z: (n,3,s,s) float32 in [-1,1] -> (n, zdim) (reference API.py:78-90)."""
        return self.encode(images)

    def get_zdim(self):
        """Integer dimension of the latent z space (reference API.py:92-96)."""
        return self.cfg['num_latents']

    def sample_at(self, z):
        """Decode images z => x: (n, zdim) float32 -> (n,3,s,s) in [-1,1] (reference API.py:98-110)."""
        z = _z(z)
        x = np.empty((z.shape[0], 3, 64, 64), np.float32)
        if z.shape[0]:
            self._check(self._lib.ian_decode_host(self._h, _fp(z), z.shape[0], _fp(x)))
        return x

    # ---- extensions (batched / reparameterised / fused) ------------------------------------------
    def encode(self, images, eps=None):
        """deterministic (eps=None): mu(x).  With eps (n,100): mu + exp(logsigma)*eps (layers.py:419-433)."""
        x = _img(images)
        n = x.shape[0]
        z = np.empty((n, 100), np.float32)
        if n:
            e = None if eps is None else _z(eps, 'eps')
            if e is not None and e.shape[0] != n:
                raise ValueError("eps must be (%d,100), got %r" % (n, e.shape))
            self._check(self._lib.ian_encode_host(self._h, _fp(x), n, _fp(e) if e is not None else None, _fp(z)))
        return z

    # ---- the reference sampling script's function set (sample_IAN.py:86-94) ---------------------------------
    def Zfn(self, images):
        """X -> l_Z_IAF, deterministic (= mu, before the MADE/IAF flow); sample_IAN.py:91."""
        x = _img(images)
        z = np.empty((x.shape[0], 100), np.float32)
        if x.shape[0]:
            self._check(self._lib.ian_encode_pre_host(self._h, _fp(x), x.shape[0], _fp(z)))
        return z

    def Z_IAF_fn(self, z_iaf):
        """l_Z_IAF -> l_Z through the MADE/IAF flow (identity for IAN_simple); sample_IAN.py:94."""
        z0 = _z(z_iaf)
        z = np.empty_like(z0)
        if z0.shape[0]:
            self._check(self._lib.ian_flow_host(self._h, _fp(z0), z0.shape[0], _fp(z), None))
        return z

    def sample(self, z_iaf):
        """l_Z_IAF -> X: flow, then decoder; sample_IAN.py:86 (what the script feeds N(0,1) noise to)."""
        z0 = _z(z_iaf)
        x = np.empty((z0.shape[0], 3, 64, 64), np.float32)
        if z0.shape[0]:
            self._check(self._lib.ian_flow_host(self._h, _fp(z0), z0.shape[0], None, _fp(x)))
        return x

    def sampleZ(self, z):
        """l_Z -> X; sample_IAN.py:88 (== sample_at)."""
        return self.sample_at(z)

    def sample_grid(self, endpoints, n_samples=27, seed=None):
        """The 6x9 grid of sample_IAN.py:173-187: n_samples random samples + 3 rows of [endpoint, 7 interpolants,
        endpoint].  `endpoints`: 6 images float32 (6,3,64,64) in [-1,1].  Returns float32 images in [-1,1]."""
        rng = np.random.RandomState(seed)
        samples = self.sample(rng.randn(n_samples, 100).astype(np.float32))
        ends = _img(endpoints, 'endpoints')
        Ze = self.Zfn(ends)
        Z = np.asarray([Ze[2 * i] * (1 - j) + Ze[2 * i + 1] * j for i in range(3) for j in [t / 6.0 for t in range(7)]],
                       dtype=np.float32)
        rows = [np.insert(ends[2 * i:2 * (i + 1)], 1, self.sample(Z[7 * i:7 * (i + 1)]), axis=0) for i in range(3)]
        return np.append(samples, np.concatenate(rows, axis=0), axis=0)

    def reconstruct(self, images, return_z=False, out=None):
        """encode -> decode in one library call (the BASELINE metric's path).  `out`: optional preallocated
        float32 (n,3,64,64) result buffer (e.g. from pinned_empty) to avoid a pageable allocation per call."""
        x = _img(images)
        n = x.shape[0]
        xh = np.empty_like(x) if out is None else self._out(out, x.shape)
        z = np.empty((n, 100), np.float32)
        if n:
            self._check(self._lib.ian_reconstruct_host(self._h, _fp(x), n, _fp(z), _fp(xh)))
        return (xh, z) if return_z else xh

    @staticmethod
    def _out(out, shape):
        if not (isinstance(out, np.ndarray) and out.dtype == np.float32 and out.shape == tuple(shape)
                and out.flags['C_CONTIGUOUS']):
            raise TypeError("out must be a C-contiguous float32 array of shape %r" % (tuple(shape),))
        return out

    def pinned_empty(self, shape):
        """float32 numpy array in page-locked host memory owned by this model (valid until close())."""
        nbytes = int(np.prod(shape)) * 4
        p = C.c_void_p()
        self._check(self._lib.ian_host_alloc(self._h, nbytes, C.byref(p)))
        buf = (C.c_float * (nbytes // 4)).from_address(p.value)
        return np.frombuffer(buf, dtype=np.float32).reshape(shape)

    def reconstruct_submit(self, images, out, z_out=None):
        """Pipelined encode -> decode: enqueue one batch (n <= 512) and return a ticket immediately; `out`
        (and `z_out`) receive the result once reconstruct_wait(ticket) returns.  Two requests may be in
        flight; use pinned_empty() buffers so the copies overlap the neighbouring requests' compute."""
        x = _img(images)
        n = x.shape[0]
        out = self._out(out, x.shape)
        if z_out is not None:
            z_out = self._out(z_out, (n, 100))
        t = C.c_int()
        self._check(self._lib.ian_reconstruct_submit(self._h, _fp(x), n, _fp(z_out) if z_out is not None else None,
                                                     _fp(out), C.byref(t)))
        return t.value

    def reconstruct_wait(self, ticket):
        self._check(self._lib.ian_reconstruct_wait(self._h, int(ticket)))

    def reconstruct_stream(self, batches):
        """Generator over an iterable of (n,3,64,64) float32 batches: yields each reconstruction in order while
        keeping two batches in flight (H2D / compute / D2H of neighbouring batches overlap).  The yielded array
        is one of two rotating pinned buffers owned by the model (allocated on first use per batch shape, reused by
        later calls): consume it before advancing the generator twice, and run one stream at a time."""
        outs, pending = self._stream_outs, None              # page-locking costs milliseconds: keep the buffers
        for i, x in enumerate(batches):
            x = _img(x)
            key = (i & 1, x.shape)
            if key not in outs:
                outs[key] = self.pinned_empty(x.shape)
            t = self.reconstruct_submit(x, outs[key])
            if pending is not None:
                self.reconstruct_wait(pending[0])
                yield pending[1]
            pending = (t, outs[key])
        if pending is not None:
            self.reconstruct_wait(pending[0])
            yield pending[1]

    def _target(self, rgb, n):
        if rgb is None:
            return None, 0
        rgb = _f32(rgb, np.asarray(rgb).ndim, 'rgb')
        if rgb.shape == (n, 3):
            return rgb, 0
        if rgb.shape == (n, 3, 64, 64):
            return rgb, 1
        raise ValueError("rgb must be (n,3) or (n,3,64,64), got %r" % (rgb.shape,))

    def grad(self, z, boxes, rgb=None):
        """Per-sample brush gradient: boxes (n,4) int32 [c1,r1,c2,r2]; rgb None (lighten), (n,3) or frames."""
        z = _z(z)
        n = z.shape[0]
        boxes = np.ascontiguousarray(np.asarray(boxes, dtype=np.int32).reshape(n, 4))
        t, is_frame = self._target(rgb, n)
        g = np.empty_like(z)
        self._check(self._lib.ian_grad_host(self._h, _fp(z), boxes.ctypes.data_as(C.POINTER(C.c_int32)),
                                            _fp(t) if t is not None else None, is_frame, n, _fp(g)))
        return g

    def decode_vjp(self, z, dx_hat):
        """Vector-Jacobian product of the decoder, dz = (d x_hat / d z)^T . dx_hat, for any pixel-space loss:
        z float32 (n,100), dx_hat float32 (n,3,64,64) = dL/dx_hat -> dz float32 (n,100).  What T.grad of any loss on
        X_hat w.r.t. l_Z gives in the reference (API.py:46); grad() is the box-loss special case.  Costs one decoder
        forward and one backward."""
        z = _z(z)
        dx = _img(dx_hat, 'dx_hat')
        n = z.shape[0]
        if dx.shape[0] != n:
            raise ValueError("dx_hat must be (%d,3,64,64), got %r" % (n, dx.shape))
        dz = np.empty_like(z)
        if n:
            self._check(self._lib.ian_decode_vjp_host(self._h, _fp(z), _fp(dx), n, _fp(dz)))
        return dz

    def decode_jvp(self, z, v, return_x_hat=False):
        """Jacobian-vector product of the decoder, dx_hat = (d x_hat / d z) . v -- how the image moves when z moves along v:
        z, v float32 (n,100) -> dx_hat float32 (n,3,64,64), and x_hat = sample_at(z) bit for bit when return_x_hat
        (returned as (x_hat, dx_hat)).  Forward mode: one decoder forward and one tangent pass.  Its derivative conventions
        are decode_vjp's, so <u, decode_jvp(z, v)> = <decode_vjp(z, u), v> up to float32 summation."""
        z = _z(z)
        v = _z(v, 'v')
        n = z.shape[0]
        if v.shape[0] != n:
            raise ValueError("v must be (%d,100), got %r" % (n, v.shape))
        dx = np.empty((n, 3, 64, 64), np.float32)
        xh = np.empty((n, 3, 64, 64), np.float32) if return_x_hat else None
        if n:
            self._check(self._lib.ian_decode_jvp_host(self._h, _fp(z), _fp(v), n, _fp(xh) if xh is not None else None, _fp(dx)))
        return (xh, dx) if return_x_hat else dx

    def decoder_jacobian(self, z):
        """The decoder's Jacobian at each latent: z float32 (n,100) -> J float32 (n,100,3,64,64) with J[k, i] = d x_hat /
        d z_i at z[k], i.e. J's 100 columns as images (NPE's latent canvas shows what each coordinate does to the picture;
        J^T J is the pull-back metric, and Gauss-Newton steps fitting z to a photo need J).  One batch-100 decode_jvp with
        the identity as tangents per row of z."""
        z = _z(z)
        n = z.shape[0]
        J = np.empty((n, 100, 3, 64, 64), np.float32)
        eye = np.eye(100, dtype=np.float32)
        for k in range(n):
            zk = np.ascontiguousarray(np.broadcast_to(z[k], (100, 100)))
            self._check(self._lib.ian_decode_jvp_host(self._h, _fp(zk), _fp(eye), 100, None, _fp(J[k])))
        return J

    def gauss_newton(self, z, images):
        """The decoder's Gauss-Newton normal equations at each latent for the target images: z float32 (n,100), images
        float32 (n,3,64,64) in [-1,1] -> (A (n,100,100), g (n,100), e (n,)) float64 with r = sample_at(z) - images,
        A = J^T J (the pull-back metric), g = J^T r and e = r^T r, J = decoder_jacobian(z)'s bits.  z is l_Z, as for
        sample_at.  Costs one batch-100 decode_jvp per sample."""
        z = _z(z)
        x = _img(images)
        n, A, g, e = self._normal_eqs(z, x)
        if n:
            self._check(self._lib.ian_decode_gauss_newton_host(self._h, _fp(z), _fp(x), n, _dp(A), _dp(g), _dp(e)))
        return A, g, e

    def fit_latent(self, images, z0=None, iters=10, return_loss=False):
        """Fit a latent to each image: `iters` Levenberg-Marquardt steps on |sample_at(z) - images|^2, every decision on the
        GPU.  images float32 (n,3,64,64) in [-1,1]; z0 float32 (n,100) the start (default: encode_images(images)) -> z
        float32 (n,100), and with return_loss the per-sample mean squared error of the start and after every step, float32
        (n, iters+1), non-increasing.  z is l_Z, as for sample_at (on IAN.py / IANv1.py after the MADE/IAF flow)."""
        x = _img(images)
        n = x.shape[0]
        iters, z, loss = self._fit_start(iters, z0, 'z0', n, lambda: self.encode_images(x))
        if n:
            self._check(self._lib.ian_fit_latent_host(self._h, _fp(x), n, _fp(z), iters, _fp(loss)))
        return (z, loss) if return_loss else z

    @staticmethod
    def _normal_eqs(u, x):
        """n and the float64 outputs A (n,100,100), g (n,100), e (n,) of the normal equations at u's n points for the
        images x, once their batch sizes agree"""
        n = u.shape[0]
        if x.shape[0] != n:
            raise ValueError("images must be (%d,3,64,64), got %r" % (n, x.shape))
        return n, np.empty((n, 100, 100), np.float64), np.empty((n, 100), np.float64), np.empty((n,), np.float64)

    @staticmethod
    def _fit_start(iters, start, name, n, default):
        """iters checked, the fit's start (a copy of `start`, default() when None) checked against the n images, and the
        (n, iters+1) float32 loss history"""
        iters = _int_scalar(iters, 'iters')
        if iters < 0:
            raise ValueError("iters must not be negative (got %d)" % iters)
        u = default() if start is None else _z(start, name).copy()
        if u.shape[0] != n:
            raise ValueError("%s must be (%d,100), got %r" % (name, n, u.shape))
        return iters, u, np.empty((n, iters + 1), np.float32)

    def _map_args(self, images, weights, prior):
        x = _img(images)
        w = None if weights is None else _img(weights, 'weights')
        if w is not None and w.shape != x.shape:
            raise ValueError("weights must be %r, got %r" % (x.shape, w.shape))
        prior = float(prior)
        if not (np.isfinite(prior) and prior >= 0):
            raise ValueError("prior must be finite and >= 0 (got %r)" % prior)
        return x, w, prior

    def gauss_newton_map(self, u, images, weights=None, prior=0.0):
        """The normal equations of the masked fit under the prior at each fit-space point u: u float32 (n,100) (l_Z on
        IAN_simple, l_Z_IAF on IAN.py / IANv1.py, as `sample` takes it), images float32 (n,3,64,64), weights float32
        (n,3,64,64) finite and >= 0 (None: all ones; pixels of weight 0 are ignored, whatever the image holds there), prior
        beta >= 0 -> (A (n,100,100), g (n,100), e (n,)) float64 with r = sample(u) - images, J_u = d sample / d u,
        A = J_u^T W J_u + beta I, g = J_u^T W r + beta u and e = r^T W r + beta |u|^2."""
        u = _z(u, 'u')
        x, w, prior = self._map_args(images, weights, prior)
        n, A, g, e = self._normal_eqs(u, x)
        if n:
            self._check(self._lib.ian_map_gauss_newton_host(self._h, _fp(u), _fp(x), _fp(w) if w is not None else None, prior,
                                                            n, _dp(A), _dp(g), _dp(e)))
        return A, g, e

    def fit_latent_map(self, images, weights=None, prior=0.0, u0=None, iters=10, return_loss=False):
        """Fit the sampling-space latent to each image under pixel weights and the N(0, I) prior: `iters`
        Levenberg-Marquardt steps on sum_p w_p (sample(u) - images)_p^2 + prior |u|^2, every decision on the GPU.  Zero
        weights mask pixels out (inpainting: the masked region is filled by the decoder).  u0 float32 (n,100) the start
        (default: Zfn of the images with every zero-weight element set to 0, so masked content never reaches it) ->
        (u float32 (n,100), z = Z_IAF_fn(u) float32 (n,100), the l_Z that sample_at / grad / paint_stroke take), and with
        return_loss the per-sample objective / 12288 of the start and after every step, float32 (n, iters+1),
        non-increasing."""
        x, w, prior = self._map_args(images, weights, prior)
        n = x.shape[0]
        iters, u, loss = self._fit_start(iters, u0, 'u0', n,
                                          lambda: self.Zfn(x if w is None else np.where(w == 0, np.float32(0), x)))
        z = np.empty((n, 100), np.float32)
        if n:
            self._check(self._lib.ian_fit_latent_map_host(self._h, _fp(x), _fp(w) if w is not None else None, prior, n, _fp(u),
                                                          _fp(z), iters, _fp(loss)))
        return (u, z, loss) if return_loss else (u, z)

    def _robust_args(self, kind, scale, n):
        if scale is None:
            return _robust_kind(kind), None
        s = np.ascontiguousarray(np.broadcast_to(np.asarray(scale, np.float64), (n,)))
        if not np.all(s > 0) or (kind == "cauchy" and not np.all(np.isfinite(s))):
            raise ValueError("scale must be > 0 (and finite for the Cauchy loss), got %r" % (scale,))
        return _robust_kind(kind), s

    def gauss_newton_robust(self, u, images, kind="huber", scale=None, weights=None, prior=0.0):
        """The normal equations of the robust fit at each fit-space point u (as for gauss_newton_map): kind "huber" or
        "cauchy", scale None (automatic: from the lower median of |sample(u) - images| over the weighted pixels), a float for
        every sample or an (n,) array, > 0 (+inf allowed for Huber: the squared loss) -> (A (n,100,100), g (n,100), e (n,),
        scale (n,)) float64 with omega = w rho'(r^2), A = J_u^T Omega J_u + prior I, g = J_u^T Omega r + prior u and
        e = sum w rho(r^2) + prior |u|^2 (include/ian_b200.h, ian_robust_gauss_newton_*)."""
        u = _z(u, 'u')
        x, w, prior = self._map_args(images, weights, prior)
        n, A, g, e = self._normal_eqs(u, x)
        k, s = self._robust_args(kind, scale, n)
        so = np.empty((n,), np.float64)
        if n:
            self._check(self._lib.ian_robust_gauss_newton_host(self._h, _fp(u), _fp(x), _fp(w) if w is not None else None,
                                                               prior, k, _dp(s), n, _dp(A), _dp(g), _dp(e), _dp(so)))
        return A, g, e, so

    def fit_latent_robust(self, images, kind="huber", scale=None, weights=None, prior=0.0, u0=None, iters=10,
                          return_loss=False, return_outliers=False):
        """Fit the sampling-space latent to each image under a robust pixel loss: `iters` reweighted Levenberg-Marquardt
        steps on sum_p w_p rho((sample(u) - images)_p^2) + prior |u|^2, so pixels the generator cannot draw (occluders,
        captions, highlights) lose their pull without being masked.  kind "huber" (convex, for mild outliers) or "cauchy"
        (redescending, for gross ones); scale as for gauss_newton_robust, automatic at the start when None; weights, prior
        and u0 as for fit_latent_map -> (u, z = Z_IAF_fn(u) float32 (n,100), scale float64 (n,)), then with return_loss the
        per-sample objective / 12288 of the start and after every step, float32 (n, iters+1), non-increasing, and with
        return_outliers rho'(r^2) at the fit, float32 (n,3,64,64): near 1 where the latent explains the pixel, near 0 on
        outliers, 0 where the weight is 0."""
        x, w, prior = self._map_args(images, weights, prior)
        n = x.shape[0]
        k, s = self._robust_args(kind, scale, n)
        iters, u, loss = self._fit_start(iters, u0, 'u0', n,
                                          lambda: self.Zfn(x if w is None else np.where(w == 0, np.float32(0), x)))
        z = np.empty((n, 100), np.float32)
        so = np.empty((n,), np.float64)
        out = np.empty((n, 3, 64, 64), np.float32) if return_outliers else None
        if n:
            self._check(self._lib.ian_fit_latent_robust_host(
                self._h, _fp(x), _fp(w) if w is not None else None, prior, k, _dp(s), n, _fp(u), _fp(z), iters, _fp(loss),
                _dp(so), _fp(out) if out is not None else None))
        res = (u, z, so)
        if return_loss:
            res += (loss,)
        if return_outliers:
            res += (out,)
        return res

    # ---- the discriminator head l_discrim --------------------------------------------------------------------------------
    def discriminator_units(self):
        """U: 3 on IAN.py (softmax over real / reconstruction / generated, train_IAN.py:482-484), else 1 (sigmoid)"""
        return 3 if self.kind == _lib.IAN_MODEL_FULL else 1

    def load_discriminator(self, weights=None):
        """Load the discriminator head's four tensors (DISCRIMINATOR_KEYS) from weights_fname, or from a {name: ndarray}
        dict.  Every key is looked up and every shape checked before anything is uploaded, so a missing key (IanError naming
        it) or a wrong shape leaves the handle as it was: a head is never half-loaded."""
        if weights is None:
            weights = np.load(self.weights_fname, allow_pickle=False)
        have = set(weights.keys() if hasattr(weights, 'keys') else weights)
        shapes = {'minibatch_discrim.theta': (1024, 500, 5), 'minibatch_discrim.log_weight_scale': (500, 5),
                  'minibatch_discrim.b': (500,), 'discrimi.W': (1524, self.discriminator_units())}
        arrs = {}
        for name in DISCRIMINATOR_KEYS:
            if name not in have:
                raise _lib.IanError("discriminator parameter '%s' is missing" % name)
            arrs[name] = np.ascontiguousarray(np.asarray(weights[name], dtype=np.float32))
            if arrs[name].shape != shapes[name]:
                raise _lib.IanError("discriminator parameter '%s' must be %r, got %r" % (name, shapes[name], arrs[name].shape))
        for name, arr in arrs.items():
            shape = (C.c_int64 * arr.ndim)(*arr.shape)
            self._check(self._lib.ian_set_discriminator_param(self._h, name.encode(), _fp(arr), shape, arr.ndim))

    def discriminate(self, images, return_logits=False):
        """l_discrim under deterministic=True: images float32 (n,3,64,64) -> p (n,U) float32, sigmoid (U = 1) or softmax
        (U = 3) of the logits [pool(enc_conv4) | minibatch features] W; (p, logits) when return_logits.  The MinibatchLayer
        compares every image of the call with every other, so one image's result depends on the rest of the batch (the
        batch is the call's, whatever the library's chunk size); at n = 1 the minibatch features are exactly b."""
        x = _img(images)
        n, U = x.shape[0], self.discriminator_units()
        p, logits = np.empty((n, U), np.float32), np.empty((n, U), np.float32)
        if n:
            self._check(self._lib.ian_discriminate_host(self._h, _fp(x), n, _fp(logits), _fp(p)))
        return (p, logits) if return_logits else p

    def discriminate_vjp(self, images, dlogits):
        """Vector-Jacobian product of the discriminator's logits over the whole coupled batch: images float32 (n,3,64,64),
        dlogits (n,U) -> dx (n,3,64,64) = (d logits / d x)^T dlogits; a cotangent on one sample reaches every image.  The
        trunk's forward runs twice (2 forwards + 1 backward)."""
        x = _img(images)
        n = x.shape[0]
        d = _f32(dlogits, 2, 'dlogits')
        if d.shape != (n, self.discriminator_units()):
            raise ValueError("dlogits must be (%d,%d), got %r" % (n, self.discriminator_units(), d.shape))
        dx = np.empty((n, 3, 64, 64), np.float32)
        if n:
            self._check(self._lib.ian_discriminate_vjp_host(self._h, _fp(x), n, _fp(d), _fp(dx)))
        return dx

    def discriminate_train(self, images, return_logits=False, return_stats=False):
        """l_discrim in training mode (deterministic=False, as train_IAN.py:139-149 evaluates it): bnorm2..4 in the trunk
        normalise with the batch's mean and biased variance over (n, h, w), inv_std = 1/sqrt(var + 1e-4); the running
        statistics are neither used nor changed.  images float32 (n,3,64,64) -> p (n,U); with return_logits also the logits,
        with return_stats also stats float32 (2,1792): row 0 the batch means of bnorm2 | bnorm3 | bnorm4, row 1 their
        inv_std (for Lasagne's running-average update, alpha = 0.1, which is the caller's).  Returns p alone, or the tuple
        (p[, logits][, stats])."""
        x = _img(images)
        n, U = x.shape[0], self.discriminator_units()
        p, logits = np.empty((n, U), np.float32), np.empty((n, U), np.float32)
        stats = np.empty((2, 1792), np.float32)
        if n:
            self._check(self._lib.ian_discriminate_train_host(self._h, _fp(x), n, _fp(logits), _fp(p), _fp(stats)))
        else:
            stats.fill(np.nan)
        res = (p,) + ((logits,) if return_logits else ()) + ((stats,) if return_stats else ())
        return res if len(res) > 1 else p

    def discriminate_train_vjp(self, images, dlogits):
        """Vector-Jacobian product of discriminate_train()'s logits over the whole batch: dx (n,3,64,64) = (d logits / d x)^T
        dlogits, through the batch statistics as Theano's T.grad gives it.  1 trunk forward + 1 backward."""
        x = _img(images)
        n = x.shape[0]
        d = _f32(dlogits, 2, 'dlogits')
        if d.shape != (n, self.discriminator_units()):
            raise ValueError("dlogits must be (%d,%d), got %r" % (n, self.discriminator_units(), d.shape))
        dx = np.empty((n, 3, 64, 64), np.float32)
        if n:
            self._check(self._lib.ian_discriminate_train_vjp_host(self._h, _fp(x), n, _fp(d), _fp(dx)))
        return dx

    # ---- the introspection features and the fit under the feature-wise loss ------------------------------------------------
    def introspect(self, images):
        """The IAN's introspection features l_introspect (IAN_simple.py:240): images float32 (n,3,64,64) -> [f1 (n,128,32,32),
        f2 (n,256,16,16), f3 (n,512,8,8), f4 (n,1024,4,4)] float32, the outputs of enc_conv1..4 after BatchNorm (inference
        statistics, as in Z_hat_fn) and LeakyReLU -- what get_output(l_introspect, deterministic=True) returns.  One encoder
        forward stopped after enc_conv4."""
        x = _img(images)
        n = x.shape[0]
        f = [np.empty((n,) + s, np.float32) for s in FEATURE_SHAPES]
        if n:
            self._check(self._lib.ian_introspect_host(self._h, _fp(x), n, *[_fp(a) for a in f]))
        return f

    def introspect_jvp(self, images, v, return_features=False):
        """Jacobian-vector product of the introspection features along image tangents: images and v float32 (n,3,64,64) ->
        the tangents [t1..t4] in introspect()'s shapes, and introspect(images) bit for bit when return_features (returned as
        (features, tangents)).  encode_jvp's tangent chain stopped after enc_conv4, with its derivative conventions."""
        x = _img(images)
        t = _img(v, 'v')
        n = x.shape[0]
        if t.shape[0] != n:
            raise ValueError("v must be (%d,3,64,64), got %r" % (n, t.shape))
        f = [np.empty((n,) + s, np.float32) for s in FEATURE_SHAPES] if return_features else [None] * 4
        dt = [np.empty((n,) + s, np.float32) for s in FEATURE_SHAPES]
        if n:
            self._check(self._lib.ian_introspect_jvp_host(self._h, _fp(x), _fp(t), n,
                                                          *([_fp(a) if a is not None else None for a in f] + [_fp(a) for a in dt])))
        return (f, dt) if return_features else dt

    def introspect_vjp(self, images, cotangents):
        """Vector-Jacobian product of the introspection features: images float32 (n,3,64,64), cotangents = 4 arrays in
        introspect()'s shapes (each may be None, a zero cotangent) -> dx = sum_i (d g_i / d x)^T c_i float32 (n,3,64,64),
        the gradient w.r.t. the images of any loss on the features with dL/dg_i = c_i.  introspect_jvp's derivative
        conventions, so <c, introspect_jvp(x, v)> = <introspect_vjp(x, c), v>.  One encoder forward to the deepest supplied
        feature and one backward from it."""
        x = _img(images)
        n = x.shape[0]
        if len(cotangents) != 4:
            raise ValueError("cotangents must hold 4 arrays or None (got %d)" % len(cotangents))
        c = []
        for i, (a, s) in enumerate(zip(cotangents, FEATURE_SHAPES)):
            if a is not None:
                a = _f32(a, 4, "cotangents[%d]" % i)
                if a.shape != (n,) + s:
                    raise ValueError("cotangents[%d] must be %r, got %r" % (i, (n,) + s, a.shape))
            c.append(a)
        dx = np.empty((n, 3, 64, 64), np.float32)
        if n:
            self._check(self._lib.ian_introspect_vjp_host(self._h, _fp(x), n, *[_fp(a) if a is not None else None for a in c],
                                                          _fp(dx)))
        return dx

    def feature_loss(self, x_hat, images):
        """The per-sample feature-wise loss of train_IAN.py:244 under deterministic=True: x_hat, images float32 (n,3,64,64)
        -> (n,) float64 l_f = (1/4) sum_i mean((g_i(x_hat) - g_i(images))^2) over the four introspect() features."""
        a, b = self.introspect(x_hat), self.introspect(images)
        if a[0].shape[0] != b[0].shape[0]:
            raise ValueError("x_hat and images must hold the same number of images")
        n = a[0].shape[0]
        return sum(((p.astype(np.float64) - q).reshape(n, -1) ** 2).mean(1) for p, q in zip(a, b)) / 4

    @staticmethod
    def _feature_weights(pixel_weight, feature_weight):
        a, b = float(pixel_weight), float(feature_weight)
        for name, w in (("pixel_weight", a), ("feature_weight", b)):
            if not (np.isfinite(w) and w >= 0):
                raise ValueError("%s must be finite and >= 0 (got %r)" % (name, w))
        if a == 0 and b == 0:
            raise ValueError("pixel_weight and feature_weight must not both be 0")
        return a, b

    def gauss_newton_features(self, z, images, pixel_weight=1.0, feature_weight=1.0):
        """The Gauss-Newton normal equations of the pixel plus feature-wise objective at each latent: z float32 (n,100) (l_Z,
        as for sample_at), images float32 (n,3,64,64), a = pixel_weight, b = feature_weight (>= 0, not both 0) ->
        (A (n,100,100), g (n,100), e (n,)) float64 for E(z) = a |x_hat - x|^2 + 12288 b feature_loss(x_hat, x), x_hat =
        sample_at(z): A = a J^T J + sum_i c_i J_i^T J_i, g = a J^T r + sum_i c_i J_i^T r_i, e = E, with J_i the Jacobian of
        feature i at x_hat along the decoder and c_i = 3072 b / M_i.  a = 1, b = 0 is gauss_newton.  Costs one batch-100
        decode_jvp and one batch-100 introspect_jvp per sample."""
        z = _z(z)
        x = _img(images)
        a, b = self._feature_weights(pixel_weight, feature_weight)
        n, A, g, e = self._normal_eqs(z, x)
        if n:
            self._check(self._lib.ian_feature_gauss_newton_host(self._h, _fp(z), _fp(x), n, a, b, _dp(A), _dp(g), _dp(e)))
        return A, g, e

    def fit_latent_features(self, images, z0=None, iters=10, pixel_weight=1.0, feature_weight=1.0, return_loss=False):
        """Fit a latent to each image under the IAN's own reconstruction objective: `iters` Levenberg-Marquardt steps on
        pixel_weight * MSE + feature_weight * feature_loss (gauss_newton_features' E / 12288), every decision on the GPU.
        images float32 (n,3,64,64) in [-1,1]; z0 float32 (n,100) the start (default: encode_images(images)) -> z float32
        (n,100), and with return_loss that objective of the start and after every step, float32 (n, iters+1),
        non-increasing.  pixel_weight = 1, feature_weight = 0 is fit_latent."""
        x = _img(images)
        a, b = self._feature_weights(pixel_weight, feature_weight)
        n = x.shape[0]
        iters, z, loss = self._fit_start(iters, z0, 'z0', n, lambda: self.encode_images(x))
        if n:
            self._check(self._lib.ian_fit_latent_features_host(self._h, _fp(x), n, _fp(z), iters, a, b, _fp(loss)))
        return (z, loss) if return_loss else z

    def param_vjp_names(self):
        """names of the parameters decode_param_vjp returns gradients for, in ian_model_param_spec order: on IAN_simple
        the 13 tensors of train_IAN_simple.py:353 (`decoder_params`); empty on IAN.py / IANv1.py."""
        return [name for i, (name, _) in enumerate(model_param_specs(self.kind))
                if self._lib.ian_param_vjp_supported(self.kind, i)]

    def _param_slots(self, names):
        specs = model_param_specs(self.kind)
        index = {name: i for i, (name, _) in enumerate(specs)}
        for name in names:
            if name not in index:
                raise KeyError("%r is not a parameter of this graph" % (name,))
        return specs, index

    def decode_param_vjp(self, z, dx_hat):
        """Gradient of a pixel-space loss with respect to the decoder's trainable parameters (IAN_simple):
        z float32 (n,100), dx_hat float32 (n,3,64,64) = dL/dx_hat -> (dz (n,100), {name: dL/dparam}) with every name of
        param_vjp_names() in the reference layout.  dz equals decode_vjp(z, dx_hat) bit for bit.  The graph is X_hat_fn's
        (API.py:46): inference BatchNorm, mean / inv_std held constant."""
        z = _z(z)
        dx = _img(dx_hat, 'dx_hat')
        n = z.shape[0]
        if dx.shape[0] != n:
            raise ValueError("dx_hat must be (%d,3,64,64), got %r" % (n, dx.shape))
        names = self.param_vjp_names()
        specs, index = self._param_slots(names)
        grads = {name: np.zeros(specs[index[name]][1], np.float32) for name in names}
        dz = np.zeros_like(z)
        ptrs = (C.c_void_p * len(specs))()
        for name, g in grads.items():
            ptrs[index[name]] = g.ctypes.data
        self._check(self._lib.ian_decode_param_vjp_host(self._h, _fp(z), _fp(dx), n, _fp(dz), ptrs))
        return dz, grads

    def decode_train(self, z, return_stats=False):
        """The IAN_simple decoder in training mode (deterministic=False, as train_IAN_simple.py:217-224 builds X_hat):
        bnorm_dec_fc2 and bnorm_dc1..3 normalise with the batch's mean and biased variance, inv_std = 1/sqrt(var + 1e-4);
        the running statistics are neither used nor changed.  z float32 (n,100) -> x_hat (n,3,64,64); with return_stats
        also stats float32 (2,17280): row 0 the batch means of bnorm_dec_fc2 (reference feature order) | bnorm_dc1 |
        bnorm_dc2 | bnorm_dc3, row 1 their inv_std (for Lasagne's running-average update, alpha = 0.1, which is the
        caller's: update_params).  The batch is coupled: every sample's x_hat depends on every z of the call."""
        z = _z(z)
        n = z.shape[0]
        x = np.empty((n, 3, 64, 64), np.float32)
        stats = np.empty((2, 17280), np.float32)
        if n:
            self._check(self._lib.ian_decode_train_host(self._h, _fp(z), n, _fp(x), _fp(stats)))
        else:
            stats.fill(np.nan)
        return (x, stats) if return_stats else x

    def decode_train_vjp(self, z, dx_hat, grads=True):
        """Reverse mode through decode_train(): (dz (n,100), {name: dL/dparam}) for dx_hat = dL/dx_hat (n,3,64,64), the
        gradient flowing through the batch statistics as Theano's T.grad gives it.  grads: True (every name of
        param_vjp_names()), False (none) or an iterable of names; weight gradients run only for those.  1 forward + 1
        backward."""
        z = _z(z)
        dx = _img(dx_hat, 'dx_hat')
        n = z.shape[0]
        if dx.shape[0] != n:
            raise ValueError("dx_hat must be (%d,3,64,64), got %r" % (n, dx.shape))
        names = self.param_vjp_names() if grads is True else [] if grads is False else list(grads)
        specs, index = self._param_slots(names)
        out = {name: np.zeros(specs[index[name]][1], np.float32) for name in names}
        dz = np.zeros_like(z)
        ptrs = (C.c_void_p * len(specs))()
        for name, g in out.items():
            ptrs[index[name]] = g.ctypes.data
        self._check(self._lib.ian_decode_train_vjp_host(self._h, _fp(z), _fp(dx), n, _fp(dz), ptrs))
        return dz, out

    def update_params(self, params):
        """Replace IAN_simple decoder parameters of this finalized model in place: {name: array in the reference shape}
        for any of param_vjp_names() and bnorm_dec_fc2 / bnorm_dc1..3 .mean / .inv_std.  Afterwards every call computes
        what a model built from the updated weights computes, bit for bit; captured graphs stay valid."""
        for name, value in params.items():
            arr = np.ascontiguousarray(np.asarray(value, dtype=np.float32))
            shape = (C.c_int64 * max(arr.ndim, 1))(*arr.shape)
            self._check(self._lib.ian_update_param_host(self._h, str(name).encode(), _fp(arr), shape, arr.ndim))

    def encode_vjp(self, images, dz, eps=None):
        """Vector-Jacobian product of the encoder, dx = (d z / d x)^T . dz, for any loss on the latent: images as for
        encode() (n,3,64,64), dz float32 (n,100) = dL/dz, eps as for encode() -> dx float32 (n,3,64,64).  z is what
        encode(images, eps) returns (on IAN.py / IANv1.py after the MADE/IAF flow), so this is what T.grad of any loss on
        Z_hat w.r.t. the image gives in the reference (API.py:50).  No gradient w.r.t. eps.  Costs one encoder forward and
        one backward."""
        x = _img(images)
        n = x.shape[0]
        d = _z(dz, 'dz')
        if d.shape[0] != n:
            raise ValueError("dz must be (%d,100), got %r" % (n, d.shape))
        dx = np.empty((n, 3, 64, 64), np.float32)
        if n:
            e = None if eps is None else _z(eps, 'eps')
            if e is not None and e.shape[0] != n:
                raise ValueError("eps must be (%d,100), got %r" % (n, e.shape))
            self._check(self._lib.ian_encode_vjp_host(self._h, _fp(x), n, _fp(e) if e is not None else None, _fp(d), _fp(dx)))
        return dx

    def encode_jvp(self, images, v, eps=None, return_z=False):
        """Jacobian-vector product of the encoder, dz = (d z / d x) . v -- how the latent moves when the image moves along
        v: images and v float32 (n,3,64,64), eps as for encode() -> dz float32 (n,100), and z = encode(images, eps) bit for
        bit when return_z (returned as (z, dz)).  z is what encode() returns (on IAN.py / IANv1.py after the MADE/IAF
        flow); eps is a constant, with no tangent.  Forward mode: one encoder forward and one tangent pass.  Its derivative
        conventions are encode_vjp's, so <u, encode_jvp(x, v)> = <encode_vjp(x, u), v> up to float32 summation."""
        x = _img(images)
        t = _img(v, 'v')
        n = x.shape[0]
        if t.shape[0] != n:
            raise ValueError("v must be (%d,3,64,64), got %r" % (n, t.shape))
        dz = np.empty((n, 100), np.float32)
        z = np.empty((n, 100), np.float32) if return_z else None
        if n:
            e = None if eps is None else _z(eps, 'eps')
            if e is not None and e.shape[0] != n:
                raise ValueError("eps must be (%d,100), got %r" % (n, e.shape))
            self._check(self._lib.ian_encode_jvp_host(self._h, _fp(x), _fp(t), n, _fp(e) if e is not None else None,
                                                      _fp(z) if z is not None else None, _fp(dz)))
        return (z, dz) if return_z else dz

    def encoder_jacobian(self, images, eps=None):
        """The encoder's Jacobian at each image: images float32 (n,3,64,64), eps as for encode() -> J float32
        (n,100,3,64,64) with J[k, i] = d z_i / d x at x[k], z as encode() returns it (on IAN.py / IANv1.py after the MADE/IAF
        flow): J's 100 rows as images, the saliency map of every latent coordinate.  One batch-100 encode_vjp with the
        identity as cotangents per image."""
        x = _img(images)
        n = x.shape[0]
        e = None if eps is None else _z(eps, 'eps')
        if e is not None and e.shape[0] != n:
            raise ValueError("eps must be (%d,100), got %r" % (n, e.shape))
        J = np.empty((n, 100, 3, 64, 64), np.float32)
        eye = np.eye(100, dtype=np.float32)
        for k in range(n):
            xk = np.ascontiguousarray(np.broadcast_to(x[k], (100, 3, 64, 64)))
            ek = None if e is None else np.ascontiguousarray(np.broadcast_to(e[k], (100, 100)))
            self._check(self._lib.ian_encode_vjp_host(self._h, _fp(xk), 100, _fp(ek) if ek is not None else None, _fp(eye),
                                                      _fp(J[k])))
        return J

    # ---- derivatives in the prior space l_Z_IAF (the sampling script's Zfn / Z_IAF_fn / sample) ------------------------
    def encode_pre_vjp(self, images, dz_iaf):
        """Vector-Jacobian product of Zfn (X -> l_Z_IAF, deterministic), dx = (d z_iaf / d x)^T . dz_iaf: images
        (n,3,64,64), dz_iaf float32 (n,100) -> dx float32 (n,3,64,64).  encode_vjp(x, dz) equals
        encode_pre_vjp(x, flow_vjp(Zfn(x), dz)) bit for bit; on IAN_simple it is encode_vjp with eps absent."""
        x = _img(images)
        n = x.shape[0]
        d = _z(dz_iaf, 'dz_iaf')
        if d.shape[0] != n:
            raise ValueError("dz_iaf must be (%d,100), got %r" % (n, d.shape))
        dx = np.empty((n, 3, 64, 64), np.float32)
        if n:
            self._check(self._lib.ian_encode_pre_vjp_host(self._h, _fp(x), n, _fp(d), _fp(dx)))
        return dx

    def encode_pre_jvp(self, images, v, return_z=False):
        """Jacobian-vector product of Zfn, dz_iaf = (d z_iaf / d x) . v: images and v float32 (n,3,64,64) -> dz_iaf float32
        (n,100), and z_iaf = Zfn(images) bit for bit when return_z (returned as (z_iaf, dz_iaf)).  encode_jvp(x, v) equals
        flow_jvp(Zfn(x), encode_pre_jvp(x, v)) bit for bit."""
        x = _img(images)
        t = _img(v, 'v')
        n = x.shape[0]
        if t.shape[0] != n:
            raise ValueError("v must be (%d,3,64,64), got %r" % (n, t.shape))
        dz = np.empty((n, 100), np.float32)
        z = np.empty((n, 100), np.float32) if return_z else None
        if n:
            self._check(self._lib.ian_encode_pre_jvp_host(self._h, _fp(x), _fp(t), n, _fp(z) if z is not None else None,
                                                          _fp(dz)))
        return (z, dz) if return_z else dz

    def flow_vjp(self, z_iaf, dz):
        """Vector-Jacobian product of the MADE/IAF flow (Z_IAF_fn: l_Z_IAF -> l_Z), dz_iaf = (d z / d z_iaf)^T . dz: z_iaf,
        dz float32 (n,100) -> dz_iaf float32 (n,100).  The gradient in the prior space: for a loss on sample(z_iaf)'s image,
        flow_vjp(z_iaf, decode_vjp(Z_IAF_fn(z_iaf), dL/dx)).  dz itself on IAN_simple (no flow)."""
        z0 = _z(z_iaf, 'z_iaf')
        d = _z(dz, 'dz')
        n = z0.shape[0]
        if d.shape[0] != n:
            raise ValueError("dz must be (%d,100), got %r" % (n, d.shape))
        out = np.empty_like(z0)
        if n:
            self._check(self._lib.ian_flow_vjp_host(self._h, _fp(z0), _fp(d), n, _fp(out)))
        return out

    def flow_jvp(self, z_iaf, v, return_z=False):
        """Jacobian-vector product of the MADE/IAF flow, dz = (d z / d z_iaf) . v: z_iaf, v float32 (n,100) -> dz float32
        (n,100), and z = Z_IAF_fn(z_iaf) bit for bit when return_z (returned as (z, dz)).  How a prior sample's image moves
        along v: decode_jvp(Z_IAF_fn(z_iaf), flow_jvp(z_iaf, v)).  v itself on IAN_simple (no flow)."""
        z0 = _z(z_iaf, 'z_iaf')
        t = _z(v, 'v')
        n = z0.shape[0]
        if t.shape[0] != n:
            raise ValueError("v must be (%d,100), got %r" % (n, t.shape))
        dz = np.empty_like(z0)
        z = np.empty_like(z0) if return_z else None
        if n:
            self._check(self._lib.ian_flow_jvp_host(self._h, _fp(z0), _fp(t), n, _fp(z) if z is not None else None, _fp(dz)))
        return (z, dz) if return_z else dz

    def edit_steps(self, z, boxes, rgb=None, n_steps=32, weight=0.05):
        """n_steps of the NPE paint rule per sample: Z <- Z - weight*g*(1+(x2-x1)) (reference NPE.py:199-209)."""
        z = _z(z).copy()
        n = z.shape[0]
        boxes = np.ascontiguousarray(np.asarray(boxes, dtype=np.int32).reshape(n, 4))
        t, is_frame = self._target(rgb, n)
        self._check(self._lib.ian_edit_loop_host(self._h, _fp(z), boxes.ctypes.data_as(C.POINTER(C.c_int32)),
                                                 _fp(t) if t is not None else None, is_frame, n, int(n_steps),
                                                 float(weight)))
        return z

    def paint_stroke(self, z, box, rgb_frame, recon_u8, error, weight=0.05):
        """One NPE paint stroke in photo mode in a single library call (reference NPE.py:199-231): brush gradient,
        latent update, re-decode, DELTA/MASK(gaussian 0.7)/ERROR blend, uint8 conversion and the 4x display upsample.
        z (1,100) float32; box = (x1,y1,x2,y2) as NPE computes it (integral floats accepted); rgb_frame (1,3,64,64)
        float32 = to_tanh(myRGB); recon_u8 (3,64,64) uint8; error (3,64,64) float32.
        Returns (z_new (1,100), IM uint8 (3,64,64), display uint8 (256,256,3) ready for PIL.Image.fromarray)."""
        z = _f32(z, 2, 'z').copy()
        frame = _f32(rgb_frame, 4, 'RGB')
        if z.shape != (1, 100) or frame.shape != (1, 3, 64, 64):
            raise TypeError("paint_stroke takes z (1,100) and RGB (1,3,64,64)")
        bx = np.array([_int_scalar(v, n) for v, n in zip(box, ('x1', 'y1', 'x2', 'y2'))], np.int32)
        recon = np.ascontiguousarray(recon_u8)
        err = _f32(error, 3, 'error')
        if recon.dtype != np.uint8 or recon.shape != (3, 64, 64) or err.shape != (3, 64, 64):
            raise TypeError("recon_u8 must be uint8 (3,64,64) and error float32 (3,64,64)")
        im = np.empty((3, 64, 64), np.uint8)
        disp = np.empty((256, 256, 3), np.uint8)
        self._check(self._lib.ian_paint_stroke_host(self._h, _fp(z), bx.ctypes.data_as(C.POINTER(C.c_int32)), _fp(frame),
                                                    float(weight), recon.ctypes.data_as(C.c_void_p), _fp(err),
                                                    im.ctypes.data_as(C.c_void_p), disp.ctypes.data_as(C.c_void_p)))
        return z, im, disp

    # ---- multi-GPU: all-gather fused into the decoder's last kernel (peer stores over NVLink) ---------------------
    def setup_fused_gather(self, n_local, group=None):
        """Collective over `group` (torch.distributed, one process per GPU): allocate the gather buffers, exchange
        their CUDA IPC handles and map the peers.  Afterwards reconstruct_gather_dev() decodes straight into every
        rank's buffer."""
        import torch
        import torch.distributed as dist
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        mine = (C.c_ubyte * 64)()
        self._check(self._lib.ian_gather_create(self._h, world, rank, int(n_local), C.cast(mine, C.c_void_p)))
        dev = torch.device("cuda", torch.cuda.current_device())
        local = torch.tensor(list(bytes(mine)), dtype=torch.uint8, device=dev)
        allh = torch.empty(world * 64, dtype=torch.uint8, device=dev)
        dist.all_gather_into_tensor(allh, local, group=group)
        blob = bytes(allh.cpu().tolist())
        self._check(self._lib.ian_gather_connect(self._h, C.cast(C.create_string_buffer(blob, len(blob)), C.c_void_p)))
        self._gather_world, self._gather_n = world, int(n_local)

    def reconstruct_gather_dev(self, x_ptr, n_local, z_ptr=0, stream=0):
        """encode -> decode of this rank's shard; returns the device pointer of the (world*n_local,3,64,64) float32
        buffer that holds EVERY rank's decoded images once the stream work (incl. the peer barrier) has run."""
        out = C.c_void_p()
        self._check(self._lib.ian_reconstruct_gather_dev(self._h, x_ptr, int(n_local), z_ptr or None, C.byref(out),
                                                         stream or None))
        return out.value

    def reconstruct_gather_async_dev(self, x_ptr, n_local, z_ptr=0, stream=0):
        """pipelined form: enqueue this rank's shard; a side stream pushes it to the peers (copy engines + stream memory
        operations; IAN_PUSH=kernel: a copy kernel) while the next call computes.  gather_wait_dev() returns the complete buffer of the most recent step."""
        self._check(self._lib.ian_reconstruct_gather_async_dev(self._h, x_ptr, int(n_local), z_ptr or None, stream or None))

    def gather_wait_dev(self, stream=0):
        out = C.c_void_p()
        self._check(self._lib.ian_gather_wait_dev(self._h, C.byref(out), stream or None))
        return out.value

    def reconstruct_sharded(self, x, group=None, stream=0, pipelined=False):
        """Data-parallel encode -> decode of a FULL batch held by every rank (torch CUDA tensor (N,3,64,64) float32, N
        divisible by the world size): this rank computes shard `parallel.shard_bounds(N, rank, world)` and the decoded
        shards are all-gathered by the library (peer stores over NVLink).  Returns a torch tensor VIEW (N,3,64,64) of
        the library's gather buffer (valid until the next call's stream work; see include/ian_b200.h)."""
        import torch
        import torch.distributed as dist
        from . import parallel
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        n = int(x.shape[0])
        lo, hi = parallel.shard_bounds(n, rank, world)
        if n % world:
            raise ValueError("reconstruct_sharded needs a batch divisible by the world size (got %d over %d ranks); "
                             "parallel.sharded_reconstruct handles ragged shards with a separate all_gather" % (n, world))
        if getattr(self, '_gather_n', None) != hi - lo or getattr(self, '_gather_world', None) != world:
            if getattr(self, '_gather_n', None) is not None:
                raise _lib.IanError("gather buffers were sized for %d images per rank" % self._gather_n)
            self.setup_fused_gather(hi - lo, group)
        shard = x[lo:hi]
        if pipelined:
            self.reconstruct_gather_async_dev(shard.data_ptr(), hi - lo, 0, stream)
            ptr = self.gather_wait_dev(stream)
        else:
            ptr = self.reconstruct_gather_dev(shard.data_ptr(), hi - lo, 0, stream)
        return parallel.as_cuda_tensor(ptr, (n, 3, 64, 64), x.device)

    # ---- device-pointer variants (ints from torch.Tensor.data_ptr(); no host copies, async) ----------
    def reconstruct_dev(self, x_ptr, n, z_ptr, xhat_ptr, stream=0):
        self._check(self._lib.ian_reconstruct_dev(self._h, x_ptr, n, z_ptr or None, xhat_ptr, stream or None))

    def encode_dev(self, x_ptr, n, z_ptr, eps_ptr=0, stream=0):
        self._check(self._lib.ian_encode_dev(self._h, x_ptr, n, eps_ptr or None, z_ptr, stream or None))

    def decode_dev(self, z_ptr, n, x_ptr, stream=0):
        self._check(self._lib.ian_decode_dev(self._h, z_ptr, n, x_ptr, stream or None))

    def grad_dev(self, z_ptr, boxes_ptr, target_ptr, target_is_frame, n, g_ptr, stream=0):
        self._check(self._lib.ian_grad_dev(self._h, z_ptr, boxes_ptr, target_ptr or None, int(target_is_frame), n,
                                           g_ptr, stream or None))

    def decode_vjp_dev(self, z_ptr, dx_ptr, n, dz_ptr, stream=0):
        self._check(self._lib.ian_decode_vjp_dev(self._h, z_ptr, dx_ptr, int(n), dz_ptr, stream or None))

    def decode_jvp_dev(self, z_ptr, v_ptr, n, dx_ptr, xhat_ptr=0, stream=0):
        """device-pointer form of decode_jvp; xhat_ptr may be 0"""
        self._check(self._lib.ian_decode_jvp_dev(self._h, z_ptr, v_ptr, int(n), xhat_ptr or None, dx_ptr, stream or None))

    def decode_param_vjp_dev(self, z_ptr, dx_ptr, n, dz_ptr, grad_ptrs, stream=0):
        """device-pointer form of decode_param_vjp: grad_ptrs {name: device pointer} (any subset of param_vjp_names()),
        dz_ptr may be 0."""
        specs, index = self._param_slots(grad_ptrs)
        ptrs = (C.c_void_p * len(specs))()
        for name, p in grad_ptrs.items():
            ptrs[index[name]] = p
        self._check(self._lib.ian_decode_param_vjp_dev(self._h, z_ptr, dx_ptr, int(n), dz_ptr or None, ptrs, stream or None))

    def decode_train_dev(self, z_ptr, n, x_ptr, stats_ptr=0, stream=0):
        """decode_train() on device pointers: x_hat (n,3,64,64) and stats (2,17280) float32 (0: not wanted)"""
        self._check(self._lib.ian_decode_train_dev(self._h, z_ptr, int(n), x_ptr, stats_ptr or None, stream or None))

    def decode_train_vjp_dev(self, z_ptr, dx_ptr, n, dz_ptr, grad_ptrs, stream=0):
        """decode_train_vjp() on device pointers: grad_ptrs {name: device pointer} (any subset of param_vjp_names()),
        dz_ptr may be 0."""
        specs, index = self._param_slots(grad_ptrs)
        ptrs = (C.c_void_p * len(specs))()
        for name, p in grad_ptrs.items():
            ptrs[index[name]] = p
        self._check(self._lib.ian_decode_train_vjp_dev(self._h, z_ptr, dx_ptr, int(n), dz_ptr or None, ptrs, stream or None))

    def encode_vjp_dev(self, x_ptr, dz_ptr, n, dx_ptr, eps_ptr=0, stream=0):
        self._check(self._lib.ian_encode_vjp_dev(self._h, x_ptr, int(n), eps_ptr or None, dz_ptr, dx_ptr, stream or None))

    def encode_jvp_dev(self, x_ptr, v_ptr, n, dz_ptr, z_ptr=0, eps_ptr=0, stream=0):
        """device-pointer form of encode_jvp; z_ptr and eps_ptr may be 0"""
        self._check(self._lib.ian_encode_jvp_dev(self._h, x_ptr, v_ptr, int(n), eps_ptr or None, z_ptr or None, dz_ptr,
                                                 stream or None))

    def Zfn_dev(self, x_ptr, n, z_iaf_ptr, stream=0):
        """device-pointer form of Zfn"""
        self._check(self._lib.ian_encode_pre_dev(self._h, x_ptr, int(n), z_iaf_ptr, stream or None))

    def flow_dev(self, z_iaf_ptr, n, z_ptr=0, x_ptr=0, stream=0):
        """device-pointer form of Z_IAF_fn (z_ptr) and sample (x_ptr); either may be 0, not both"""
        self._check(self._lib.ian_flow_dev(self._h, z_iaf_ptr, int(n), z_ptr or None, x_ptr or None, stream or None))

    def flow_vjp_dev(self, z_iaf_ptr, dz_ptr, n, dz_iaf_ptr, stream=0):
        self._check(self._lib.ian_flow_vjp_dev(self._h, z_iaf_ptr, dz_ptr, int(n), dz_iaf_ptr, stream or None))

    def flow_jvp_dev(self, z_iaf_ptr, v_ptr, n, dz_ptr, z_ptr=0, stream=0):
        """device-pointer form of flow_jvp; z_ptr may be 0"""
        self._check(self._lib.ian_flow_jvp_dev(self._h, z_iaf_ptr, v_ptr, int(n), z_ptr or None, dz_ptr, stream or None))

    def encode_pre_vjp_dev(self, x_ptr, dz_iaf_ptr, n, dx_ptr, stream=0):
        self._check(self._lib.ian_encode_pre_vjp_dev(self._h, x_ptr, int(n), dz_iaf_ptr, dx_ptr, stream or None))

    def encode_pre_jvp_dev(self, x_ptr, v_ptr, n, dz_iaf_ptr, z_iaf_ptr=0, stream=0):
        """device-pointer form of encode_pre_jvp; z_iaf_ptr may be 0"""
        self._check(self._lib.ian_encode_pre_jvp_dev(self._h, x_ptr, v_ptr, int(n), z_iaf_ptr or None, dz_iaf_ptr,
                                                     stream or None))

    def gauss_newton_dev(self, z_ptr, x_ptr, n, A_ptr, g_ptr, e_ptr=0, stream=0):
        """device-pointer form of gauss_newton: A (n,100,100), g (n,100), e (n) float64; e_ptr may be 0"""
        self._check(self._lib.ian_decode_gauss_newton_dev(self._h, z_ptr, x_ptr, int(n), A_ptr, g_ptr, e_ptr or None,
                                                          stream or None))

    def fit_latent_dev(self, x_ptr, n, z_ptr, iters, loss_ptr=0, stream=0):
        """device-pointer form of fit_latent: z (n,100) in place (in: the start), loss (n, iters+1) float32; loss_ptr may be 0"""
        self._check(self._lib.ian_fit_latent_dev(self._h, x_ptr, int(n), z_ptr, int(iters), loss_ptr or None, stream or None))

    def gauss_newton_map_dev(self, u_ptr, x_ptr, w_ptr, prior, n, A_ptr, g_ptr, e_ptr=0, stream=0):
        """device-pointer form of gauss_newton_map: A (n,100,100), g (n,100), e (n) float64; w_ptr and e_ptr may be 0"""
        self._check(self._lib.ian_map_gauss_newton_dev(self._h, u_ptr, x_ptr, w_ptr or None, float(prior), int(n), A_ptr, g_ptr,
                                                       e_ptr or None, stream or None))

    def fit_latent_map_dev(self, x_ptr, w_ptr, prior, n, u_ptr, iters, z_ptr=0, loss_ptr=0, stream=0):
        """device-pointer form of fit_latent_map: u (n,100) in place (in: the start), z (n,100) = F(u), loss (n, iters+1)
        float32; w_ptr, z_ptr and loss_ptr may be 0"""
        self._check(self._lib.ian_fit_latent_map_dev(self._h, x_ptr, w_ptr or None, float(prior), int(n), u_ptr, z_ptr or None,
                                                     int(iters), loss_ptr or None, stream or None))

    def gauss_newton_robust_dev(self, u_ptr, x_ptr, w_ptr, prior, kind, scale_ptr, n, A_ptr, g_ptr, e_ptr=0, scale_out_ptr=0,
                                stream=0):
        """device-pointer form of gauss_newton_robust: kind "huber" / "cauchy", scale (n) float64 or 0 (automatic), A
        (n,100,100), g (n,100), e (n), scale_out (n) float64; w_ptr, e_ptr and scale_out_ptr may be 0"""
        self._check(self._lib.ian_robust_gauss_newton_dev(self._h, u_ptr, x_ptr, w_ptr or None, float(prior), _robust_kind(kind),
                                                          scale_ptr or None, int(n), A_ptr, g_ptr, e_ptr or None,
                                                          scale_out_ptr or None, stream or None))

    def fit_latent_robust_dev(self, x_ptr, w_ptr, prior, kind, scale_ptr, n, u_ptr, iters, z_ptr=0, loss_ptr=0,
                              scale_out_ptr=0, outliers_ptr=0, stream=0):
        """device-pointer form of fit_latent_robust: u (n,100) in place (in: the start), z (n,100) = F(u), loss (n, iters+1)
        float32, scale_out (n) float64, outliers (n,3,64,64) float32; every pointer but x_ptr and u_ptr may be 0"""
        self._check(self._lib.ian_fit_latent_robust_dev(self._h, x_ptr, w_ptr or None, float(prior), _robust_kind(kind),
                                                        scale_ptr or None, int(n), u_ptr, z_ptr or None, int(iters),
                                                        loss_ptr or None, scale_out_ptr or None, outliers_ptr or None,
                                                        stream or None))

    def introspect_dev(self, x_ptr, n, f_ptrs, stream=0):
        """introspect() on device pointers: f_ptrs = 4 pointers (0: not wanted) to float32 outputs in FEATURE_SHAPES"""
        self._check(self._lib.ian_introspect_dev(self._h, x_ptr, int(n), *[p or None for p in f_ptrs], stream or None))

    def introspect_jvp_dev(self, x_ptr, v_ptr, n, t_ptrs, f_ptrs=(0, 0, 0, 0), stream=0):
        """introspect_jvp() on device pointers: t_ptrs = the 4 tangent outputs, f_ptrs the features (0: not wanted)"""
        self._check(self._lib.ian_introspect_jvp_dev(self._h, x_ptr, v_ptr, int(n), *([p or None for p in f_ptrs] + list(t_ptrs)),
                                                     stream or None))

    def introspect_vjp_dev(self, x_ptr, n, c_ptrs, dx_ptr, stream=0):
        """introspect_vjp() on device pointers: c_ptrs = 4 pointers to float32 cotangents in FEATURE_SHAPES (0: zero)"""
        self._check(self._lib.ian_introspect_vjp_dev(self._h, x_ptr, int(n), *[p or None for p in c_ptrs], dx_ptr, stream or None))

    def discriminate_dev(self, x_ptr, n, logits_ptr, p_ptr=0, stream=0):
        """discriminate() on device pointers: logits (n,U) float32, p (n,U) float32 (0: not wanted)"""
        self._check(self._lib.ian_discriminate_dev(self._h, x_ptr, int(n), logits_ptr, p_ptr or None, stream or None))

    def discriminate_vjp_dev(self, x_ptr, dlogits_ptr, n, dx_ptr, stream=0):
        """discriminate_vjp() on device pointers"""
        self._check(self._lib.ian_discriminate_vjp_dev(self._h, x_ptr, int(n), dlogits_ptr, dx_ptr, stream or None))

    def discriminate_train_dev(self, x_ptr, n, logits_ptr, p_ptr=0, stats_ptr=0, stream=0):
        """discriminate_train() on device pointers: logits (n,U), p (n,U) and stats (2,1792) float32 (0: not wanted)"""
        self._check(self._lib.ian_discriminate_train_dev(self._h, x_ptr, int(n), logits_ptr, p_ptr or None, stats_ptr or None,
                                                         stream or None))

    def discriminate_train_vjp_dev(self, x_ptr, dlogits_ptr, n, dx_ptr, stream=0):
        """discriminate_train_vjp() on device pointers"""
        self._check(self._lib.ian_discriminate_train_vjp_dev(self._h, x_ptr, int(n), dlogits_ptr, dx_ptr, stream or None))

    def gauss_newton_features_dev(self, z_ptr, x_ptr, n, A_ptr, g_ptr, e_ptr=0, pixel_weight=1.0, feature_weight=1.0, stream=0):
        """gauss_newton_features() on device pointers: A (n,100,100), g (n,100), e (n,) float64 (e optional)"""
        self._check(self._lib.ian_feature_gauss_newton_dev(self._h, z_ptr, x_ptr, int(n), float(pixel_weight), float(feature_weight),
                                                           A_ptr, g_ptr, e_ptr or None, stream or None))

    def fit_latent_features_dev(self, x_ptr, n, z_ptr, iters, loss_ptr=0, pixel_weight=1.0, feature_weight=1.0, stream=0):
        """fit_latent_features() on device pointers, in place on z (n,100); loss (n, iters+1) float32 optional"""
        self._check(self._lib.ian_fit_latent_features_dev(self._h, x_ptr, int(n), z_ptr, int(iters), float(pixel_weight),
                                                          float(feature_weight), loss_ptr or None, stream or None))

    def edit_loop_dev(self, z_ptr, boxes_ptr, target_ptr, target_is_frame, n, n_steps, weight, stream=0):
        self._check(self._lib.ian_edit_loop_dev(self._h, z_ptr, boxes_ptr, target_ptr or None, int(target_is_frame),
                                                n, int(n_steps), float(weight), stream or None))

"""torch autograd binding of the IAN decoder and encoder, through the C-ABI of libian_b200.so (include/ian_b200.h):

  * decode(model, z) = X_hat of the reference (API.py:46, sample_at) as a differentiable torch op.  Its backward is the
    decoder's vector-Jacobian product (ian_decode_vjp_dev), so any loss torch can write on the decoded images -- soft or
    per-pixel weighted brushes, L1, losses on the whole frame, refining a latent against a photo -- drives the latent
    through torch.autograd, as any loss on X_hat was one T.grad away in the reference.  Its jvp is the decoder's
    Jacobian-vector product (ian_decode_jvp_dev), so torch.autograd.forward_ad's make_dual / unpack_dual work through it.
  * encode(model, x, eps=None) = Z_hat of the reference (API.py:50) -- on IAN.py / IANv1.py after the MADE/IAF flow -- as a
    differentiable torch op.  Its backward is the encoder's vector-Jacobian product (ian_encode_vjp_dev): latent-consistency
    losses such as |E(G(z)) - z| or |E(x_hat) - E(x)|, saliency of a latent coordinate, optimising a photo against the
    encoder, and a differentiable decode(encode(x)).  Its jvp is the encoder's Jacobian-vector product (ian_encode_jvp_dev),
    so forward mode works through encode and through decode(encode(x)).  eps is a constant input: it gets no gradient or
    tangent, and an eps that requires grad or carries a tangent is refused.
  * encode_pre(model, x) = Zfn and flow(model, z_iaf) = Z_IAF_fn of the reference's sampling script (sample_IAN.py:91-94):
    the encoder split at l_Z_IAF, the input of the MADE/IAF flow where the generative prior lives.  Both are differentiable
    in reverse and forward mode, so decode(model, flow(model, z_iaf)) -- the script's `sample` -- optimises in prior space,
    and flow(model, encode_pre(model, x)) is encode(model, x) with eps absent.

  * introspect(model, x) = the IAN's introspection features l_introspect = [enc_conv1..4] (IAN_simple.py:240, what
    model.introspect returns) as a differentiable torch op.  Its backward is the features' vector-Jacobian product
    (ian_introspect_vjp_dev, one call for all four features; an unused feature costs nothing and the chain starts at the
    deepest one used), its jvp ian_introspect_jvp_dev.  feature_loss(model, x_hat, x) is the per-sample feature-wise loss
    of train_IAN.py:244 built on it, so feature_loss(model, decode(model, z), x).sum().backward() drives z -- or, with
    params, the IAN_simple decoder's parameters -- under the generator's own reconstruction objective.

  * discriminate(model, x, training=False) = the logits of the IAN's discriminator head l_discrim (what model.discriminate(x,
    return_logits=True) returns) as a differentiable torch op; F.logsigmoid / log_softmax of them is the realism score.  Its
    backward is one ian_discriminate_vjp_dev call over the whole batch: the MinibatchLayer couples the samples, so a
    loss on one sample's logits moves every image of the call.  Reverse mode only.  training=True evaluates it as the
    reference's trainers do (batch-statistics BatchNorm in the trunk), for the generator's adversarial term.

  * decoder_parameters(model, weights) + decode(model, z, params): the IAN_simple decoder's 13 trainable tensors
    (train_IAN_simple.py:353, `decoder_params`) as leaf CUDA tensors, differentiable through one parameter VJP
    (ian_decode_param_vjp_dev) that also returns dz.  Before each forward, every tensor whose in-place version moved since
    its last upload is written back into the handle (ian_update_param_host), so a plain torch.optim loop over
    params.values() fine-tunes the generator with no extra call.  decode(model, z, params, training=True) is the decoder
    as the reference's trainers run it (batch-statistics BatchNorm: ian_decode_train_dev forward, one
    ian_decode_train_vjp_dev backward), so that loop trains the reference's function.

A backward costs one forward plus one backward of that half of the model: the library recomputes the forward from the
saved input instead of keeping the activations of the forward call.  The op is once-differentiable (no double backward).  Inputs and outputs are
torch CUDA float32 tensors on the model's device; torch only carries the device memory and the stream.
"""
from __future__ import annotations

from .train_ops import _lib_stream

_Decode = None
_Encode = None
_DecodeParams = None
_Introspect = None
_Discriminate = None


def _check_tensor(model, t, what):
    import torch
    if not (t.is_cuda and t.dtype == torch.float32):
        raise TypeError("%s must be a float32 CUDA tensor (got %s on %s)" % (what, t.dtype, t.device))
    if t.device.index != model.device:
        raise ValueError("%s is on %s but the model's handle is bound to cuda:%d" % (what, t.device, model.device))


def _function():
    global _Decode
    if _Decode is not None:
        return _Decode
    import torch
    from torch.autograd.function import once_differentiable

    class Decode(torch.autograd.Function):
        @staticmethod
        def forward(ctx, model, z):
            _check_tensor(model, z, "z")
            if z.dim() != 2 or z.shape[1] != 100:
                raise ValueError("z must be (n,100), got %r" % (tuple(z.shape),))
            z = z.contiguous()
            n = int(z.shape[0])
            x = torch.empty(n, 3, 64, 64, dtype=torch.float32, device=z.device)
            if n:
                with _lib_stream(model, z) as st:
                    model.decode_dev(z.data_ptr(), n, x.data_ptr(), st)
            ctx.model = model
            ctx.save_for_backward(z)
            ctx.save_for_forward(z)
            return x

        @staticmethod
        @once_differentiable
        def backward(ctx, g):
            (z,) = ctx.saved_tensors
            model = ctx.model
            _check_tensor(model, g, "grad_output")
            g = g.contiguous()
            n = int(z.shape[0])
            dz = torch.empty_like(z)
            if n:
                with _lib_stream(model, z) as st:
                    model.decode_vjp_dev(z.data_ptr(), g.data_ptr(), n, dz.data_ptr(), st)
            return None, dz

        @staticmethod
        def jvp(ctx, _model_t, v):
            (z,) = ctx.saved_tensors
            model = ctx.model
            _check_tensor(model, v, "tangent")
            v = v.contiguous()
            n = int(z.shape[0])
            dx = torch.empty(n, 3, 64, 64, dtype=torch.float32, device=z.device)
            if n:
                with _lib_stream(model, z) as st:
                    model.decode_jvp_dev(z.data_ptr(), v.data_ptr(), n, dx.data_ptr(), 0, st)
            return dx

    _Decode = Decode
    return Decode


def _encode_function():
    global _Encode
    if _Encode is not None:
        return _Encode
    import torch
    from torch.autograd.function import once_differentiable

    class Encode(torch.autograd.Function):
        @staticmethod
        def forward(ctx, model, x, eps):
            _check_tensor(model, x, "x")
            if x.dim() != 4 or tuple(x.shape[1:]) != (3, 64, 64):
                raise ValueError("x must be (n,3,64,64), got %r" % (tuple(x.shape),))
            x = x.contiguous()
            n = int(x.shape[0])
            if eps is not None:
                _check_tensor(model, eps, "eps")
                if tuple(eps.shape) != (n, 100):
                    raise ValueError("eps must be (%d,100), got %r" % (n, tuple(eps.shape)))
                eps = eps.contiguous()
            z = torch.empty(n, 100, dtype=torch.float32, device=x.device)
            if n:
                with _lib_stream(model, x) as st:
                    model.encode_dev(x.data_ptr(), n, z.data_ptr(), eps.data_ptr() if eps is not None else 0, st)
            ctx.model = model
            ctx.has_eps = eps is not None
            saved = (x, eps if eps is not None else x.new_empty(0))
            ctx.save_for_backward(*saved)
            ctx.save_for_forward(*saved)
            return z

        @staticmethod
        @once_differentiable
        def backward(ctx, g):
            x, eps = ctx.saved_tensors
            model = ctx.model
            _check_tensor(model, g, "grad_output")
            g = g.contiguous()
            n = int(x.shape[0])
            dx = torch.empty_like(x)
            if n:
                with _lib_stream(model, x) as st:
                    model.encode_vjp_dev(x.data_ptr(), g.data_ptr(), n, dx.data_ptr(),
                                         eps.data_ptr() if ctx.has_eps else 0, st)
            return None, dx, None

        @staticmethod
        def jvp(ctx, _model_t, v, _eps_t):
            x, eps = ctx.saved_tensors
            model = ctx.model
            n = int(x.shape[0])
            dz = torch.zeros(n, 100, dtype=torch.float32, device=x.device)
            if v is None:
                return dz
            _check_tensor(model, v, "tangent")
            v = v.contiguous()
            if n:
                with _lib_stream(model, x) as st:
                    model.encode_jvp_dev(x.data_ptr(), v.data_ptr(), n, dz.data_ptr(), 0,
                                         eps.data_ptr() if ctx.has_eps else 0, st)
            return dz

    _Encode = Encode
    return Encode


def encode(model, x, eps=None):
    """z = encoder(x) (what model.encode returns) for x (n,3,64,64) float32 CUDA on the model's device, eps (n,100) or None;
    differentiable w.r.t. x (one encoder forward + one backward per backward call).  It also supports forward mode: under
    torch.autograd.forward_ad a dual x (make_dual(x, v)) gives z with the tangent (d z / d x) . v, from one
    ian_encode_jvp_dev call, so forward mode runs through decode(encode(x)) too.  eps is not differentiated: pass a
    tensor that neither requires grad nor carries a forward-mode tangent."""
    if eps is not None and getattr(eps, "requires_grad", False):
        raise ValueError("torch_ops.encode does not differentiate w.r.t. eps; pass eps.detach() (eps.requires_grad is set)")
    if eps is not None:
        import torch.autograd.forward_ad as fwAD
        if fwAD.unpack_dual(eps).tangent is not None:
            raise ValueError("torch_ops.encode does not differentiate w.r.t. eps; pass its primal (eps carries a forward-mode "
                             "tangent)")
    return _encode_function().apply(model, x, eps)


_Prior = {}


def _prior_function(kind):
    """the Function of encode_pre (x (n,3,64,64) -> z_iaf) or flow (z_iaf -> z): forward, backward and jvp are one library
    call each"""
    if kind in _Prior:
        return _Prior[kind]
    import torch
    from torch.autograd.function import once_differentiable
    pre = kind == "encode_pre"
    in_shape, what = ((3, 64, 64), "x") if pre else ((100,), "z_iaf")

    class Prior(torch.autograd.Function):
        @staticmethod
        def forward(ctx, model, a):
            _check_tensor(model, a, what)
            if tuple(a.shape[1:]) != in_shape or a.dim() != 1 + len(in_shape):
                raise ValueError("%s must be (n,%s), got %r" % (what, ",".join(map(str, in_shape)), tuple(a.shape)))
            a = a.contiguous()
            n = int(a.shape[0])
            z = torch.empty(n, 100, dtype=torch.float32, device=a.device)
            if n:
                with _lib_stream(model, a) as st:
                    if pre:
                        model.Zfn_dev(a.data_ptr(), n, z.data_ptr(), st)
                    else:
                        model.flow_dev(a.data_ptr(), n, z.data_ptr(), 0, st)
            ctx.model = model
            ctx.save_for_backward(a)
            ctx.save_for_forward(a)
            return z

        @staticmethod
        @once_differentiable
        def backward(ctx, g):
            (a,) = ctx.saved_tensors
            model = ctx.model
            _check_tensor(model, g, "grad_output")
            g = g.contiguous()
            n = int(a.shape[0])
            da = torch.empty_like(a)
            if n:
                with _lib_stream(model, a) as st:
                    if pre:
                        model.encode_pre_vjp_dev(a.data_ptr(), g.data_ptr(), n, da.data_ptr(), st)
                    else:
                        model.flow_vjp_dev(a.data_ptr(), g.data_ptr(), n, da.data_ptr(), st)
            return None, da

        @staticmethod
        def jvp(ctx, _model_t, v):
            (a,) = ctx.saved_tensors
            model = ctx.model
            _check_tensor(model, v, "tangent")
            v = v.contiguous()
            n = int(a.shape[0])
            dz = torch.empty(n, 100, dtype=torch.float32, device=a.device)
            if n:
                with _lib_stream(model, a) as st:
                    if pre:
                        model.encode_pre_jvp_dev(a.data_ptr(), v.data_ptr(), n, dz.data_ptr(), 0, st)
                    else:
                        model.flow_jvp_dev(a.data_ptr(), v.data_ptr(), n, dz.data_ptr(), 0, st)
            return dz

    _Prior[kind] = Prior
    return Prior


def encode_pre(model, x):
    """z_iaf = Zfn(x) (model.Zfn: X -> l_Z_IAF, deterministic, before the MADE/IAF flow; encode itself on IAN_simple) for x
    (n,3,64,64) float32 CUDA on the model's device.  Differentiable w.r.t. x in reverse mode (one ian_encode_pre_vjp_dev call
    per backward) and forward mode (one ian_encode_pre_jvp_dev call).  flow(model, encode_pre(model, x)) is encode(model, x)
    with eps absent, in both modes."""
    return _prior_function("encode_pre").apply(model, x)


def flow(model, z_iaf):
    """z = Z_IAF_fn(z_iaf) (model.Z_IAF_fn: the MADE/IAF flow l_Z_IAF -> l_Z; the identity on IAN_simple) for z_iaf (n,100)
    float32 CUDA on the model's device.  Differentiable in reverse mode (one ian_flow_vjp_dev call per backward) and forward
    mode (one ian_flow_jvp_dev call).  decode(model, flow(model, z_iaf)) is the sampling script's `sample` (sample_IAN.py:86),
    so losses on a prior sample's image -- fitting z_iaf to a photo, a brush loss plus a |z_iaf|^2 prior term -- drive z_iaf
    through torch.autograd."""
    return _prior_function("flow").apply(model, z_iaf)


def _introspect_function():
    global _Introspect
    if _Introspect is not None:
        return _Introspect
    import torch
    from torch.autograd.function import once_differentiable
    from .API import FEATURE_SHAPES

    class Introspect(torch.autograd.Function):
        @staticmethod
        def forward(ctx, model, x):
            _check_tensor(model, x, "x")
            if x.dim() != 4 or tuple(x.shape[1:]) != (3, 64, 64):
                raise ValueError("x must be (n,3,64,64), got %r" % (tuple(x.shape),))
            x = x.contiguous()
            n = int(x.shape[0])
            f = [torch.empty((n,) + s, dtype=torch.float32, device=x.device) for s in FEATURE_SHAPES]
            if n:
                with _lib_stream(model, x) as st:
                    model.introspect_dev(x.data_ptr(), n, [a.data_ptr() for a in f], st)
            ctx.model = model
            ctx.set_materialize_grads(False)              # an unused feature reaches backward as None: a NULL cotangent
            ctx.save_for_backward(x)
            ctx.save_for_forward(x)
            return tuple(f)

        @staticmethod
        @once_differentiable
        def backward(ctx, *gs):
            (x,) = ctx.saved_tensors
            model = ctx.model
            cs = []
            for g in gs:
                if g is not None:
                    _check_tensor(model, g, "grad_output")
                    g = g.contiguous()
                cs.append(g)
            n = int(x.shape[0])
            dx = torch.empty_like(x)
            if n:
                with _lib_stream(model, x) as st:
                    model.introspect_vjp_dev(x.data_ptr(), n, [c.data_ptr() if c is not None else 0 for c in cs],
                                             dx.data_ptr(), st)
            return None, dx

        @staticmethod
        def jvp(ctx, _model_t, v):
            (x,) = ctx.saved_tensors
            model = ctx.model
            n = int(x.shape[0])
            if v is None:
                return tuple(torch.zeros((n,) + s, dtype=torch.float32, device=x.device) for s in FEATURE_SHAPES)
            _check_tensor(model, v, "tangent")
            v = v.contiguous()
            t = [torch.empty((n,) + s, dtype=torch.float32, device=x.device) for s in FEATURE_SHAPES]
            if n:
                with _lib_stream(model, x) as st:
                    model.introspect_jvp_dev(x.data_ptr(), v.data_ptr(), n, [a.data_ptr() for a in t], (0, 0, 0, 0), st)
            return tuple(t)

    _Introspect = Introspect
    return Introspect


def introspect(model, x):
    """(f1, f2, f3, f4) = the IAN's introspection features of x (n,3,64,64) float32 CUDA on the model's device: enc_conv1..4
    after inference BatchNorm and LeakyReLU, shapes (n,128,32,32), (n,256,16,16), (n,512,8,8), (n,1024,4,4) -- what
    model.introspect returns.  Differentiable w.r.t. x in reverse mode (one ian_introspect_vjp_dev call per backward; a
    feature the loss does not use passes a NULL cotangent, so the chain starts at the deepest feature used) and forward mode
    (one ian_introspect_jvp_dev call)."""
    return _introspect_function().apply(model, x)


def feature_loss(model, x_hat, x):
    """Per-sample feature-wise loss of train_IAN.py:244, (1/4) sum_i mean((g_i(x_hat) - g_i(x))^2) over introspect's four
    features, (n,) float32; differentiable w.r.t. x_hat and x through introspect (the same formula as
    model.feature_loss)."""
    fa, fb = introspect(model, x_hat), introspect(model, x)
    n = int(fa[0].shape[0])
    if int(fb[0].shape[0]) != n:
        raise ValueError("x_hat and x must hold the same number of images")
    return sum(((a - b) ** 2).reshape(n, -1).mean(1) for a, b in zip(fa, fb)) / 4


def _discriminate_function():
    global _Discriminate
    if _Discriminate is not None:
        return _Discriminate
    import torch
    from torch.autograd.function import once_differentiable

    class Discriminate(torch.autograd.Function):
        @staticmethod
        def forward(ctx, model, x, training):
            _check_tensor(model, x, "x")
            if x.dim() != 4 or tuple(x.shape[1:]) != (3, 64, 64):
                raise ValueError("x must be (n,3,64,64), got %r" % (tuple(x.shape),))
            x = x.contiguous()
            n = int(x.shape[0])
            logits = torch.empty(n, model.discriminator_units(), dtype=torch.float32, device=x.device)
            if n:
                with _lib_stream(model, x) as st:
                    if training:
                        model.discriminate_train_dev(x.data_ptr(), n, logits.data_ptr(), 0, 0, st)
                    else:
                        model.discriminate_dev(x.data_ptr(), n, logits.data_ptr(), 0, st)
            ctx.model = model
            ctx.training = training
            ctx.save_for_backward(x)
            return logits

        @staticmethod
        @once_differentiable
        def backward(ctx, g):
            (x,) = ctx.saved_tensors
            model = ctx.model
            _check_tensor(model, g, "grad_output")
            g = g.contiguous()
            n = int(x.shape[0])
            dx = torch.empty_like(x)
            if n:
                with _lib_stream(model, x) as st:
                    vjp = model.discriminate_train_vjp_dev if ctx.training else model.discriminate_vjp_dev
                    vjp(x.data_ptr(), g.data_ptr(), n, dx.data_ptr(), st)
            return None, dx, None

        @staticmethod
        def jvp(ctx, *tangents):
            raise NotImplementedError("torch_ops.discriminate has no forward mode (the library has no JVP of the discriminator)")

    _Discriminate = Discriminate
    return Discriminate


def discriminate(model, x, training=False):
    """logits (n,U) of the discriminator head for x (n,3,64,64) float32 CUDA on the model's device, after
    model.load_discriminator(): U = 1 (sigmoid) on IAN_simple / IANv1, 3 (softmax: real, reconstruction, generated) on IAN.py.
    Differentiable w.r.t. x in reverse mode (one ian_discriminate_vjp_dev per backward: two trunk forwards and one
    backward).  The batch is coupled: every sample's logits depend on every image of the call.
    training=True: l_discrim as the reference's trainers evaluate it (deterministic=False): bnorm2..4 normalise with the
    batch's statistics, and the backward (ian_discriminate_train_vjp_dev: one trunk forward and one backward) flows through
    them.  The model's running statistics are neither used nor changed."""
    return _discriminate_function().apply(model, x, bool(training))


def _params_function():
    global _DecodeParams
    if _DecodeParams is not None:
        return _DecodeParams
    import torch
    from torch.autograd.function import once_differentiable

    class DecodeParams(torch.autograd.Function):
        @staticmethod
        def forward(ctx, model, z, training, names, *tensors):
            _check_tensor(model, z, "z")
            if z.dim() != 2 or z.shape[1] != 100:
                raise ValueError("z must be (n,100), got %r" % (tuple(z.shape),))
            _sync_params(model, names, tensors)
            z = z.contiguous()
            n = int(z.shape[0])
            x = torch.empty(n, 3, 64, 64, dtype=torch.float32, device=z.device)
            if n:
                with _lib_stream(model, z) as st:
                    if training:
                        model.decode_train_dev(z.data_ptr(), n, x.data_ptr(), 0, st)
                    else:
                        model.decode_dev(z.data_ptr(), n, x.data_ptr(), st)
            ctx.model, ctx.names, ctx.training = model, names, training
            ctx.save_for_backward(z, *tensors)
            return x

        @staticmethod
        @once_differentiable
        def backward(ctx, g):
            z, *tensors = ctx.saved_tensors
            model = ctx.model
            _check_tensor(model, g, "grad_output")
            g = g.contiguous()
            n = int(z.shape[0])
            want_z = ctx.needs_input_grad[1]
            dz = torch.zeros_like(z) if want_z else None
            grads = [torch.zeros_like(t) if ctx.needs_input_grad[4 + i] else None for i, t in enumerate(tensors)]
            if n:
                ptrs = {name: gr.data_ptr() for name, gr in zip(ctx.names, grads) if gr is not None}
                vjp = model.decode_train_vjp_dev if ctx.training else model.decode_param_vjp_dev
                with _lib_stream(model, z) as st:
                    vjp(z.data_ptr(), g.data_ptr(), n, dz.data_ptr() if want_z else 0, ptrs, st)
            return (None, dz, None, None) + tuple(grads)

    _DecodeParams = DecodeParams
    return DecodeParams


def _sync_params(model, names, tensors):
    """write every tensor whose identity or in-place version changed since its last upload back into the handle"""
    seen = getattr(model, "_param_uploads", None)
    if seen is None:
        seen = model._param_uploads = {}
    changed = {}
    for name, t in zip(names, tensors):
        _check_tensor(model, t, name)
        key = (id(t), t._version)
        if seen.get(name) != key:
            changed[name] = t.detach().cpu().numpy()
            seen[name] = key
    if changed:
        model.update_params(changed)


def decoder_parameters(model, weights):
    """{name: leaf float32 CUDA tensor with requires_grad} for the IAN_simple decoder's trainable tensors
    (model.param_vjp_names()), built from the checkpoint mapping `weights` and uploaded into the handle once, so that the
    handle provably holds their values."""
    import torch
    names = model.param_vjp_names()
    if not names:
        raise ValueError("this graph has no parameter gradients (IAN_simple only)")
    params = {n: torch.tensor(weights[n], dtype=torch.float32, device="cuda:%d" % model.device).requires_grad_(True)
              for n in names}
    _sync_params(model, names, [params[n] for n in names])
    return params


def decode(model, z, params=None, training=False):
    """x_hat = decoder(z) for z (n,100) float32 CUDA on the model's device; differentiable w.r.t. z (one decoder forward +
    one backward per backward call).  Without params it also supports forward mode: under torch.autograd.forward_ad a
    dual z (make_dual(z, v)) gives x_hat with the tangent (d x_hat / d z) . v, from one ian_decode_jvp_dev call.
    With params (from decoder_parameters), also differentiable w.r.t. those tensors: one ian_decode_param_vjp_dev returns
    dz and every gradient; tensors that do not require grad get None.  That form is reverse mode only.
    training=True (IAN_simple): the decoder as the reference's trainers evaluate it (deterministic=False): its four
    BatchNorms normalise with the batch's statistics, so every sample's x_hat depends on every z of the call.  The forward
    is ian_decode_train_dev and the backward one ian_decode_train_vjp_dev, for z and the params alike; reverse mode only.
    The model's running statistics are neither used nor changed."""
    if params is None and not training:
        return _function().apply(model, z)
    names = list(params or ())
    return _params_function().apply(model, z, bool(training), tuple(names), *[params[n] for n in names])

"""torch autograd binding of the IAN decoder, through the C-ABI of libian_b200.so (include/ian_b200.h):

  * decode(model, z) = X_hat of the reference (API.py:46, sample_at) as a differentiable torch op.  Its backward is the
    decoder's vector-Jacobian product (ian_decode_vjp_dev), so any loss torch can write on the decoded images -- soft or
    per-pixel weighted brushes, L1, losses on the whole frame, refining a latent against a photo -- drives the latent
    through torch.autograd, as any loss on X_hat was one T.grad away in the reference.

A backward costs one decoder forward plus one backward: the library recomputes the forward from the saved z instead of
keeping the activations of the forward call.  The op is once-differentiable (no double backward).  Inputs and outputs are
torch CUDA float32 tensors on the model's device; torch only carries the device memory and the stream.
"""
from __future__ import annotations

from .train_ops import _lib_stream

_Decode = None


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

    _Decode = Decode
    return Decode


def decode(model, z):
    """x_hat = decoder(z) for z (n,100) float32 CUDA on the model's device; differentiable w.r.t. z (one decoder forward +
    one backward per backward call)."""
    return _function().apply(model, z)

"""Training-mode pieces next to the IAN hot path, through the C-ABI of libian_b200.so (include/ian_b200.h):

  * batch_norm_train  = lasagne BatchNormLayer.get_output_for(deterministic=False), i.e. `BN(...)` of the reference graphs
    (IAN_simple.py:12,84-170; layers.py:411-416) in training, with the running `mean` / `inv_std` update; statistics
    can be synchronised over a torch.distributed group (sum / sum-of-squares all-reduce between the two library calls).
  * minibatch_layer   = reference layers.py:486-524 (MinibatchLayer forward).

Both are torch autograd ops (DESIGN §5.6b): batch_norm_train is differentiable in x, gamma and beta, minibatch_layer in x,
theta, log_weight_scale and b, so a torch trainer gets the gradients Theano's T.grad gives the reference.  The backward
recomputes what it needs from the saved input (BatchNorm keeps x, its 2*c float64 sums and the count; MinibatchLayer
keeps its inputs) and is once-differentiable.  With `group=`, the BatchNorm backward all-reduces its 2*c float64 sums over
the same group, as the forward does; dgamma / dbeta stay this rank's, for DDP to reduce with the other parameters.
When no input requires grad, the ops run exactly the forward calls they always ran.

Inputs and outputs are torch CUDA tensors (float32); torch only carries the device memory and the optional all-reduce.
The trainers themselves (train_IAN*.py) are out of scope and stay the reference's.
"""
from __future__ import annotations

import contextlib


@contextlib.contextmanager
def _lib_stream(model, x):
    """The raw CUDA stream the library call is enqueued on, ordered with torch's current stream.  A non-default torch
    stream is used as is; the legacy default stream (handle 0, which the C-ABI reads as "the handle's own stream") is
    bridged through a side stream with wait_stream on both sides."""
    import torch
    cur = torch.cuda.current_stream(x.device)
    if cur.cuda_stream != 0:
        yield cur.cuda_stream
        return
    side = getattr(model, "_train_stream", None)
    if side is None:
        side = model._train_stream = torch.cuda.Stream(device=x.device)
    side.wait_stream(cur)
    yield side.cuda_stream
    cur.wait_stream(side)


_BatchNorm = None
_Minibatch = None


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _all_reduce(t, group):
    import torch.distributed as dist
    g = None if group is True else group
    dist.all_reduce(t, group=g)
    return dist.get_world_size(g)


def _bn_forward(model, x, gamma, beta, running_mean, running_inv_std, eps, alpha, group):
    """the two forward calls; returns y, the (global) sums and the global element count"""
    import torch
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() >= 2
    n, c = int(x.shape[0]), int(x.shape[1])
    hw = int(x[0, 0].numel()) if x.dim() > 2 else 1
    sums = torch.empty(2, c, dtype=torch.float64, device=x.device)
    with _lib_stream(model, x) as st:
        model._check(model._lib.ian_bn_batch_stats_dev(model._h, x.data_ptr(), n, c, hw, sums[0].data_ptr(), sums[1].data_ptr(), st))
    count = float(n * hw)
    if group is not None:                                   # cross-GPU synchronised BN: one all-reduce of 2*c float64
        count *= _all_reduce(sums, group)
    y = torch.empty_like(x)
    with _lib_stream(model, x) as st:
        model._check(model._lib.ian_bn_train_normalize_dev(model._h, x.data_ptr(), n, c, hw, sums[0].data_ptr(), sums[1].data_ptr(),
                                                           count, _ptr(gamma), _ptr(beta), float(eps), float(alpha),
                                                           _ptr(running_mean), _ptr(running_inv_std), y.data_ptr(), st))
    return y, sums, count


def _mb_forward(model, x2, theta, lws, b):
    import torch
    n, d = int(x2.shape[0]), int(x2.shape[1])
    K, P = int(theta.shape[1]), int(theta.shape[2])
    out = torch.empty(n, d + K, dtype=torch.float32, device=x2.device)
    with _lib_stream(model, x2) as st:
        model._check(model._lib.ian_minibatch_discrim_dev(model._h, x2.data_ptr(), n, d, theta.data_ptr(), lws.data_ptr(), b.data_ptr(),
                                                          K, P, out.data_ptr(), st))
    return out


def _bn_function():
    global _BatchNorm
    if _BatchNorm is not None:
        return _BatchNorm
    import torch
    from torch.autograd.function import once_differentiable

    class BatchNormTrain(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, gamma, beta, model, running_mean, running_inv_std, eps, alpha, group):
            y, sums, count = _bn_forward(model, x, gamma, beta, running_mean, running_inv_std, eps, alpha, group)
            ctx.model, ctx.count, ctx.eps, ctx.group = model, count, eps, group
            ctx.save_for_backward(x, gamma, sums)
            return y

        @staticmethod
        @once_differentiable
        def backward(ctx, dy):
            x, gamma, sums = ctx.saved_tensors
            model = ctx.model
            n, c = int(x.shape[0]), int(x.shape[1])
            hw = int(x[0, 0].numel()) if x.dim() > 2 else 1
            dy = dy.contiguous()
            want_x, want_g, want_b = ctx.needs_input_grad[:3]
            bsums = torch.empty(2, c, dtype=torch.float64, device=x.device)
            dgamma = torch.empty(c, dtype=torch.float32, device=x.device) if want_g else None
            dbeta = torch.empty(c, dtype=torch.float32, device=x.device) if want_b else None
            with _lib_stream(model, x) as st:
                model._check(model._lib.ian_bn_backward_sums_dev(
                    model._h, x.data_ptr(), dy.data_ptr(), n, c, hw, sums[0].data_ptr(), sums[1].data_ptr(), ctx.count,
                    float(ctx.eps), bsums[0].data_ptr(), bsums[1].data_ptr(), _ptr(dgamma), _ptr(dbeta), st))
            dx = None
            if want_x:
                if ctx.group is not None:
                    _all_reduce(bsums, ctx.group)
                dx = torch.empty_like(x)
                with _lib_stream(model, x) as st:
                    model._check(model._lib.ian_bn_backward_dx_dev(
                        model._h, x.data_ptr(), dy.data_ptr(), n, c, hw, sums[0].data_ptr(), sums[1].data_ptr(), ctx.count,
                        bsums[0].data_ptr(), bsums[1].data_ptr(), _ptr(gamma), float(ctx.eps), dx.data_ptr(), st))
            return dx, dgamma, dbeta, None, None, None, None, None, None

    _BatchNorm = BatchNormTrain
    return _BatchNorm


def _mb_function():
    global _Minibatch
    if _Minibatch is not None:
        return _Minibatch
    import torch
    from torch.autograd.function import once_differentiable

    class MinibatchLayer(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x2, theta, lws, b, model):
            ctx.model = model
            ctx.save_for_backward(x2, theta, lws, b)
            return _mb_forward(model, x2, theta, lws, b)

        @staticmethod
        @once_differentiable
        def backward(ctx, g):
            x2, theta, lws, b = ctx.saved_tensors
            model = ctx.model
            n, d = int(x2.shape[0]), int(x2.shape[1])
            K, P = int(theta.shape[1]), int(theta.shape[2])
            g = g.contiguous()
            grads = [torch.empty_like(t) if want else None for t, want in zip((x2, theta, lws, b), ctx.needs_input_grad[:4])]
            with _lib_stream(model, x2) as st:
                model._check(model._lib.ian_minibatch_discrim_bwd_dev(model._h, x2.data_ptr(), n, d, theta.data_ptr(), lws.data_ptr(),
                                                                      b.data_ptr(), K, P, g.data_ptr(), *[_ptr(t) for t in grads], st))
            return tuple(grads) + (None,)

    _Minibatch = MinibatchLayer
    return _Minibatch


def _needs_grad(*ts):
    import torch
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ts)


def batch_norm_train(model, x, gamma, beta, running_mean=None, running_inv_std=None, eps=1e-4, alpha=0.1, group=None):
    """x (n, c, ...) float32 CUDA, contiguous.  Returns y; running_mean / running_inv_std are updated IN PLACE.
    `model`: any finalized IAN handle on x's device (it owns the workspace).  `group`: torch.distributed group (or True
    for the default group) to synchronise the batch statistics across ranks, in the forward and in the backward.
    Differentiable in x, gamma and beta (torch autograd)."""
    if not _needs_grad(x, gamma, beta):
        return _bn_forward(model, x, gamma, beta, running_mean, running_inv_std, eps, alpha, group)[0]
    return _bn_function().apply(x, gamma, beta, model, running_mean, running_inv_std, eps, alpha, group)


def minibatch_layer(model, x, theta, log_weight_scale, b):
    """x (n, ...) float32 CUDA (flattened to (n, d) like layers.py:504-507); theta (d, K, P); log_weight_scale (K, P); b (K).
    Returns (n, d + K) = [x | f].  Differentiable in x, theta, log_weight_scale and b (torch autograd)."""
    x2 = x.reshape(x.shape[0], -1).contiguous()
    n, d = int(x2.shape[0]), int(x2.shape[1])
    K, P = int(theta.shape[1]), int(theta.shape[2])
    assert tuple(theta.shape) == (d, K, P) and tuple(log_weight_scale.shape) == (K, P) and tuple(b.shape) == (K,)
    th, lw, bb = theta.contiguous(), log_weight_scale.contiguous(), b.contiguous()
    if _needs_grad(x, theta, log_weight_scale, b):
        return _mb_function().apply(x2, th, lw, bb, model)
    return _mb_forward(model, x2, th, lw, bb)

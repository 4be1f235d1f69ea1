"""Float64 torch-autograd restatement of the training-mode ops, and the closed forms of their reverse mode (DESIGN §5.6b).

  * bn_train / mb_layer restate oracle/train_numpy.py's forward in torch, so torch.autograd differentiates them the way
    Theano's T.grad differentiates the reference: through the batch mean and variance, and through |.| with sgn(0) = 0
    (torch's abs backward, as Theano's).  tests/test_train_grad_oracle.py pins them to the numpy forward and to the
    executed reference's central differences (tests/golden/ref_exec_train_grad.npz).
  * bn_backward / mb_backward are the closed forms the CUDA kernels evaluate, in float64.
Only tests/ import this module.  Every function takes and returns torch float64 tensors on any device.
"""
import torch

F64 = torch.float64


def _axes(x):
    return (0,) + tuple(range(2, x.dim()))


def _shape(x):
    return [1, -1] + [1] * (x.dim() - 2)


def bn_train(x, gamma, beta, eps=1e-4):
    """lasagne BatchNormLayer.get_output_for(deterministic=False); gamma / beta None mean 1 / 0"""
    axes, shp = _axes(x), _shape(x)
    mean = x.mean(axes)
    inv_std = 1.0 / torch.sqrt(x.var(axes, unbiased=False) + eps)
    y = (x - mean.reshape(shp)) * inv_std.reshape(shp)
    if gamma is not None:
        y = y * gamma.reshape(shp)
    if beta is not None:
        y = y + beta.reshape(shp)
    return y


def mb_layer(x, theta, lws, b):
    """reference layers.py:495, :503-524 (init=False): x (n, d) -> (n, d + K)"""
    x = x.reshape(x.shape[0], -1)
    W = theta * (torch.exp(lws) / torch.sqrt((theta * theta).sum(0)))[None]
    act = torch.tensordot(x, W, dims=([1], [0]))                                      # (n, K, P)
    n = x.shape[0]
    abs_dif = (act[:, :, :, None] - act.permute(1, 2, 0)[None]).abs().sum(2)          # (n, K, n)
    abs_dif = abs_dif + 1e6 * torch.eye(n, dtype=x.dtype, device=x.device)[:, None, :]
    f = torch.exp(-abs_dif).sum(2) + b[None]
    return torch.cat([x, f], 1)


def bn_stats(x, eps=1e-4):
    axes = _axes(x)
    mean = x.mean(axes)
    return mean, 1.0 / torch.sqrt(x.var(axes, unbiased=False) + eps)


def bn_backward(x, gamma, dy, eps=1e-4):
    """(dx, dgamma, dbeta): dx = gamma s (dy - mean(dy) - x̂ mean(dy x̂)), dgamma = Σ dy x̂, dbeta = Σ dy"""
    axes, shp = _axes(x), _shape(x)
    mean, s = bn_stats(x, eps)
    xh = (x - mean.reshape(shp)) * s.reshape(shp)
    g = torch.ones_like(mean) if gamma is None else gamma
    dx = (g * s).reshape(shp) * (dy - dy.mean(axes).reshape(shp) - xh * (dy * xh).mean(axes).reshape(shp))
    return dx, (dy * xh).sum(axes), dy.sum(axes)


def mb_backward(x, theta, lws, b, g):
    """(dx, dtheta, dlws, db) of Σ g·mb_layer(x, theta, lws, b), by the closed forms of DESIGN §5.6b"""
    x = x.reshape(x.shape[0], -1)
    n, d = x.shape
    K, P = theta.shape[1:]
    r = torch.sqrt((theta * theta).sum(0))                                            # (K, P)
    cs = torch.exp(lws) / r
    W = theta * cs[None]
    A = torch.tensordot(x, W, dims=([1], [0]))                                        # (n, K, P)
    gx, gf = g[:, :d], g[:, d:]
    diff = A[:, None] - A[None]                                                       # (i, j, K, P)
    e = torch.exp(-diff.abs().sum(-1))                                                # (i, j, K)
    e = e * (1 - torch.eye(n, dtype=x.dtype, device=x.device))[:, :, None]
    c = (gf[:, None] + gf[None]) * e
    dA = -(c[..., None] * torch.sign(diff)).sum(1)                                    # (n, K, P)
    dx = gx + torch.tensordot(dA, W, dims=([1, 2], [1, 2]))
    dW = torch.tensordot(x, dA, dims=([0], [0]))                                      # (d, K, P)
    S = (theta * dW).sum(0)
    dtheta = cs[None] * (dW - theta * (S / (r * r))[None])
    dlws = (dW * W).sum(0)
    return dx, dtheta, dlws, gf.sum(0)

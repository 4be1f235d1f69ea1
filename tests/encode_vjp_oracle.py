"""float64 numpy reference of the encoder vector-Jacobian product dx = (dz/dx)^T dz (ian_encode_vjp_*): reverse mode through
the encoder of oracle/ian_numpy.py / oracle/ian_full_numpy.py, written out layer by layer so that it is a second
formulation next to torch autograd of oracle/ian_torch.py.  The test modules import it; the product never does.

Rectifier derivatives follow Theano's T.grad of lasagne's forms (assumption C.5 of oracle/ian_numpy.py):
  rectify 0.5 (x + |x|)             -> 0.5 (1 + sgn x)       (1/2 at exactly 0)
  LeakyRectify(0.2) 0.6 x + 0.4 |x| -> 0.6 + 0.4 sgn x
  elu where(x > 0, x, exp(x) - 1)   -> where(x > 0, 1, exp(x))
torch autograd of the same forms gives the same values, abs'(0) = 0 included."""
from __future__ import annotations

import numpy as np

from oracle import ian_full_numpy as fn
from oracle import ian_numpy as on

F64 = np.float64


def rectify_grad(x):
    return 0.5 * (1.0 + np.sign(x))


def lrelu_grad(x, alpha=0.2):
    return 0.5 * (1 + alpha) + 0.5 * (1 - alpha) * np.sign(x)


def elu_grad(x):
    return np.where(x > 0, 1.0, np.exp(np.minimum(x, 0)))


def conv5x5_s2_bwd_data(dy, W, hw):
    """Adjoint of on.conv5x5_s2 (IAN_simple.py:73-116) w.r.t. its input of spatial size hw:
    dx[n,c,2p+i-2,2q+j-2] += sum_o dy[n,o,p,q] W[o,c,i,j]."""
    dy = np.asarray(dy, F64)
    W = np.asarray(W, F64)
    n, _, ho, wo = dy.shape
    dxp = np.zeros((n, W.shape[1], hw + 4, hw + 4), F64)
    for i in range(5):
        for j in range(5):
            dxp[:, :, i:i + 2 * ho:2, j:j + 2 * wo:2] += np.einsum("nohw,oc->nchw", dy, W[:, :, i, j], optimize=True)
    return dxp[:, :, 2:2 + hw, 2:2 + hw]


def _bn_scale(P, name):
    return np.asarray(P[name + ".gamma"], F64) * np.asarray(P[name + ".inv_std"], F64)


def _encoder_vjp(P, x, fc1_act, fc1_grad, dmu, dls):
    """reverse mode through enc_conv1..enc_fc1 and the mu / logsigma heads (IAN_simple.py:72-126, IAN.py:71-125) given the
    cotangents of mu and logsigma."""
    x = np.asarray(x, F64)
    bn = lambda t, name: on.batchnorm_inf(t, on._bn(P, name))
    u1 = on.conv5x5_s2(x, P["enc_conv1.W"], P["enc_conv1.b"]); a1 = on.lrelu(u1)
    u2 = bn(on.conv5x5_s2(a1, P["enc_conv2.W"]), "bnorm2"); a2 = on.lrelu(u2)
    u3 = bn(on.conv5x5_s2(a2, P["enc_conv3.W"]), "bnorm3"); a3 = on.lrelu(u3)
    u4 = bn(on.conv5x5_s2(a3, P["enc_conv4.W"]), "bnorm4"); a4 = on.lrelu(u4)
    u5 = bn(on.dense(a4, P["enc_fc1.W"]), "bnorm_enc_fc1")
    dh = (dmu * _bn_scale(P, "mu_bnorm")) @ np.asarray(P["enc_mu.W"], F64).T
    dh = dh + (dls * _bn_scale(P, "ls_bnorm")) @ np.asarray(P["enc_logsigma.W"], F64).T
    d5 = dh * fc1_grad(u5) * _bn_scale(P, "bnorm_enc_fc1")
    da4 = (d5 @ np.asarray(P["enc_fc1.W"], F64).T).reshape(a4.shape)
    d4 = da4 * lrelu_grad(u4) * _bn_scale(P, "bnorm4")[None, :, None, None]
    da3 = conv5x5_s2_bwd_data(d4, P["enc_conv4.W"], 8)
    d3 = da3 * lrelu_grad(u3) * _bn_scale(P, "bnorm3")[None, :, None, None]
    da2 = conv5x5_s2_bwd_data(d3, P["enc_conv3.W"], 16)
    d2 = da2 * lrelu_grad(u2) * _bn_scale(P, "bnorm2")[None, :, None, None]
    da1 = conv5x5_s2_bwd_data(d2, P["enc_conv2.W"], 32)
    d1 = da1 * lrelu_grad(u1)
    return conv5x5_s2_bwd_data(d1, P["enc_conv1.W"], 64)


def _sample_vjp(ls, dz, eps):
    """GaussianSampleLayer (layers.py:419-433): z = mu (+ exp(logsigma) eps) -> (dmu, dlogsigma); no gradient w.r.t. eps."""
    dz = np.asarray(dz, F64)
    if eps is None:
        return dz, np.zeros_like(dz)
    return dz, dz * np.exp(ls) * np.asarray(eps, F64)


def simple_encode_vjp(P, x, dz, eps=None):
    """dx of IAN_simple's Z_hat (API.py:50 on IAN_simple.py): z = mu, or mu + exp(logsigma) eps."""
    _, ls = on.simple_encode_mu_ls(P, x)
    dmu, dls = _sample_vjp(ls, dz, eps)
    return _encoder_vjp(P, x, on.elu, elu_grad, dmu, dls)


def made_vjp(P, name, z, masks, g):
    """reverse mode of fn.made_forward (layers.py:653-853 as wired in IAN.py:127): the `<name>_input` MaskedLayer runs twice,
    u = rect(z W0 + b0), h = rect(u W0 + b0), out = h W1 + b1 + u Wd + bd; returns d out / d z applied to g."""
    M0, M1, Md = [np.asarray(m, F64) for m in masks]
    W0 = np.asarray(P[name + "_input.W"], F64) * M0
    b0 = np.asarray(P[name + "_input.b"], F64)
    W1 = np.asarray(P[name + "_output_W.W"], F64) * M1
    Wd = np.asarray(P[name + "_output_D.W"], F64) * Md
    z = np.asarray(z, F64)
    pu = z @ W0 + b0
    u = on.rectify(pu)
    ph = u @ W0 + b0
    dph = (g @ W1.T) * rectify_grad(ph)
    du = g @ Wd.T + dph @ W0.T
    return (du * rectify_grad(pu)) @ W0.T


def flow_vjp(P, z_iaf, masks, dz):
    """reverse mode of fn.full_latent (IAFLayer layers.py:641-650): z = (z_iaf - MADE_mu(z_iaf)) / exp(MADE_ls(z_iaf))."""
    z_iaf = np.asarray(z_iaf, F64)
    dz = np.asarray(dz, F64)
    o_mu = fn.made_forward(P, "l_IAF_mu", z_iaf, masks)
    o_ls = fn.made_forward(P, "l_IAF_ls", z_iaf, masks)
    e = np.exp(o_ls)
    z = (z_iaf - o_mu) / e
    return dz / e + made_vjp(P, "l_IAF_mu", z_iaf, masks, -dz / e) + made_vjp(P, "l_IAF_ls", z_iaf, masks, -dz * z)


def full_encode_vjp(P, x, masks, dz, eps=None):
    """dx of IAN.py's Z_hat (API.py:50: l_Z, IAN.py:126-128): the MADE/IAF flow applied to mu (+ exp(logsigma) eps)."""
    mu, ls = fn.full_encode_mu_ls(P, x)
    z_iaf = on.gaussian_sample(mu, ls, eps, eps is None)
    dmu, dls = _sample_vjp(ls, flow_vjp(P, z_iaf, masks, dz), eps)
    return _encoder_vjp(P, x, on.rectify, rectify_grad, dmu, dls)


def v1_encode_vjp(P, x, masks, dz, eps=None):
    """IANv1.py's encoder and latent flow (IANv1.py:71-123) are IAN.py's: the same chain."""
    return full_encode_vjp(P, x, masks, dz, eps)

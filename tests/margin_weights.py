"""Well-conditioned weights for the gradient tests: every rectifier pre-activation of a fixed input pool is at least
delta away from its kink, on a side fixed per channel, and every sigmoid of the RGB-Beta head sees an argument in
[-2, 2].  On the synthetic weights some rectifier sits within ~1e-6 of its kink and the Beta ratio is steep, so a
float32 forward error of 1e-5 flips masks and moves a gradient by up to 5e-2 (DESIGN section 5.6c); on these weights a
gradient moves with the float32 error of the kernels alone, and a tight bound can tell the hi|lo scheme from a
single-pass bf16 slip.

margin_weights(graph, P, pool) walks the graph in forward order in float64 torch (CPU or CUDA).  At each rectifier it
picks a sign s_c per channel or unit (-1 for one in four, (c + crc32(knob)) % 4 == 3) and shifts the bias or BatchNorm beta
feeding it by just enough that s_c * pre >= delta on every element of every pool sample: LeakyRectify channels run at
slope 0.2 and ReLU channels die where s_c = -1.  Every BatchNorm first gets the pool's float64 statistics as its
inference mean / inv_std, so activations do not grow layer after layer (ls_bnorm gets a third of its inv_std, so that
exp(logsigma) stays near 1).  The knobs (checkpoint names):
  encoder       enc_conv1.b; beta of bnorm2-4; beta of bnorm_enc_fc1 (ReLU on the flow graphs; IAN_simple's ELU is C1
                and gets statistics only)
  MADE          l_IAF_{mu,ls}_input.b (ReLU).  The input MaskedLayer runs twice with the same bias (DESIGN section 2),
                so the shift is iterated until both applications hold, for z = mu and z = mu + exp(logsigma) eps; if
                that does not settle, the MADE signs fall back to all +1
  IAN.py dec    l_dec_fc2.b per unit; dec_conv{2,3,4}a bnorm0 / bnorm1 / bnorm2 (bnorm2 after the residual add); bnorm_dc4
  IANv1 dec     beta of bnorm_dc1-4 (its l_dec_fc2 is linear)
  IAN_simple    beta of bnorm_dec_fc2, bnorm_dc1-3
  RGB-Beta head the _coeff_* vectors of R, G_a / G_b and B_a / B_b, scaled per output channel until every sigmoid argument
                of the pool lies in [-1.9, 1.9]; then a + b >= 0.26 and the Beta ratio is well-conditioned.
certificate() runs the same walk without changing anything and reports, per rectifier, min s_c * pre and the counts of
each sign, the head's largest sigmoid argument and how many output pixels are saturated (|x_hat| >= 0.99).

The pool is pool(n): x, z, eps, rgb, frame and the boxes of tests/scale_inputs.py (1x1, the full width, random
<= 17), so a batch of n samples of it is pool(POOL)[:n]."""
from __future__ import annotations

import os
import zlib

import numpy as np
import torch
import torch.nn.functional as F

from oracle import ian_full_numpy as fn
from oracle import ian_torch as ot

import scale_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POOL = 130
POOL_SEED = 7130
DELTA = 0.5
HEAD_ARG = 1.9
DECODER = {"simple": ot.decode, "full": ot.full_decode, "v1": ot.v1_decode}
_MADE_ITERS = 60


def pool(n=POOL, seed=POOL_SEED):
    """the input pool: tests/scale_inputs.py's inputs, drawn with this module's seed"""
    return scale_inputs.inputs(n, seed)


def signs(n, knob):
    """+1 / -1 per channel, -1 for one in four in a pattern that moves from layer to layer"""
    s = np.ones(n)
    s[(np.arange(n) + zlib.crc32(knob.encode())) % 4 == 3] = -1.0
    return s


def made_masks(device="cpu"):
    return [torch.from_numpy(m.astype(np.float64)).to(device) for m in fn.made_masks(fn.made_ordering())]


def _chan(t):
    """per-channel (dim 1) min and max over every other dimension"""
    d = [0] + list(range(2, t.dim()))
    return t.amin(dim=d), t.amax(dim=d)


class _Walk:
    """one forward pass in float64 that either fits the knobs (fit=True: Q is changed in place) or only records"""

    def __init__(self, Q, fit, delta, head_arg=HEAD_ARG):
        self.Q, self.fit, self.delta, self.head_arg = Q, fit, delta, head_arg
        self.report, self.slip = {}, None

    def _slip(self, name, t):
        return _BF16Grad.apply(t) if self.slip == name else t

    def _shape(self, v, t):
        return v.reshape((1, -1) + (1,) * (t.dim() - 2))

    def bn(self, name, x, inv_scale=1.0):
        if self.fit:
            d = [0] + list(range(2, x.dim()))
            self.Q[name + ".mean"] = x.mean(dim=d)
            self.Q[name + ".inv_std"] = inv_scale / x.std(dim=d)
        return ot._bn(self.Q, name, x)

    def rect(self, knob, pre, leaky):
        """pre = ... + Q[knob] (a bias or a beta); returns the rectified value"""
        s = torch.from_numpy(signs(pre.shape[1], knob)).to(pre)
        lo, hi = _chan(pre.detach())
        if self.fit:
            d = self.delta * 1.001                                   # float32 rounding of the knob keeps >= delta
            shift = torch.where(s > 0, (d - lo).clamp(min=0), -(d + hi).clamp(min=0))
            self.Q[knob] = self.Q[knob] + shift
            pre = pre + self._shape(shift, pre)
            lo, hi = lo + shift, hi + shift
        m = torch.where(s > 0, lo, -hi)
        self.report[knob] = {"min_margin": float(m.min()), "pos": int((s > 0).sum()), "neg": int((s < 0).sum())}
        return ot._lrelu(pre) if leaky else ot._relu(pre)

    # ---- encoder ----
    def encode_mu_ls(self, x, graph):
        Q = self.Q
        h = self.rect("enc_conv1.b", F.conv2d(x, Q["enc_conv1.W"], Q["enc_conv1.b"], stride=2, padding=2), True)
        for i in (2, 3, 4):
            name = "bnorm%d" % i
            y = F.conv2d(h, Q["enc_conv%d.W" % i], None, stride=2, padding=2)
            h = self.rect(name + ".beta", self.bn(name, self._slip("enc", y) if i == 3 else y), True)
        u = self.bn("bnorm_enc_fc1", h.flatten(1) @ Q["enc_fc1.W"])
        h = F.elu(u) if graph == "simple" else self.rect("bnorm_enc_fc1.beta", u, False)
        return self.bn("mu_bnorm", h @ Q["enc_mu.W"]), self.bn("ls_bnorm", h @ Q["enc_logsigma.W"], 1.0 / 3.0)

    def made(self, name, zs, masks):
        """both applications of `<name>_input` on every z of zs; fits by iteration (module docstring)"""
        Q, M0 = self.Q, masks[0]
        knob = name + "_input.b"
        W0 = Q[name + "_input.W"] * M0

        def margins(s):
            m = None
            for z in zs:
                pu = z @ W0 + Q[knob]
                ph = ot._relu(pu) @ W0 + Q[knob]
                for pre in (pu, ph):
                    lo, hi = _chan(pre)
                    v = torch.where(s > 0, lo, -hi)
                    m = v if m is None else torch.minimum(m, v)
            return m
        s = torch.from_numpy(signs(W0.shape[1], knob)).to(W0)
        if self.fit:
            b0 = Q[knob].clone()
            for signed in (True, False):
                if not signed:
                    s, Q[knob] = torch.ones_like(s), b0.clone()
                for _ in range(_MADE_ITERS):
                    m = margins(s)
                    if float(m.min()) >= self.delta:
                        break
                    Q[knob] = Q[knob] + s * (self.delta * 1.001 - m).clamp(min=0)
                if float(margins(s).min()) >= self.delta:
                    break
        m = margins(s)
        if not self.fit and float(m.min()) < self.delta:             # the all-positive fallback
            s = torch.ones_like(s)
            m = margins(s)
        self.report[knob] = {"min_margin": float(m.min()), "pos": int((s > 0).sum()), "neg": int((s < 0).sum())}

    # ---- decoders ----
    def deconv_bn_rect(self, h, conv, name, leaky):
        y = ot.deconv(h, self.Q[conv])
        return self.rect(name + ".beta", self.bn(name, self._slip("block", y) if conv == "dec_conv2.W" else y), leaky)

    def mdblock(self, name, x, scales):
        t = self.rect(name + "bnorm0.beta", self.bn(name + "bnorm0", x), True)
        t = self.rect(name + "bnorm1.beta", self.bn(name + "bnorm1", ot.mdcl(self.Q, name, t, scales)), True)
        t = ot.mdcl(self.Q, name + "2", t, scales)
        t = self._slip("block", t) if name == "dec_conv3a" else t
        return self.rect(name + "bnorm2.beta", self.bn(name + "bnorm2", x + t), True)

    def sigmoid(self, names, args):
        """sigmoid of sum(args), each arg linear in the _coeff_* vectors of the matching name"""
        a = self._slip("head", sum(args))
        top = a.detach().abs().amax(dim=(0, 2, 3))
        if self.fit:
            scale = torch.clamp(self.head_arg / top, max=1.0)
            for name in names:
                for k in [k for k in self.Q if k.startswith(name + "_coeff_")]:
                    self.Q[k] = self.Q[k] * scale
            a, top = a * self._shape(scale, a), top * scale
        self.report.setdefault("head_max_arg", 0.0)
        self.report["head_max_arg"] = max(self.report["head_max_arg"], float(top.max()))
        return torch.sigmoid(a)

    def head(self, h):
        Q, sc = self.Q, [2, 3, 4]
        R = self.sigmoid(["R"], [ot.mdcl(Q, "R", h, sc)])
        G = self.sigmoid(["G_a", "G_b"], [ot.mdcl(Q, "G_a", h, sc), ot.mdcl(Q, "G_b", R, sc)])
        B = self.sigmoid(["B_a", "B_b"], [ot.mdcl(Q, "B_a", h, sc), ot.mdcl(Q, "B_b", torch.cat([R, G], 1), sc)])
        beta = lambda a, b: 2.0 * (a / (a + b + 1e-8)) - 1.0
        return torch.stack([beta(R[:, 0], R[:, 1]), beta(G[:, 0], G[:, 1]), beta(B[:, 0], B[:, 1])], 1)

    def decode(self, z, graph):
        Q = self.Q
        if graph == "simple":
            h = self.rect("bnorm_dec_fc2.beta", self.bn("bnorm_dec_fc2", z @ Q["l_dec_fc2.W"]), False).reshape(-1, 1024, 4, 4)
            for i in (1, 2, 3):
                h = self.deconv_bn_rect(h, "dec_conv%d.W" % i, "bnorm_dc%d" % i, False)
            return torch.tanh(self._slip("head", ot.deconv(h, Q["dec_out.W"])))
        if graph == "v1":
            h = (z @ Q["l_dec_fc2.W"] + Q["l_dec_fc2.b"]).reshape(-1, 1024, 4, 4)
            for i in (1, 2, 3, 4):
                h = self.deconv_bn_rect(h, "dec_conv%d.W" % i, "bnorm_dc%d" % i, False)
            return self.head(h)
        h = self.rect("l_dec_fc2.b", z @ Q["l_dec_fc2.W"] + Q["l_dec_fc2.b"], True).reshape(-1, 512, 4, 4)
        h = self.mdblock("dec_conv2a", ot.deconv(h, Q["dec_conv1.W"]), [0, 2])
        h = self.mdblock("dec_conv3a", ot.deconv(h, Q["dec_conv2.W"]), [0, 2, 3])
        h = self.mdblock("dec_conv4a", ot.deconv(h, Q["dec_conv3.W"]), [0, 2, 3])
        return self.head(self.deconv_bn_rect(h, "dec_conv4.W", "bnorm_dc4", True))

    def run(self, graph, x, z, eps, masks):
        """the encoder (x; x with eps), the MADE/IAF flow on both, the decoder on z; returns x_hat"""
        mu, ls = self.encode_mu_ls(x, graph)
        if graph != "simple":
            zs = [mu, mu + torch.exp(ls) * eps]
            self.made("l_IAF_mu", zs, masks)
            self.made("l_IAF_ls", zs, masks)
            self.report["latent_max_abs"] = max(float(ot.full_latent(self.Q, v, masks).abs().max()) for v in zs)
        self.report["exp_logsigma_max"] = float(torch.exp(ls).max())
        xh = self.decode(z, graph)
        self.report["saturated_fraction"] = float((xh.abs() >= 0.99).double().mean())
        self.report["x_hat_finite"] = bool(torch.isfinite(xh).all())
        return xh


_WEIGHTS = {}


def weights(graph, device="cpu"):
    """margin_weights of the graph's test checkpoint (the seed of tests/golden/ian_<graph>_golden.npz) on pool()"""
    if (graph, device) not in _WEIGHTS:
        from oracle import weights as ow
        make = {"simple": ow.make_simple_weights, "full": ow.make_full_weights, "v1": ow.make_v1_weights}[graph]
        seed = int(np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % graph))["weight_seed"])
        _WEIGHTS[(graph, device)] = margin_weights(graph, make(seed), pool(), device=device)
    return _WEIGHTS[(graph, device)]


def _inputs64(inp, device):
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64)).to(device)
    return t(inp["x"]), t(inp["z"]), t(inp["eps"])


@torch.no_grad()
def margin_weights(graph, P, inp, delta=DELTA, device="cpu"):
    """P (float32 numpy, a graph's checkpoint) with the knobs of the module docstring fitted to the pool inp (a dict with
    x, z, eps as pool() returns) -> float32 numpy weights"""
    Q = ot.to_torch(P, torch.float64)
    Q = {k: v.to(device) for k, v in Q.items()}
    x, z, eps = _inputs64(inp, device)
    _Walk(Q, True, delta).run(graph, x, z, eps, made_masks(device))
    return {k: (Q[k].cpu().numpy().astype(np.float32) if k in Q else v) for k, v in P.items()}


@torch.no_grad()
def certificate(graph, P, inp, device="cpu"):
    """the walk of margin_weights on P without changes: {knob: {min_margin, pos, neg}, head_max_arg, saturated_fraction,
    x_hat_finite, exp_logsigma_max, latent_max_abs}"""
    Q = {k: v.to(device) for k, v in ot.to_torch(P, torch.float64).items()}
    x, z, eps = _inputs64(inp, device)
    w = _Walk(Q, False, DELTA)
    w.run(graph, x, z, eps, made_masks(device))
    return w.report


@torch.no_grad()
def decoder_margin(graph, P, z, device="cpu"):
    """min over rectifiers of min s_c * pre for the decoder alone at latents z (the edit loop moves z off the pool)"""
    Q = {k: v.to(device) for k, v in ot.to_torch(P, torch.float64).items()}
    w = _Walk(Q, False, DELTA)
    w.decode(torch.from_numpy(np.asarray(z, np.float64)).to(device), graph)
    return min(v["min_margin"] for v in w.report.values() if isinstance(v, dict)), w.report.get("head_max_arg", 0.0)


# ---- bounds and metrics -------------------------------------------------------------------------------------------
# Per sample: relative L2 <= the first and max-abs / max|ref| <= the second bound of the path's kind.  Set from one run on
# an H100 80GB HBM3 at 700 W (worst of every sample, run and batch; the GPU results are the same bits on every rerun) and
# from the float64 discrimination floor of tests/test_margin_weights.py: the smallest move of any of the pool's 130
# samples when one backward operand is rounded to bf16.
#   decoder  (decoder VJP, grad)   worst 8.1e-5 / 7.4e-5; floor 5.2e-4 / 3.4e-4 (IAN.py's MDC block, samples 122 / 90)
#   encoder  (encoder VJP)         worst 2.1e-4 / 3.0e-4 (IAN_simple, whole tiles; flow graphs 1.0e-4 / 1.2e-4);
#                                  floor 1.58e-3 / 1.11e-3 (IAN_simple, samples 71 / 104)
#   edit     (the move of two edit-loop steps) worst 4.1e-4 / 1.2e-3: the float32 rounding of z itself, next to a move of
#            5e-3 to 1.3e-2, not a gradient error
# Each bound is at most a third of its floor.  The relative L2 bounds have >= 2x headroom over the worst sample; the max-abs
# bounds cannot have both: the decoder's has 1.5x, the encoder's 1.2x (2x would be within 3x of the floor).
BOUNDS = {"decoder": (1.7e-4, 1.1e-4), "encoder": (5.2e-4, 3.65e-4), "edit": (8.5e-4, 2.5e-3)}
# The edit-loop tests step with this weight: at NPE's 0.05 a step moves z by ~3e-4, near the float32 rounding of z itself;
# at 1.0 two steps move it by 5e-3 to 1.3e-2 and keep every rectifier >= 0.48 from its kink.
EDIT_WEIGHT = 1.0


def rel_l2(got, ref):
    """per-sample ||got - ref|| / ||ref||"""
    n = len(ref)
    d = (np.asarray(got, np.float64) - ref).reshape(n, -1)
    return np.linalg.norm(d, axis=1) / np.linalg.norm(np.asarray(ref, np.float64).reshape(n, -1), axis=1)


def rel_max(got, ref):
    """per-sample max|got - ref| / max|ref|"""
    n = len(ref)
    d = np.abs(np.asarray(got, np.float64) - ref).reshape(n, -1)
    return d.max(axis=1) / np.abs(np.asarray(ref, np.float64)).reshape(n, -1).max(axis=1)


def bf16_round(a):
    """float32 -> bfloat16 (round to nearest even) -> float32, in numpy"""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    return u.view(np.float32)


class _BF16Grad(torch.autograd.Function):
    """identity forward; the backward rounds the incoming gradient to bf16, as a single-pass bf16 tap-GEMM would round
    the operand of that layer's backward contraction"""

    @staticmethod
    def forward(ctx, t):
        return t.view_as(t)

    @staticmethod
    def backward(ctx, g):
        return torch.from_numpy(bf16_round(g.detach().cpu().numpy()).astype(np.float64)).to(g)


# ---- the float64 reference of every gradient path ------------------------------------------------------------------
class Oracle:
    """float64 torch autograd through the walk above (no fitting) on weights P, on `device`.  slip = "head", "block" or
    "enc" rounds one backward operand to bf16 (_BF16Grad): the head's backward GEMM (dec_out's on IAN_simple), the
    backward of dec_conv3a's second MDC conv (IAN.py) or of dec_conv2 (IANv1, IAN_simple), enc_conv3's adjoint."""

    def __init__(self, graph, P, device="cpu"):
        self.graph, self.device = graph, device
        self.Q = {k: v.to(device) for k, v in ot.to_torch(P, torch.float64).items()}
        self.masks = made_masks(device)

    def _t(self, a):
        return torch.from_numpy(np.asarray(a, np.float64)).to(self.device)

    def _walk(self, slip):
        w = _Walk(self.Q, False, DELTA)
        w.slip = slip
        return w

    def _decode(self, z, slip=None):
        return self._walk(slip).decode(z, self.graph)

    def _encode(self, x, eps=None, slip=None):
        mu, ls = self._walk(slip).encode_mu_ls(x, self.graph)
        z = mu if eps is None else mu + torch.exp(ls) * eps
        return z if self.graph == "simple" else ot.full_latent(self.Q, z, self.masks)

    def decode(self, z):
        with torch.no_grad():
            return self._decode(self._t(z)).cpu().numpy()

    def encode(self, x, eps=None):
        with torch.no_grad():
            return self._encode(self._t(x), None if eps is None else self._t(eps)).cpu().numpy()

    def decode_vjp(self, z, dx, slip=None):
        zt = self._t(z).requires_grad_(True)
        (g,) = torch.autograd.grad(self._decode(zt, slip), zt, self._t(dx))
        return g.cpu().numpy()

    def encode_vjp(self, x, dz, eps=None, slip=None):
        xt = self._t(x).requires_grad_(True)
        (g,) = torch.autograd.grad(self._encode(xt, None if eps is None else self._t(eps), slip), xt, self._t(dz))
        return g.cpu().numpy()

    def grads(self, z, boxes, targets):
        """per-sample brush gradients {kind: dz} of grad(z, boxes, target) for each target kind (None, (n,3), frames)"""
        zt = self._t(z).requires_grad_(True)
        xh = self._decode(zt)
        out = {}
        for name, tgt in targets.items():
            loss = 0.0
            for k in range(len(z)):
                c1, r1, c2, r2 = [int(v) for v in boxes[k]]
                patch = xh[k, :, r1:r2, c1:c2]
                if tgt is None:
                    loss = loss + patch.mean()
                elif tgt.ndim == 2:
                    loss = loss + ((self._t(tgt[k]).reshape(3, 1, 1) - patch) ** 2).mean()
                else:
                    loss = loss + ((self._t(tgt[k, :, r1:r2, c1:c2]) - patch) ** 2).mean()
            (g,) = torch.autograd.grad(loss, zt, retain_graph=True)
            out[name] = g.cpu().numpy()
        return out

    def edit(self, z, boxes, rgb, n_steps, weight=EDIT_WEIGHT):
        """the NPE step rule of edit_steps: z <- z - weight g (1 + (c2 - c1)), all in float64"""
        z = np.asarray(z, np.float64)
        fac = (1.0 + (boxes[:, 2] - boxes[:, 0]))[:, None]
        for _ in range(n_steps):
            z = z - weight * self.grads(z, boxes, {"t": rgb})["t"] * fac
        return z


def cotangents(n, seed):
    """three pixel-space cotangents per sample: a Gaussian, a soft mask (a smooth blob in [0, 1] times a colour) and a
    one-hot pixel"""
    rng = np.random.default_rng(seed)
    gauss = rng.standard_normal((n, 3, 64, 64)).astype(np.float32)
    yy, xx = np.mgrid[0:64, 0:64]
    soft = np.empty_like(gauss)
    onehot = np.zeros_like(gauss)
    for k in range(n):
        cy, cx, r = rng.uniform(8, 56), rng.uniform(8, 56), rng.uniform(4, 16)
        blob = 1.0 / (1.0 + np.exp(((yy - cy) ** 2 + (xx - cx) ** 2) ** 0.5 - r))
        soft[k] = blob[None] * rng.uniform(-1, 1, (3, 1, 1))
        onehot[k, k % 3, (7 * k + 5) % 64, (13 * k + 11) % 64] = 1.0
    return {"gauss": gauss, "soft": soft, "onehot": onehot}

"""CPU tests of the decoder vector-Jacobian product's oracle, dz = (d X_hat / d Z)^T dx (the reverse mode of reference
API.py:46 for any cotangent dx; include/ian_b200.h ian_decode_vjp_*):
  * the float64 numpy form (the IAN_simple decoder backward of oracle/ian_numpy.py fed dx * (1 - x_hat^2)) and float64
    torch autograd with grad_outputs=dx agree to 1e-10;
  * with the box-loss cotangent the VJP is imgrad / imgradRGB -- the gradients already pinned to the executed reference
    -- to 1e-12, on all three graphs;
  * one central-difference directional derivative per graph agrees to 1e-7 relative.
The two oracle functions live here (and in tests/test_gpu_decode_vjp.py) because they are three lines over the oracle's
public pieces."""
import os

import numpy as np
import pytest
import torch

from oracle import ian_numpy as on
from oracle import ian_torch as ot
from oracle import weights as ow

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def simple_decode_vjp(P, z, dx):
    """float64 numpy: the IAN_simple decoder backward of oracle/ian_numpy.py seeded with dx * (1 - x_hat^2)."""
    xh, cache = on.simple_decode(P, z, return_cache=True)
    return on._decoder_backward(P, cache, np.asarray(dx, np.float64) * (1 - xh ** 2))


def torch_decode_vjp(P, z, dx, decode_fn=None):
    """autograd of the torch restatement with grad_outputs=dx (run it on float64 parameters)."""
    z = z.clone().requires_grad_(True)
    (g,) = torch.autograd.grad((decode_fn or ot.decode)(P, z), z, grad_outputs=dx)
    return g


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def _seed(name):
    return int(np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % name))["weight_seed"])


GRAPHS = {"simple": (ow.make_simple_weights, ot.decode), "full": (ow.make_full_weights, ot.full_decode),
          "v1": (ow.make_v1_weights, ot.v1_decode)}


@pytest.fixture(scope="module")
def params():
    out = {}
    for name, (make, dec) in GRAPHS.items():
        P = make(_seed(name))
        out[name] = (P, ot.to_torch(P, torch.float64), dec)
    return out


def test_numpy_and_torch_vjp_agree(params):
    P, P64, dec = params["simple"]
    rng = np.random.default_rng(0)
    z = rng.standard_normal((2, 100))
    dx = rng.standard_normal((2, 3, 64, 64))
    a = simple_decode_vjp(P, z, dx)
    b = torch_decode_vjp(P64, torch.from_numpy(z), torch.from_numpy(dx), dec).numpy()
    assert a.shape == (2, 100) and _rel(a, b) <= 1e-10


@pytest.mark.parametrize("graph", ["simple", "full", "v1"])
def test_box_loss_cotangent_gives_the_brush_gradients(params, graph):
    P, P64, dec = params[graph]
    rng = np.random.default_rng(1)
    z = rng.standard_normal((1, 100))
    zt = torch.from_numpy(z)
    c1, r1, c2, r2 = 11, 7, 29, 20
    cnt = 3 * (r2 - r1) * (c2 - c1)
    frame = rng.uniform(-1, 1, (1, 3, 64, 64))
    xh = dec(P64, zt).numpy()
    light = np.zeros_like(xh)
    light[0, :, r1:r2, c1:c2] = 1.0 / cnt
    rgb = np.zeros_like(xh)
    rgb[0, :, r1:r2, c1:c2] = 2.0 * (xh[0, :, r1:r2, c1:c2] - frame[0, :, r1:r2, c1:c2]) / cnt
    g_light = ot.imgrad(P64, c1, r1, c2, r2, zt, decode_fn=dec).numpy()
    g_rgb = ot.imgradRGB(P64, c1, r1, c2, r2, torch.from_numpy(frame), zt, decode_fn=dec).numpy()
    assert _rel(torch_decode_vjp(P64, zt, torch.from_numpy(light), dec).numpy(), g_light) <= 1e-12
    assert _rel(torch_decode_vjp(P64, zt, torch.from_numpy(rgb), dec).numpy(), g_rgb) <= 1e-12
    if graph == "simple":
        assert _rel(simple_decode_vjp(P, z, light), on.simple_imgrad(P, c1, r1, c2, r2, z)) <= 1e-12
        assert _rel(simple_decode_vjp(P, z, rgb), on.simple_imgradRGB(P, c1, r1, c2, r2, frame, z)) <= 1e-12


@pytest.mark.parametrize("graph", ["simple", "full", "v1"])
def test_vjp_matches_central_differences(params, graph):
    """<dz, v> = d/dt <dx, decode(z + t v)> at t = 0, central differences in float64.  The flow graphs' Beta ratio
    2a/(a+b+1e-8) is steep where both sigmoids are small, so at some pixels the function bends on a 1e-6 scale: the check
    takes the closest of the step sizes 1e-6, 1e-7 and 1e-8 (on this input all three graphs reach <= 4e-8 at one of them)."""
    P, P64, dec = params[graph]
    rng = np.random.default_rng(4)
    z = torch.from_numpy(rng.standard_normal((1, 100)))
    v = torch.from_numpy(rng.standard_normal((1, 100)))
    dx = torch.from_numpy(rng.standard_normal((1, 3, 64, 64)))
    an = float((torch_decode_vjp(P64, z, dx, dec) * v).sum())
    rel = []
    with torch.no_grad():
        for h in (1e-6, 1e-7, 1e-8):
            fd = float(((dx * dec(P64, z + h * v)).sum() - (dx * dec(P64, z - h * v)).sum()) / (2 * h))
            rel.append(abs(an - fd) / abs(fd))
    assert min(rel) <= 1e-7, (an, rel)

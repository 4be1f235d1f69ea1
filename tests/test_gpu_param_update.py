"""GPU tests of in-place parameter updates of a finalized IAN_simple handle (ian_update_param_host, API.IAN.update_params)
and of the torch binding over the decoder's parameters (torch_ops.decoder_parameters, torch_ops.decode(model, z, params)).

  * A handle updated in place computes every entry point -- decode, grad, decode_vjp, the parameter VJP, the edit loop
    and a paint stroke -- bit for bit like a fresh handle finalized from the updated parameters, on both paths, and a
    CUDA graph captured before the update replays the new weights.
  * torch: the gradients of decode(model, z, params) equal the C-ABI's bit for bit; 20 Adam steps on a photo's
    reconstruction loss lower it; an edited tensor is re-uploaded and an untouched one is not; wrong dtype or device is
    refused.
  * errors: a name that cannot be updated, a wrong shape, IANv1.py."""
import numpy as np
import pytest

from oracle import weights as ow

from test_gpu_param_vjp import PARAM_VJP_NAMES, handles, path  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu
STATS = ["%s.%s" % (b, f) for b in ("bnorm_dec_fc2", "bnorm_dc1", "bnorm_dc2", "bnorm_dc3") for f in ("mean", "inv_std")]


def _perturbed(P, seed=3):
    rng = np.random.default_rng(seed)
    Q = {k: np.array(v) for k, v in P.items()}
    for k in PARAM_VJP_NAMES + STATS:
        f = np.exp(0.05 * rng.standard_normal(Q[k].shape)) if k.endswith("inv_std") else 1 + 0.05 * rng.standard_normal(Q[k].shape)
        Q[k] = (Q[k] * f).astype(np.float32)
    return Q


def _entry_points(m, rng_seed=4):
    rng = np.random.default_rng(rng_seed)
    z2, z40 = rng.standard_normal((2, 100)).astype(np.float32), rng.standard_normal((40, 100)).astype(np.float32)
    dx = rng.standard_normal((3, 3, 64, 64)).astype(np.float32)
    boxes = np.array([[3, 5, 20, 17], [40, 30, 41, 31], [0, 47, 64, 64]], np.int32)
    rgb = rng.uniform(-1, 1, (3, 3)).astype(np.float32)
    frame = rng.uniform(-1, 1, (1, 3, 64, 64)).astype(np.float32)
    recon = rng.integers(0, 256, (3, 64, 64)).astype(np.uint8)
    err = rng.uniform(-0.1, 0.1, (3, 64, 64)).astype(np.float32)
    out = {"decode2": m.sample_at(z2), "decode40": m.sample_at(z40), "grad": m.grad(z40[:3], boxes, rgb),
           "decode_vjp": m.decode_vjp(z40[:3], dx), "edit": m.edit_steps(z40[:3], boxes, rgb, n_steps=4)}
    dz, g = m.decode_param_vjp(z40[:3], dx)
    out["param_dz"] = dz
    out.update({"param_" + k: v for k, v in g.items()})
    z_new, im, disp = m.paint_stroke(z2[:1], (8, 8, 24, 20), frame, recon, err)
    out.update({"stroke_z": z_new, "stroke_im": im, "stroke_disp": disp})
    return out


def test_updated_handle_matches_fresh_handle(handles, weights, path):  # noqa: F811
    Q = _perturbed(weights)
    a = handles(IAN_PATH=path)
    before = _entry_points(a)                     # also captures the small-batch graphs with the old weights
    a.update_params({k: Q[k] for k in PARAM_VJP_NAMES + STATS})
    after, fresh = _entry_points(a), _entry_points(handles(Q, IAN_PATH=path))
    for k in fresh:
        assert np.array_equal(after[k], fresh[k]), k
    assert not np.array_equal(before["decode2"], after["decode2"])   # the replayed graph sees the new weights
    a.update_params({k: weights[k] for k in PARAM_VJP_NAMES + STATS})
    restored = _entry_points(a)
    for k in before:
        assert np.array_equal(restored[k], before[k]), k


def test_update_errors(npe, model, weights):
    with pytest.raises(npe.IanError):
        model.update_params({"enc_conv2.W": weights["enc_conv2.W"]})
    with pytest.raises(npe.IanError):
        model.update_params({"dec_conv2.W": weights["dec_conv2.W"][:, :128]})
    v1 = npe.IAN("IANv1.py", True, weights=ow.make_v1_weights(0))
    try:
        with pytest.raises(npe.IanError, match="IAN_simple only"):
            v1.update_params({"dec_conv2.W": np.zeros((512, 256, 5, 5), np.float32)})
    finally:
        v1.close()


def _torch_ops():
    import importlib
    return importlib.import_module("neural-photo-editor_b200.torch_ops")


def test_torch_gradients_equal_the_c_abi(handles, weights, path):  # noqa: F811
    import torch
    ops = _torch_ops()
    m = handles(IAN_PATH=path)
    params = ops.decoder_parameters(m, weights)
    rng = np.random.default_rng(6)
    z = rng.standard_normal((5, 100)).astype(np.float32)
    dx = rng.standard_normal((5, 3, 64, 64)).astype(np.float32)
    zt = torch.from_numpy(z).cuda().requires_grad_(True)
    x = ops.decode(m, zt, params)
    (x * torch.from_numpy(dx).cuda()).sum().backward()
    dz, g = m.decode_param_vjp(z, dx)
    assert np.array_equal(zt.grad.cpu().numpy(), dz)
    for k in PARAM_VJP_NAMES:
        assert np.array_equal(params[k].grad.cpu().numpy(), g[k]), k
    assert np.array_equal(x.detach().cpu().numpy(), m.sample_at(z))
    frozen = dict(params)
    frozen["dec_conv1.W"] = params["dec_conv1.W"].detach()          # does not require grad -> no gradient
    zt2 = torch.from_numpy(z).cuda()
    ops.decode(m, zt2, frozen).sum().backward()
    assert frozen["dec_conv1.W"].grad is None and params["dec_out.W"].grad is not None


def test_torch_adam_fine_tunes_the_decoder(handles, weights):  # noqa: F811
    import torch
    ops = _torch_ops()
    m = handles()
    params = ops.decoder_parameters(m, weights)
    rng = np.random.default_rng(7)
    z = torch.from_numpy(rng.standard_normal((4, 100)).astype(np.float32)).cuda()
    photo = torch.from_numpy(np.tanh(rng.standard_normal((4, 3, 64, 64))).astype(np.float32)).cuda()
    opt = torch.optim.Adam(params.values(), lr=1e-3)
    losses = []
    for _ in range(20):
        opt.zero_grad()
        loss = ((ops.decode(m, z, params) - photo) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    final = ((ops.decode(m, z, params) - photo) ** 2).mean().item()
    assert final < 0.9 * losses[0], (losses, final)


def test_torch_reuploads_only_edited_tensors(handles, weights):  # noqa: F811
    import torch
    ops = _torch_ops()
    m = handles()
    params = ops.decoder_parameters(m, weights)
    sent = []
    orig = m.update_params
    m.update_params = lambda d: (sent.append(sorted(d)), orig(d))
    z = torch.from_numpy(np.random.default_rng(8).standard_normal((2, 100)).astype(np.float32)).cuda()
    ops.decode(m, z, params)
    assert sent == []
    with torch.no_grad():
        params["dec_conv2.W"].mul_(1.01)
    x = ops.decode(m, z, params)
    assert sent == [["dec_conv2.W"]]
    Q = dict(weights)
    Q["dec_conv2.W"] = params["dec_conv2.W"].detach().cpu().numpy()
    assert np.array_equal(x.detach().cpu().numpy(), handles(Q).sample_at(z.cpu().numpy()))
    with pytest.raises(TypeError):
        ops.decode(m, z.double(), params)
    bad = dict(params)
    bad["dec_out.W"] = params["dec_out.W"].detach().cpu()
    with pytest.raises(TypeError):
        ops.decode(m, z, bad)

"""A batch keeps its samples apart: replacing some samples of a batch -- by other data, by extreme finite values, by a
NaN or an Inf -- never changes one bit of any other sample's result, on every batch entry point of all three graphs.

Nothing of the reference graphs mixes samples (inference BatchNorm), but the kernels put several images into one tile: a
128-row tap-GEMM tile holds 2 images of an 8x8 layer and 8 of a 4x4 layer, dense layers take 128 images per tile,
head_tc_kernel gives a CTA several (image, conv) items, dec_out / conv1_bwd run col2im on-chip, stream-K cuts tiles
across CTAs and host calls run in plan chunks of 512 (IAN_CHUNK).  A halo row of the next image, a tap or col2im index
across an image edge, or an out-of-image operand zeroed by a multiply (0 * NaN = NaN) instead of a select would show up
here and nowhere else: the oracle tests hold probe samples to bounds of 1e-4 - 1e-2 and feed no non-finite value.

The check needs no oracle.  Summation order depends on n and the layer shape, never on the data (the rerun tests of
tests/test_gpu_parity.py rely on it, and stream-K cuts K ranges by tile index), so at a fixed n and schedule every sample
that stays in place and unchanged must come back with the same bits.  A tracer batch is the clean batch with some probe
positions replaced; the tracer kinds, cycled over the entry point's inputs and the probe positions:
  new     another random sample;
  const   an image at constant +1 or -1 (images only);
  big     every pixel +-1e3, a latent scaled to max |z| = 1e3, a colour +-1e3;
  nan0 / nan1    one NaN at pixel (0, 0) / (63, 63) of one channel (where a halo or col2im leak starts), in latent 0 / 99;
  inf0 / ninf1   +Inf / -Inf placed the same way;
  corner0 / corner1   brush boxes (0,0,1,1) / (63,63,64,64); the device form also takes an empty box, whose gradient is
                      NaN (the reference's mean over an empty slice; the host form refuses an empty box).
Tracers sit on the even probe samples in one batch and on the odd ones in the next, so both sides of every tile, chunk
and CTA-round edge among the probes are a clean sample next to a tracer once.  Probes: tests/test_gpu_flow_scale.py's
(first, middle, last, both sides of every 128-image tile and of head_tc_kernel's CTA rounds) plus both sides of the
2- and 8-image tile edges and the chunk edges at the start, middle and end of the batch.

After the tracer calls the clean call is repeated on the same handle and must give the first clean call's bits, and a
fresh handle must give them too (default schedule at n = 3, and the chunked runs): nothing non-finite may stay in
split-K slabs, stream-K partial slots, the padded borders of activation planes or captured CUDA graphs.

Reference semantics checked on the way:
  - a frame target that is NaN outside every sample's box leaves grad and edit_steps bit-unchanged (the reference slices
    RGB[0,:,r1:r2,c1:c2] and never reads those pixels);
  - fit_latent on a target with a NaN (an Inf) keeps that sample's z bit-unchanged -- gn_solve_kernel rejects a
    non-finite step and gn_accept_kernel never accepts against a NaN / Inf error -- and its loss history is NaN (Inf);
  - a permuted batch comes back permuted bit for bit on whole tiles (IAN_SPLITK=0 IAN_STREAMK=0) and on the SIMT path;
    under forced stream-K a sample changes tile and so its K cut, and is held to the bounds that compare two schedules
    (test_permuted_batch).
Runs: every graph on the tensor-core path under the default, whole-tile and stream-K schedules and on the SIMT path,
IAN.py in bf16 mode, at n = 3 (the host form replays a CUDA graph), SMs/3 + 3 (47 on a 132-SM H100) and 130 as _plan
picks them, and IAN_CHUNK=16 at n = 40.  The fit entry points (one batch-100 decoder JVP per sample) run at n = 3 and,
chunked, at n = 20.  The device forms and the pipelined calls run at SMs/3 + 3."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_flow_scale import EPS_K, SCHEDULES, X_TOL, Z_K, _probes
from test_gpu_launch_forms import _Dev, _inputs, handle  # noqa: F401  (handle: the fixture)
from test_gpu_parity import X_RERUN, Z_RERUN

pytestmark = pytest.mark.gpu

GRAPHS = ("simple", "full", "v1")
KINDS = {"img": ("new", "const", "big", "nan0", "nan1", "inf0", "ninf1"),
         "lat": ("new", "big", "nan0", "nan1", "inf0", "ninf1"),
         "rgb": ("new", "big", "nan0", "nan1", "inf0", "ninf1"),
         "box": ("corner0", "corner1")}
INPUT_KIND = {"x": "img", "frame": "img", "dx": "img", "z": "lat", "eps": "lat", "dz": "lat", "rgb": "rgb", "boxes": "box"}


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- probes and tracers -------------------------------------------------------------------------------------------
def _probe_set(n, sms, chunk=512):
    """_probes plus both sides of the 2- and 8-image tile edges and of the chunk edges at the batch's start, middle
    and end"""
    s = set(_probes(n, sms))
    for t in (2, 8, chunk):
        for b in (t, (n // 2) // t * t, (n - 1) // t * t):
            if 0 < b < n:
                s |= {b - 1, b}
    return sorted(s)


def _apply(a, k, kind, rng):
    """replace sample k of input array `a` (in place) by a tracer of `kind`"""
    latent = a.ndim == 2 and a.shape[1] == 100
    first = (k, 0) if a.ndim == 2 else (k, k % 3, 0, 0)
    last = (k, a.shape[1] - 1) if a.ndim == 2 else (k, k % 3, 63, 63)
    if kind == "new":
        a[k] = rng.standard_normal(a.shape[1:]) if latent else rng.uniform(-1, 1, a.shape[1:])
    elif kind == "const":
        a[k] = 1.0 if k % 2 == 0 else -1.0
    elif kind == "big":
        a[k] = a[k] * (1e3 / np.abs(a[k]).max()) if latent else 1e3 * rng.choice([-1.0, 1.0], a.shape[1:])
    elif kind in ("nan0", "nan1"):
        a[first if kind == "nan0" else last] = np.nan
    elif kind == "inf0":
        a[first] = np.inf
    elif kind == "ninf1":
        a[last] = -np.inf
    elif kind == "corner0":
        a[k] = (0, 0, 1, 1)
    elif kind == "corner1":
        a[k] = (63, 63, 64, 64)
    elif kind == "empty":
        a[k] = (10, 20, 10, 30) if k % 2 == 0 else (5, 9, 21, 9)
    else:
        raise ValueError(kind)


def _trace(inp, names, positions, start, seed, kinds=KINDS):
    """the tracer batch: a copy of inp with sample positions[j] of input combos[start + j] replaced.  Returns the batch
    and {position: 'input:kind'}."""
    combos = [(nm, kd) for nm in names for kd in kinds[INPUT_KIND[nm]]]
    rng = np.random.default_rng(seed)
    out = dict(inp)
    for nm in names:
        out[nm] = inp[nm].copy()
    tags = {}
    for j, k in enumerate(positions):
        nm, kd = combos[(start + j) % len(combos)]
        _apply(out[nm], k, kd, rng)
        tags[k] = "%s:%s" % (nm, kd)
    return out, tags


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.reshape(len(a), -1).view(np.uint8)


def _changed(got, want):
    """samples whose result bits differ, over every output of the call"""
    bad = np.zeros(len(want[0]), bool)
    for g, w in zip(got, want):
        assert g.shape == w.shape and g.dtype == w.dtype, (g.shape, w.shape)
        bad |= (_bits(g) != _bits(w)).any(axis=1)
    return np.nonzero(bad)[0]


def _assert_isolated(what, got, want, tags):
    """every sample that is not a tracer has want's bits; the message names each changed sample and its nearest tracer"""
    moved = [int(k) for k in _changed(got, want) if k not in tags]
    if moved:
        tr = sorted(tags)
        near = lambda k: min(tr, key=lambda t: abs(t - k))
        desc = ["%d (nearest tracer %d = %s)" % (k, near(k), tags[near(k)]) for k in moved[:12]]
        pytest.fail("%s: clean samples changed: %s%s" % (what, ", ".join(desc), " ..." if len(moved) > 12 else ""))


def _assert_same(what, got, want):
    moved = _changed(got, want)
    assert len(moved) == 0, "%s: samples %s differ from the first clean call" % (what, moved[:12].tolist())


# ---- entry points ---------------------------------------------------------------------------------------------------
def _recon_no_z(m, x):
    """the host form without z_out (the API always passes one)"""
    xh = np.empty_like(x)
    m._check(m._lib.ian_reconstruct_host(m._h, x.ctypes.data_as(C.POINTER(C.c_float)), len(x), None,
                                         xh.ctypes.data_as(C.POINTER(C.c_float))))
    return (xh,)


def _fit_check(tin, tags, got):
    """a non-finite target: z stays the start's bits and the loss history is that non-finite value"""
    z, loss = got
    for k, tag in tags.items():
        nm, kd = tag.split(":")
        if nm != "x" or kd in ("new", "const", "big"):
            continue
        assert np.array_equal(_bits(z[k:k + 1]), _bits(tin["z"][k:k + 1])), ("fit_latent moved z", k, tag)
        if kd.startswith("nan"):
            assert np.isnan(loss[k]).all(), ("fit_latent loss", k, tag, loss[k])
        else:
            assert not np.isfinite(loss[k]).any(), ("fit_latent loss", k, tag, loss[k])


def _entries(graph, main, fit):
    """(name, traced inputs, call(m, inp) -> tuple of per-sample arrays, extra check or None) of the host-form batch
    entry points: all but the fit when `main`, gauss_newton and fit_latent when `fit`"""
    e = [("encode", ("x",), lambda m, d: (m.encode(d["x"]),), None),
         ("encode_eps", ("x", "eps"), lambda m, d: (m.encode(d["x"], d["eps"]),), None),
         ("sample_at", ("z",), lambda m, d: (m.sample_at(d["z"]),), None),
         ("reconstruct", ("x",), lambda m, d: m.reconstruct(d["x"], return_z=True), None),
         ("reconstruct_no_z", ("x",), lambda m, d: _recon_no_z(m, d["x"]), None)]
    for t in ("light", "rgb", "frame"):
        names = ("z", "boxes") + (() if t == "light" else (t,))
        tg = (lambda d: None) if t == "light" else (lambda d, t=t: d[t])
        e += [("grad_" + t, names, lambda m, d, tg=tg: (m.grad(d["z"], d["boxes"], tg(d)),), None),
              ("edit_" + t, names, lambda m, d, tg=tg: (m.edit_steps(d["z"], d["boxes"], tg(d), n_steps=2, weight=0.05),),
               None)]
    e += [("decode_vjp", ("z", "dx"), lambda m, d: (m.decode_vjp(d["z"], d["dx"]),), None),
          ("decode_jvp", ("z", "dz"), lambda m, d: m.decode_jvp(d["z"], d["dz"], return_x_hat=True), None),
          ("encode_vjp", ("x", "dz"), lambda m, d: (m.encode_vjp(d["x"], d["dz"]),), None),
          ("encode_vjp_eps", ("x", "dz", "eps"), lambda m, d: (m.encode_vjp(d["x"], d["dz"], d["eps"]),), None),
          ("encode_jvp", ("x", "dx"), lambda m, d: m.encode_jvp(d["x"], d["dx"], return_z=True), None),
          ("encode_jvp_eps", ("x", "dx", "eps"), lambda m, d: m.encode_jvp(d["x"], d["dx"], d["eps"], return_z=True), None)]
    if graph == "simple":
        e.append(("param_vjp_dz", ("z", "dx"), lambda m, d: (m.decode_param_vjp(d["z"], d["dx"])[0],), None))
    else:
        e += [("encode_pre", ("x",), lambda m, d: (m.Zfn(d["x"]),), None),
              ("flow", ("z",), lambda m, d: (m.Z_IAF_fn(d["z"]),), None),
              ("sample", ("z",), lambda m, d: (m.sample(d["z"]),), None),
              ("flow_vjp", ("z", "dz"), lambda m, d: (m.flow_vjp(d["z"], d["dz"]),), None),
              ("flow_jvp", ("z", "dz"), lambda m, d: m.flow_jvp(d["z"], d["dz"], return_z=True), None),
              ("encode_pre_vjp", ("x", "dz"), lambda m, d: (m.encode_pre_vjp(d["x"], d["dz"]),), None),
              ("encode_pre_jvp", ("x", "dx"), lambda m, d: m.encode_pre_jvp(d["x"], d["dx"], return_z=True), None)]
    if not main:
        e = []
    if fit:
        e += [("gauss_newton", ("z", "x"), lambda m, d: m.gauss_newton(d["z"], d["x"]), None),
              ("fit_latent", ("x", "z"), lambda m, d: m.fit_latent(d["x"], d["z"], iters=2, return_loss=True), _fit_check)]
    return e


def _outside_nan(inp):
    """the frame target with NaN at every pixel outside each sample's box"""
    f = np.full_like(inp["frame"], np.nan)
    for k, (c1, r1, c2, r2) in enumerate(inp["boxes"]):
        f[k, :, r1:r2, c1:c2] = inp["frame"][k, :, r1:r2, c1:c2]
    return f


def _isolation(m, graph, plan, sms, chunk=512):
    """plan: [(n, with_main, with_fit)].  Every entry point of the plan: the clean call, two tracer calls (clean samples
    keep their bits; the checks of the entry point on the tracers), then the clean call again (the first call's bits:
    nothing of the tracers stayed behind).  Returns {(name, n): clean result} for the fresh-handle check."""
    want_all = {}
    for n, with_main, with_fit in plan:
        inp = _inputs(n, 7100 + n)
        probes = _probe_set(n, sms, chunk)
        groups = [[k for k in probes if k % 2 == p] for p in (0, 1)]
        for name, names, call, check in _entries(graph, with_main, with_fit):
            want = call(m, inp)
            want_all[(name, n)] = want
            start = n
            for gi, pos in enumerate(groups):
                tin, tags = _trace(inp, names, pos, start, 100 * n + gi)
                start += len(pos)
                got = call(m, tin)
                _assert_isolated("%s n=%d tracers %d" % (name, n, gi), got, want, tags)
                if check is not None:
                    check(tin, tags, got)
            _assert_same("%s n=%d clean after tracers" % (name, n), call(m, inp), want)
            if name in ("grad_frame", "edit_frame"):
                out = dict(inp, frame=_outside_nan(inp))
                _assert_same("%s n=%d NaN frame outside the boxes" % (name, n), call(m, out), want)
    return want_all


def _fresh_equal(m, graph, want_all):
    calls = {e[0]: e[2] for e in _entries(graph, True, True)}
    for (name, n), want in want_all.items():
        _assert_same("%s n=%d fresh handle" % (name, n), calls[name](m, _inputs(n, 7100 + n)), want)


# ---- 1-3. tracers, every host entry point, every run ------------------------------------------------------------------
RUNS = [(g, s, "tc", "fp32") for g in GRAPHS for s in SCHEDULES] + [(g, "default", "simt", "fp32") for g in GRAPHS]
RUNS += [("full", "default", "tc", "bf16")]


def _plan(sched, path, sms):
    """[(n, with_main, with_fit)] of a run.  n = 3: the host form replays a CUDA graph, and the fit entry points run
    there; SMs/3 + 3: the ragged 2-image tile and head_tc_kernel's second CTA round; 130: the 128-image tile edge.  Trimmed
    so that the module takes about as long as tests/test_gpu_flow_scale.py: the default schedule (split-K and stream-K
    as the library chooses) runs n = 3 and 130, whole tiles, forced stream-K (every tap-GEMM but the head's cut at any
    n) and the SIMT path run SMs/3 + 3."""
    nm = sms // 3 + 3
    if sched == "default" and path == "tc":
        return [(3, True, True), (130, True, False)]
    return [(nm, True, False)]


@pytest.mark.parametrize("graph,sched,path,precision", RUNS, ids=["-".join(r) for r in RUNS])
def test_tracers_leave_other_samples_alone(handle, sms, graph, sched, path, precision):
    """the tracer batches of every host entry point; on the default schedule also a fresh handle at n = 3 (split-K
    slabs and captured graphs)"""
    m = handle(graph, path, precision, **SCHEDULES[sched])
    want = _isolation(m, graph, _plan(sched, path, sms), sms)
    m.close()
    if sched == "default" and path == "tc":
        want = {k: v for k, v in want.items() if k[1] == 3 and k[0] not in ("gauss_newton", "fit_latent")}
        _fresh_equal(handle(graph, path, precision), graph, want)


@pytest.mark.parametrize("graph", GRAPHS)
def test_tracers_across_plan_chunks(handle, sms, graph):
    """IAN_CHUNK=16: n = 40 runs as chunks of 16, 16 and 8, the fit entry points at n = 20 as 16 and 4"""
    m = handle(graph, "tc", "fp32", IAN_CHUNK=16)
    want = _isolation(m, graph, [(20, False, True), (40, True, False)], sms, chunk=16)
    m.close()
    _fresh_equal(handle(graph, "tc", "fp32", IAN_CHUNK=16), graph, want)


# ---- the device form --------------------------------------------------------------------------------------------------
def _dev_entries(graph):
    """(name, traced inputs, call(m, inp) -> tuple of numpy results) of the device forms"""
    def run(m, d, fn, outs):
        dev = _Dev()
        n = len(d["z"])
        t = [dev.empty((n,) + s) for s in outs]
        dev.run(lambda: fn(m, dev, n, [o.data_ptr() for o in t]))
        return tuple(o.cpu().numpy() for o in t)
    X, Z = (3, 64, 64), (100,)
    e = [("encode", ("x",), lambda m, d: run(m, d, lambda m, v, n, o: m.encode_dev(v.put(d["x"]), n, o[0]), [Z])),
         ("encode_eps", ("x", "eps"),
          lambda m, d: run(m, d, lambda m, v, n, o: m.encode_dev(v.put(d["x"]), n, o[0], v.put(d["eps"])), [Z])),
         ("decode", ("z",), lambda m, d: run(m, d, lambda m, v, n, o: m.decode_dev(v.put(d["z"]), n, o[0]), [X])),
         ("reconstruct", ("x",), lambda m, d: run(m, d, lambda m, v, n, o: m.reconstruct_dev(v.put(d["x"]), n, o[1], o[0]),
                                                  [X, Z])),
         ("decode_vjp", ("z", "dx"),
          lambda m, d: run(m, d, lambda m, v, n, o: m.decode_vjp_dev(v.put(d["z"]), v.put(d["dx"]), n, o[0]), [Z])),
         ("decode_jvp", ("z", "dz"),
          lambda m, d: run(m, d, lambda m, v, n, o: m.decode_jvp_dev(v.put(d["z"]), v.put(d["dz"]), n, o[0], o[1]), [X, X])),
         ("encode_vjp_eps", ("x", "dz", "eps"),
          lambda m, d: run(m, d, lambda m, v, n, o: m.encode_vjp_dev(v.put(d["x"]), v.put(d["dz"]), n, o[0], v.put(d["eps"])),
                           [X])),
         ("encode_jvp_eps", ("x", "dx", "eps"),
          lambda m, d: run(m, d, lambda m, v, n, o: m.encode_jvp_dev(v.put(d["x"]), v.put(d["dx"]), n, o[0], o[1],
                                                                     v.put(d["eps"])), [Z, Z]))]
    for t in ("light", "rgb", "frame"):
        names = ("z", "boxes") + (() if t == "light" else (t,))
        tg = (lambda d: None) if t == "light" else (lambda d, t=t: d[t])

        def grad(m, d, tg=tg):
            return run(m, d, lambda m, v, n, o: m.grad_dev(v.put(d["z"]), v.put(d["boxes"]), v.put(tg(d)),
                                                           int(tg(d) is not None and tg(d).ndim == 4), n, o[0]), [Z])

        def edit(m, d, tg=tg):
            dev = _Dev()
            zt = dev.empty(d["z"].shape, like=d["z"])
            tgt = tg(d)
            dev.run(lambda: m.edit_loop_dev(zt.data_ptr(), dev.put(d["boxes"]), dev.put(tgt),
                                            int(tgt is not None and tgt.ndim == 4), len(d["z"]), 2, 0.05))
            return (zt.cpu().numpy(),)
        e += [("grad_" + t, names, grad), ("edit_" + t, names, edit)]
    if graph != "simple":
        e += [("encode_pre", ("x",), lambda m, d: run(m, d, lambda m, v, n, o: m.Zfn_dev(v.put(d["x"]), n, o[0]), [Z])),
              ("flow", ("z",), lambda m, d: run(m, d, lambda m, v, n, o: m.flow_dev(v.put(d["z"]), n, o[0], o[1]), [Z, X])),
              ("flow_vjp", ("z", "dz"),
               lambda m, d: run(m, d, lambda m, v, n, o: m.flow_vjp_dev(v.put(d["z"]), v.put(d["dz"]), n, o[0]), [Z])),
              ("flow_jvp", ("z", "dz"),
               lambda m, d: run(m, d, lambda m, v, n, o: m.flow_jvp_dev(v.put(d["z"]), v.put(d["dz"]), n, o[0], o[1]), [Z, Z])),
              ("encode_pre_vjp", ("x", "dz"),
               lambda m, d: run(m, d, lambda m, v, n, o: m.encode_pre_vjp_dev(v.put(d["x"]), v.put(d["dz"]), n, o[0]), [X])),
              ("encode_pre_jvp", ("x", "dx"),
               lambda m, d: run(m, d, lambda m, v, n, o: m.encode_pre_jvp_dev(v.put(d["x"]), v.put(d["dx"]), n, o[0], o[1]),
                                [Z, Z]))]
    return e


@pytest.mark.parametrize("graph", GRAPHS)
def test_device_form_tracers(handle, sms, graph):
    """the device forms at n = SMs/3 + 3, also with empty boxes (a NaN gradient for that sample)"""
    n = sms // 3 + 3
    inp = _inputs(n, 7300 + n)
    probes = _probe_set(n, sms)
    kinds = dict(KINDS, box=("corner0", "empty", "corner1"))
    m = handle(graph, "tc", "fp32")
    for name, names, call in _dev_entries(graph):
        want = call(m, inp)
        for gi, pos in enumerate([k for k in probes if k % 2 == p] for p in (0, 1)):
            tin, tags = _trace(inp, names, pos, 3 * gi, 300 + gi, kinds)
            got = call(m, tin)
            _assert_isolated("%s (device form) tracers %d" % (name, gi), got, want, tags)
            if name.startswith("grad_"):
                for k, tag in tags.items():
                    if tag == "boxes:empty":
                        assert np.isnan(got[0][k]).all(), (name, k, "empty box: NaN gradient")
            _assert_same("%s (device form) clean after tracers %d" % (name, gi), call(m, inp), want)


# ---- pipelining -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", GRAPHS)
def test_pipelined_tracer_batches(handle, sms, graph):
    """reconstruct_stream / reconstruct_submit with tracer batches between clean ones: every clean batch gives its
    synchronous call's bits, every tracer batch its clean samples' bits"""
    n = sms // 3 + 3
    inp = _inputs(n, 7400 + n)
    probes = _probe_set(n, sms)
    m = handle(graph, "tc", "fp32")
    want = m.reconstruct(inp["x"], return_z=True)
    batches, tags = [], []
    for j in range(5):
        if j % 2 == 0:
            batches.append(inp["x"])
            tags.append(None)
        else:
            tin, tg = _trace(inp, ("x",), [k for k in probes if k % 2 == j // 2], 5 * j, 400 + j)
            batches.append(tin["x"])
            tags.append(tg)
    for j, xh in enumerate(m.reconstruct_stream(batches)):
        got = (xh.copy(),)
        if tags[j] is None:
            _assert_same("reconstruct_stream batch %d" % j, got, want[:1])
        else:
            _assert_isolated("reconstruct_stream batch %d" % j, got, want[:1], tags[j])
    outs = [(m.pinned_empty((n, 3, 64, 64)), m.pinned_empty((n, 100))) for _ in batches]
    pending = []
    for j, x in enumerate(batches):                        # two tickets in flight
        pending.append((j, m.reconstruct_submit(x, outs[j][0], outs[j][1])))
        if len(pending) == 2:
            jj, t = pending.pop(0)
            m.reconstruct_wait(t)
    for jj, t in pending:
        m.reconstruct_wait(t)
    for j in range(len(batches)):
        got = (outs[j][0].copy(), outs[j][1].copy())
        if tags[j] is None:
            _assert_same("reconstruct_submit ticket %d" % j, got, want)
        else:
            _assert_isolated("reconstruct_submit ticket %d" % j, got, want, tags[j])


# ---- 4. permutation ---------------------------------------------------------------------------------------------------
FORWARD = ("encode", "encode_eps", "sample_at", "reconstruct", "reconstruct_no_z")


@pytest.mark.parametrize("graph", GRAPHS)
def test_permuted_batch(handle, sms, graph):
    """a permuted batch comes back permuted: bit for bit on whole tiles (every entry point) and on the SIMT path (the
    forward).  Under forced stream-K a sample's K cut follows its tile, so there the forward is held to the bounds
    that compare two schedules: X_RERUN / Z_RERUN of test_gpu_parity on IAN_simple, test_gpu_flow_scale's X_TOL and
    Z_K (1 + |z|) on the flow graphs, and for encode with eps its EPS_K (1 + |z| + |exp(logsigma) eps|), since eps
    multiplies the change of logsigma.  Measured with the default schedule at n = 47: IAN.py's sample_at moves by
    8.4e-5 (above X_RERUN), encode with eps by 1.3e-3 - 1.9e-3."""
    n = sms // 3 + 3
    inp = _inputs(n, 7500 + n)
    perm = np.random.default_rng(n).permutation(n)
    pin = {k: v[perm] for k, v in inp.items()}
    xtol, zk = (X_RERUN, 0.0) if graph == "simple" else (X_TOL, Z_K)
    for sched, path in (("whole", "tc"), ("default", "simt"), ("sk", "tc")):
        m = handle(graph, path, "fp32", **SCHEDULES[sched])
        got = {}
        for name, _, call, _ in _entries(graph, True, False):
            if sched != "whole" and name not in FORWARD:
                continue
            want = tuple(a[perm] for a in call(m, inp))
            got[name] = call(m, pin)
            if sched == "whole" or path == "simt":
                _assert_same("%s %s/%s permuted" % (name, sched, path), got[name], want)
                continue
            for g, w in zip(got[name], want):
                if name == "encode_eps":
                    bound = EPS_K * (1.0 + np.abs(w) + np.abs(w - got["encode"][0]))
                elif g.ndim == 2:
                    bound = np.maximum(Z_RERUN, zk * (1.0 + np.abs(w)))
                else:
                    bound = xtol
                assert (np.abs(g - w) <= bound).all(), (name, sched, path, "permuted", float(np.abs(g - w).max()))
        m.close()

"""The flow graphs (IAN.py, IANv1.py) at production batch sizes, under every tap-GEMM schedule, both CUDA paths and both
precisions.  The other flow-graph GPU tests run n <= 4, where every MDC block layer is split-K and its epilogue runs only
in splitk_finalize_kernel, and where head_tc_kernel never gives a CTA a second (image, conv) item.

Three handles per graph, built with the schedule in the environment:
  default  the library's own choice: split-K for layers with <= 74 output tiles (mark_splitk_candidates, choose_ksplit),
           stream-K where launch_tapgemm_tc's makespan test asks for it (ksplit 1, >= SMs/2 tiles of 128 columns);
  whole    IAN_SPLITK=0 IAN_STREAMK=0: every tap-GEMM runs whole tiles, the epilogue in tapgemm_tc_kernel;
  sk       IAN_SPLITK=0 IAN_STREAMK=2: every tap-GEMM but the head's runs stream-K, the epilogue in the finisher CTA.
n_multi = SMs // 3 + 3 (47 on a 132-SM H100): odd, so the last 8x8 MDC tile (2 images per tile) is ragged, and the
head's items 3n > SMs, so CTAs 0 .. 3n - SMs - 1 run a second item (weight-buffer hand-off, A-ring counter carried
over, accumulator reset per item).

Which epilogue runs where (IAN.py; S split-K + finalize kernel, W whole tiles in tapgemm_tc_kernel, H whole or
stream-K as the makespan test decides, K stream-K forced; fp32 mode = <128, 3, *> instances, bf16 = <128, 1, *>):
  layer group                                   n<=4   n_multi   128/130   512    whole   sk
  enc_fc1, enc_head                             S      S         S         S      W       K
  enc_conv4, bwd_conv1                          S      S         S/H       H      W       K
  dec_fc2 (2 K steps: ksplit stays 1)           W      W         W/H       H      W       K
  dec_conv1 + md1a/b (out_raw; res before BN)   S      H         H         H      W       K
  dec_conv2/3 + md2/md3 (out_raw; res)          S      H         H         H      W       K
  bwd md*a (res_after, mask slope 0.2)          S      md1: H    H         H      W       K
  head GEMM (tile table out_f32_t)              W      W         W         W      W       W
No layer has Cout = 16, so launch_one<16, ...> is unreachable and not tested here.  IANv1 has the same encoder and a
plain deconv decoder (no out_raw / res / res_after); its layers fall in the same columns by tile count.

Bounds are the standing ones of tests/test_gpu_full.py (x_hat max-abs 2e-4; z |dz| <= 3e-4 (1 + |z|); encode with eps
1e-3 (1 + |z| + |exp(logsigma) eps|)), of test_flow_model_brush_gradients for IANv1 brush gradients (max-abs / max|g|
<= 2e-2 per case, half of the cases <= 1e-4: a ReLU flip inside the box moves one case by 0.3-1 %), and of bench.py's
bf16 line (max-abs 0.1, mean-abs 5e-3).  IAN.py brush gradients are held to every case <= 5e-2 (the flow-graph bound
of tests/test_gpu_decode_vjp.py) and a median <= 5e-3, not to the 1e-3 its three fixed cases meet in
test_flow_model_brush_gradients: on random latents and boxes the box-loss gradient crosses LeakyRectify kinks and the
steep Beta ratio the same way the dense VJP does (DESIGN section 5.6c).  In float64 alone, moving z so that x_hat moves
by 6e-6 -- 30x less than the float32 forward is allowed -- moves the gradient of a 1x1 box by 1.8e-3 and that of a
17x12 box by 7.8e-4; two float32 GPU runs that differ only in summation order (the chunked test) differ by up to 3.8e-2.  The float64 oracle (oracle/ian_torch.py, oracle/ian_full_numpy.py)
runs on probe samples -- first, middle, last, both sides of every 128-image dense tile, of the head's first and second
CTA rounds and of every plan chunk -- and is computed once per (graph, inputs); every schedule, path and precision is
compared with the same values.  Schedules and paths are compared with each other on every sample.
Measured values go to flow_scale_parity.json when IAN_TEST_RECORD names a directory."""
import json
import os

import numpy as np
import pytest

from oracle import ian_full_numpy as fn
from oracle import weights as ow

import scale_inputs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
X_TOL, Z_K, EPS_K, BF16_MAX, BF16_MEAN = 2e-4, 3e-4, 1e-3, 0.1, 5e-3
CONFIG = {"full": "IAN.py", "v1": "IANv1.py"}
SCHEDULES = {"default": {}, "whole": {"IAN_SPLITK": "0", "IAN_STREAMK": "0"}, "sk": {"IAN_SPLITK": "0", "IAN_STREAMK": "2"}}
ENV = ("IAN_STREAMK", "IAN_SPLITK", "IAN_GRAPHS", "IAN_PDL", "IAN_FINALIZE8", "IAN_CHUNK", "IAN_PATH")
RECORD = {}


def _record(key, value):
    RECORD[key] = value
    if os.environ.get("IAN_TEST_RECORD"):
        os.makedirs(os.environ["IAN_TEST_RECORD"], exist_ok=True)
        with open(os.path.join(os.environ["IAN_TEST_RECORD"], "flow_scale_parity.json"), "w") as f:
            json.dump(RECORD, f, indent=1, sort_keys=True)


_WEIGHTS = {}


def _weights(graph):
    if graph not in _WEIGHTS:
        seed = int(np.load(os.path.join(ROOT, "tests", "golden", "ian_%s_golden.npz" % graph))["weight_seed"])
        _WEIGHTS[graph] = (ow.make_full_weights if graph == "full" else ow.make_v1_weights)(seed)
    return _WEIGHTS[graph]


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _n(nkey, sms):
    return sms // 3 + 3 if nkey == "multi" else int(nkey)


@pytest.fixture
def handles(npe, monkeypatch):
    """make(graph, **env) builds a handle with exactly `env` set among the library's schedule variables; every handle
    made is closed when the test ends, so plans of large batches do not outlive their test."""
    made = []

    def make(graph, **env):
        for k in ENV:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, str(v))
        try:
            m = npe.IAN(CONFIG[graph], True, weights=_weights(graph))
        finally:
            for k in env:
                monkeypatch.delenv(k, raising=False)
        made.append(m)
        return m
    try:
        yield make
    finally:
        for m in made:
            m.close()


# ---- inputs and probes ----------------------------------------------------------------------------------------------
_inputs = scale_inputs.inputs


def _probes(n, sms):
    """first, middle, last (alone in the ragged last 8x8 tile when n is odd) and both sides of every 128-image dense
    tile and of head_tc_kernel's second and third CTA rounds.  Chunk edges: test_chunked_batch."""
    s = {0, n // 2, n - 1, n - 2}
    for b in range(128, n, 128):
        s |= {b - 1, b}
    for r in (1, 2):
        b = (r * sms + 2) // 3                               # the first image with an item in CTA round r + 1
        s |= {b - 1, b}
    return sorted(k for k in s if 0 <= k < n)


def _targets(inp):
    return {"light": None, "colour": inp["rgb"], "frame": inp["frame"]}


# ---- float64 oracle, cached per (graph, inputs) --------------------------------------------------------------------
class _Oracle:
    def __init__(self, graph):
        import torch
        from oracle import ian_torch as ot
        self.torch, self.ot = torch, ot
        self.P = _weights(graph)
        self.P64 = ot.to_torch(self.P, torch.float64)
        self.masks = fn.made_masks(fn.made_ordering())
        self.masks_t = [torch.from_numpy(m.astype(np.float64)) for m in self.masks]
        self.dec = ot.full_decode if graph == "full" else ot.v1_decode

    def _t(self, a):
        return self.torch.from_numpy(np.asarray(a, np.float64))

    def encode(self, x, eps=None):
        """l_Z of encode_images; with eps also (l_Z of encode(x, eps), |exp(logsigma) eps|) from the same encoder pass"""
        with self.torch.no_grad():
            mu, ls = self.ot.full_encode_mu_ls(self.P64, self._t(x))
            z = self.ot.full_latent(self.P64, mu, self.masks_t).numpy()
            if eps is None:
                return z
            amp = self.torch.exp(ls) * self._t(eps)
            zeps = self.ot.full_latent(self.P64, mu + amp, self.masks_t).numpy()
            return z, zeps, np.abs(amp.numpy())

    def mu(self, x):
        with self.torch.no_grad():
            return self.ot.full_encode_mu_ls(self.P64, self._t(x))[0].numpy()

    def latent(self, z_iaf):
        return fn.full_latent(self.P, np.asarray(z_iaf, np.float64), self.masks)

    def decode(self, z):
        with self.torch.no_grad():
            return self.dec(self.P64, self._t(z)).numpy()

    def grads(self, z, boxes, targets):
        """per-sample brush gradients for every target kind: one float64 forward, one backward per kind (the samples
        are independent, so the gradient of the summed loss is each sample's own)."""
        torch = self.torch
        zt = self._t(z).requires_grad_(True)
        xh = self.dec(self.P64, zt)
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
            out[name] = g.numpy()
        return out


_ORACLES, _CACHE = {}, {}


def _oracle(graph):
    if graph not in _ORACLES:
        _ORACLES[graph] = _Oracle(graph)
    return _ORACLES[graph]


def _cached(key, fn_):
    if key not in _CACHE:
        _CACHE[key] = fn_()
    return _CACHE[key]


def _forward_ref(graph, n, seed, probe):
    def make():
        o, inp = _oracle(graph), _inputs(n, seed)
        z, zeps, amp = o.encode(inp["x"][probe], inp["eps"][probe])
        return {"z": z, "zeps": zeps, "amp": amp, "xh": o.decode(inp["z"][probe])}
    return _cached((graph, "fwd", n, seed, tuple(probe)), make)


def _grad_ref(graph, n, seed, probe):
    def make():
        inp = _inputs(n, seed)
        tg = {k: (None if v is None else v[probe]) for k, v in _targets(inp).items()}
        return _oracle(graph).grads(inp["z"][probe], inp["boxes"][probe], tg)
    return _cached((graph, "grad", n, seed, tuple(probe)), make)


# ---- comparisons ------------------------------------------------------------------------------------------------------
def _zerr(z, ref, k=Z_K):
    """the largest |dz| / (1 + |z_ref|), to be held <= k"""
    return float((np.abs(z - ref) / (1.0 + np.abs(ref))).max())


def _xerr(x, ref):
    return float(np.abs(x - ref).max())


def _grad_rel(g, ref):
    n = len(ref)
    return np.abs(g - ref).reshape(n, -1).max(axis=1) / np.abs(ref).reshape(n, -1).max(axis=1)


def _assert_grads(graph, rel, what):
    """per-case max-abs / max|g| (module docstring): IAN.py every case <= 5e-2 and the median <= 5e-3; IANv1 every case
    <= 2e-2 and at least half of the cases <= 1e-4"""
    rel = np.asarray(rel)
    if graph == "full":
        assert rel.max() <= 5e-2 and np.median(rel) <= 5e-3, (what, rel)
    else:
        assert rel.max() <= 2e-2 and (rel <= 1e-4).sum() * 2 >= rel.size, (what, rel)


def _box_cotangent(xh, boxes, target):
    """the box loss's dL/dx_hat in float32, formed exactly as the seed kernels form it"""
    dx = np.zeros_like(xh)
    for k, (c1, r1, c2, r2) in enumerate(boxes):
        inv = np.float32(1) / np.float32(3 * (r2 - r1) * (c2 - c1))
        if target is None:
            dx[k, :, r1:r2, c1:c2] = inv
        else:
            t = target[k].reshape(3, 1, 1) if target.ndim == 2 else target[k, :, r1:r2, c1:c2]
            dx[k, :, r1:r2, c1:c2] = (np.float32(2) * inv) * (xh[k, :, r1:r2, c1:c2] - t)
    return dx


def _forward(m, inp):
    xr, zr = m.reconstruct(inp["x"], return_z=True)
    return {"z": m.encode_images(inp["x"]), "zeps": m.encode(inp["x"], eps=inp["eps"]), "xh": m.sample_at(inp["z"]),
            "xr": xr, "zr": zr}


# ---- 1. forward at scale --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph,nkey", [("full", "multi"), ("full", 130), ("full", 512), ("v1", "multi"), ("v1", 130)])
def test_forward_at_scale(handles, sms, graph, nkey):
    n = _n(nkey, sms)
    seed = 1000 + n
    inp, probe = _inputs(n, seed), _probes(n, sms)
    ref = _forward_ref(graph, n, seed, probe)
    scheds = ["default"] if n == 512 else list(SCHEDULES)
    hs = {s: handles(graph, **SCHEDULES[s]) for s in scheds}
    runs, rec = {}, {}
    for s, path in [(s, "tc") for s in scheds] + [("default", "simt")]:
        m = hs[s]
        m.set_path(path)
        try:
            out = _forward(m, inp)
            again = _forward(m, inp)
            for k in out:
                assert np.array_equal(out[k], again[k]), (s, path, k, "rerun")
            xs = m.sample_at(out["zr"])
        finally:
            m.set_path("tc")
        e = {"z": _zerr(out["z"][probe], ref["z"]), "zr": _zerr(out["zr"][probe], ref["z"]),
             "xh": _xerr(out["xh"][probe], ref["xh"]), "recon_vs_decode": _xerr(out["xr"], xs),
             "zeps": float((np.abs(out["zeps"][probe] - ref["zeps"]) / (1.0 + np.abs(ref["zeps"]) + ref["amp"])).max())}
        rec["%s_%s" % (s, path)] = e
        assert e["z"] <= Z_K and e["zr"] <= Z_K and e["zeps"] <= EPS_K, (s, path, e)
        assert e["xh"] <= X_TOL and e["recon_vs_decode"] <= X_TOL, (s, path, e)
        runs[(s, path)] = out
    base = runs[("default", "tc")]
    amp = np.abs(base["zeps"] - base["z"])
    for (s, path), out in runs.items():
        c = {"z": _zerr(out["z"], base["z"]), "zr": _zerr(out["zr"], base["zr"]), "xh": _xerr(out["xh"], base["xh"]),
             "xr": _xerr(out["xr"], base["xr"]),
             "zeps": float((np.abs(out["zeps"] - base["zeps"]) / (1.0 + np.abs(base["zeps"]) + amp)).max())}
        rec["%s_%s_vs_default_all" % (s, path)] = c
        assert c["z"] <= Z_K and c["zr"] <= Z_K and c["zeps"] <= EPS_K, (s, path, c)
        assert c["xh"] <= X_TOL and c["xr"] <= X_TOL, (s, path, c)
    _record("forward_%s_n%d" % (graph, n), rec)


# ---- 2. brush gradients, edit loop and VJP at scale -----------------------------------------------------------------
@pytest.mark.parametrize("nkey", ["multi", 128])
@pytest.mark.parametrize("graph", ["full", "v1"])
def test_brush_gradients_at_scale(handles, sms, graph, nkey):
    n = _n(nkey, sms)
    seed = 2000 + n
    inp, probe = _inputs(n, seed), _probes(n, sms)
    z, boxes, targets = inp["z"], inp["boxes"], _targets(inp)
    ref = _grad_ref(graph, n, seed, probe)
    rec = {}
    for s, env in SCHEDULES.items():
        m = handles(graph, **env)
        try:
            for precision in ("fp32", "bf16"):
                m.set_precision(precision)
                xh = m.sample_at(z)
                g = {t: m.grad(z, boxes, tgt) for t, tgt in targets.items()}
                for t, tgt in targets.items():
                    dz = m.decode_vjp(z, _box_cotangent(xh, boxes, tgt))
                    assert np.array_equal(dz, g[t]), (s, precision, t, "box-cotangent VJP == grad")
                assert np.array_equal(g["colour"], m.grad(z, boxes, inp["rgb"])), (s, precision, "rerun")
                if precision == "bf16":
                    continue
                rel = {t: _grad_rel(g[t][probe], ref[t]) for t in targets}
                rec["%s_grad" % s] = {t: v.tolist() for t, v in rel.items()}
                _record("grad_%s_n%d" % (graph, n), rec)
                _assert_grads(graph, np.concatenate(list(rel.values())), (s, rel))
                # the NPE step rule: edit steps equal manual gradient steps.  One step at the bound of
                # test_flow_model_brush_gradients; after two, a 1-ulp difference in the first step's z can cross a kink
                # of IAN.py's second gradient (module docstring), so IAN.py's second step is held relative to the move.
                zm = [z]
                for _ in range(2):
                    zm.append((zm[-1] - np.float32(0.05) * m.grad(zm[-1], boxes, inp["rgb"]) * (1.0 + (boxes[:, 2] - boxes[:, 0]))[:, None]).astype(np.float32))
                z1, z2 = (m.edit_steps(z, boxes, inp["rgb"], n_steps=k, weight=0.05) for k in (1, 2))
                e1, e2 = float(np.abs(z1 - zm[1]).max()), np.abs(z2 - zm[2]).max(axis=1)
                move = np.abs(zm[2] - z).max(axis=1)
                rec["%s_edit" % s] = {"step1": e1, "step2": float(e2.max()), "step2_over_move": float((e2 / move).max())}
                assert e1 <= 1e-5 * max(1.0, np.abs(zm[1]).max()), (s, rec["%s_edit" % s])
                if graph == "full":
                    assert (e2 <= 2e-2 * move).all(), (s, rec["%s_edit" % s])
                else:
                    assert e2.max() <= 1e-5 * max(1.0, np.abs(zm[2]).max()), (s, rec["%s_edit" % s])
        finally:
            m.set_precision("fp32")
            m.close()
    _record("grad_%s_n%d" % (graph, n), rec)


# ---- 3. bf16 mode -----------------------------------------------------------------------------------------------------
def _bf16_stats(a, b):
    d = np.abs(a - b)
    return float(d.max()), float(d.mean())


def _assert_bf16(stats, what):
    assert stats[0] <= BF16_MAX and stats[1] <= BF16_MEAN, (what, stats)


def test_bf16_full_batch512(handles, sms):
    """BASELINE configs[2]: IAN.py at batch 512 on the default schedule, bf16 mode against float32 mode on every sample
    and against the float64 oracle on the probes."""
    n = 512
    seed = 1000 + n
    inp, probe = _inputs(n, seed), _probes(n, sms)
    ref = _forward_ref("full", n, seed, probe)
    m = handles("full")
    x32 = m.sample_at(inp["z"])
    m.set_precision("bf16")
    x16 = m.sample_at(inp["z"])
    assert np.array_equal(x16, m.sample_at(inp["z"])), "bf16 rerun"
    xr16 = m.reconstruct(inp["x"])
    assert np.array_equal(xr16, m.reconstruct(inp["x"])), "bf16 reconstruct rerun"
    rec = {"vs_fp32_all": _bf16_stats(x16, x32), "vs_oracle_probes": _bf16_stats(x16[probe], ref["xh"]),
           "fp32_vs_oracle_probes": _xerr(x32[probe], ref["xh"])}
    _record("bf16_full_n512", rec)
    _assert_bf16(rec["vs_fp32_all"], "bf16 vs fp32")
    _assert_bf16(rec["vs_oracle_probes"], "bf16 vs oracle")
    assert np.isfinite(xr16).all()
    assert rec["fp32_vs_oracle_probes"] <= X_TOL, rec


@pytest.mark.parametrize("graph", ["full", "v1"])
def test_bf16_whole_tiles_and_stream_k_agree(handles, sms, graph):
    """n_multi in bf16 mode: tapgemm_tc_kernel<128, 1, false> (whole) against <128, 1, true> (stream-K), both against the
    oracle on the probes; reruns bit-identical.  IAN.py also checks the box-cotangent VJP == grad identity in bf16 here."""
    n = _n("multi", sms)
    seed = 1000 + n
    inp, probe = _inputs(n, seed), _probes(n, sms)
    ref = _forward_ref(graph, n, seed, probe)
    out, rec = {}, {}
    for s in ("whole", "sk"):
        m = handles(graph, **SCHEDULES[s])
        m.set_precision("bf16")
        out[s] = m.sample_at(inp["z"])
        assert np.array_equal(out[s], m.sample_at(inp["z"])), (s, "rerun")
        xr, zr = m.reconstruct(inp["x"], return_z=True)
        xr2, zr2 = m.reconstruct(inp["x"], return_z=True)
        assert np.array_equal(xr, xr2) and np.array_equal(zr, zr2), (s, "reconstruct rerun")
        rec[s + "_vs_oracle"] = _bf16_stats(out[s][probe], ref["xh"])
        _assert_bf16(rec[s + "_vs_oracle"], (s, "vs oracle"))
        m.close()
    rec["whole_vs_sk"] = _bf16_stats(out["whole"], out["sk"])
    _record("bf16_schedules_%s_n%d" % (graph, n), rec)
    _assert_bf16(rec["whole_vs_sk"], "whole vs sk")


# ---- 4. launch forms: exact -------------------------------------------------------------------------------------------
def _calls(inp):
    """every host entry point the flow graphs capture into CUDA graphs, as (name, call) pairs"""
    x, z, boxes, rgb, frame = inp["x"], inp["z"], inp["boxes"], inp["rgb"], inp["frame"]
    dx = np.random.default_rng(len(z)).standard_normal(x.shape).astype(np.float32)
    return [("reconstruct", lambda m: m.reconstruct(x, return_z=True)), ("encode_images", lambda m: m.encode_images(x)),
            ("sample_at", lambda m: m.sample_at(z)), ("grad_light", lambda m: m.grad(z, boxes, None)),
            ("grad_colour", lambda m: m.grad(z, boxes, rgb)), ("grad_frame", lambda m: m.grad(z, boxes, frame)),
            ("edit_steps", lambda m: m.edit_steps(z, boxes, rgb, n_steps=2)), ("decode_vjp", lambda m: m.decode_vjp(z, dx))]


def _equal(a, b):
    if isinstance(a, tuple):
        return all(np.array_equal(u, v) for u, v in zip(a, b))
    return np.array_equal(a, b)


def _launch_forms(handles, graph, precision, ref_env, other_env, sizes, reps):
    ref_m, other = handles(graph, **ref_env), handles(graph, **other_env)
    for m in (ref_m, other):
        m.set_precision(precision)
    for n in sizes:
        inp = _inputs(n, 3000 + n)
        for name, call in _calls(inp):
            want = call(ref_m)
            for rep in range(reps):                       # with graphs on: the capture call, then replays
                assert _equal(want, call(other)), (graph, precision, n, name, rep)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("graph", ["full", "v1"])
def test_graph_replay_equals_plain_launches(handles, graph, precision):
    _launch_forms(handles, graph, precision, {"IAN_GRAPHS": "0"}, {}, (1, 6, 32), 3)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("graph", ["full", "v1"])
def test_pdl_equals_plain_launches(handles, sms, graph, precision):
    _launch_forms(handles, graph, precision, {"IAN_GRAPHS": "0", "IAN_PDL": "0"}, {"IAN_GRAPHS": "0"},
                  (5, _n("multi", sms), 130), 2)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("graph", ["full", "v1"])
def test_sequential_finalize_equals_cooperative(handles, graph, precision):
    _launch_forms(handles, graph, precision, {}, {"IAN_FINALIZE8": "0"}, (1, 5), 2)


# ---- 5. plan chunks and the flow function set -------------------------------------------------------------------------
@pytest.mark.parametrize("graph", ["full", "v1"])
def test_chunked_batch(handles, sms, graph):
    """IAN_CHUNK=48 at n = 100: chunks of 48, 48 and 4 images, against an unchunked handle and the oracle on the samples
    at the chunk edges."""
    n, seed = 100, 4100
    inp = _inputs(n, seed)
    probe = [47, 48, 95, 96, 99]
    chunked, whole = handles(graph, IAN_CHUNK="48"), handles(graph)
    xc, zc = chunked.reconstruct(inp["x"], return_z=True)
    xw, zw = whole.reconstruct(inp["x"], return_z=True)
    o = _oracle(graph)
    zref = _cached((graph, "chunk_z", n, seed), lambda: o.encode(inp["x"][probe]))
    rec = {"z_vs_unchunked": _zerr(zc, zw), "x_vs_unchunked": _xerr(xc, xw), "z_vs_oracle": _zerr(zc[probe], zref),
           "x_vs_oracle": _xerr(xc[probe], o.decode(zc[probe]))}
    gc, gw = chunked.grad(inp["z"], inp["boxes"], inp["rgb"]), whole.grad(inp["z"], inp["boxes"], inp["rgb"])
    gref = _cached((graph, "chunk_g", n, seed), lambda: o.grads(inp["z"][probe], inp["boxes"][probe],
                                                               {"colour": inp["rgb"][probe]})["colour"])
    rel_u, rel_o = _grad_rel(gc, gw), _grad_rel(gc[probe], gref)
    rec.update(grad_vs_unchunked_max=float(rel_u.max()), grad_vs_oracle=rel_o.tolist())
    _record("chunk48_%s_n100" % graph, rec)
    assert rec["z_vs_unchunked"] <= Z_K and rec["z_vs_oracle"] <= Z_K, rec
    assert rec["x_vs_unchunked"] <= X_TOL and rec["x_vs_oracle"] <= X_TOL, rec
    _assert_grads(graph, rel_u, "chunked vs unchunked")
    _assert_grads(graph, rel_o, "chunked vs oracle")


@pytest.mark.parametrize("graph", ["full", "v1"])
def test_flow_function_set_at_scale(handles, sms, graph):
    """Zfn / Z_IAF_fn / sample of sample_IAN.py at n = 130 against the oracle on the probes.  made_iaf_kernel runs one
    block per sample with a fixed loop order and reads nothing of other samples, so Z_IAF_fn of a sample is the same bits
    at n = 130 and n = 1."""
    n = 130
    seed = 5000 + n
    inp, probe = _inputs(n, seed), _probes(n, sms)
    o = _oracle(graph)

    def make():
        lat = o.latent(inp["z"][probe])
        return {"mu": o.mu(inp["x"][probe]), "lat": lat, "xs": o.decode(lat)}
    ref = _cached((graph, "flowset", n, seed), make)
    m = handles(graph)
    mu, lat, xs = m.Zfn(inp["x"]), m.Z_IAF_fn(inp["z"]), m.sample(inp["z"])
    rec = {"Zfn": _xerr(mu[probe], ref["mu"]), "Z_IAF_fn": _zerr(lat[probe], ref["lat"]), "sample": _xerr(xs[probe], ref["xs"])}
    _record("flowset_%s_n%d" % (graph, n), rec)
    assert rec["Zfn"] <= 2e-4 and rec["Z_IAF_fn"] <= Z_K and rec["sample"] <= 3e-4, rec
    for k in probe:
        assert np.array_equal(m.Z_IAF_fn(inp["z"][k:k + 1]), lat[k:k + 1]), k

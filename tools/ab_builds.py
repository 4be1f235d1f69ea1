"""A/B of two builds of the library on one GPU, in one command.

    python tools/ab_builds.py build REV
        (no GPU needed) builds the sources of git revision REV into build/ab/<REV>/libian_b200.so (git-ignored).
    python tools/ab_builds.py run REV [--rounds 3] [--steps 30] [--warmup 5] [--variant NAME:ENV=V,...] [--out DIR]
        runs bench.py alternately against build/ab/<REV> ("base") and the in-tree build ("head"), plus any --variant (the
        in-tree build under extra environment settings, e.g. head_wholetiles:IAN_STREAMK=0), A B A B ... for --rounds
        rounds.  Prints, per build, the median and range of `value`, of each `roofline.layer_ms` entry and of the
        secondary blocks, with the card name, power limit and sampled SM clock of every run, and compares the
        --dump-outputs arrays (z.npy, xhat.npy of the last timed step) of every build with "base" bit for bit.
        Raw result lines go to DIR/ab_<steps>.jsonl (default DIR: build/ab/results).
    python tools/ab_builds.py outputs REV
        runs every batch entry point in its host and its device form (the calls of tests/test_gpu_launch_forms.py) on
        seeded inputs and synthetic oracle.weights, in one child process per build, and prints per array whether
        build/ab/<REV> ("base") and the in-tree build ("head") give the same bits: the three graphs; the tensor-core path
        by default and with IAN_STREAMK=0, IAN_STREAMK=2 and IAN_GRAPHS=0; the SIMT path; batches 1, 3, 47, 130 and 513.
        Also the host forms of the sampling script's Zfn, Z_IAF_fn and sample on seeded images and N(0,1) latents, and
        the eight latent-fit entry points (normal equations and fits: plain; masked with and without weights; robust,
        Huber and Cauchy, automatic and given scale, with outliers; features at weights (1, 1), (0, 1), (1, 0)) in both
        forms with 3 steps, each call's launch_count() delta one more array, at batches 1 and 3, and 20 under IAN_CHUNK=16.
        And the entry points whose batch is coupled, in both forms, each call's launch_count() delta one more array, at
        every batch above and at 20 under IAN_CHUNK=16: the discriminator (tests/test_gpu_discriminate_train.py's seeded
        head) in inference and in training mode, forward with the statistics and VJP; on IAN_simple the training-mode
        decoder, x_hat with the statistics and its VJP with all 13 gradients and with l_dec_fc2.W's alone.
"""
import argparse
import hashlib
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEAD_LIB = os.path.join(ROOT, "neural-photo-editor_b200", "libian_b200.so")


def ab_dir(rev):
    return os.path.join(ROOT, "build", "ab", rev)


def cmd_build(rev):
    out = ab_dir(rev)
    os.makedirs(out, exist_ok=True)
    with tempfile.TemporaryDirectory(prefix="ian_ab_") as tmp:
        arch = subprocess.run(["git", "-C", ROOT, "archive", rev, "neural-photo-editor_b200", "include"], check=True,
                              capture_output=True).stdout
        subprocess.run(["tar", "-x", "-C", tmp], input=arch, check=True)
        pkg = os.path.join(tmp, "neural-photo-editor_b200")
        code = "import sys; sys.path.insert(0, %r); import build; build.build(force=True)" % pkg
        subprocess.run([sys.executable, "-c", code], check=True, cwd=pkg)
        shutil.copy2(os.path.join(pkg, "libian_b200.so"), os.path.join(out, "libian_b200.so"))
    print(os.path.join(out, "libian_b200.so"))


def _bench(lib, env_extra, steps, warmup, dump):
    env = dict(os.environ, IAN_B200_LIB=lib, **env_extra)
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
           "--no-cpu-baseline"]
    if dump:
        cmd += ["--dump-outputs", dump]
    p = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=ROOT)
    if p.returncode != 0:
        raise SystemExit("bench.py failed for %s %s:\n%s" % (lib, env_extra, p.stderr[-3000:]))
    return json.loads([l for l in p.stdout.splitlines() if l.startswith("{")][-1])


def _secondary(line):
    """the bench blocks besides `value` (higher is better unless the key says ms)"""
    out = {}
    if line.get("edit"):
        out["edit steps/s"] = line["edit"]["value"]
    f = line.get("full_ian")
    if f:
        out["full_ian bf16 img/s"] = f["bf16"]["value"]
        out["full_ian fp32 img/s"] = f["fp32_split"]["value"]
    if line.get("config5"):
        out["config5 img/s"] = line["config5"]["value"]
    if line.get("e2e"):
        out["e2e img/s"] = line["e2e"]["value"]
    lat = line.get("single_image_latency")
    if lat:
        out["latency b1 ms"] = lat["median_ms"]
        out["paint_stroke ms"] = lat["paint_stroke_median_ms"]
    return out


def _fmt(vals):
    return "median %.4g  range [%.4g, %.4g]" % (statistics.median(vals), min(vals), max(vals))


def cmd_run(args):
    import numpy as np
    builds = [("base", os.path.join(ab_dir(args.rev), "libian_b200.so"), {}), ("head", HEAD_LIB, {})]
    for v in args.variant:
        name, _, envs = v.partition(":")
        builds.append((name, HEAD_LIB, dict(kv.split("=", 1) for kv in envs.split(",") if kv)))
    for _, lib, _ in builds:
        if not os.path.exists(lib):
            raise SystemExit("missing %s (python tools/ab_builds.py build %s)" % (lib, args.rev))
    os.makedirs(args.out, exist_ok=True)
    lines = {b[0]: [] for b in builds}
    raw = open(os.path.join(args.out, "ab_%d.jsonl" % args.steps), "w")
    for r in range(args.rounds):
        for name, lib, env in builds:
            dump = os.path.join(args.out, "dump_%s" % name) if r == 0 else None
            line = _bench(lib, env, args.steps, args.warmup, dump)
            line["ab_build"], line["ab_round"] = name, r
            raw.write(json.dumps(line) + "\n")
            raw.flush()
            lines[name].append(line)
            g, c = line.get("gpu", {}), line.get("clocks") or {}
            print("round %d %-16s value %.1f  (%s, %s W, SM clock median %s MHz)" % (r, name, line["value"], g.get("name"),
                  g.get("power_limit_w"), c.get("sm_mhz")), flush=True)
    print("\n== --steps %d --warmup %d, %d rounds, builds alternated" % (args.steps, args.warmup, args.rounds))
    for name, _, env in builds:
        ls = lines[name]
        print("%s %s" % (name, env or ""))
        print("  value (images/s)      %s" % _fmt([l["value"] for l in ls]))
        print("  SM clock (MHz)        %s" % _fmt([(l.get("clocks") or {}).get("sm_mhz") or 0 for l in ls]))
        for k in ls[0]["roofline"]["layer_ms"]:
            print("  layer_ms %-12s %s" % (k, _fmt([l["roofline"]["layer_ms"][k] for l in ls])))
        for k in _secondary(ls[0]):
            print("  %-21s %s" % (k, _fmt([_secondary(l)[k] for l in ls])))
    base_dump = os.path.join(args.out, "dump_base")
    for name, _, _ in builds[1:]:
        for f in ("z.npy", "xhat.npy"):
            a, b = np.load(os.path.join(base_dump, f)), np.load(os.path.join(args.out, "dump_%s" % name, f))
            same = a.shape == b.shape and np.array_equal(a, b)
            diff = float(np.abs(a.astype(np.float64) - b).max()) if a.shape == b.shape else float("nan")
            print("outputs %s vs base %s: %s (max abs diff %.3g)" % (name, f, "bit-identical" if same else "DIFFER", diff))


OUTPUT_CONFIGS = [("tc", {}), ("tc", {"IAN_STREAMK": "0"}), ("tc", {"IAN_STREAMK": "2"}), ("tc", {"IAN_GRAPHS": "0"}),
                  ("simt", {})]
OUTPUT_BATCHES = (1, 3, 47, 130, 513)
FIT_BATCHES = (1, 3)                       # a fit costs one batch-100 JVP pass per sample and step
FIT_ITERS = 3


def _counted(m, out, name, f, *res):
    """runs f(), one entry point; appends to out its arrays -- what f returns (host form) or the device tensors res (device
    form) -- and its launch_count() delta; returns what f returned"""
    import numpy as np
    import torch
    c0 = m.launch_count()
    torch.cuda.synchronize()
    r = f()
    torch.cuda.synchronize()
    arrays = [a.cpu().numpy() for a in res] if res else list(r if isinstance(r, tuple) else (r,))
    out.extend(("%s %d" % (name, i), a) for i, a in enumerate(arrays))
    out.append((name + " launches", np.array([m.launch_count() - c0])))
    return r


def _fit_arrays(m, n, seed):
    """(name, array) of every latent-fit entry point in its host and its device form on seeded inputs, each call
    followed by its launch_count() delta"""
    import numpy as np
    import torch
    import test_gpu_launch_forms as lf
    rng = np.random.default_rng(seed)
    x = np.tanh(rng.standard_normal((n, 3, 64, 64))).astype(np.float32)
    u = (0.5 * rng.standard_normal((n, 100))).astype(np.float32)
    w = np.where(rng.uniform(size=x.shape) < 0.25, 0, rng.uniform(size=x.shape)).astype(np.float32)
    scale = rng.uniform(0.05, 0.5, n)
    d = lf._Dev()
    xp, up, wp, sp = d.put(x), d.put(u), d.put(w), d.put(scale)
    it, prior = FIT_ITERS, 1e-2
    out = []

    def t(*shape, like=None, f64=False):
        a = torch.zeros(shape, dtype=torch.float64 if f64 else torch.float32, device="cuda") if like is None else \
            torch.from_numpy(like.copy()).cuda()
        d.keep.append(a)
        return a

    def call(name, f, *res):
        _counted(m, out, name, f, *res)

    def gn(name, host, dev):
        A, g, e = t(n, 100, 100, f64=True), t(n, 100, f64=True), t(n, f64=True)
        call(name + " host", host)
        call(name + " dev", lambda: dev(A.data_ptr(), g.data_ptr(), e.data_ptr()), A, g, e)

    gn("gauss_newton", lambda: m.gauss_newton(u, x), lambda A, g, e: m.gauss_newton_dev(up, xp, n, A, g, e))
    z, loss = t(like=u), t(n, it + 1)
    call("fit_latent host", lambda: m.fit_latent(x, u, iters=it, return_loss=True))
    call("fit_latent dev", lambda: m.fit_latent_dev(xp, n, z.data_ptr(), it, loss.data_ptr()), z, loss)
    for tag, wa, wd in (("", None, 0), ("_w", w, wp)):
        gn("gauss_newton_map" + tag, lambda: m.gauss_newton_map(u, x, wa, prior),
           lambda A, g, e: m.gauss_newton_map_dev(up, xp, wd, prior, n, A, g, e))
        uu, z, loss = t(like=u), t(n, 100), t(n, it + 1)
        call("fit_latent_map%s host" % tag, lambda: m.fit_latent_map(x, wa, prior, u, iters=it, return_loss=True))
        call("fit_latent_map%s dev" % tag,
             lambda: m.fit_latent_map_dev(xp, wd, prior, n, uu.data_ptr(), it, z.data_ptr(), loss.data_ptr()), uu, z, loss)
    for kind in ("huber", "cauchy"):
        for tag, sa, sd in (("auto", None, 0), ("given", scale, sp)):
            name = "%s_%s" % (kind, tag)
            so = t(n, f64=True)
            gn("gauss_newton_robust_" + name, lambda: m.gauss_newton_robust(u, x, kind, sa, w, prior),
               lambda A, g, e: m.gauss_newton_robust_dev(up, xp, wp, prior, kind, sd, n, A, g, e, so.data_ptr()))
            out.append(("gauss_newton_robust_%s dev scale_out" % name, so.cpu().numpy()))
            uu, z, loss, so, ow = t(like=u), t(n, 100), t(n, it + 1), t(n, f64=True), t(n, 3, 64, 64)
            call("fit_latent_robust_%s host" % name,
                 lambda: m.fit_latent_robust(x, kind, sa, w, prior, u, iters=it, return_loss=True, return_outliers=True))
            call("fit_latent_robust_%s dev" % name,
                 lambda: m.fit_latent_robust_dev(xp, wp, prior, kind, sd, n, uu.data_ptr(), it, z.data_ptr(), loss.data_ptr(),
                                                 so.data_ptr(), ow.data_ptr()), uu, z, so, loss, ow)
    for a, b in ((1.0, 1.0), (0.0, 1.0), (1.0, 0.0)):
        name = "features_%g_%g" % (a, b)
        gn("gauss_newton_" + name, lambda: m.gauss_newton_features(u, x, a, b),
           lambda A, g, e: m.gauss_newton_features_dev(up, xp, n, A, g, e, a, b))
        z, loss = t(like=u), t(n, it + 1)
        call("fit_latent_%s host" % name, lambda: m.fit_latent_features(x, u, it, a, b, return_loss=True))
        call("fit_latent_%s dev" % name,
             lambda: m.fit_latent_features_dev(xp, n, z.data_ptr(), it, loss.data_ptr(), a, b), z, loss)
    return out


def _train_arrays(m, n, seed):
    """(name, array) of the discriminator's entry points, inference and training mode (the head loaded), and on IAN_simple
    of the training-mode decoder's (x_hat with stats; dz with all 13 gradients, and with l_dec_fc2.W's alone), in their host
    and their device form on seeded inputs, each call followed by its launch_count() delta"""
    import importlib
    import numpy as np
    import test_gpu_launch_forms as lf
    rng = np.random.default_rng(seed)
    U = m.discriminator_units()
    x = np.tanh(rng.standard_normal((n, 3, 64, 64))).astype(np.float32)
    dl = rng.standard_normal((n, U)).astype(np.float32)
    d = lf._Dev()
    xp, dlp = d.put(x), d.put(dl)
    out = []

    def call(name, f, *res):
        return _counted(m, out, name, f, *res)

    lg, p = d.empty((n, U)), d.empty((n, U))
    call("discriminate host", lambda: m.discriminate(x, return_logits=True))
    call("discriminate dev", lambda: m.discriminate_dev(xp, n, lg.data_ptr(), p.data_ptr()), lg, p)
    dx = d.empty((n, 3, 64, 64))
    call("discriminate_vjp host", lambda: m.discriminate_vjp(x, dl))
    call("discriminate_vjp dev", lambda: m.discriminate_vjp_dev(xp, dlp, n, dx.data_ptr()), dx)
    lg, p, st = d.empty((n, U)), d.empty((n, U)), d.empty((2, 1792))
    call("discriminate_train host", lambda: m.discriminate_train(x, return_logits=True, return_stats=True))
    call("discriminate_train dev", lambda: m.discriminate_train_dev(xp, n, lg.data_ptr(), p.data_ptr(), st.data_ptr()), lg, p, st)
    dx = d.empty((n, 3, 64, 64))
    call("discriminate_train_vjp host", lambda: m.discriminate_train_vjp(x, dl))
    call("discriminate_train_vjp dev", lambda: m.discriminate_train_vjp_dev(xp, dlp, n, dx.data_ptr()), dx)
    if m.kind != importlib.import_module("neural-photo-editor_b200._lib").IAN_MODEL_SIMPLE:
        return out
    z = rng.standard_normal((n, 100)).astype(np.float32)
    dxh = rng.standard_normal((n, 3, 64, 64)).astype(np.float32)
    zp, dxhp = d.put(z), d.put(dxh)
    xh, st = d.empty((n, 3, 64, 64)), d.empty((2, 17280))
    call("decode_train host", lambda: m.decode_train(z, return_stats=True))
    call("decode_train dev", lambda: m.decode_train_dev(zp, n, xh.data_ptr(), st.data_ptr()), xh, st)
    def vjp_host(names):
        dz, g = m.decode_train_vjp(z, dxh, names)
        return (dz,) + tuple(g[k] for k in names)

    for tag, names in (("all", m.param_vjp_names()), ("fc2_W", ["l_dec_fc2.W"])):
        r = call("decode_train_vjp_%s host" % tag, lambda: vjp_host(names))
        dz, g = d.empty((n, 100)), [d.empty(a.shape) for a in r[1:]]
        call("decode_train_vjp_%s dev" % tag,
             lambda: m.decode_train_vjp_dev(zp, dxhp, n, dz.data_ptr(), {k: t.data_ptr() for k, t in zip(names, g)}), dz, *g)
    return out


def cmd_dump(out):
    """child of `outputs`: sha256 and sum of |a| of every array, for the build IAN_B200_LIB names"""
    import importlib
    import numpy as np
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    import ctypes
    import discrim_train_oracle as dto
    import test_gpu_launch_forms as lf
    lib = importlib.import_module("neural-photo-editor_b200._lib")
    so = ctypes.CDLL(lib.LIB_PATH)
    for name in list(lib.SIGNATURES):      # an older build lacks the entry points added after it; none of them is called here
        if not hasattr(so, name):
            del lib.SIGNATURES[name]
    npe = importlib.import_module("neural-photo-editor_b200")
    heads = {g: f[2] for g, f in dto.fixture().items()}    # tests/test_gpu_discriminate_train.py's seeded heads
    res = {}

    def record(cfg, n, arrays):
        for name, a in arrays:
            a = np.ascontiguousarray(a)
            res["%s n=%d %s" % (cfg, n, name)] = [hashlib.sha256(a.tobytes()).hexdigest(), list(a.shape),
                                                  float(np.abs(a.astype(np.float64)).sum())]
    for graph in ("simple", "full", "v1"):
        for path, env in OUTPUT_CONFIGS:
            for k in lf.ENV:
                os.environ.pop(k, None)
            os.environ.update(env)
            m = npe.IAN(lf.CONFIG[graph], True, weights=lf._weights(graph), path=path)
            m.load_discriminator(heads[graph])
            cfg = "%s-%s%s" % (graph, path, "".join("-%s=%s" % kv for kv in env.items()))
            for n in OUTPUT_BATCHES:
                arrays = [("%s %s" % (name, form), a) for name, host, dev in lf._pairs(m, npe, lf._inputs(n, 7000 + n))
                          for form, a in (("host", host), ("dev", dev))]
                # the sampling script's function set (host forms: the only ones older builds have)
                rng = np.random.default_rng(7100 + n)
                x = np.tanh(rng.standard_normal((n, 3, 64, 64))).astype(np.float32)
                zi = rng.standard_normal((n, 100)).astype(np.float32)
                arrays += [("Zfn host", m.Zfn(x)), ("Z_IAF_fn host", m.Z_IAF_fn(zi)), ("sample host", m.sample(zi))]
                if n in FIT_BATCHES:
                    arrays += _fit_arrays(m, n, 7200 + n)
                arrays += _train_arrays(m, n, 7300 + n)
                record(cfg, n, arrays)
            m.close()
        # the fits and the coupled-batch entries over two chunks, of 16 and 4 samples
        for k in lf.ENV:
            os.environ.pop(k, None)
        os.environ["IAN_CHUNK"] = "16"
        m = npe.IAN(lf.CONFIG[graph], True, weights=lf._weights(graph), path="tc")
        m.load_discriminator(heads[graph])
        record("%s-tc-IAN_CHUNK=16" % graph, 20, _fit_arrays(m, 20, 7220) + _train_arrays(m, 20, 7320))
        m.close()
        os.environ.pop("IAN_CHUNK")
    with open(out, "w") as f:
        json.dump(res, f)


def cmd_outputs(rev):
    libs = [("base", os.path.join(ab_dir(rev), "libian_b200.so")), ("head", HEAD_LIB)]
    res = {}
    with tempfile.TemporaryDirectory(prefix="ian_ab_out_") as tmp:
        for name, lib in libs:
            if not os.path.exists(lib):
                raise SystemExit("missing %s (python tools/ab_builds.py build %s)" % (lib, rev))
            out = os.path.join(tmp, name + ".json")
            subprocess.run([sys.executable, os.path.abspath(__file__), "_dump", out], check=True, cwd=ROOT, stdout=subprocess.DEVNULL,
                           env=dict(os.environ, IAN_B200_LIB=lib))
            res[name] = json.load(open(out))
    base, head = res["base"], res["head"]
    ndiff = 0
    for key in sorted(set(base) | set(head)):
        same = key in base and key in head and base[key][:2] == head[key][:2]
        ndiff += not same
        print("%-70s %s" % (key, "bit-identical" if same else "DIFFER (sum|a| base %s, head %s)" % (
            base.get(key, [None] * 3)[2], head.get(key, [None] * 3)[2])))
    print("\n%d arrays, %d DIFFER (base %s, head in-tree)" % (len(set(base) | set(head)), ndiff, rev))
    if ndiff:
        raise SystemExit(1)


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    b = sub.add_parser("build")
    b.add_argument("rev")
    sub.add_parser("outputs").add_argument("rev")
    sub.add_parser("_dump").add_argument("out")
    r = sub.add_parser("run")
    r.add_argument("rev")
    r.add_argument("--rounds", type=int, default=3)
    r.add_argument("--steps", type=int, default=30)
    r.add_argument("--warmup", type=int, default=5)
    r.add_argument("--variant", action="append", default=[], metavar="NAME:ENV=V,...")
    r.add_argument("--out", default=os.path.join(ROOT, "build", "ab", "results"))
    a = ap.parse_args()
    if a.cmd == "build":
        cmd_build(a.rev)
    elif a.cmd == "outputs":
        cmd_outputs(a.rev)
    elif a.cmd == "_dump":
        cmd_dump(a.out)
    else:
        cmd_run(a)


if __name__ == "__main__":
    main()

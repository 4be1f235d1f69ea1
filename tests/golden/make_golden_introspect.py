"""Generate tests/golden/ref_exec_introspect.npz: the reference's own introspection features l_introspect
(IAN_simple.py:240, IAN.py:227, IANv1.py:220) and their directional derivatives, by EXECUTING the reference's Python files
on the numpy stand-ins of oracle/refshim, in float64 -- the fixture the feature entry points (ian_introspect_*,
ian_introspect_jvp_*) and their float64 restatement (tests/introspect_oracle.py) are pinned to.

The staging is make_golden_encvjp.py's (make_golden_ref.py's synthetic checkpoints, the reference's API.IAN for IAN_simple,
get_model + GANcheckpoints.load_weights for IAN.py / IANv1.py).  The compiled function is
    get_output(model['l_introspect'], {l_in: X}, deterministic=True)
on a float64 input variable.  Per graph and golden image (the first two of ian_<graph>_golden.npz) and feature layer i:
  * f_<graph>_<i>:  the features at channels CHANNELS[i] (all pixels), (N_IMG, len(CHANNELS[i]), H, W);
  * p_<graph>_<i>:  <probe_j, g_i(x)> for PROBES seeded probes (N_IMG, PROBES);
  * dp_<graph>_<i>: <probe_j, (g_i(x + h v) - g_i(x - h v)) / 2h>, h = 1e-7, along a seeded image tangent v;
  * df_<graph>_<i>: that central difference at channels CHANNELS[i].
The probes and tangents are drawn from the stored seed (draws()), which keeps the file small.

    python tests/golden/make_golden_introspect.py            # ~1 min

The GPU box has no /root/reference: tests read only the committed .npz file.
"""
import logging
import os
import shutil
import sys
import time

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_ref as mgr   # noqa: E402  (puts oracle/refshim and the reference on sys.path)

SEED = 20261018
H = 1e-7
N_IMG = 2
PROBES = 4
SHAPES = ((128, 32, 32), (256, 16, 16), (512, 8, 8), (1024, 4, 4))
CHANNELS = ((0, 77), (5, 200), (31, 444), (2, 1000))
GRAPHS = ('simple', 'full', 'v1')


def draws(seed=SEED):
    """per graph: image tangents v (N_IMG,3,64,64) and per layer probes (PROBES, C, H, W), float64"""
    rng = np.random.RandomState(seed)
    return {g: (rng.standard_normal((N_IMG, 3, 64, 64)), [rng.standard_normal((PROBES,) + s) for s in SHAPES]) for g in GRAPHS}


def images(which):
    gold = np.load(os.path.join(mgr.ROOT, 'tests', 'golden', 'ian_%s_golden.npz' % which))
    return mgr.on.to_tanh(gold['images'][:N_IMG].astype(np.float64)).astype(np.float32), int(gold['weight_seed'])


def introspect_fn(which):
    """the compiled l_introspect function of the reference graph"""
    import imp
    import theano
    import theano.tensor as T
    import lasagne
    _, seed = images(which)
    X = T.TensorType('float64', [False] * 4)('X')
    if which == 'simple':
        from API import IAN                               # the reference's API.py
        link = mgr._stage('IAN_simple.py', mgr.ow.make_simple_weights(seed))
        model = IAN(config_path=link, dnn=True).model
    else:
        import GANcheckpoints
        config = {'v1': 'IANv1.py', 'full': 'IAN.py'}[which]
        link = mgr._stage(config, (mgr.ow.make_v1_weights if which == 'v1' else mgr.ow.make_full_weights)(seed))
        model = imp.load_source('config', link).get_model()
        params = list(set(lasagne.layers.get_all_params(model['l_out'], trainable=True) +
                          lasagne.layers.get_all_params(model['l_discrim'], trainable=True) +
                          [x for x in lasagne.layers.get_all_params(model['l_out']) + lasagne.layers.get_all_params(model['l_discrim'])
                           if x.name[-4:] == 'mean' or x.name[-7:] == 'inv_std']))
        GANcheckpoints.load_weights(link[:-3] + '.npz', params)
    return theano.function([X], lasagne.layers.get_output(model['l_introspect'], {model['l_in']: X}, deterministic=True))


def main():
    logging.basicConfig(level=logging.ERROR)
    d = draws()
    out = {'seed': np.int64(SEED), 'h': np.float64(H), 'n_img': np.int64(N_IMG), 'probes': np.int64(PROBES)}
    try:
        for which in GRAPHS:
            t0 = time.time()
            fn = introspect_fn(which)
            x, _ = images(which)
            v, probes = d[which]
            x = x.astype(np.float64)
            F = lambda xx: [np.asarray(a, np.float64) for a in fn(xx)]
            f, fp, fm = F(x), F(x + H * v), F(x - H * v)
            for i in range(4):
                assert f[i].shape == (N_IMG,) + SHAPES[i], f[i].shape
                df = (fp[i] - fm[i]) / (2 * H)
                ch = list(CHANNELS[i])
                out['f_%s_%d' % (which, i)] = f[i][:, ch]
                out['df_%s_%d' % (which, i)] = df[:, ch]
                out['p_%s_%d' % (which, i)] = np.einsum('nchw,jchw->nj', f[i], probes[i])
                out['dp_%s_%d' % (which, i)] = np.einsum('nchw,jchw->nj', df, probes[i])
            print(which, [float(np.abs(out['dp_%s_%d' % (which, i)]).max()) for i in range(4)],
                  'in %.1f s' % (time.time() - t0), flush=True)
    finally:
        shutil.rmtree(mgr.WORK, ignore_errors=True)
    path = os.path.join(mgr.OUT, 'ref_exec_introspect.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()

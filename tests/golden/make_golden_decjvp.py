"""Generate tests/golden/ref_exec_decjvp.npz: directional derivatives of the reference's own X_hat (API.py:46) by
EXECUTING the reference's Python files on the numpy stand-ins of oracle/refshim, in float64 -- the fixture the decoder
Jacobian-vector product (ian_decode_jvp_*) is pinned to.

The staging (synthetic checkpoint next to a config symlink, the reference's API.IAN for IAN_simple, get_model +
GANcheckpoints.load_weights for IAN.py / IANv1.py) is make_golden_ref.py's, reused by import, as in make_golden_encvjp.py.
Per graph, N_PAIRS latent / direction pairs (z, v) drawn from the stored seed:
    dx = (X(z + h v) - X(z - h v)) / 2h,      h = 1e-7
where X is get_output(l_out, {l_Z: Z}, deterministic=True) compiled on a float64 input variable (the decoder from l_Z, no
MADE/IAF), evaluated in float64 by the stand-in.  The (N_PAIRS,3,64,64) float64 images are stored; z and v are redrawn
from the seed by the tests.

    python tests/golden/make_golden_decjvp.py            # ~1 min

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

SEED = 20261016
H = 1e-7
N_PAIRS = 2


def draws(seed=SEED):
    """per graph: latents z and directions v, (N_PAIRS,100) float64 each"""
    rng = np.random.RandomState(seed)
    return {g: (rng.standard_normal((N_PAIRS, 100)), rng.standard_normal((N_PAIRS, 100))) for g in ('simple', 'full', 'v1')}


def weight_seed(which):
    return int(np.load(os.path.join(mgr.ROOT, 'tests', 'golden', 'ian_%s_golden.npz' % which))['weight_seed'])


def x_hat_function(which):
    """X_hat_fn of the reference graph (API.py:46), compiled on a float64 latent"""
    import imp
    import theano
    import theano.tensor as T
    import lasagne
    seed = weight_seed(which)
    Z = T.TensorType('float64', [False] * 2)('Z')
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
    return theano.function([Z], lasagne.layers.get_output(model['l_out'], {model['l_Z']: Z}, deterministic=True))


def main():
    logging.basicConfig(level=logging.ERROR)
    d = draws()
    out = {'seed': np.int64(SEED), 'h': np.float64(H), 'n_pairs': np.int64(N_PAIRS)}
    try:
        for which in ('simple', 'full', 'v1'):
            t0 = time.time()
            X = x_hat_function(which)
            z, v = d[which]
            dx = np.zeros((N_PAIRS, 3, 64, 64))
            for k in range(N_PAIRS):
                xp = np.asarray(X(z[k:k + 1] + H * v[k:k + 1]), np.float64)
                xm = np.asarray(X(z[k:k + 1] - H * v[k:k + 1]), np.float64)
                dx[k] = ((xp - xm) / (2 * H))[0]
            out['dx_' + which] = dx
            print(which, np.abs(dx).max(axis=(1, 2, 3)), 'in %.1f s' % (time.time() - t0), flush=True)
    finally:
        shutil.rmtree(mgr.WORK, ignore_errors=True)
    path = os.path.join(mgr.OUT, 'ref_exec_decjvp.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()

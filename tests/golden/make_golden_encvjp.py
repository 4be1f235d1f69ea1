"""Generate tests/golden/ref_exec_encvjp.npz: directional derivatives of the reference's own Z_hat (API.py:50-51) by
EXECUTING the reference's Python files on the numpy stand-ins of oracle/refshim, in float64 -- the fixture the encoder
vector-Jacobian product (ian_encode_vjp_*) is pinned to.

The staging (synthetic checkpoint next to a config symlink, the reference's API.IAN for IAN_simple, get_model +
GANcheckpoints.load_weights + MADE reset("Once") for IAN.py / IANv1.py) is make_golden_ref.py's, reused by import.
Per graph and golden image (the first two of ian_<graph>_golden.npz), without and with eps:
    d = dz . (Z(x + h v) - Z(x - h v)) / 2h,      h = 1e-7
where Z is the compiled Z_hat function (no eps) or, with eps, Z_IAF_fn (sample_IAN.py:92) of mu + exp(logsigma) eps
from the compiled mu / logsigma functions (GaussianSampleLayer, layers.py:419-433, with the noise injected: its MRG
stream is not reproducible).  The functions are compiled on float64 input variables and the stand-in evaluates in
float64 (refshim theano.config.floatX), so x +- h v reaches the graph without a float32 round trip.  v and dz are drawn
from the stored seed, which keeps the file a few KB.

    python tests/golden/make_golden_encvjp.py            # ~2 min

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

SEED = 20261015
H = 1e-7
N_IMG = 2


def draws(seed=SEED):
    """per graph: directions v (N_IMG,3,64,64), cotangents dz (N_IMG,100) and eps (N_IMG,100), float64"""
    rng = np.random.RandomState(seed)
    out = {}
    for g in ('simple', 'full', 'v1'):
        out[g] = (rng.standard_normal((N_IMG, 3, 64, 64)), rng.standard_normal((N_IMG, 100)), rng.standard_normal((N_IMG, 100)))
    return out


def images(which):
    gold = np.load(os.path.join(mgr.ROOT, 'tests', 'golden', 'ian_%s_golden.npz' % which))
    return mgr.on.to_tanh(gold['images'][:N_IMG].astype(np.float64)).astype(np.float32), int(gold['weight_seed'])


def functions(which):
    """(Z_hat, mu_ls, flow) compiled from the reference graph; flow is None for IAN_simple (l_Z = the sample layer)"""
    import imp
    import theano
    import theano.tensor as T
    import lasagne
    _, seed = images(which)
    go = lasagne.layers.get_output
    X = T.TensorType('float64', [False] * 4)('X')
    Z = T.TensorType('float64', [False] * 2)('Z')
    if which == 'simple':
        from API import IAN                               # the reference's API.py
        link = mgr._stage('IAN_simple.py', mgr.ow.make_simple_weights(seed))
        model = IAN(config_path=link, dnn=True).model
        flow = None
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
        model['l_IAF_mu'].reset("Once")
        model['l_IAF_ls'].reset("Once")
        flow = theano.function([Z], go(model['l_Z'], {model['l_Z_IAF']: Z}, deterministic=True))      # sample_IAN.py:92
    z_hat = theano.function([X], go(model['l_Z'], {model['l_in']: X}, deterministic=True))          # API.py:50-51
    mu_ls = theano.function([X], [go(model['l_mu'], {model['l_in']: X}, deterministic=True),
                                  go(model['l_ls'], {model['l_in']: X}, deterministic=True)])
    return z_hat, mu_ls, flow


def main():
    logging.basicConfig(level=logging.ERROR)
    d = draws()
    out = {'seed': np.int64(SEED), 'h': np.float64(H), 'n_img': np.int64(N_IMG)}
    try:
        for which in ('simple', 'full', 'v1'):
            t0 = time.time()
            z_hat, mu_ls, flow = functions(which)
            x, _ = images(which)
            v, dz, eps = d[which]
            dd = np.zeros((2, N_IMG))
            for k in range(N_IMG):
                xk = x[k:k + 1].astype(np.float64)
                for j, with_eps in enumerate((False, True)):
                    def Z(xx):
                        if not with_eps:
                            return np.asarray(z_hat(xx), np.float64)
                        mu, ls = (np.asarray(a, np.float64) for a in mu_ls(xx))
                        zi = mu + np.exp(ls) * eps[k:k + 1]
                        return zi if flow is None else np.asarray(flow(zi), np.float64)
                    zp, zm = Z(xk + H * v[k:k + 1]), Z(xk - H * v[k:k + 1])
                    dd[j, k] = float((dz[k:k + 1] * (zp - zm)).sum() / (2 * H))
            out['dd_' + which] = dd                       # [without eps, with eps][image]
            print(which, dd, 'in %.1f s' % (time.time() - t0), flush=True)
    finally:
        shutil.rmtree(mgr.WORK, ignore_errors=True)
    path = os.path.join(mgr.OUT, 'ref_exec_encvjp.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()

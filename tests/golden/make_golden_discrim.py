"""Generate tests/golden/ref_exec_discrim.npz: the reference's own discriminator head l_discrim (IAN_simple.py:225-231,
IAN.py:210-216, IANv1.py:203-209) and its directional derivatives, by EXECUTING the reference's Python files on the numpy
stand-ins of oracle/refshim, in float64 -- the fixture the discriminator entry points (ian_discriminate_*,
ian_discriminate_vjp_*) and their float64 restatement (tests/discrim_oracle.py) are pinned to.

The staging is make_golden_introspect.py's, with the head's four tensors added to each synthetic checkpoint so that the
reference's loaders (API.py:26, GANcheckpoints.load_weights) read them by name.  The head is
tests/discrim_oracle.make_discriminator_weights(graph, HEAD_SEED[graph]) with log_weight_scale set by the reference's own
data-dependent rule (MinibatchLayer init=True, layers.py:510-513) on the fixture's batch: with it at 0 the pair terms of
these features could all underflow, and the coupling would go untested.  The batch is the first N_IMG = 4 images of
ian_simple_golden.npz on every graph, so the MinibatchLayer couples them.  The compiled functions are
    get_output(model['l_discrim'], {l_in: X}, deterministic=True)           (p)
and the same with l_discrim's nonlinearity set to the identity (the logits), on a float64 input.  Per graph it stores the
logits and p, log_weight_scale (float32, as loaded), b, W, theta's seed, and dp[t] = <probe_t, (logits(x + h v_t) -
logits(x - h v_t)) / 2h>, h = 1e-7, along discrim_oracle.draws()'s tangents of all 4 images (the third moves one image
and reads another sample).

    python tests/golden/make_golden_discrim.py            # ~1 min

The GPU box has no /root/reference: tests read only the committed .npz file.
"""
import logging
import os
import shutil
import sys
import time

import numpy as np

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]
import make_golden_ref as mgr   # noqa: E402  (puts oracle/refshim and the reference on sys.path)
import discrim_oracle as do     # noqa: E402

SEED = 20261018
HEAD_SEED = {'simple': 11, 'full': 12, 'v1': 13}
H = 1e-7
N_IMG = 4
GRAPHS = ('simple', 'full', 'v1')


def images(which):
    """the first N_IMG images of ian_simple_golden.npz (the other graphs' files hold two) and the graph's weight seed"""
    imgs = np.load(os.path.join(mgr.ROOT, 'tests', 'golden', 'ian_simple_golden.npz'))['images'][:N_IMG]
    seed = int(np.load(os.path.join(mgr.ROOT, 'tests', 'golden', 'ian_%s_golden.npz' % which))['weight_seed'])
    return mgr.on.to_tanh(imgs.astype(np.float64)).astype(np.float32), seed


def model_of(which, head):
    """the reference graph, loaded from a staged checkpoint of the graph's synthetic weights plus `head`"""
    import imp
    import lasagne
    _, seed = images(which)
    if which == 'simple':
        from API import IAN                               # the reference's API.py
        link = mgr._stage('IAN_simple.py', dict(mgr.ow.make_simple_weights(seed), **head))
        return IAN(config_path=link, dnn=True).model
    import GANcheckpoints
    config = {'v1': 'IANv1.py', 'full': 'IAN.py'}[which]
    link = mgr._stage(config, dict((mgr.ow.make_v1_weights if which == 'v1' else mgr.ow.make_full_weights)(seed), **head))
    model = imp.load_source('config', link).get_model()
    params = list(set(lasagne.layers.get_all_params(model['l_out'], trainable=True) +
                      lasagne.layers.get_all_params(model['l_discrim'], trainable=True) +
                      [x for x in lasagne.layers.get_all_params(model['l_out']) + lasagne.layers.get_all_params(model['l_discrim'])
                       if x.name[-4:] == 'mean' or x.name[-7:] == 'inv_std']))
    GANcheckpoints.load_weights(link[:-3] + '.npz', params)
    return model


def functions(model):
    """(pooled, logits, p): compiled functions of the GlobalPoolLayer, of l_discrim before and after its nonlinearity"""
    import theano
    import theano.tensor as T
    import lasagne
    X = T.TensorType('float64', [False] * 4)('X')
    l = model['l_discrim']
    get = lambda layer: theano.function([X], lasagne.layers.get_output(layer, {model['l_in']: X}, deterministic=True))
    pool = get(l.input_layer.input_layer)
    nl = l.nonlinearity
    l.nonlinearity = lasagne.nonlinearities.identity
    lg = get(l)
    l.nonlinearity = nl
    return pool, lg, get(l)


def main():
    logging.basicConfig(level=logging.ERROR)
    d = do.draws(SEED, N_IMG)
    out = {'seed': np.int64(SEED), 'h': np.float64(H), 'n_img': np.int64(N_IMG)}
    try:
        for which in GRAPHS:
            t0 = time.time()
            x, _ = images(which)
            x = x.astype(np.float64)
            head = do.make_discriminator_weights(which, HEAD_SEED[which])
            pool, _, _ = functions(model_of(which, head))
            pooled = np.asarray(pool(x), np.float64)
            lws = do.init_log_weight_scale(pooled, head[do.NAMES[0]], head[do.NAMES[1]]).astype(np.float32)
            head[do.NAMES[1]] = lws
            _, lg, pf = functions(model_of(which, head))
            L = lambda xx: np.asarray(lg(xx), np.float64)
            out['logits_%s' % which] = L(x)
            out['p_%s' % which] = np.asarray(pf(x), np.float64)
            v, probe = d[which]
            out['dp_%s' % which] = np.array([np.sum(probe[t] * (L(x + H * v[t]) - L(x - H * v[t])) / (2 * H)) for t in range(len(v))])
            out['head_seed_%s' % which] = np.int64(HEAD_SEED[which])
            for k in do.NAMES[1:]:
                out['%s_%s' % (k, which)] = head[k]
            print(which, out['logits_%s' % which].ravel()[:6], out['dp_%s' % which], 'in %.1f s' % (time.time() - t0), flush=True)
    finally:
        shutil.rmtree(mgr.WORK, ignore_errors=True)
    path = os.path.join(mgr.OUT, 'ref_exec_discrim.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()

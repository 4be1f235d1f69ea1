"""Generate tests/golden/ref_exec_discrim_train.npz: the reference's own discriminator head l_discrim in TRAINING mode --
get_output(l_discrim, {l_in: X}) without deterministic, as train_IAN.py:139-149 and train_IAN_simple.py:405 build it --
and its directional derivatives, by EXECUTING the reference's Python files on the numpy stand-ins of oracle/refshim, in
float64: the fixture the training-mode entry points (ian_discriminate_train_*, ian_discriminate_train_vjp_*) and their
float64 restatement (tests/discrim_train_oracle.py) are pinned to.

The staging, the graphs' synthetic weights and the head's seeded tensors are make_golden_discrim.py's; log_weight_scale
comes from the reference's data-dependent rule (MinibatchLayer init=True, layers.py:510-513) on the training-mode pooled
features of the fixture's batch, so the pair terms stay alive.  The batch is the first N_IMG = 4 images of
ian_simple_golden.npz on every graph: bnorm2..4 (the stand-in's BatchNormLayer with deterministic=False) normalise with
its statistics and the MinibatchLayer compares its samples.  Per graph it stores the logits and p of the batch, the logits
of image 0 alone (n = 1: a batch of one normalises over its own pixels), stats (2,1792) -- row 0 the batch means of
bnorm2 | bnorm3 | bnorm4's inputs as the executed graph computes them, row 1 1/sqrt(var + 1e-4) --, log_weight_scale (float32,
as loaded), b, W, and dp[t] = <probe_t, (logits(x + h v_t) - logits(x - h v_t)) / 2h>, h = 1e-7, along
discrim_train_oracle.draws()'s tangents (the third moves image 1 alone and reads sample 0).

    python tests/golden/make_golden_discrim_train.py            # ~1 min

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
import make_golden_ref as mgr           # noqa: E402  (puts oracle/refshim and the reference on sys.path)
import make_golden_discrim as mgd       # noqa: E402
import discrim_oracle as do             # noqa: E402
import discrim_train_oracle as dto      # noqa: E402

SEED = 20261019
H = 1e-7
N_IMG = mgd.N_IMG
GRAPHS = mgd.GRAPHS


def functions(model):
    """(pooled, logits, p, bn_inputs): compiled training-mode functions of the GlobalPoolLayer, of l_discrim before and
    after its nonlinearity, and of the inputs of the trunk's three BatchNormLayers (bnorm2, bnorm3, bnorm4 in order)"""
    import theano
    import theano.tensor as T
    import lasagne
    X = T.TensorType('float64', [False] * 4)('X')
    l = model['l_discrim']
    get = lambda layer: theano.function([X], lasagne.layers.get_output(layer, {model['l_in']: X}))
    pool = get(l.input_layer.input_layer)
    bns = [b for b in lasagne.layers.get_all_layers(l) if isinstance(b, lasagne.layers.BatchNormLayer)]
    assert len(bns) == 3, len(bns)
    raw = [get(b.input_layer) for b in bns]
    nl = l.nonlinearity
    l.nonlinearity = lasagne.nonlinearities.identity
    lg = get(l)
    l.nonlinearity = nl
    return pool, lg, get(l), raw


def main():
    logging.basicConfig(level=logging.ERROR)
    d = dto.draws(SEED, N_IMG)
    out = {'seed': np.int64(SEED), 'h': np.float64(H), 'n_img': np.int64(N_IMG)}
    try:
        for which in GRAPHS:
            t0 = time.time()
            x, _ = mgd.images(which)
            x = x.astype(np.float64)
            head = do.make_discriminator_weights(which, mgd.HEAD_SEED[which])
            pool, _, _, _ = functions(mgd.model_of(which, head))
            pooled = np.asarray(pool(x), np.float64)
            head[do.NAMES[1]] = do.init_log_weight_scale(pooled, head[do.NAMES[0]], head[do.NAMES[1]]).astype(np.float32)
            _, lg, pf, raw = functions(mgd.model_of(which, head))
            L = lambda xx: np.asarray(lg(xx), np.float64)
            out['logits_%s' % which] = L(x)
            out['logits1_%s' % which] = L(x[:1])
            out['p_%s' % which] = np.asarray(pf(x), np.float64)
            st = []
            for f in raw:
                r = np.asarray(f(x), np.float64)
                st.append((r.mean(axis=(0, 2, 3)), 1.0 / np.sqrt(r.var(axis=(0, 2, 3)) + dto.BN_EPS)))
            out['stats_%s' % which] = np.stack([np.concatenate([m for m, _ in st]), np.concatenate([s for _, s in st])])
            v, probe = d[which]
            out['dp_%s' % which] = np.array([np.sum(probe[t] * (L(x + H * v[t]) - L(x - H * v[t])) / (2 * H)) for t in range(len(v))])
            out['head_seed_%s' % which] = np.int64(mgd.HEAD_SEED[which])
            for k in do.NAMES[1:]:
                out['%s_%s' % (k, which)] = head[k]
            print(which, out['logits_%s' % which].ravel()[:6], out['dp_%s' % which], 'in %.1f s' % (time.time() - t0), flush=True)
    finally:
        shutil.rmtree(mgr.WORK, ignore_errors=True)
    path = os.path.join(mgr.OUT, 'ref_exec_discrim_train.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()

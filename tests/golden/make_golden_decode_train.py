"""Generate tests/golden/ref_exec_decode_train.npz: the reference's own IAN_simple decoder in TRAINING mode --
get_output(l_out, {l_Z: Z}) without deterministic, as train_IAN_simple.py:217-224 and 253 build X_hat and the generated
samples -- and its directional derivatives, by EXECUTING the reference's Python files on the numpy stand-ins of
oracle/refshim, in float64: the fixture the training-mode entry points (ian_decode_train_*, ian_decode_train_vjp_*) and
their float64 restatement (tests/decode_train_oracle.py) are pinned to.

The staging (synthetic checkpoint next to a config symlink, the reference's API.IAN) is make_golden_ref.py's.  The batch
is decode_train_oracle.draws()'s N_IMG = 4 latents: bnorm_dec_fc2 and bnorm_dc1..3 (the stand-in's BatchNormLayer with
deterministic=False) normalise with its statistics.  Stored: x_hat of the batch and of sample 0 alone (n = 1), stats
(2,17280) -- row 0 the batch means of the four BatchNorms' inputs (bnorm_dec_fc2 in the reference's feature order), row 1
1/sqrt(var + 1e-4) --, dp[t] = <probe_t, (X(z + h v_t) - X(z - h v_t)) / 2h> along the three z-directions (the third moves
sample 1 alone and reads sample 0), and dq[k] the same along one direction of trainable tensor k, h = 1e-7.

    python tests/golden/make_golden_decode_train.py            # ~1 min

Only this script needs the reference's sources: the tests read the committed .npz file alone.
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
import make_golden_decjvp as mgj        # noqa: E402
import decode_train_oracle as dto       # noqa: E402

SEED = 20261020
H = 1e-7
N_IMG = 4


def functions(model):
    """(x_hat, bn_inputs, params): compiled training-mode functions of l_out and of the inputs of the decoder's four
    BatchNormLayers (bnorm_dec_fc2, bnorm_dc1..3 in order), and {name: shared variable} of the trainable tensors"""
    import theano
    import theano.tensor as T
    import lasagne
    Z = T.TensorType('float64', [False] * 2)('Z')
    lz, lo = model['l_Z'], model['l_out']
    get = lambda layer: theano.function([Z], lasagne.layers.get_output(layer, {lz: Z}))
    layers = lasagne.layers.get_all_layers(lo, treat_as_input=[lz])
    bns = [b for b in layers if isinstance(b, lasagne.layers.BatchNormLayer)]
    assert len(bns) == 4, len(bns)
    params = {p.name: p for p in lasagne.layers.get_all_params(lo, trainable=True) if p.name in dto.PARAM_NAMES}
    assert sorted(params) == sorted(dto.PARAM_NAMES), sorted(params)
    return get(lo), [get(b.input_layer) for b in bns], params


def main():
    logging.basicConfig(level=logging.ERROR)
    from API import IAN                                   # the reference's API.py
    seed = mgj.weight_seed('simple')
    z, v, probe, pdir, pprobe = dto.draws(SEED, N_IMG)
    out = {'seed': np.int64(SEED), 'h': np.float64(H), 'n_img': np.int64(N_IMG), 'weight_seed': np.int64(seed)}
    try:
        t0 = time.time()
        link = mgr._stage('IAN_simple.py', mgr.ow.make_simple_weights(seed))
        X, raw, params = functions(IAN(config_path=link, dnn=True).model)
        L = lambda zz: np.asarray(X(zz), np.float64)
        out['x_hat'] = L(z)
        out['x_hat1'] = L(z[:1])
        st = []
        for k, f in enumerate(raw):
            r = np.asarray(f(z), np.float64)
            axes = (0,) if r.ndim == 2 else (0, 2, 3)
            st.append((r.mean(axis=axes), 1.0 / np.sqrt(r.var(axis=axes) + dto.BN_EPS)))
        out['stats'] = np.stack([np.concatenate([m for m, _ in st]), np.concatenate([s for _, s in st])])
        out['dp'] = np.array([np.sum(probe[t] * (L(z + H * v[t]) - L(z - H * v[t])) / (2 * H)) for t in range(len(v))])
        dq = []
        for k, name in enumerate(dto.PARAM_NAMES):
            p = params[name]
            w = np.array(p.get_value(), np.float64)
            p.set_value(w + H * pdir[name])
            xp = L(z)
            p.set_value(w - H * pdir[name])
            xm = L(z)
            p.set_value(w)
            dq.append(np.sum(pprobe[k] * (xp - xm) / (2 * H)))
        out['dq'] = np.array(dq)
        print(out['x_hat'].ravel()[:4], out['dp'], out['dq'], 'in %.1f s' % (time.time() - t0), flush=True)
    finally:
        shutil.rmtree(mgr.WORK, ignore_errors=True)
    path = os.path.join(mgr.OUT, 'ref_exec_decode_train.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()

"""tests/golden/ref_exec_train_grad.npz: directional derivatives of the training-mode ops, from the executed reference.

The reference's own MinibatchLayer (layers.py:486-524) and the stand-in BatchNormLayer (training mode, as `BN(...)` of the
reference graphs runs it) are evaluated unmodified on the numpy stand-ins of oracle/refshim, in float64, as
make_golden_train.py does for their forward.  For each case the file keeps the inputs, a seeded probe R of the output's
shape, L = Σ R·out, and for every differentiable input p a seeded direction v_p with the float64 central difference
dL[p] = (8 (L(p + h v) - L(p - h v)) - (L(p + 2h v) - L(p - 2h v))) / (12 h), fourth order.  MinibatchLayer takes
h = 1e-5, small enough that no |A_ikp - A_jkp| changes sign inside the stencil (|.| has a kink at 0).  BatchNorm takes
h = 3e-5: the constant channel's inv_std bends on the scale sqrt(eps) = 1e-2, so a larger step truncates, and the offset
channel's x - mean loses the difference to cancellation at a smaller one.

Cases are the forward fixtures' edges: MinibatchLayer on a (4, 4, 4) feature map with K = 7, P = 5, and with d = 33 at
n = 1 (f = b), K = P = 1 and K = 13, P = 5; BatchNorm on a conv and a dense input, and on a conv input with one channel
offset far from zero (mean 1000, std 1) and one constant channel (1000.1).

    python tests/golden/make_golden_train_grad.py
"""
import os
import sys

import numpy as np

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = '/root/reference'
sys.path[:0] = [os.path.join(ROOT, 'oracle', 'refshim'), REF, ROOT]
OUT = os.environ.get('REF_EXEC_OUT', os.path.join(ROOT, 'tests', 'golden'))


def directional(fn, args, key, v, h):
    """fourth-order central difference of fn(**args) along v in args[key]"""
    def at(t):
        a = dict(args)
        a[key] = args[key] + t * v
        return fn(**a)
    return (8 * (at(h) - at(-h)) - (at(2 * h) - at(-2 * h))) / (12 * h)


def main():
    import theano
    import theano.tensor as T
    import lasagne
    import layers as ref_layers                           # the reference's layers.py
    rng = np.random.default_rng(21)
    out = {}

    def mb_case(tag, x, K, P, lws_mean):
        n, shape = len(x), x.shape[1:]
        d = int(np.prod(shape))
        l_in = lasagne.layers.InputLayer((None,) + shape)
        mb = ref_layers.MinibatchLayer(l_in, num_kernels=K, dim_per_kernel=P, name='minibatch_discrim')
        X = T.TensorType('float64', [False] * x.ndim)('X')
        f = theano.function([X], lasagne.layers.get_output(mb, {l_in: X}))
        args = dict(x=x, theta=rng.normal(0, 0.05, (d, K, P)), lws=rng.normal(lws_mean, 0.2, (K, P)), b=rng.normal(-1, 0.2, K))
        R = rng.standard_normal((n, d + K))

        def L(x, theta, lws, b):
            mb.theta.set_value(theta); mb.log_weight_scale.set_value(lws); mb.b.set_value(b)
            return float(np.sum(R * f(x)))
        scale = dict(x=1.0, theta=0.05, lws=0.2, b=0.2)
        res = {'x': x, 'theta': args['theta'], 'lws': args['lws'], 'b': args['b'], 'R': R, 'L': L(**args)}
        for key in ('x', 'theta', 'lws', 'b'):
            v = scale[key] * rng.standard_normal(np.shape(args[key]))
            res['v_' + key], res['dL_' + key] = v, directional(L, args, key, v, 1e-5)
        out.update({'mb_%s_%s' % (tag, k): val for k, val in res.items()})

    mb_case('main', rng.standard_normal((6, 4, 4, 4)), 7, 5, 0.0)
    for tag, n, K, P in (('n1', 1, 13, 5), ('k1p1', 6, 1, 1), ('k13p5', 17, 13, 5)):
        mb_case(tag, rng.standard_normal((n, 33)), K, P, np.log(0.1))

    def bn_case(tag, x):
        shape = x.shape[1:]
        c = shape[0]
        l_in = lasagne.layers.InputLayer((None,) + shape)
        bn = lasagne.layers.BatchNormLayer(l_in, name='bn_' + tag)
        X = T.TensorType('float64', [False] * x.ndim)('X')
        f = theano.function([X], lasagne.layers.get_output(bn, {l_in: X}, deterministic=False))
        args = dict(x=x, gamma=rng.uniform(0.5, 1.5, c), beta=rng.normal(0, 0.1, c))
        R = rng.standard_normal(x.shape)

        def L(x, gamma, beta):
            bn.gamma.set_value(gamma); bn.beta.set_value(beta)
            return float(np.sum(R * f(x)))
        res = {'x': x, 'gamma': args['gamma'], 'beta': args['beta'], 'R': R, 'L': L(**args)}
        for key in ('x', 'gamma', 'beta'):
            v = rng.standard_normal(np.shape(args[key]))
            res['v_' + key], res['dL_' + key] = v, directional(L, args, key, v, 3e-5)
        out.update({'bn_%s_%s' % (tag, k): val for k, val in res.items()})

    bn_case('conv', rng.standard_normal((5, 8, 6, 6)) * 2 + 0.5)
    bn_case('dense', rng.standard_normal((9, 20)) * 3 - 1)
    xe = np.empty((6, 2, 17, 19))
    xe[:, 0] = 1000.0 + rng.standard_normal((6, 17, 19))
    xe[:, 1] = 1000.1
    bn_case('edges', xe)
    path = os.path.join(OUT, 'ref_exec_train_grad.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()

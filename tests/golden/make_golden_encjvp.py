"""Generate tests/golden/ref_exec_encjvp.npz: Jacobian-vector products of the reference's own Z_hat (API.py:50-51) by
EXECUTING the reference's Python files on the numpy stand-ins of oracle/refshim, in float64 -- the fixture the encoder
Jacobian-vector product (ian_encode_jvp_*) is pinned to.

The staging and the compiled functions are make_golden_encvjp.py's, reused by import.  Per graph and golden image (the
first two of ian_<graph>_golden.npz), without and with eps, the full 100-vector central difference
    Jv = (Z(x + h v) - Z(x - h v)) / 2h,      h = 1e-7
where Z is the compiled Z_hat function (no eps) or, with eps, Z_IAF_fn (sample_IAN.py:92) of mu + exp(logsigma) eps.
v and eps are drawn from the stored seed (make_golden_encvjp.draws), which keeps the file a few KB.

    python tests/golden/make_golden_encjvp.py            # ~2 min

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
import make_golden_encvjp as mge   # noqa: E402  (and, through it, make_golden_ref's staging)

SEED = 20261016
H = mge.H
N_IMG = mge.N_IMG


def main():
    logging.basicConfig(level=logging.ERROR)
    d = mge.draws(SEED)
    out = {'seed': np.int64(SEED), 'h': np.float64(H), 'n_img': np.int64(N_IMG)}
    try:
        for which in ('simple', 'full', 'v1'):
            t0 = time.time()
            z_hat, mu_ls, flow = mge.functions(which)
            x, _ = mge.images(which)
            v, _, eps = d[which]
            jv = np.zeros((2, N_IMG, 100))
            for k in range(N_IMG):
                xk = x[k:k + 1].astype(np.float64)
                for j, with_eps in enumerate((False, True)):
                    def Z(xx):
                        if not with_eps:
                            return np.asarray(z_hat(xx), np.float64)
                        mu, ls = (np.asarray(a, np.float64) for a in mu_ls(xx))
                        zi = mu + np.exp(ls) * eps[k:k + 1]
                        return zi if flow is None else np.asarray(flow(zi), np.float64)
                    jv[j, k] = ((Z(xk + H * v[k:k + 1]) - Z(xk - H * v[k:k + 1])) / (2 * H))[0]
            out['jv_' + which] = jv                       # [without eps, with eps][image][100]
            print(which, np.abs(jv).max(axis=2), 'in %.1f s' % (time.time() - t0), flush=True)
    finally:
        shutil.rmtree(mge.mgr.WORK, ignore_errors=True)
    path = os.path.join(mge.mgr.OUT, 'ref_exec_encjvp.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()

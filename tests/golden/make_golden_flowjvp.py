"""Generate tests/golden/ref_exec_flowjvp.npz: Jacobian-vector products of the reference's own Zfn and Z_IAF_fn
(sample_IAN.py:91-94) by EXECUTING the reference's Python files on the numpy stand-ins of oracle/refshim, in float64 -- the
fixture the prior-space derivatives (ian_encode_pre_jvp_*, ian_flow_jvp_*) are pinned to.

The staging and the compiled functions are make_golden_encvjp.py's, reused by import: Zfn is the compiled mu function
(deterministic l_Z_IAF = mu), Z_IAF_fn the compiled flow.  Per flow graph (IAN.py, IANv1.py) and golden image (the first
two of ian_<graph>_golden.npz), the full 100-vector central differences
    Zfn:       (mu(x + h vx) - mu(x - h vx)) / 2h
    Z_IAF_fn:  (F(z + h vz) - F(z - h vz)) / 2h    at z = mu(x) and at an N(0,1) prior draw,     h = 1e-7
vx, vz and the prior draws come from the stored seed (draws()); mu(x) is stored, so the file stays a few KB.

    python tests/golden/make_golden_flowjvp.py            # ~1 min

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

SEED = 20261017
H = mge.H
N_IMG = mge.N_IMG
GRAPHS = ('full', 'v1')


def draws(seed=SEED):
    """per flow graph: image directions vx (N_IMG,3,64,64), prior draws z (N_IMG,100) and latent directions vz (N_IMG,100)"""
    rng = np.random.RandomState(seed)
    return {g: (rng.standard_normal((N_IMG, 3, 64, 64)), rng.standard_normal((N_IMG, 100)), rng.standard_normal((N_IMG, 100)))
            for g in GRAPHS}


def main():
    logging.basicConfig(level=logging.ERROR)
    d = draws()
    out = {'seed': np.int64(SEED), 'h': np.float64(H), 'n_img': np.int64(N_IMG)}
    try:
        for which in GRAPHS:
            t0 = time.time()
            _, mu_ls, flow = mge.functions(which)
            x, _ = mge.images(which)
            vx, zp, vz = d[which]
            mu = lambda xx: np.asarray(mu_ls(xx)[0], np.float64)
            F = lambda zz: np.asarray(flow(zz), np.float64)
            z_zfn = np.zeros((N_IMG, 100))
            jv = {k: np.zeros((N_IMG, 100)) for k in ('zfn', 'flow_zfn', 'flow_prior')}
            for k in range(N_IMG):
                xk = x[k:k + 1].astype(np.float64)
                z_zfn[k] = mu(xk)[0]
                jv['zfn'][k] = ((mu(xk + H * vx[k:k + 1]) - mu(xk - H * vx[k:k + 1])) / (2 * H))[0]
                for name, z in (('flow_zfn', z_zfn[k:k + 1]), ('flow_prior', zp[k:k + 1])):
                    jv[name][k] = ((F(z + H * vz[k:k + 1]) - F(z - H * vz[k:k + 1])) / (2 * H))[0]
            out['z_zfn_' + which] = z_zfn
            for name, a in jv.items():
                out['jv_%s_%s' % (name, which)] = a
            print(which, {k: float(np.abs(a).max()) for k, a in jv.items()}, 'in %.1f s' % (time.time() - t0), flush=True)
    finally:
        shutil.rmtree(mge.mgr.WORK, ignore_errors=True)
    path = os.path.join(mge.mgr.OUT, 'ref_exec_flowjvp.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()

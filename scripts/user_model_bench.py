"""What does a user likelihood cost on the C2 random walk?  One C2-shaped queue fill (Q = 2000 chains, walks 70,
n = 50, the correlated Gaussian behind U(-5, 5)) timed three ways on the same start points and bound:

  registry        LIKE_GAUSS_PREC on the default kernel (the lock-step DMMA kernel at n = 50)
  registry-warp   the same model forced onto the warp-per-chain kernel (B2N_RWALK_IMPL=warp)
  user            the precision-matrix Gaussian restated as user CUDA code (DeviceModel.from_cuda), which always
                  runs on the warp-per-chain kernel
  user-prior      the same user likelihood with the U(-5, 5) box restated as a user prior (b2n_user_prior): the
                  prior moves out of the fused per-element proposal loop into one warp call per accepted-cube
                  proposal; the outputs must equal the user row's bit for bit (same_as_user)

Kernel time per fill from CUDA events around the chain kernel (b2n_set_timing), median of --reps fills after
--warmup; the card name and power limit are read in the same run.  usage: python scripts/user_model_bench.py"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dynesty_b200 import _lib, ops, likelihoods as DL                  # noqa: E402
from dynesty_b200.likelihoods import DeviceModel                         # noqa: E402
from oracle import bounding as OB                                        # noqa: E402

PREC = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    for (int i = lane; i < n; i += 32) work[i] = v[i] - p[i];
    __syncwarp();
    const double* P = p + n;
    double s = 0.0;
    for (int i = lane; i < n; i += 32) {
        double y = 0.0;
        for (int j = 0; j < n; j++) y = fma(P[(size_t)j * n + i], work[j], y);
        s = fma(work[i], y, s);
    }
    s = b2n_warp_sum(s);
    __syncwarp();
    return fma(-0.5, s, p[n + n * n]);
}
'''

PRIOR_UNIFORM = r'''
__device__ void b2n_user_prior(const double* u, double* v, double* work, int n, const double* p, int lane) {
    for (int i = lane; i < n; i += 32) v[i] = fma(p[n + i], u[i], p[i]);
}
'''


def card():
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, plim = [x.strip() for x in out.split(',')[:2]]
        return name, plim
    except Exception as e:                                              # noqa: BLE001
        return 'unknown (%r)' % (e,), 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--Q', type=int, default=2000)
    ap.add_argument('--walks', type=int, default=70)
    ap.add_argument('--n', type=int, default=50)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    a = ap.parse_args()
    n = a.n
    reg = DL.gauss_corr(n, 0.4, 5.0)
    user = DeviceModel.from_cuda(n, PREC, params=np.concatenate([reg.like_vec0, reg.like_mat.T.ravel(), [reg.s[0]]]),
                                 prior_kind=_lib.PRIOR_UNIFORM, prior_p0=-5.0, prior_p1=10.0, name='user_gauss_corr')
    user_prior = DeviceModel.from_cuda(n, PREC, params=user.params, prior_source=PRIOR_UNIFORM,
                                       prior_params=np.concatenate([np.full(n, -5.0), np.full(n, 10.0)]),
                                       name='user_prior_gauss_corr')
    rng = np.random.default_rng(1)
    Cm = np.full((n, n), 0.4)
    np.fill_diagonal(Cm, 1.0)
    pts = 0.5 + 0.08 * rng.standard_normal((4000, n)) @ np.linalg.cholesky(Cm).T
    _, logl = reg.evaluate(pts)
    loglstar = float(np.quantile(logl, 0.2))
    good = pts[logl > loglstar]
    ell = OB.bounding_ellipsoid(good)
    ops.bound_set(ell.axes[None])
    u0 = np.ascontiguousarray(good[rng.integers(len(good), size=a.Q)])
    ctx = _lib.default_context()
    ctx.set_timing(True)
    name, plim = card()
    res, outs = {}, {}
    for label, m, env in (('registry', reg, None), ('registry-warp', reg, 'warp'), ('user', user, None),
                          ('user-prior', user_prior, None)):
        if env:
            os.environ['B2N_RWALK_IMPL'] = env
        else:
            os.environ.pop('B2N_RWALK_IMPL', None)
        mid = m.model_id()
        ms = []
        for r in range(a.warmup + a.reps):
            o = ops.rwalk_batch(mid, u0, loglstar, 0.5, a.walks, 7, chain0=0)
            outs[label] = {k: np.array(o[k]) for k in ('u', 'v', 'logl', 'n_accept')}
            if r >= a.warmup:
                ms.append(ctx.last_kernel_ms())
        res[label] = dict(ms_per_fill=round(float(np.median(ms)), 4), ms_min=round(float(np.min(ms)), 4))
    res['user-prior']['same_as_user'] = all(np.array_equal(outs['user'][k], outs['user-prior'][k])
                                            for k in ('u', 'v', 'logl', 'n_accept'))
    os.environ.pop('B2N_RWALK_IMPL', None)
    print(json.dumps(dict(card=name, power_limit=plim, Q=a.Q, walks=a.walks, n=n, reps=a.reps, results=res)))


if __name__ == '__main__':
    main()

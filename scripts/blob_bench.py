"""What does saving a blob cost?  Two measurements on a user model with blobs:

  kernel   b2n_model_blob over a C2-shaped record (M = 52 000 points, n = 50, nblob = 8): the blob is the
           log-likelihood of the precision-matrix Gaussian (one n x n mat-vec per point, as in the chains) plus
           seven coordinates.  Kernel time from CUDA events around the launch (b2n_set_timing), median of --reps
           calls after --warmup.
  run      one C2 device run (nlive 2000, multi / rwalk, walks 70, n = 50, the user Gaussian behind U(-5, 5)) with
           blob=False and blob=True, alternated --runs times; wall time of run_nested, and whether every other result
           key has the same bits.

The blob pass makes niter evaluations where the run makes ncall (about walks x niter for rwalk).  The card name and
power limit are read in the same run.  usage: python scripts/blob_bench.py"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dynesty_b200 import _lib, nested, likelihoods as DL                # noqa: E402
from dynesty_b200.likelihoods import DeviceModel                         # noqa: E402

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

__device__ void b2n_user_blob(const double* v, double* work, int n, const double* p, int lane, double* blob,
                              int nblob) {
    const double l = b2n_user_loglike(v, work, n, p, lane);
    if (lane == 0) blob[0] = l;
    for (int j = 1 + lane; j < nblob; j += 32) blob[j] = v[j - 1];
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
    ap.add_argument('--M', type=int, default=52000)
    ap.add_argument('--n', type=int, default=50)
    ap.add_argument('--nblob', type=int, default=8)
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--runs', type=int, default=2, help='C2 runs per setting (0: kernel only)')
    ap.add_argument('--nlive', type=int, default=2000)
    a = ap.parse_args()
    n = a.n
    reg = DL.gauss_corr(n, 0.4, 5.0)
    user = DeviceModel.from_cuda(n, PREC, params=np.concatenate([reg.like_vec0, reg.like_mat.T.ravel(), [reg.s[0]]]),
                                 prior_kind=_lib.PRIOR_UNIFORM, prior_p0=-5.0, prior_p1=10.0, nblob=a.nblob,
                                 name='user_gauss_corr_blob')
    ctx = _lib.default_context()
    name, plim = card()
    v = np.random.default_rng(1).uniform(-5.0, 5.0, (a.M, n))
    ctx.set_timing(True)
    ms = []
    for r in range(a.warmup + a.reps):
        b = user.blob(v)
        if r >= a.warmup:
            ms.append(ctx.last_kernel_ms())
    ctx.set_timing(False)
    ok = bool(np.array_equal(b[:, 0], user.loglikelihood(v)) and np.array_equal(b[:, 1:], v[:, :a.nblob - 1]))
    out = dict(card=name, power_limit=plim, kernel=dict(M=a.M, n=n, nblob=a.nblob, reps=a.reps,
                                                        ms_median=round(float(np.median(ms)), 4),
                                                        ms_min=round(float(np.min(ms)), 4),
                                                        ms_max=round(float(np.max(ms)), 4), matches=ok))
    runs = {False: [], True: []}
    res = {}
    for _ in range(a.runs):
        for blob in (False, True):
            s = nested.NestedSampler(user, nlive=a.nlive, bound='multi', sample='rwalk', seed=7, blob=blob)
            t0 = time.perf_counter()
            res[blob] = s.run_nested(loop='device')
            runs[blob].append(time.perf_counter() - t0)
    if a.runs:
        same = all(np.array_equal(np.asarray(res[True][k]), np.asarray(res[False][k])) if
                   isinstance(res[False][k], np.ndarray) else res[True][k] == res[False][k] for k in res[False])
        out['run'] = dict(nlive=a.nlive, niter=int(res[True]['niter']), ncall=int(res[True]['ncall']),
                          samples=len(res[True]['logl']), wall_s_plain=[round(t, 3) for t in runs[False]],
                          wall_s_blob=[round(t, 3) for t in runs[True]], other_keys_identical=bool(same),
                          blob_is_model_blob=bool(np.array_equal(res[True]['blob'], user.blob(res[True]['samples']))))
    print(json.dumps(out))


if __name__ == '__main__':
    main()

"""What does a likelihood written in PyTorch cost?  One C2-shaped fill (50-D correlated Gaussian, prior U(-5, 5)^50,
2000 chains x 70 walks, one ellipsoid) three ways, then a whole C2 run with the torch model:

  registry   rwalk_batch with the registry's GAUSS_PREC model (the fused kernel the planner picks)
  user       rwalk_batch with the same likelihood as user CUDA (DeviceModel.from_cuda, warp-per-chain kernel)
  torch      rwalk_stepped with the same likelihood as a TorchModel: 71 stepped launches and 71 torch calls
  profile    one torch fill under torch.profiler: the share of the fill's GPU time in the stepped kernel and in the
             torch calls' kernels
  run        NestedSampler(TorchModel, nlive 2000, multi / rwalk, walks 70).run_nested(loop='device'): wall time, and
             ln Z against the analytic -115.129

Proposals/s = chains x walks / fill time; fill time = median over --reps fills after --warmup, each ended by a device
synchronise.  The card's name and power limit are read in the same process.  usage: python
scripts/torch_model_bench.py [--reps 20] [--no-run]"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dynesty_b200 import TorchModel, _lib, nested, ops, likelihoods as DL      # noqa: E402
from dynesty_b200.likelihoods import DeviceModel                               # noqa: E402

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
N, Q, WALKS, H = 50, 2000, 70, 5.0


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:            # (the measurement itself does not depend on nvidia-smi)
        return 'unknown (%s)' % e


def models():
    reg = DL.gauss_corr(N, 0.4, H)
    prec = reg.like_mat
    user = DeviceModel.from_cuda(N, PREC, params=np.concatenate([np.zeros(N), prec.T.ravel(), [reg.s[0]]]),
                                 prior_kind=_lib.PRIOR_UNIFORM, prior_p0=-H, prior_p1=2 * H, name='user_c2')
    dev = torch.device('cuda', _lib.default_context().device)
    P = torch.as_tensor(prec.copy(), device=dev)
    lnorm = reg.s[0]
    tm = TorchModel(N, lambda v: -0.5 * torch.sum((v @ P) * v, 1) + lnorm, lambda u: 2 * H * u - H, name='torch_c2')
    return reg, user, tm


def fill_inputs(reg, rng):
    """Start points and threshold of a fill in the middle of a C2 run: points of the posterior bulk."""
    v = rng.multivariate_normal(np.zeros(N), np.linalg.inv(reg.like_mat), size=4 * Q)
    u = (v + H) / (2 * H)
    _, l = reg.evaluate(u)
    loglstar = float(np.quantile(l, 0.2))
    good = u[l > loglstar]
    cov = np.cov(good, rowvar=False)
    axes = np.linalg.cholesky(cov * (N + 2))
    return np.ascontiguousarray(good[rng.integers(len(good), size=Q)]), loglstar, axes


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--no-run', action='store_true')
    a = ap.parse_args()
    out = dict(card=card(), shape=dict(ndim=N, chains=Q, walks=WALKS))
    reg, user, tm = models()
    rng = np.random.default_rng(1)
    u0, loglstar, axes = fill_inputs(reg, rng)
    ops.bound_set(axes)
    scale = 0.5
    cases = dict(
        registry=lambda: ops.rwalk_batch(reg.model_id(), u0, loglstar, scale, WALKS, 7),
        user=lambda: ops.rwalk_batch(user.model_id(), u0, loglstar, scale, WALKS, 7),
        torch=lambda: ops.rwalk_stepped(tm, u0, loglstar, scale, WALKS, 7))
    fills = {}
    for k, fn in cases.items():
        t = timed(fn, a.reps, a.warmup)
        fills[k] = dict(fill_ms=1e3 * t, proposals_per_s=Q * WALKS / t)
    out['fill'] = fills
    # profile: share of the fill's GPU time
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cases['torch']()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type.name == 'CUDA']
    tot = sum(e.time_range.elapsed_us() for e in ev) or 1.0
    step = sum(e.time_range.elapsed_us() for e in ev if e.name.startswith('rwalk_step_kernel'))
    cp = sum(e.time_range.elapsed_us() for e in ev if 'memcpy' in e.name.lower() or 'memset' in e.name.lower())
    out['profile'] = dict(gpu_us=tot, stepped_kernel_share=step / tot, torch_kernels_share=(tot - step - cp) / tot,
                          copies_share=cp / tot, stepped_launches=sum(1 for e in ev if e.name.startswith('rwalk_step_kernel')))
    if not a.no_run:
        t0 = time.perf_counter()
        r = nested.NestedSampler(tm, nlive=2000, bound='multi', sample='rwalk', walks=WALKS, seed=11).run_nested(
            loop='device')
        out['run'] = dict(wall_s=time.perf_counter() - t0, logz=float(r['logz'][-1]),
                          logzerr=float(r['logzerr'][-1]), logz_truth=-N * math.log(2 * H),
                          niter=int(r['niter']), ncall=int(r['ncall']))
    print(json.dumps(out))


if __name__ == '__main__':
    main()

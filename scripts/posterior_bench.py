"""Time b2n_jitter_posterior / b2n_resample_posterior on a C2-shaped record (nlive 2000, rounds of K = 50, add_live
tail, N ~ 52 000) with n = 50 synthesised positions, R = 128 realisations.

    python scripts/posterior_bench.py [--R 128] [--n 50] [--calls 10] [--oracle]

Kernel time: CUDA events around each call's launches (b2n_set_timing), median over `calls` calls after warm-up, for
the producer alone (b2n_jitter_runs / b2n_resample_runs), the producer with the moments (q = None), and everything
(q = 5 quantiles).  The stage times are the differences: moments = shift + GEMM + finish, sort + quantiles = the CUB
sort, its key kernel and the two quantile kernels.  The moment GEMM's FP64 rate counts 2 R N P flops (P = 1 + n +
n(n+1)/2) over the whole moments stage, against b2n_fp64_peak (MMA) measured in the same run.  The card's name and
power limit are read in the same call.  --oracle adds the host time of the numpy loop over the realisations
(oracle/posterior.py).  Prints one JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dynesty_b200 import _lib, ops, utils as DU  # noqa: E402
from dynesty_b200.nested import Results  # noqa: E402
from oracle import posterior as OP, resample as ORS  # noqa: E402
from scripts.jitter_bench import card  # noqa: E402

Q = [0.0, 0.025, 0.5, 0.975, 1.0]


def record(n):
    rec = ORS.synthetic_strand_record(2000, 50, seed=0)
    rng = np.random.default_rng(7)
    u = rng.standard_normal((len(rec['logl']), n))
    u /= np.linalg.norm(u, axis=1)[:, None]
    rec['samples'] = 0.5 + 1e-3 * np.sqrt(-2.0 * rec['logl'])[:, None] * u
    return Results(rec)


def timed(ctx, fn, warmup, calls):
    ms = []
    for i in range(warmup + calls):
        fn()
        if i >= warmup:
            ms.append(ctx.last_kernel_ms())
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--R', type=int, default=128)
    ap.add_argument('--n', type=int, default=50)
    ap.add_argument('--calls', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--oracle', action='store_true')
    a = ap.parse_args()
    res = record(a.n)
    N, n, R = len(res['logl']), a.n, a.R
    P = 1 + n + n * (n + 1) // 2
    ctx = _lib.default_context()
    ctx.set_timing(True)
    name, plim = card()
    peak = ops.fp64_peak('mma', 20000, ctx=ctx)[0]
    out = dict(card=name, power_limit=plim, N=N, n=n, R=R, P=P, nq=len(Q), calls=a.calls,
               fp64_mma_peak_tflops=peak, gemm_gflop=2.0 * R * N * P / 1e9)
    plan = DU.strand_plan(res)
    pp, ps = DU._piece_csr(np.asarray(res['logl']), plan)
    sargs = (res['logl'], plan['strand'], plan['base'], pp, ps, plan['end'])
    x, kw = np.asarray(res['samples']), dict(logwt_ref=res['logwt'], logz_ref=res['logz'][-1], ctx=ctx)
    for error in ('jitter', 'resample'):
        if error == 'jitter':
            prod = lambda: ops.jitter_runs(res['logl'], res['samples_n'], R, 1234, **kw)
            post = lambda q: ops.jitter_posterior(res['logl'], res['samples_n'], x, R, 1234, q=q, **kw)
        else:
            prod = lambda: ops.resample_runs(*sargs, R, 1234, **kw)
            post = lambda q: ops.resample_posterior(*sargs, x, R, 1234, q=q, **kw)
        t0 = timed(ctx, prod, a.warmup, a.calls)
        t1 = timed(ctx, lambda: post(None), a.warmup, a.calls)
        t2 = timed(ctx, lambda: post(Q), a.warmup, a.calls)
        mom = t1 - t0
        out[error] = dict(producer_ms=t0, moments_ms=mom, sort_quantiles_ms=t2 - t1, total_ms=t2,
                          moments_tflops=2.0 * R * N * P / (mom * 1e-3) / 1e12,
                          moments_share_of_mma_peak=2.0 * R * N * P / (mom * 1e-3) / 1e12 / peak)
    if a.oracle:
        t = time.perf_counter()
        OP.jitter_posterior(res['logl'], res['samples_n'], x, R, 1234, q=Q, logwt_ref=res['logwt'],
                            logz_ref=res['logz'][-1])
        out['oracle_jitter_host_s'] = time.perf_counter() - t
    print(json.dumps(out))


if __name__ == '__main__':
    main()

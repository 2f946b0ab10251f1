"""Time the equal-weight draws on a merged record: R = 64 C2-shaped records (nlive 2000, rounds of K = 50, add_live
tail; oracle.jitter.synthetic_record with seeds 0..63) merged into one by b2n_merge_runs, as scripts/merge_bench.py
builds it.

    python scripts/equal_bench.py [--R 64] [--n-mc 128] [--calls 10] [--warmup 2] [--ref-calls 3]

  resample_equal      utils.resample_equal of the merged record's importance weights (M = N): wall time of the call
                      (host arrays in and out, synchronised) and kernel time (CUDA events, b2n_set_timing), medians over
                      `calls` after `warmup`; against the reference's resample_equal (oracle/_ref, when present) with a
                      numpy Generator, median wall time over `ref-calls`, and the reference through
                      oracle.equal.ScriptedEqualGenerator checked bit for bit against the GPU's indices.
  equal_realisations  n_mc jitter realisations with M draws each (b2n_jitter_equal; M = 10^5 and M = N by default),
                      kernel and wall time, next to b2n_jitter_runs alone (the realisations without the draws).
The card's name and power limit are printed with the numbers.  Prints one JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np

T0 = time.perf_counter()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from dynesty_b200 import _lib, ops, utils as DU  # noqa: E402
from dynesty_b200.nested import Results  # noqa: E402
from oracle import equal as OE, jitter as OJ, refshim  # noqa: E402
from jitter_bench import card  # noqa: E402


def merged_record(R):
    recs = [OJ.synthetic_record(seed=s) for s in range(R)]
    logl = np.concatenate([r[0] for r in recs])
    n = np.concatenate([r[1] for r in recs])
    run_ptr = np.r_[0, np.cumsum([len(r[0]) for r in recs])]
    o = ops.merge_runs(logl, n, run_ptr, R, arrays=True)
    return Results(dict(logl=logl[o['perm']], samples_n=o['samples_n'], logwt=o['logwt'], logz=o['logz']))


def log(msg):
    sys.stderr.write('%.1f s  %s\n' % (time.perf_counter() - T0, msg))
    sys.stderr.flush()


def timed(fn, ctx, calls, warmup):
    wall, kern = [], []
    for i in range(warmup + calls):
        t = time.perf_counter()
        out = fn()
        dt = time.perf_counter() - t
        if i >= warmup:
            wall.append(dt * 1e3)
            kern.append(ctx.last_kernel_ms())
    return out, float(np.median(wall)), float(np.median(kern))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--R', type=int, default=64)
    ap.add_argument('--n-mc', type=int, default=128)
    ap.add_argument('--calls', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--ref-calls', type=int, default=3)
    ap.add_argument('--nsamples', type=int, nargs='+', default=[100000, 0],
                    help='draws per realisation of equal_realisations (0: the record length)')
    a = ap.parse_args()
    ctx = _lib.default_context()
    ctx.set_timing(True)
    res = merged_record(a.R)
    N = len(res['logl'])
    log('merged record: N = %d' % N)
    name, plim = card()
    out = dict(card=name, power_limit=plim, nlive=2000, K=50, R=a.R, N=N, n_mc=a.n_mc, calls=a.calls)

    w = res.importance_weights()
    x = np.arange(N)
    seed = 12345
    idx, out['resample_equal_wall_ms'], out['resample_equal_kernel_ms'] = timed(
        lambda: DU.resample_equal(x, w, seed=seed, ctx=ctx), ctx, a.calls, a.warmup)
    log('resample_equal: %.2f ms' % out['resample_equal_wall_ms'])
    if refshim.available():
        U = refshim.import_reference().utils
        ts = []
        for i in range(a.ref_calls):
            g = np.random.default_rng(i)
            t = time.perf_counter()
            U.resample_equal(x, w, rstate=g)
            ts.append((time.perf_counter() - t) * 1e3)
        out['reference_wall_ms'] = float(np.median(ts))
        out['speedup_wall'] = out['reference_wall_ms'] / out['resample_equal_wall_ms']
        ref = U.resample_equal(x, w, rstate=OE.ScriptedEqualGenerator(seed, 0))
        out['reference_bit_equal'] = bool(np.array_equal(ref, idx))
        log('reference: %.1f ms' % out['reference_wall_ms'])

    lz = float(res['logz'][-1])
    _, out['jitter_runs_wall_ms'], out['jitter_runs_kernel_ms'] = timed(
        lambda: ops.jitter_runs(res['logl'], res['samples_n'], a.n_mc, 7, logwt_ref=res['logwt'], logz_ref=lz,
                                ctx=ctx), ctx, a.calls, a.warmup)
    log('jitter_runs: %.2f ms' % out['jitter_runs_wall_ms'])
    for M in a.nsamples:
        M = M or N
        l0 = ctx.launch_count()
        o, wall, kern = timed(lambda: DU.equal_realisations(res, a.n_mc, 7, nsamples=M, ctx=ctx), ctx, a.calls,
                              a.warmup)
        out['equal_realisations_M%d' % M] = dict(wall_ms=wall, kernel_ms=kern, idx_shape=list(o['idx'].shape),
                                                 launches=(ctx.launch_count() - l0) // (a.calls + a.warmup))
        del o
        log('equal_realisations M = %d: %.2f ms' % (M, wall))
    print(json.dumps(out))


if __name__ == '__main__':
    main()

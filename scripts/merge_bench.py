"""Time b2n_merge_runs: R = 64 C2-shaped records (nlive 2000, rounds of K = 50, add_live tail;
oracle.jitter.synthetic_record with seeds 0..63) merged into one, all as base runs.

    python scripts/merge_bench.py [--R 64] [--calls 20] [--warmup 3] [--oracle]

Kernel time: CUDA events around the call's launches (b2n_set_timing), median over `calls` calls after `warmup`; the
summary-only path (perm, merged counts and the last logz / logzerr / h) and the path that also returns the five full
arrays.  The card's name and power limit are printed with the numbers.  --oracle adds the host CPU time of the numpy
restatement (oracle/merge.py) for the same input.  Prints one JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from dynesty_b200 import _lib, ops  # noqa: E402
from oracle import jitter as OJ, merge as OM  # noqa: E402
from jitter_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--R', type=int, default=64)
    ap.add_argument('--calls', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--oracle', action='store_true')
    a = ap.parse_args()
    recs = [OJ.synthetic_record(seed=s) for s in range(a.R)]
    logl = np.concatenate([r[0] for r in recs])
    n = np.concatenate([r[1] for r in recs])
    run_ptr = np.r_[0, np.cumsum([len(r[0]) for r in recs])]
    ctx = _lib.default_context()
    ctx.set_timing(True)
    name, plim = card()
    out = dict(card=name, power_limit=plim, nlive=2000, K=50, R=a.R, N=int(len(logl)), calls=a.calls)
    ref = None
    for arrays in (False, True):
        ms, launches = [], []
        for i in range(a.warmup + a.calls):
            l0 = ctx.launch_count()
            o = ops.merge_runs(logl, n, run_ptr, a.R, arrays=arrays, ctx=ctx)
            if i >= a.warmup:
                ms.append(ctx.last_kernel_ms())
                launches.append(ctx.launch_count() - l0)
        key = 'arrays' if arrays else 'summary'
        out[key + '_kernel_ms_median'] = float(np.median(ms))
        out[key + '_launches'] = int(launches[0])
        ref = o
    if a.oracle:
        t = time.perf_counter()
        q = OM.merge_runs(logl, n, run_ptr, a.R)
        out['oracle_host_cpu_s'] = time.perf_counter() - t
        out['perm_equal'] = bool(np.array_equal(q['perm'], ref['perm']))
        out['logz_diff'] = float(abs(q['logz'][-1] - ref['logz'][-1]))
    print(json.dumps(out))


if __name__ == '__main__':
    main()

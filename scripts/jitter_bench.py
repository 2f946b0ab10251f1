"""Time b2n_jitter_runs: R prior-volume realisations of a C2-shaped record (nlive 2000, rounds of K = 50, add_live
tail; oracle.jitter.synthetic_record), approx off and on.

    python scripts/jitter_bench.py [--R 128] [--calls 20] [--oracle]

Kernel time: CUDA events around the call's launches (b2n_set_timing), median over `calls` calls after warm-up; the
summary-only path (no R x N buffer) and the path that also returns the four R x N arrays.  The card's name and power
limit are printed with the numbers.  --oracle adds the host CPU time of the numpy restatement for the same R.
Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dynesty_b200 import _lib, ops  # noqa: E402
from oracle import jitter as OJ  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim = [s.strip() for s in q.split(',')[:2]]
        return name, plim
    except Exception as e:                                   # the numbers still stand; say why the card is unknown
        return 'unknown (%r)' % (e,), 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--R', type=int, default=128)
    ap.add_argument('--calls', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--oracle', action='store_true')
    a = ap.parse_args()
    logl, n = OJ.synthetic_record()
    logwt = np.log(np.ones(len(logl)) / len(logl))            # a reference weighting so that kld is computed too
    ctx = _lib.default_context()
    ctx.set_timing(True)
    name, plim = card()
    out = dict(card=name, power_limit=plim, nlive=2000, K=50, N=int(len(logl)), R=a.R, calls=a.calls)
    for approx in (False, True):
        for arrays in (False, True):
            ms, launches = [], []
            for i in range(a.warmup + a.calls):
                l0 = ctx.launch_count()
                ops.jitter_runs(logl, n, a.R, 1234, chain0=0, approx=approx, logwt_ref=logwt, logz_ref=0.0,
                                arrays=arrays, ctx=ctx)
                if i >= a.warmup:
                    ms.append(ctx.last_kernel_ms())
                    launches.append(ctx.launch_count() - l0)
            key = 'approx%d_%s' % (approx, 'arrays' if arrays else 'summary')
            out[key + '_kernel_ms_median'] = float(np.median(ms))
            out[key + '_launches'] = int(launches[0])
        if a.oracle:
            t = time.perf_counter()
            OJ.jitter_runs(logl, n, a.R, 1234, 0, approx, logwt, 0.0)
            out['approx%d_oracle_host_cpu_s' % approx] = time.perf_counter() - t
    print(json.dumps(out))


if __name__ == '__main__':
    main()

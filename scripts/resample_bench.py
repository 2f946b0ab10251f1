"""Time b2n_resample_runs: R bootstrap realisations of a C2-shaped record with strands (nlive 2000, rounds of K = 50,
add_live tail; oracle.resample.synthetic_strand_record).

    python scripts/resample_bench.py [--R 128] [--calls 20] [--oracle]

Kernel time: CUDA events around the call's launches (b2n_set_timing), median over `calls` calls after warm-up, with
the multiplicities returned and without.  The card's name and power limit are read in the same call and printed with
the numbers.  --oracle adds the host CPU time of the numpy restatement for the same R.  Prints one JSON line."""
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
from oracle import resample as OR  # noqa: E402
from scripts.jitter_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--R', type=int, default=128)
    ap.add_argument('--calls', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--oracle', action='store_true')
    a = ap.parse_args()
    res = Results(OR.synthetic_strand_record())
    plan = DU.strand_plan(res)
    pp, ps = DU._piece_csr(res.logl, plan)
    args = (res.logl, plan['strand'], plan['base'], pp, ps, plan['end'])
    ctx = _lib.default_context()
    ctx.set_timing(True)
    name, plim = card()
    out = dict(card=name, power_limit=plim, nlive=2000, K=50, N=int(len(res.logl)), S=int(len(plan['ids'])), R=a.R,
               calls=a.calls)
    for mult in (False, True):
        ms, launches = [], []
        for i in range(a.warmup + a.calls):
            l0 = ctx.launch_count()
            ops.resample_runs(*args, a.R, 1234, chain0=0, logwt_ref=res.logwt, logz_ref=res.logz[-1],
                              multiplicities=mult, ctx=ctx)
            if i >= a.warmup:
                ms.append(ctx.last_kernel_ms())
                launches.append(ctx.launch_count() - l0)
        key = 'mult' if mult else 'summary'
        out[key + '_kernel_ms_median'] = float(np.median(ms))
        out[key + '_launches'] = int(launches[0])
    if a.oracle:
        t = time.perf_counter()
        OR.resample_runs(*args, a.R, 1234, 0, res.logwt, res.logz[-1])
        out['oracle_host_cpu_s'] = time.perf_counter() - t
    print(json.dumps(out))


if __name__ == '__main__':
    main()

"""Time importance reweighting on a C2-shaped record with positions (nlive 2000, rounds of K = 50, add_live tail,
N ~ 52 000, n = 50 synthesised positions inside the prior of gauss_corr(50)).

    python scripts/reweight_bench.py [--R 128] [--calls 20] [--warmup 3] [--reference]

  eval_ms            gauss_corr(50)'s likelihood at every sample in one launch (ops.model_eval, the model's
                     likelihood-only twin): host clock around the synchronising call, so it includes the copies of the
                     N x n positions in and the N values out;
  integrals_ms       b2n_compute_integrals with the log-reweight;
  jitter / resample  b2n_jitter_runs / b2n_resample_runs at R realisations with and without the log-reweight
                     (b2n_set_reweight), the two calls alternated;
all but eval_ms are CUDA events around each call's launches (b2n_set_timing), median of `calls` calls after `warmup`.
--reference adds the reference route on the host: a Python loop of the same likelihood over the samples and the
reference's reweight_run (needs the reference copy oracle/_ref).  The card's name and power limit are read in the same
call.  Prints one JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dynesty_b200 import _lib, likelihoods as DL, ops, utils as DU  # noqa: E402
from dynesty_b200.nested import Results  # noqa: E402
from oracle import likelihoods as OL, resample as ORS  # noqa: E402
from scripts.jitter_bench import card  # noqa: E402


def record(n):
    rec = ORS.synthetic_strand_record(2000, 50, seed=0)
    rng = np.random.default_rng(7)
    u = rng.standard_normal((len(rec['logl']), n))
    u /= np.linalg.norm(u, axis=1)[:, None]
    rec['samples'] = 0.5 + 0.1 * np.sqrt(-2.0 * rec['logl'])[:, None] * u
    return Results(rec)


def median_ms(ctx, fns, warmup, calls):
    """Each fn's median kernel time, the fns called in turn (alternated) every round."""
    ms = [[] for _ in fns]
    for i in range(warmup + calls):
        for k, fn in enumerate(fns):
            fn()
            if i >= warmup:
                ms[k].append(ctx.last_kernel_ms())
    return [float(np.median(m)) for m in ms]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--R', type=int, default=128)
    ap.add_argument('--n', type=int, default=50)
    ap.add_argument('--calls', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reference', action='store_true')
    a = ap.parse_args()
    res = record(a.n)
    N, R = len(res['logl']), a.R
    ctx = _lib.default_context()
    name, plim = card()
    model = DL.gauss_corr(a.n)
    x = np.asarray(res['samples'])
    mid = model.ids(ctx)[1]
    ts = []
    for i in range(a.warmup + a.calls):
        t = time.perf_counter()
        logp_new = ops.model_eval(mid, x, want_v=False, ctx=ctx)[1]
        if i >= a.warmup:
            ts.append(1e3 * (time.perf_counter() - t))
    logl = np.asarray(res['logl'], dtype=float)
    rw = logp_new - logl
    out = dict(card=name, power_limit=plim, N=N, n=a.n, R=R, calls=a.calls, warmup=a.warmup,
               eval_ms=float(np.median(ts)))
    ctx.set_timing(True)
    out['integrals_ms'] = median_ms(ctx, [lambda: ops.compute_integrals(logl, res['logvol'], rw, ctx=ctx)],
                                    a.warmup, a.calls)[0]
    new = DU.reweight_run(res, logp_new, ctx=ctx)
    kw = dict(logwt_ref=new['logwt'], logz_ref=float(new['logz'][-1]), ctx=ctx)
    sargs = DU._strand_inputs(res)[1]
    for error in ('jitter', 'resample'):
        if error == 'jitter':
            run = lambda lrw: ops.jitter_runs(logl, res['samples_n'], R, 1234, logrwt=lrw, **kw)
        else:
            run = lambda lrw: ops.resample_runs(*sargs, R, 1234, logrwt=lrw, **kw)
        plain, rwt = median_ms(ctx, [lambda: run(None), lambda: run(rw)], a.warmup, a.calls)
        out[error] = dict(plain_ms=plain, reweighted_ms=rwt, ratio=rwt / plain)
    ctx.set_timing(False)
    if a.reference:
        from oracle import refshim
        refshim.import_reference()
        from dynesty import utils as U
        om = OL.gauss_corr(a.n, 0.4, 5.0)
        t = time.perf_counter()
        lp = np.array([om.loglike(v) for v in x])
        t_loop = time.perf_counter() - t
        rr = U.Results(dict(samples=x, logl=logl, logvol=np.asarray(res['logvol']), logwt=np.asarray(res['logwt']),
                            logz=np.asarray(res['logz']), logzerr=np.asarray(res['logzerr']),
                            information=np.asarray(res['information']), samples_u=x, samples_id=res['samples_id'],
                            samples_it=res['samples_it'], ncall=np.ones(N, dtype=int), nlive=2000,
                            niter=int(res['niter']), eff=1.0, blob=np.zeros(N)))
        t = time.perf_counter()
        ref = U.reweight_run(rr, lp)
        t_rw = time.perf_counter() - t
        out['reference'] = dict(likelihood_loop_s=t_loop, reweight_run_s=t_rw,
                                max_abs_logl_diff=float(np.max(np.abs(lp - logp_new))),
                                logz_diff=float(ref['logz'][-1] - new['logz'][-1]))
    print(json.dumps(out))


if __name__ == '__main__':
    main()

"""Generate tests/golden/posterior.npz by running the UNMODIFIED reference's mean_and_cov / quantile on its own
jitter_run / resample_run realisations.

TEST INFRASTRUCTURE.  Run where the reference copy oracle/_ref exists (oracle/install_ref.py):

    python -m oracle.make_golden_posterior

Records with positions: the four oracle-backed runs of make_golden_resample.py (3-D, strands=True: host loop, device
rounds with and without the final live points, dynamic) and one seeded 12-D strand record
(oracle.posterior.positioned_strand_record).  Per realisation r (streams (SEED, POST_CHAIN0 + r), scripted with
ScriptedJitterGenerator / ScriptedResampleGenerator):
  jitter     mean_and_cov(samples, exp(logwt - logz[-1])) and quantile of every coordinate, of jitter_run's result;
  resample   mean_and_cov of resample_run's expanded sample set (copies included) -- the reference's call -- and
             quantile on the distinct samples drawn, each with the sum of its copies' weights (np.bincount over
             return_idx): the reference's quantile on the copies depends on argsort's order among equal values.
"""
import os

import numpy as np

from . import jitter, posterior, refshim, resample
from .make_golden import OUT, SEED
from .make_golden_resample import records, ref_results

POST_CHAIN0, POST_R = 11000, (0, 1, 3)
POST_Q = np.array([0.0, 0.025, 0.5, 0.975, 1.0])
KEYS = ('logl', 'samples_id', 'samples_it', 'samples_n', 'logwt', 'logz', 'logvol', 'ncall_per_it', 'samples_batch',
        'samples')


def _with(U, rr, **extra):
    d = {k: rr[k] for k in rr.keys()}
    d.update(extra)
    return U.Results(d)


def gen_posterior(U):
    from dynesty_b200.utils import samples_n_of
    recs = records()
    recs['hd'] = posterior.positioned_strand_record()
    out = dict(post_seed=np.int64(SEED), post_chain0=np.int64(POST_CHAIN0), post_r=np.array(POST_R, dtype=np.int64),
               post_q=POST_Q, post_names=np.array(sorted(recs)))
    for name, res in sorted(recs.items()):
        p = 'post_%s_' % name
        for k in KEYS:
            if k in res:
                out[p + k] = np.asarray(res[k])
        out[p + 'niter'] = np.int64(res['niter'])
        if 'batch_bounds' in res:
            out[p + 'batch_bounds'] = np.array(res['batch_bounds'], dtype=float)
        x = np.asarray(res['samples'], dtype=float)
        N, n = x.shape
        base = ref_results(U, res)
        rr_res = _with(U, base, samples=x)
        rr_jit = _with(U, base, samples=x, samples_n=samples_n_of(res))
        for r in POST_R:
            new = U.jitter_run(rr_jit, rstate=jitter.ScriptedJitterGenerator(SEED, POST_CHAIN0 + r))
            w = np.exp(np.asarray(new['logwt']) - np.asarray(new['logz'])[-1])
            mean, cov = U.mean_and_cov(np.asarray(new['samples']), w)
            q = p + 'j%d_' % r
            out[q + 'logz'] = np.float64(np.asarray(new['logz'])[-1])
            out[q + 'mean'], out[q + 'cov'] = mean, cov
            out[q + 'quant'] = np.array([U.quantile(x[:, j], POST_Q, weights=w) for j in range(n)])

            new, idx = U.resample_run(rr_res, rstate=resample.ScriptedResampleGenerator(SEED, POST_CHAIN0 + r),
                                      return_idx=True)
            wc = np.exp(np.asarray(new['logwt']) - np.asarray(new['logz'])[-1])
            mean, cov = U.mean_and_cov(np.asarray(new['samples']), wc)
            W = np.bincount(idx, weights=wc, minlength=N)
            present = np.bincount(idx, minlength=N) > 0
            q = p + 's%d_' % r
            out[q + 'idx'] = np.asarray(idx)
            out[q + 'logz'] = np.float64(np.asarray(new['logz'])[-1])
            out[q + 'mean'], out[q + 'cov'] = mean, cov
            out[q + 'quant'] = np.array([U.quantile(x[present, j], POST_Q, weights=W[present]) for j in range(n)])
    np.savez_compressed(os.path.join(OUT, 'posterior.npz'), **out)
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    refshim.import_reference()
    from dynesty import utils as U
    gen_posterior(U)
    print('wrote', os.path.join(OUT, 'posterior.npz'), os.path.getsize(os.path.join(OUT, 'posterior.npz')))


if __name__ == '__main__':
    main()

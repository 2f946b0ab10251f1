"""Generate tests/golden/reweight.npz by running the UNMODIFIED reference's reweight_run, and its compute_integrals(
reweight=) on its own jitter_run / resample_run realisations.

TEST INFRASTRUCTURE.  Run where the reference copy oracle/_ref exists (oracle/install_ref.py):

    python -m oracle.make_golden_reweight

Records: those of make_golden_posterior.py (the four 3-D strand records of make_golden_resample.py and the seeded 12-D
record of oracle.posterior.positioned_strand_record), plus 'cut': the host-loop record under a truncated target, -inf
beyond the 70th percentile of the first coordinate.  The new target logp_new is a second Gaussian, its mean moved by
a quarter of a standard deviation from the run's weighted mean, its variances the run's scaled by 1.3 and every
correlation 0.2, evaluated at res['samples'].  Stored per record:
  rw_<name>_*     the reference's reweight_run(res, logp_new): logwt, logz, logzerr, information (the input's: the
                  reference drops its h) and importance_weights();
  per realisation r (streams (SEED, RW_CHAIN0 + r), scripted with ScriptedJitterGenerator / ScriptedResampleGenerator):
  ..j<r>_*        compute_integrals(logl, logvol_r, reweight=logrwt) on the logvol of the reference's own jitter_run;
  ..s<r>_*        compute_integrals(logl[idx], logvol_r, reweight=logrwt[idx]) on its resample_run(return_idx=True);
                  both as logwt and `last` = (logz[-1], sqrt(max(logzvar[-1], 0)), h[-1], kld[-1]), kld_error's KL
                  divergence against the reweighted run's weights (a term of zero weight set
                  to 0, where the formula gives 0 * -inf = NaN) and mean_and_cov / quantile as make_golden_posterior.py
                  builds them.
"""
import os

import numpy as np

from . import jitter, posterior, refshim, resample
from .make_golden import OUT, SEED
from .make_golden_posterior import KEYS, POST_Q, _with
from .make_golden_resample import records, ref_results

RW_CHAIN0, RW_R = 13000, (0, 1, 3)


def second_gaussian(x, logwt, logz_end):
    """logp_new at the samples x (N x n): the Gaussian described in the module docstring."""
    w = np.exp(np.asarray(logwt) - logz_end)
    w /= w.sum()
    mu = w @ x
    C = np.cov(x.T, aweights=w).reshape(x.shape[1], x.shape[1])
    sd = np.sqrt(np.diag(C))
    C2 = np.diag(1.3 * sd ** 2) + 0.2 * np.outer(sd, sd) * (1.0 - np.eye(len(sd)))
    d = x - (mu + 0.25 * sd)
    L = np.linalg.cholesky(C2)
    z = np.linalg.solve(L, d.T)
    return -0.5 * np.sum(z * z, axis=0) - np.sum(np.log(np.diag(L))) - 0.5 * len(sd) * np.log(2 * np.pi)


def _kld(logwt, logz, logp2):
    logp1 = logwt - logz[-1]
    with np.errstate(invalid='ignore'):
        return np.cumsum(np.where(logp1 == -np.inf, 0.0, np.exp(logp1) * (logp1 - logp2)))


def cases():
    """name -> (record, logp_new)."""
    recs = records()
    recs['hd'] = posterior.positioned_strand_record()
    out = {}
    for name, res in recs.items():
        x = np.asarray(res['samples'], dtype=float)
        out[name] = (res, second_gaussian(x, res['logwt'], float(np.asarray(res['logz'])[-1])))
    res, lp = out['host']
    x0 = np.asarray(res['samples'], dtype=float)[:, 0]
    out['cut'] = (res, np.where(x0 > np.quantile(x0, 0.7), -np.inf, lp))
    return out


def gen_reweight(U):
    from dynesty_b200.utils import samples_n_of
    cs = cases()
    out = dict(rw_seed=np.int64(SEED), rw_chain0=np.int64(RW_CHAIN0), rw_r=np.array(RW_R, dtype=np.int64),
               rw_q=POST_Q, rw_names=np.array(sorted(cs)))
    for name, (res, logp_new) in sorted(cs.items()):
        p = 'rw_%s_' % name
        for k in KEYS:
            if k in res:
                out[p + k] = np.asarray(res[k])
        out[p + 'niter'] = np.int64(res['niter'])
        if 'batch_bounds' in res:
            out[p + 'batch_bounds'] = np.array(res['batch_bounds'], dtype=float)
        out[p + 'logp_new'] = logp_new
        out[p + 'information'] = np.asarray(res['information'])
        x = np.asarray(res['samples'], dtype=float)
        N, n = x.shape
        logl = np.asarray(res['logl'], dtype=float)
        base = ref_results(U, res)
        rr_res = _with(U, base, samples=x)
        rr_jit = _with(U, base, samples=x, samples_n=samples_n_of(res))
        new = U.reweight_run(rr_res, logp_new)
        for k in ('logwt', 'logz', 'logzerr', 'information'):
            out[p + 'ref_' + k] = np.asarray(new[k])
        out[p + 'ref_impw'] = np.asarray(new.importance_weights())
        logrwt = logp_new - logl
        logp2 = np.asarray(new['logwt']) - np.asarray(new['logz'])[-1]
        for r in RW_R:
            jr = U.jitter_run(rr_jit, rstate=jitter.ScriptedJitterGenerator(SEED, RW_CHAIN0 + r))
            logwt, logz, logzvar, h = U.compute_integrals(logl=logl, logvol=np.asarray(jr['logvol']), reweight=logrwt)
            w = np.exp(logwt - logz[-1])
            q = p + 'j%d_' % r
            out[q + 'logwt'] = logwt
            out[q + 'last'] = np.array([logz[-1], np.sqrt(max(logzvar[-1], 0.)), h[-1], _kld(logwt, logz, logp2)[-1]])
            out[q + 'mean'], out[q + 'cov'] = U.mean_and_cov(x, w)
            out[q + 'quant'] = np.array([U.quantile(x[:, j], POST_Q, weights=w) for j in range(n)])

            sr, idx = U.resample_run(rr_res, rstate=resample.ScriptedResampleGenerator(SEED, RW_CHAIN0 + r),
                                     return_idx=True)
            logwt, logz, logzvar, h = U.compute_integrals(logl=logl[idx], logvol=np.asarray(sr['logvol']),
                                                          reweight=logrwt[idx])
            wc = np.exp(logwt - logz[-1])
            W = np.bincount(idx, weights=wc, minlength=N)
            present = np.bincount(idx, minlength=N) > 0
            q = p + 's%d_' % r
            out[q + 'idx'] = np.asarray(idx)
            out[q + 'logwt'] = logwt
            out[q + 'last'] = np.array([logz[-1], np.sqrt(max(logzvar[-1], 0.)), h[-1],
                                        _kld(logwt, logz, logp2[idx])[-1]])
            out[q + 'mean'], out[q + 'cov'] = U.mean_and_cov(x[idx], wc)
            out[q + 'quant'] = np.array([U.quantile(x[present, j], POST_Q, weights=W[present]) for j in range(n)])
    np.savez_compressed(os.path.join(OUT, 'reweight.npz'), **out)
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    refshim.import_reference()
    from dynesty import utils as U
    gen_reweight(U)
    print('wrote', os.path.join(OUT, 'reweight.npz'), os.path.getsize(os.path.join(OUT, 'reweight.npz')))


if __name__ == '__main__':
    main()

"""Importance reweighting of a run and of its jitter / resample realisations (the reference's reweight_run and
compute_integrals(reweight=)), restated in numpy.

TEST INFRASTRUCTURE (see oracle/__init__.py).  What is restated (reference py/dynesty/utils.py):
  reweight_run       :1663-1708   logrwt = logp_new - logp_old, compute_integrals(logl, logvol, reweight=logrwt)
  compute_integrals  :1411-1467   dynesty_b200.nested._integrate(..., reweight=)
and the realisations of oracle.jitter / oracle.resample / oracle.posterior with the reweight carried, which the
reference's own jitter_run / resample_run drop (include/b200nest.h, b2n_set_reweight; DESIGN.md section 15.4):
  logwt_i = logaddexp(L_i, L_{i-1}) + logdvol2_i + logrwt_i   for every sample or copy of a sample,
h keeps the unreweighted L and logdvol2, and a KL term of zero weight (logrwt = -inf) is 0.
"""
import numpy as np

from . import jitter, posterior, resample


def integrate(logl, logvol, reweight=None):
    """compute_integrals(logl, logvol, reweight=) (utils.py:1411-1467): logwt, logz, logzvar, h."""
    from dynesty_b200.nested import _integrate
    return _integrate(np.asarray(logl, dtype=float), logvol, reweight=reweight)


def kld(logp1, logp2):
    """The cumulative KL divergence cumsum(p1 (ln p1 - ln p2)) of kld_error (utils.py:1976-1992), ln p1 = logwt -
    logz[-1] of the realisation; a term of zero weight is 0."""
    logp1 = np.asarray(logp1)
    with np.errstate(invalid='ignore'):
        return np.cumsum(np.where(logp1 == -np.inf, 0.0, np.exp(logp1) * (logp1 - logp2)))


def reweight_run(logl, logvol, logp_new, logp_old=None):
    """dict(logrwt, logwt, logz, logzvar, h, logzerr) of reweight_run (h: the reweighted one the reference computes
    and then drops)."""
    logl = np.asarray(logl, dtype=float)
    logrwt = np.asarray(logp_new, dtype=float) - (logl if logp_old is None else np.asarray(logp_old, dtype=float))
    logwt, logz, logzvar, h = integrate(logl, logvol, logrwt)
    return dict(logrwt=logrwt, logwt=logwt, logz=logz, logzvar=logzvar, h=h, logzerr=np.sqrt(np.maximum(logzvar, 0)))


def importance_weights(logwt, logz):
    """Results.importance_weights (utils.py:886-893)."""
    wt = np.exp(np.asarray(logwt) - np.asarray(logz)[-1])
    return wt / wt.sum()


def jitter_realisation(logl, samples_n, seed, chain, reweight, approx=False, logwt_ref=None, logz_ref=None):
    """oracle.jitter.realisation with the reweight: dict(logvol, logwt, logz, logzvar, h[, kld])."""
    logvol = np.cumsum(jitter.log_t(samples_n, seed, chain, approx))
    logwt, logz, logzvar, h = integrate(logl, logvol, reweight)
    out = dict(logvol=logvol, logwt=logwt, logz=logz, logzvar=logzvar, h=h)
    if logwt_ref is not None:
        out['kld'] = kld(logwt - logz[-1], np.asarray(logwt_ref) - logz_ref)
    return out


def resample_realisation(logl, strand, base, piece_ptr, piece_strand, end, seed, chain, reweight, logwt_ref=None,
                         logz_ref=None):
    """oracle.resample.realisation of the draw (seed, chain) with the reweight of each copy's sample: dict(idx,
    samples_n, logvol, logwt, logz, logzvar, h[, kld])."""
    strand = np.asarray(strand, dtype=np.int64)
    m = resample.draw_multiplicities(base, seed, chain)
    c = resample.csr_counts(strand, piece_ptr, np.asarray(piece_strand, dtype=np.int64), m)
    o = resample.realisation(logl, strand, m, c, end)
    rw = np.asarray(reweight)[o['idx']]
    o['logwt'], o['logz'], o['logzvar'], o['h'] = integrate(np.asarray(logl)[o['idx']], o['logvol'], rw)
    if logwt_ref is not None:
        o['kld'] = kld(o['logwt'] - o['logz'][-1], np.asarray(logwt_ref)[o['idx']] - logz_ref)
    return o


def _summaries(rs, kl):
    out = dict(logz=np.array([o['logz'][-1] for o in rs]),
               logzerr=np.array([np.sqrt(max(o['logzvar'][-1], 0.)) for o in rs]),
               h=np.array([o['h'][-1] for o in rs]))
    if kl:
        out['kld'] = np.array([o['kld'][-1] for o in rs])
    return out


def jitter_runs(logl, samples_n, R, seed, chain0=0, approx=False, logwt_ref=None, logz_ref=None, arrays=False,
                logrwt=None):
    """Same contract as ``dynesty_b200.ops.jitter_runs`` with logrwt."""
    if logrwt is None:
        return jitter.jitter_runs(logl, samples_n, R, seed, chain0, approx, logwt_ref, logz_ref, arrays)
    rs = [jitter_realisation(logl, samples_n, seed, chain0 + r, logrwt, approx, logwt_ref, logz_ref)
          for r in range(R)]
    out = _summaries(rs, logwt_ref is not None)
    if arrays:
        for k in ('logvol', 'logwt', 'logz') + (('kld',) if logwt_ref is not None else ()):
            out[k + '_arr'] = np.array([o[k] for o in rs])
    return out


def resample_runs(logl, strand, base, piece_ptr, piece_strand, end, R, seed, chain0=0, logwt_ref=None, logz_ref=None,
                  multiplicities=False, logrwt=None):
    """Same contract as ``dynesty_b200.ops.resample_runs`` with logrwt."""
    if logrwt is None:
        return resample.resample_runs(logl, strand, base, piece_ptr, piece_strand, end, R, seed, chain0, logwt_ref,
                                      logz_ref, multiplicities)
    rs = [resample_realisation(logl, strand, base, piece_ptr, piece_strand, end, seed, chain0 + r, logrwt, logwt_ref,
                               logz_ref) for r in range(R)]
    out = _summaries(rs, logwt_ref is not None)
    if multiplicities:
        out['mult'] = np.array([resample.draw_multiplicities(base, seed, chain0 + r) for r in range(R)])
    return out


def jitter_weights(logl, samples_n, seed, chain, reweight, approx=False):
    """w (N) of the reweighted jitter realisation (seed, chain)."""
    o = jitter_realisation(logl, samples_n, seed, chain, reweight, approx)
    return np.exp(o['logwt'] - o['logz'][-1])


def resample_weights(logl, strand, base, piece_ptr, piece_strand, end, seed, chain, reweight):
    """(W (N), w2sum, present (N)) of the reweighted resample realisation (seed, chain)."""
    o = resample_realisation(logl, strand, base, piece_ptr, piece_strand, end, seed, chain, reweight)
    wc = np.exp(o['logwt'] - o['logz'][-1])
    N = len(strand)
    return (np.bincount(o['idx'], weights=wc, minlength=N), float(np.sum(wc ** 2)),
            np.bincount(o['idx'], minlength=N) > 0)


def jitter_posterior(logl, samples_n, x, R, seed, chain0=0, approx=False, logwt_ref=None, logz_ref=None, q=None,
                     logrwt=None):
    """Same contract as ``dynesty_b200.ops.jitter_posterior`` with logrwt."""
    if logrwt is None:
        return posterior.jitter_posterior(logl, samples_n, x, R, seed, chain0, approx, logwt_ref, logz_ref, q)
    o = jitter_runs(logl, samples_n, R, seed, chain0, approx, logwt_ref, logz_ref, logrwt=logrwt)
    x = np.asarray(x, dtype=np.float64)
    rs = [posterior.stats(x, jitter_weights(logl, samples_n, seed, chain0 + r, logrwt, approx), q) for r in range(R)]
    o.update(posterior._collect(rs, q))
    return o


def resample_posterior(logl, strand, base, piece_ptr, piece_strand, end, x, R, seed, chain0=0, logwt_ref=None,
                       logz_ref=None, q=None, logrwt=None):
    """Same contract as ``dynesty_b200.ops.resample_posterior`` with logrwt."""
    if logrwt is None:
        return posterior.resample_posterior(logl, strand, base, piece_ptr, piece_strand, end, x, R, seed, chain0,
                                            logwt_ref, logz_ref, q)
    o = resample_runs(logl, strand, base, piece_ptr, piece_strand, end, R, seed, chain0, logwt_ref, logz_ref,
                      logrwt=logrwt)
    x = np.asarray(x, dtype=np.float64)
    rs = []
    for r in range(R):
        W, w2, present = resample_weights(logl, strand, base, piece_ptr, piece_strand, end, seed, chain0 + r, logrwt)
        rs.append(posterior.stats(x, W, q, w2, present))
    o.update(posterior._collect(rs, q))
    return o


def compute_integrals(logl, logvol, logrwt=None):
    """Same contract as ``dynesty_b200.ops.compute_integrals``."""
    logwt, logz, logzvar, h = integrate(logl, np.asarray(logvol, dtype=float), logrwt)
    return dict(logwt=logwt, logz=logz, logzvar=logzvar, h=h)

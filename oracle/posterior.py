"""Posterior means, covariances and weighted quantiles of jitter / resample realisations (the reference's mean_and_cov
and quantile, utils.py:1081-1117, 1196-1233, applied to jitter_run / resample_run realisations), restated in numpy.

TEST INFRASTRUCTURE (see oracle/__init__.py).  The semantics are those of include/b200nest.h (b2n_weighted_stats,
b2n_jitter_posterior, b2n_resample_posterior) and DESIGN.md section 15.3:
  weights     jitter: w_i = exp(logwt_i - logz[-1]) of oracle.jitter's realisation, every sample present;
              resample: W_i = the sum over sample i's copies of exp(logwt - logz[-1]) of oracle.resample's realisation,
              w2sum over the copies, a sample drawn 0 times absent;
  moments     mean = sum w x / wsum, cov = wsum / (wsum^2 - w2sum) sum w (x - mean)(x - mean)^T;
  quantiles   nodes = the present samples sorted stably by (x, record index), C_k = sum_{l<k} w_l / sum_{l<M-1} w_l,
              p = the largest k with C_k <= q: x_p if q == C_p or p is the last node, else the line towards node p + 1.
"""
import numpy as np

from . import jitter, resample


def moments(x, w, w2sum=None):
    """(mean, cov) of the samples x (N x n) under weights w (N); w2sum defaults to sum(w^2)."""
    x = np.asarray(x, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    wsum = w.sum()
    w2 = np.sum(w ** 2) if w2sum is None else w2sum
    mean = w @ x / wsum
    dx = x - mean
    return mean, wsum / (wsum ** 2 - w2) * np.einsum('i,ij,ik', w, dx, dx)


def quantile_nodes(x, q, w, present=None):
    """The weighted quantiles q of one coordinate x (N) under weights w (N); present (N bool, default all): the nodes.
    NaN where sum_{l<M-1} w_l is 0."""
    x = np.asarray(x, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    keep = np.ones(len(x), dtype=bool) if present is None else np.asarray(present, dtype=bool)
    xs, ws = x[keep], w[keep]
    order = np.argsort(xs, kind='stable')
    xs, ws = xs[order], ws[order]
    M = len(xs)
    out = np.full(len(np.atleast_1d(q)), np.nan)
    if M == 0:
        return out
    cum = np.r_[0.0, np.cumsum(ws)[:-1]]
    S = cum[-1]
    if not S > 0:
        return out
    C = cum / S
    for t, qq in enumerate(np.atleast_1d(q)):
        p = int(np.searchsorted(C, qq, side='right')) - 1
        if p < 0:
            continue
        if qq == C[p] or p == M - 1:
            out[t] = xs[p]
        else:
            out[t] = (xs[p + 1] - xs[p]) / (C[p + 1] - C[p]) * (qq - C[p]) + xs[p]
    return out


def stats(x, w, q=None, w2sum=None, present=None):
    """dict(mean, cov[, quantiles (n x nq)]) of one weight vector."""
    mean, cov = moments(x, w, w2sum)
    o = dict(mean=mean, cov=cov)
    if q is not None:
        o['quantiles'] = np.array([quantile_nodes(x[:, j], q, w, present) for j in range(x.shape[1])])
    return o


def weighted_stats(x, w, shift=None, q=None, moments=True):
    """Same contract as ``dynesty_b200.ops.weighted_stats`` (the shift only rounds, so it is not used here)."""
    x = np.asarray(x, dtype=np.float64)
    w = np.atleast_2d(np.asarray(w, dtype=np.float64))
    rs = [stats(x, wr, q, present=~np.signbit(wr)) for wr in w]
    o = {}
    if moments:
        o.update(mean=np.array([r['mean'] for r in rs]), cov=np.array([r['cov'] for r in rs]))
    if q is not None:
        o['quantiles'] = np.array([r['quantiles'] for r in rs])
    return o


def jitter_weights(logl, samples_n, seed, chain, approx=False):
    """w (N) of the jitter realisation (seed, chain)."""
    o = jitter.realisation(logl, samples_n, seed, chain, approx)
    return np.exp(o['logwt'] - o['logz'][-1])


def resample_weights(logl, strand, base, piece_ptr, piece_strand, end, seed, chain):
    """(W (N), w2sum, present (N)) of the resample realisation (seed, chain): sums over each sample's copies."""
    strand = np.asarray(strand, dtype=np.int64)
    m = resample.draw_multiplicities(base, seed, chain)
    c = resample.csr_counts(strand, piece_ptr, np.asarray(piece_strand, dtype=np.int64), m)
    o = resample.realisation(logl, strand, m, c, end)
    wc = np.exp(o['logwt'] - o['logz'][-1])
    return np.bincount(o['idx'], weights=wc, minlength=len(strand)), float(np.sum(wc ** 2)), m[strand] > 0


def _collect(rs, q):
    o = dict(mean=np.array([r['mean'] for r in rs]), cov=np.array([r['cov'] for r in rs]))
    if q is not None:
        o['quantiles'] = np.array([r['quantiles'] for r in rs])
    return o


def jitter_posterior(logl, samples_n, x, R, seed, chain0=0, approx=False, logwt_ref=None, logz_ref=None, q=None):
    """Same contract as ``dynesty_b200.ops.jitter_posterior``."""
    o = jitter.jitter_runs(logl, samples_n, R, seed, chain0, approx, logwt_ref, logz_ref)
    x = np.asarray(x, dtype=np.float64)
    o.update(_collect([stats(x, jitter_weights(logl, samples_n, seed, chain0 + r, approx), q) for r in range(R)], q))
    return o


def resample_posterior(logl, strand, base, piece_ptr, piece_strand, end, x, R, seed, chain0=0, logwt_ref=None,
                       logz_ref=None, q=None):
    """Same contract as ``dynesty_b200.ops.resample_posterior``."""
    o = resample.resample_runs(logl, strand, base, piece_ptr, piece_strand, end, R, seed, chain0, logwt_ref, logz_ref)
    x = np.asarray(x, dtype=np.float64)
    rs = []
    for r in range(R):
        W, w2, present = resample_weights(logl, strand, base, piece_ptr, piece_strand, end, seed, chain0 + r)
        rs.append(stats(x, W, q, w2, present))
    o.update(_collect(rs, q))
    return o


def positioned_strand_record(ndim=12, nlive=200, K=1, lnx_end=-12.0, offset=3.0, seed=3):
    """``oracle.resample.synthetic_strand_record`` with sample positions: sample i sits at radius sqrt(-2 logl_i) (a
    unit Gaussian's logl) in a seeded random direction, about the point (offset, .., offset)."""
    rec = resample.synthetic_strand_record(nlive, K, lnx_end=lnx_end, seed=seed)
    rng = np.random.default_rng(seed + 2)
    u = rng.standard_normal((len(rec['logl']), ndim))
    u /= np.linalg.norm(u, axis=1)[:, None]
    rec['samples'] = offset + np.sqrt(-2.0 * np.asarray(rec['logl']))[:, None] * u
    return rec

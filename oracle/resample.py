"""Bootstrap realisations of a strand-labelled record (the reference's resample_run / kld_error(error='resample')),
restated in numpy.

TEST INFRASTRUCTURE (see oracle/__init__.py).  What is restated (reference py/dynesty/utils.py):
  resample_run       :1495-1660   strand draws, live counts of the resampled points, ln X, integrals
  compute_integrals  :1411-1467   dynesty_b200.nested._integrate (same quadrature)
  kld_error          :1932-1997   cumulative KL divergence against the input run's weights

Live counts, two rules (include/b200nest.h, b2n_resample_runs; DESIGN.md section 15):
  piece rule      (what b2n_resample_runs computes) point p is live on (birth_p, logl_p], i.e. from the first sample
                  after its birth to itself; the count at a sample is the sum over the pieces covering it of the
                  multiplicity of their strand, added up piece by piece here instead of the kernel's scan of
                  per-sample differences;
  reference rule  (utils.py:1601-1622) strand s is live on the open range (its batch's lower bound, its largest logl);
                  only right where every round removes one point.
Both give a final live point's m copies n, n-1, .., n-m+1.

Random stream of realisation r: the B2N chain (seed, chain0 + r) -- tick 0: one uniform event over the nbase base
strands, the e-th draw is base_ids[min(floor(U_e nbase), nbase - 1)]; tick 1: the same over the nadd add-on strands
(only when nadd > 0).  ``ScriptedResampleGenerator(seed, chain0 + r)`` drives the unmodified reference with the same
numbers.
"""
import numpy as np

from . import philox


class ScriptedResampleGenerator(philox.ScriptedGenerator):
    """``philox.ScriptedGenerator`` whose ``integers(0, high, size)`` -- the draw resample_run makes (utils.py:1576-1579)
    -- is one uniform vector event: element e -> min(floor(U_e * high), high - 1)."""

    def integers(self, low, high=None, size=None, **k):
        if high is None:
            return super().integers(low, high, size, **k)
        assert low == 0 and size is not None
        return self._s.integers(int(high), int(np.prod(size))).reshape(size)


def draw_multiplicities(base, seed, chain):
    """m per strand of realisation (seed, chain): base strands drawn at tick 0, add-on strands at tick 1."""
    base = np.asarray(base, dtype=bool)
    m = np.zeros(len(base), dtype=np.int64)
    for tick, ids in ((0, np.nonzero(base)[0]), (1, np.nonzero(~base)[0])):
        if len(ids):
            u = philox.event_uniforms(seed, chain, tick, len(ids))
            np.add.at(m, ids[np.minimum((u * len(ids)).astype(np.int64), len(ids) - 1)], 1)
    return m


def live_counts(start, strand, m, open_start=None):
    """Piece rule: n_i = sum of m[strand_p] over the points p with start_p <= i <= p (start_p: the first sample the
    piece covers), plus the unrecorded live points (open_start per strand, or None) with open_start <= i."""
    N = len(strand)
    n = np.zeros(N, dtype=np.int64)
    for p in range(N):
        n[start[p]:p + 1] += m[strand[p]]
    if open_start is not None:
        for s, q in enumerate(open_start):
            n[q:] += m[s]
    return n


def reference_counts(logl, strand, lower, m):
    """Reference rule: n_i = sum of m_s over the strands with lower_s < logl_i < upper_s (without the end-point
    share-out, which both rules apply alike)."""
    logl = np.asarray(logl, dtype=float)
    S = len(m)
    upper = np.full(S, -np.inf)
    np.maximum.at(upper, strand, logl)
    lo = np.full(S, np.inf)
    np.minimum.at(lo, strand, lower)
    inside = (logl[:, None] > lo[None, :]) & (logl[:, None] < upper[None, :])
    return inside.astype(np.int64) @ m


def realisation(logl, strand, m, counts, end=None, logwt_ref=None, logz_ref=None, dtype=np.float64):
    """One realisation from its multiplicities and the live counts of the record's samples: dict(idx, samples_n,
    logvol, logwt, logz, logzvar, h[, kld]), in `dtype` (np.longdouble: a reference for records so long that float64's
    running sums round at the bars the kernel is held to)."""
    from dynesty_b200.nested import _integrate
    logl = np.asarray(logl, dtype=float)
    ms = m[strand]
    idx = np.repeat(np.arange(len(logl)), ms)
    copy = np.arange(len(idx)) - np.repeat(np.cumsum(ms) - ms, ms)
    n = counts[idx] - (copy * np.asarray(end)[idx] if end is not None else 0)
    logvol = np.cumsum(np.log(n.astype(dtype) / (n + 1)))
    logwt, logz, logzvar, h = _integrate(logl[idx], logvol)
    out = dict(idx=idx, samples_n=n, logvol=logvol, logwt=logwt, logz=logz, logzvar=logzvar, h=h)
    if logwt_ref is not None:
        logp2 = np.asarray(logwt_ref)[idx] - logz_ref
        logp1 = logwt - logz[-1]
        out['kld'] = np.cumsum(np.exp(logp1) * (logp1 - logp2))
    return out


def csr_counts(strand, piece_ptr, piece_strand, m):
    """Piece rule from the piece plan b2n_resample_runs takes (pieces listed at their first covered sample): the
    pieces started at or before i minus the samples' own pieces ended before i."""
    start = np.repeat(np.arange(len(strand)), np.diff(piece_ptr))
    started = np.cumsum(np.bincount(start, weights=m[piece_strand], minlength=len(strand)))
    ended = np.r_[0.0, np.cumsum(m[strand])[:-1]]
    return np.rint(started - ended).astype(np.int64)


def resample_runs(logl, strand, base, piece_ptr, piece_strand, end, R, seed, chain0=0, logwt_ref=None, logz_ref=None,
                  multiplicities=False, dtype=np.float64):
    """Same contract as ``dynesty_b200.ops.resample_runs`` (computed in `dtype`, returned in float64)."""
    strand = np.asarray(strand, dtype=np.int64)
    base = np.asarray(base, dtype=bool)
    piece_strand = np.asarray(piece_strand, dtype=np.int64)
    S = len(base)
    rs, ms = [], []
    for r in range(R):
        m = draw_multiplicities(base, seed, chain0 + r)
        c = csr_counts(strand, piece_ptr, piece_strand, m)
        rs.append(realisation(logl, strand, m, c, end, logwt_ref, logz_ref, dtype))
        ms.append(m)
    out = dict(logz=np.array([o['logz'][-1] for o in rs], dtype=np.float64),
               logzerr=np.array([np.sqrt(max(o['logzvar'][-1], 0.)) for o in rs], dtype=np.float64),
               h=np.array([o['h'][-1] for o in rs], dtype=np.float64))
    if logwt_ref is not None:
        out['kld'] = np.array([o['kld'][-1] for o in rs], dtype=np.float64)
    if multiplicities:
        out['mult'] = np.array(ms).reshape(R, S)
    return out


def synthetic_strand_record(nlive=2000, K=50, lnx_end=-25.0, seed=0):
    """``oracle.jitter.synthetic_record`` (rounds of K removals, then the add_live tail) with strands: each round
    frees K slots drawn at random, whose new points enter after its K dead rows.  Returns a dict with the keys of a
    static run's results that resample_run reads."""
    from dynesty_b200.nested import _integrate
    from .jitter import synthetic_record
    logl, n = synthetic_record(nlive, K, lnx_end=lnx_end, seed=seed)
    rng = np.random.default_rng(seed + 1)
    ndead = len(logl) - nlive
    live_it = np.zeros(nlive, dtype=np.int64)
    ids, its = np.empty(len(logl), dtype=np.int64), np.empty(len(logl), dtype=np.int64)
    for r in range(ndead // K):
        slots = rng.choice(nlive, K, replace=False)
        ids[r * K:(r + 1) * K], its[r * K:(r + 1) * K] = slots, live_it[slots]
        live_it[slots] = (r + 1) * K
    tail = rng.permutation(nlive)
    ids[ndead:], its[ndead:] = tail, live_it[tail]
    logvol = -np.cumsum(np.log((n + 1.) / n))
    logwt, logz, logzvar, h = _integrate(logl, logvol)
    return dict(logl=logl, samples_n=n, samples_id=ids, samples_it=its, niter=ndead, logvol=logvol, logwt=logwt,
                logz=logz, logzerr=np.sqrt(logzvar), information=h, ncall_per_it=np.ones(len(logl), dtype=np.int64))

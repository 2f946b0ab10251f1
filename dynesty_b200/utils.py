"""Run uncertainties from simulated prior volumes and from bootstrapped strands, computed on the GPU.

What is mirrored (reference py/dynesty/utils.py, same names / meaning):
  jitter_run    :1317-1408   one realisation of the prior volumes of a run's dead points
  resample_run  :1495-1660   one bootstrap realisation of a run's strands (the points that occupied one live slot)
  unravel_run   :1711-1814   a run split into its strands
  kld_error     :1932-1997   the KL divergence from the run to such a realisation
  merge_runs    :1817-1929   several runs merged into one (``b2n_merge_runs``)
  mean_and_cov  :1081-1117   weighted mean and covariance (``b2n_weighted_stats``)
  quantile      :1196-1233   weighted quantiles (``b2n_weighted_stats``; unweighted: np.percentile)
  resample_equal :1120-1187  equal-weight draws by systematic resampling (``b2n_resample_equal``)
  reweight_run  :1663-1708   a run's weights for a new target (``b2n_compute_integrals``)
and the batched forms the dynamic sampler's stopping function needs: ``jitter_realisations`` (``b2n_jitter_runs``) and
``resample_realisations`` (``b2n_resample_runs``), n_mc realisations in one call and a fixed number of kernel launches,
and ``posterior_realisations``: the same realisations with the posterior mean, covariance and quantiles of each
(``b2n_jitter_posterior`` / ``b2n_resample_posterior``), and ``equal_realisations``: equal-weight draws of each
(``b2n_jitter_equal`` / ``b2n_resample_equal_runs``).

Randomness: realisation r of a call is the B2N Philox stream (seed, chain0 + r) (include/b200nest.h), so a (seed,
chain) pair names one realisation: it is the same whether it is computed alone or in a batch of any size.
``seed=None`` draws a fresh seed, like the reference's ``rstate=None``.

A record that ``reweight_run`` made carries its log-reweight as ``logrwt`` (N).  Every realisation of it -- jitter,
resample, posterior, kld_error -- then carries that reweight too (``b2n_set_reweight``), so the reweighted evidence and
posterior get the same error bars the original target has; the reference's realisations drop it.  ``merge_runs``
refuses such records: the reweight is per sample, so merge first, then reweight.

Strands need a record with samples_id / samples_it (``run_nested(strands=True)``).  The live count of a resampled
point follows the strand rule of include/b200nest.h (b2n_resample_runs, DESIGN.md section 15): every point is live
from the threshold it entered above to its own logl.  For runs that remove one point at a time this is the
reference's rule; for the device rounds, which remove `batch` points at once, it keeps the run's own live counts
where the reference's rule would count every slot as occupied.
"""
import math
import warnings

import numpy as np

from . import ops
from .nested import Results, _integrate


def _seed(seed):
    return int(np.random.default_rng().integers(1 << 63)) if seed is None else int(seed)


def samples_n_of(res):
    """_get_nsamps_samples_n (utils.py:1231-1270): the live-point count at every dead point."""
    if 'samples_n' in res:
        return np.asarray(res['samples_n'], dtype=np.int64)
    niter, nlive, nsamps = int(res['niter']), int(res['nlive']), len(res['logvol'])
    if nsamps == niter:
        return np.full(niter, nlive, dtype=np.int64)
    if nsamps == niter + nlive:
        return np.minimum(np.arange(nsamps, 0, -1), nlive).astype(np.int64)
    raise ValueError("Final number of samples differs from number of iterations and number of live points.")


def _logrwt(res):
    """The record's log-reweight (reweight_run), or None."""
    return np.asarray(res['logrwt'], dtype=float) if 'logrwt' in res else None


def _rw(res):
    """The ops keyword of the record's log-reweight: none for a record without one, which is called as before."""
    return {} if 'logrwt' not in res else dict(logrwt=_logrwt(res))


def _logz_end(res):
    """The record's own logz[-1] (the reference weights' normalisation)."""
    return float(np.asarray(res['logz'])[-1])


def jitter_realisations(res, n_mc, seed, chain0=0, approx=False, arrays=False, ctx=None):
    """n_mc realisations of `res` in one call.  Returns dict(logz, logzerr, h, kld): the last element of each
    realisation's logz / logzerr / information / cumulative KL divergence (n_mc values each); with arrays=True also
    logvol_arr, logwt_arr, logz_arr, kld_arr (n_mc x nsamps).  Realisation r uses the stream (seed, chain0 + r)."""
    return ops.jitter_runs(res['logl'], samples_n_of(res), int(n_mc), int(seed), chain0=int(chain0),
                           approx=approx, logwt_ref=res['logwt'], logz_ref=_logz_end(res), arrays=arrays,
                           ctx=ctx, **_rw(res))


def _realisation(res, seed, chain, approx, ctx):
    o = jitter_realisations(res, 1, _seed(seed), chain, approx, arrays=True, ctx=ctx)
    logvol = o['logvol_arr'][0]
    # logzerr and information as arrays: the quadrature of compute_integrals on the realisation's volumes (host,
    # O(nsamps) for the one realisation; their last elements are the kernel's)
    _, _, logzvar, h = _integrate(np.asarray(res['logl'], dtype=float), logvol, reweight=_logrwt(res))
    new = Results(res)
    new.update(logvol=logvol, logwt=o['logwt_arr'][0], logz=o['logz_arr'][0],
               logzerr=np.sqrt(np.maximum(logzvar, 0)), information=h)
    return new, o['kld_arr'][0]


def jitter_run(res, seed=None, chain=0, approx=False, ctx=None):
    """jitter_run (utils.py:1317-1408): a copy of `res` whose logvol, logwt, logz, logzerr and information come from
    one realisation of the prior volumes -- Beta(n, 1) shrinkage where the live-point count is constant or
    increasing, uniform order statistics over each decreasing stretch (approx=True: Beta(n, 1) everywhere).  The
    realisation is the stream (seed, chain)."""
    return _realisation(res, seed, chain, approx, ctx)[0]


def kld_error(res, error='jitter', seed=None, chain=0, return_new=False, approx=False, ctx=None):
    """kld_error (utils.py:1932-1997): the cumulative KL divergence from `res` to the realisation (seed, chain) of
    jitter_run (error='jitter') or of resample_run (error='resample'); with return_new, also that realisation."""
    if error == 'resample':
        new, idx = resample_run(res, seed, chain, return_idx=True, ctx=ctx)
        logp2 = (np.asarray(res['logwt']) - np.asarray(res['logz'])[-1])[idx]
        logp1 = new['logwt'] - new['logz'][-1]
        with np.errstate(invalid='ignore'):            # a term of zero weight (a -inf reweight) is 0
            kld = np.cumsum(np.where(logp1 == -np.inf, 0.0, np.exp(logp1) * (logp1 - logp2)))
        return (kld, new) if return_new else kld
    if error != 'jitter':
        raise ValueError("Input `'error'` option '{}' is not valid.".format(error))
    new, kld = _realisation(res, seed, chain, approx, ctx)
    return (kld, new) if return_new else kld


# ---------------------------------------------------------------------------------------------- strands
def strand_plan(res):
    """The strands of a record and the thresholds its points entered above.  Returns dict(
      ids      the distinct samples_id (strand s is ids[s]),
      strand   per sample, its strand s,
      base     per strand, True if one of its samples is in a batch whose lower bound is -inf (utils.py:1563-1570),
      birth    per sample, the threshold it entered the live set above: the lower bound of its batch if samples_it
               is 0, else the logl of its batch's (samples_it - 1)-th sample in record order,
      start    per sample, the first sample its piece covers: the one after that (samples_it - 1)-th sample, or the
               first whose logl is above the lower bound (positions, so that equal logl values keep the run's order),
      end      per sample, True at a strand's last sample when the record ends with its final live points, else None,
      open     per strand, the first sample covered by its live point that the record does not hold (no final live
               points: the one after the last point of the round its last recorded point died in), else None)."""
    if 'samples_id' not in res or 'samples_it' not in res:
        raise NotImplementedError("error='resample' / resample_run need every sample's strand (samples_id / "
                                  "samples_it): run the sampler with run_nested(strands=True).")
    logl = np.asarray(res['logl'], dtype=float)
    N = len(logl)
    ids, strand = np.unique(np.asarray(res['samples_id']), return_inverse=True)
    sit = np.asarray(res['samples_it'], dtype=np.int64)
    if 'samples_batch' in res:                      # a dynamic record: every batch ends with its live points
        batch = np.asarray(res['samples_batch'], dtype=np.int64)
        lower = np.array([b[0] for b in res['batch_bounds']], dtype=float)
        final_live = True
    else:
        batch, lower = np.zeros(N, dtype=np.int64), np.array([-np.inf])
        final_live = N > int(res['niter'])
    S = len(ids)
    base = np.zeros(S, dtype=bool)
    base[strand[lower[batch] == -np.inf]] = True
    # the k-th sample of batch b in record order is rec_pos[first[b] + k]
    rec_pos = np.argsort(batch, kind='stable')
    cnt = np.bincount(batch, minlength=len(lower))
    first = np.cumsum(cnt) - cnt
    birth = lower[batch].copy()
    start = np.searchsorted(logl, birth, side='right')
    later = sit > 0
    prev = rec_pos[first[batch[later]] + sit[later] - 1]
    birth[later] = logl[prev]
    start[later] = prev + 1
    last = np.full(S, -1, dtype=np.int64)
    np.maximum.at(last, strand, np.arange(N))
    end = opened = None
    if final_live:
        end = np.zeros(N, dtype=bool)
        end[last] = True
    else:
        # a round ends where the live count stops falling (samples_n: nlive in a host loop, N - j in device rounds);
        # its threshold is the logl of its last point
        n = np.asarray(res['samples_n'], dtype=np.int64)
        stops = np.nonzero(np.r_[n[1:] >= n[:-1], True])[0]
        opened = stops[np.searchsorted(stops, last)] + 1
    return dict(ids=ids, strand=strand.astype(np.int64), base=base, birth=birth, start=np.minimum(start, np.arange(N)),
                end=end, open=opened)


def _pieces(logl, plan):
    """Every piece's first covered sample (the first whose logl is above its birth) and its strand: one per sample,
    then one per strand whose unrecorded live point covers samples of the record."""
    start, pstr = plan['start'], plan['strand']
    if plan['open'] is not None:
        keep = plan['open'] < len(logl)
        start, pstr = np.r_[start, plan['open'][keep]], np.r_[pstr, np.nonzero(keep)[0]]
    return start, pstr


def _piece_csr(logl, plan):
    """(piece_ptr, piece_strand) as b2n_resample_runs takes them: the pieces by their first covered sample."""
    start, pstr = _pieces(logl, plan)
    ptr_ = np.zeros(len(logl) + 1, dtype=np.int64)
    ptr_[1:] = np.cumsum(np.bincount(start, minlength=len(logl)))
    return ptr_, pstr[np.argsort(start, kind='stable')]


def _strand_inputs(res):
    """(plan, record): the strand plan of `res` and the record as b2n_resample_runs takes it, (logl, strand, base,
    piece_ptr, piece_strand, end).  The record must hold a strand started from the prior."""
    plan = strand_plan(res)
    if not plan['base'].any():
        raise ValueError("The provided `Results` does not include any points initially sampled from the prior!")
    logl = np.asarray(res['logl'], dtype=float)
    return plan, (logl, plan['strand'], plan['base']) + _piece_csr(logl, plan) + (plan['end'],)


def resample_realisations(res, n_mc, seed, chain0=0, multiplicities=False, ctx=None):
    """n_mc resample_run realisations of `res` in one call.  Returns dict(logz, logzerr, h, kld): the last element of
    each realisation's logz / logzerr / information / cumulative KL divergence (n_mc values each); with
    multiplicities=True also mult (n_mc x nstrands): the times each strand (in the order of np.unique(samples_id)) is
    drawn.  Realisation r uses the stream (seed, chain0 + r)."""
    rec = _strand_inputs(res)[1]
    return ops.resample_runs(*rec, int(n_mc), int(seed), chain0=int(chain0), logwt_ref=res['logwt'],
                             logz_ref=_logz_end(res), multiplicities=multiplicities, ctx=ctx, **_rw(res))


def resample_run(res, seed=None, chain=0, return_idx=False, ctx=None):
    """resample_run (utils.py:1495-1660): a copy of `res` made of a bootstrap draw of its strands -- base strands
    (started from the prior) drawn with replacement among themselves, add-on strands (started inside a dynamic
    batch) among themselves -- with the live counts of the strand rule and the integrals of those.  The draw is the
    stream (seed, chain) (b2n_resample_runs computes it and the summaries; the arrays are built here).  With
    return_idx, also the index in `res` of every sample of the new run."""
    plan, rec = _strand_inputs(res)
    m = ops.resample_runs(*rec, 1, _seed(seed), chain0=int(chain), logwt_ref=res['logwt'], logz_ref=_logz_end(res),
                          multiplicities=True, ctx=ctx)['mult'][0]
    logl = rec[0]
    N = len(logl)
    start, pstr = _pieces(logl, plan)
    ms = m[plan['strand']]
    # live count: the pieces covering each sample, weighted by the multiplicity of their strand
    diff = np.bincount(start, weights=m[pstr], minlength=N)
    diff[1:] -= ms[:-1]
    n = np.rint(np.cumsum(diff)).astype(np.int64)
    idx = np.repeat(np.arange(N), ms)
    copy = np.arange(len(idx)) - np.repeat(np.cumsum(ms) - ms, ms)
    samp_n = n[idx] - (0 if plan['end'] is None else copy * plan['end'][idx])     # a final live point's copies
    logvol = np.cumsum(np.log(samp_n / (samp_n + 1.)))
    lnew = logl[idx]
    rw = _logrwt(res)
    logwt, logz, logzvar, h = _integrate(lnew, logvol, reweight=None if rw is None else rw[idx])
    new = Results(res)
    nc = np.asarray(res['ncall_per_it'])[idx]
    new.update(niter=len(idx), ncall_per_it=nc, eff=100. * len(idx) / max(int(nc.sum()), 1), logl=lnew,
               samples_n=samp_n, logvol=logvol, logwt=logwt, logz=logz, logzerr=np.sqrt(np.maximum(logzvar, 0)),
               information=h)
    for k in ('samples', 'samples_u', 'samples_id', 'samples_it', 'samples_batch', 'samples_scale', 'logrwt', 'blob'):
        if k in res and len(res[k]) == N:
            new[k] = np.asarray(res[k])[idx]
    return (new, idx) if return_idx else new


def unravel_run(res):
    """unravel_run (utils.py:1711-1814): the run split into its strands, each a run with one live point (host only).
    Their volumes are those of a one-point run: valid only for strands that started from the prior."""
    plan = strand_plan(res)
    ids = np.asarray(res['samples_id'])
    added_live = plan['end'] is not None
    logl_all = np.asarray(res['logl'], dtype=float)
    rw_all = _logrwt(res)
    out = []
    for s in plan['ids']:
        sel = ids == s
        logl = logl_all[sel]
        nsamps = len(logl)
        niter = nsamps - 1 if added_live else nsamps
        logvol = -math.log(2) * (1. + np.arange(niter))
        if added_live:
            logvol = np.append(logvol, (logvol[-1] if niter else 0.0) + math.log(0.5))
        logwt, logz, logzvar, h = _integrate(logl, logvol, reweight=None if rw_all is None else rw_all[sel])
        nc = np.asarray(res['ncall_per_it'])[sel]
        r = Results(nlive=1, niter=niter, ncall_per_it=nc, eff=100. * nsamps / max(int(nc.sum()), 1), logl=logl,
                    logvol=logvol, logwt=logwt, logz=logz, logzerr=np.sqrt(logzvar), information=h)
        for k in ('samples', 'samples_u', 'samples_id', 'samples_it', 'samples_batch', 'logrwt', 'blob'):
            if k in res and len(res[k]) == len(ids):
                r[k] = np.asarray(res[k])[sel]
        if 'batch_bounds' in res:
            r['batch_bounds'] = res['batch_bounds']
        out.append(r)
    return out


# ---------------------------------------------------------------------------------------------- posterior summaries
def mean_and_cov(samples, weights, ctx=None):
    """mean_and_cov (utils.py:1081-1117): the weighted mean (ndim) and covariance (ndim x ndim) of samples (nsamples x
    ndim), cov = wsum / (wsum^2 - w2sum) sum w (x - mean)(x - mean)^T.  weights may also be R x nsamples: then R
    weight vectors at once, returning (R x ndim, R x ndim x ndim).  Computed on the GPU in FP64 (b2n_weighted_stats),
    second moments about the mean under the summed weights."""
    x = np.ascontiguousarray(samples, dtype=np.float64)
    w = np.asarray(weights, dtype=np.float64)
    if x.ndim != 2:
        raise ValueError("samples must be an array of shape (nsamples, ndim)")
    if w.ndim not in (1, 2) or w.shape[-1] != len(x):
        raise ValueError("Dimension mismatch: the weights must have shape (nsamples,) or (R, nsamples).")
    wt = np.atleast_2d(w).sum(axis=0)
    shift = wt @ x / wt.sum() if wt.sum() > 0 else x.mean(axis=0)
    o = ops.weighted_stats(x, np.atleast_2d(w), shift, ctx=ctx)
    return (o['mean'][0], o['cov'][0]) if w.ndim == 1 else (o['mean'], o['cov'])


def quantile(x, q, weights=None, ctx=None):
    """quantile (utils.py:1196-1233): the weighted quantiles q of the samples x, as a list (np.interp's rule on the
    cdf of the sorted samples, include/b200nest.h b2n_weighted_stats; computed on the GPU); without weights,
    np.percentile(x, 100 q), as the reference does."""
    x = np.atleast_1d(x)
    q = np.atleast_1d(q)
    if np.any(q < 0.0) or np.any(q > 1.0):
        raise ValueError("Quantiles must be between 0. and 1.")
    if weights is None:
        return np.percentile(x, list(100.0 * q))
    weights = np.atleast_1d(weights)
    if len(x) != len(weights):
        raise ValueError("Dimension mismatch: len(weights) != len(x).")
    x = np.asarray(x, dtype=np.float64).reshape(-1, 1)
    o = ops.weighted_stats(x, np.asarray(weights, dtype=np.float64)[None, :], x.mean(axis=0), q=q, moments=False,
                           ctx=ctx)
    return o['quantiles'][0, 0].tolist()


def posterior_realisations(res, n_mc, seed, chain0=0, error='jitter', approx=False, q=None, of='samples', ctx=None):
    """n_mc realisations of `res` -- jitter_run's (error='jitter') or resample_run's (error='resample') -- with the
    posterior summaries of each over res[of]: the sample positions (of='samples') or the blobs the run saved
    (of='blob', NestedSampler(..., blob=True)), whose summaries are the error bars of derived quantities.  Returns the dict of jitter_realisations / resample_realisations
    (logz, logzerr, h, kld; n_mc values each) plus mean (n_mc x ndim), cov (n_mc x ndim x ndim) and, with q,
    quantiles (n_mc x ndim x nq): mean_and_cov / quantile of each realisation's samples and weights
    exp(logwt - logz[-1]), a resampled point's copies counted each.  Realisation r is the stream (seed, chain0 + r):
    the one jitter_run(res, seed, chain0 + r) / resample_run(res, seed, chain0 + r) returns."""
    if error not in ('jitter', 'resample'):
        raise ValueError("Input `'error'` option '{}' is not valid.".format(error))
    if of not in ('samples', 'blob'):
        raise ValueError("of must be 'samples' or 'blob', not %r" % (of,))
    logl = np.asarray(res['logl'], dtype=float)
    x = np.asarray(res[of]) if of in res else np.empty((0, 0))
    if x.ndim != 2 or len(x) != len(logl) or x.shape[1] < 1:
        if of == 'blob':
            raise ValueError("posterior_realisations(of='blob') needs the blob of every point (res['blob']): run the "
                             "sampler with blob=True")
        raise ValueError("posterior_realisations needs the sample positions of every point (res['samples']); "
                         "a run made with keep_samples=False has none")
    logz_ref = _logz_end(res)
    if error == 'jitter':
        return ops.jitter_posterior(logl, samples_n_of(res), x, int(n_mc), int(seed), chain0=int(chain0),
                                    approx=approx, logwt_ref=res['logwt'], logz_ref=logz_ref, q=q,
                                    ctx=ctx, **_rw(res))
    return ops.resample_posterior(*_strand_inputs(res)[1], x, int(n_mc), int(seed), chain0=int(chain0),
                                  logwt_ref=res['logwt'], logz_ref=logz_ref, q=q, ctx=ctx, **_rw(res))


# ---------------------------------------------------------------------------------------------- equal-weight samples
SQRTEPS = math.sqrt(float(np.finfo(np.float64).eps))
EQUAL_MAX_BYTES = 8 << 30       # the largest gathered output equal_realisations returns (n_mc x nsamples x k float64)


def resample_equal(samples, weights, rstate=None, seed=None, chain=0, ctx=None):
    """resample_equal (utils.py:1120-1187): len(weights) equal-weight draws of samples, in random order, by systematic
    resampling -- each sample appears floor(N w_i) or ceil(N w_i) times -- computed on the GPU with the reference's
    rounding (b2n_resample_equal).  The draw is the B2N stream (seed, chain); with a numpy Generator rstate and no seed
    the seed is rstate.integers(2**63), with neither a fresh one.  Warns, as the reference does, when the weights do not
    sum to 1 within sqrt(eps); they are then renormalised.  Where the reference raises IndexError (a position that
    rounds to 1.0) the last sample is drawn."""
    w = np.asarray(weights, dtype=np.float64)
    if w.ndim != 1 or len(w) < 1:
        raise ValueError("weights must be a non-empty 1-d array")
    if len(samples) != len(w):
        raise ValueError("Dimension mismatch: len(weights) != len(samples).")
    if not np.isfinite(w).all() or (w < 0).any():
        raise ValueError("weights must be finite and non-negative")
    if not (w > 0).any():
        raise ValueError("weights sum to zero")
    if seed is None:
        seed = int(rstate.integers(1 << 63)) if rstate is not None else _seed(None)
    o = ops.resample_equal(w[None, :], len(w), int(seed), chain0=int(chain), ctx=ctx)
    if abs(o['wsum'][0] - 1.) > SQRTEPS:
        warnings.warn("Weights do not sum to 1 and have been renormalized.")
    return np.asarray(samples)[o['idx'][0]]


def equal_realisations(res, n_mc, seed, chain0=0, error='jitter', nsamples=None, approx=False, of=None, ctx=None):
    """n_mc realisations of `res` -- jitter_run's (error='jitter') or resample_run's (error='resample') -- each turned
    into nsamples (default: the record's length) equal-weight draws of the record's samples by resample_equal's
    algorithm.  Returns the dict of jitter_realisations / resample_realisations (logz, logzerr, h, kld; n_mc values
    each) plus idx (n_mc x nsamples): the drawn rows of the record, in random order, and wsum (n_mc): the sum of each
    realisation's weights exp(logwt - logz[-1]) (on the resample path, a row's weight is the sum over its copies).
    With of='samples' or 'blob', also that key: res[of][idx] (n_mc x nsamples x k), gathered on the GPU; it may not
    exceed EQUAL_MAX_BYTES.  Realisation r is the one jitter_run(res, seed, chain0 + r) / resample_run(res, seed,
    chain0 + r) returns; its draws use the stream (seed, ops.EQUAL_CHAIN0 + chain0 + r), so row r is the same whatever
    n_mc.  resample_run(res).samples_equal() would draw over the copies as rows of their own: the same distribution,
    not the same bits."""
    if error not in ('jitter', 'resample'):
        raise ValueError("Input `'error'` option '{}' is not valid.".format(error))
    if of not in (None, 'samples', 'blob'):
        raise ValueError("of must be None, 'samples' or 'blob', not %r" % (of,))
    logl = np.asarray(res['logl'], dtype=float)
    N, R = len(logl), int(n_mc)
    M = N if nsamples is None else int(nsamples)
    if M < 1 or R < 1:
        raise ValueError("n_mc and nsamples must be positive")
    if R * M >= 1 << 31:
        raise ValueError("n_mc x nsamples must be below 2^31")
    x = None
    if of is not None:
        x = np.asarray(res[of]) if of in res else np.empty((0, 0))
        if x.ndim != 2 or len(x) != N or x.shape[1] < 1:
            raise ValueError("equal_realisations(of=%r) needs res[%r] with one row per sample" % (of, of))
        if R * M * x.shape[1] * 8 > EQUAL_MAX_BYTES:
            raise ValueError("the gathered rows (n_mc x nsamples x %d float64) would exceed %d bytes; gather "
                             "res[%r][idx] in pieces instead" % (x.shape[1], EQUAL_MAX_BYTES, of))
    logz_ref = _logz_end(res)
    if error == 'jitter':
        o = ops.jitter_equal(logl, samples_n_of(res), R, M, int(seed), chain0=int(chain0), approx=approx,
                             logwt_ref=res['logwt'], logz_ref=logz_ref, x=x, ctx=ctx, **_rw(res))
    else:
        o = ops.resample_equal_runs(*_strand_inputs(res)[1], R, M, int(seed), chain0=int(chain0),
                                    logwt_ref=res['logwt'], logz_ref=logz_ref, x=x, ctx=ctx, **_rw(res))
    if of is not None:
        o[of] = o.pop('x')
    return o


# ---------------------------------------------------------------------------------------------- merging runs
def _batches(res):
    """(per-sample batch, batch bounds) of a record: its own, or batch 0 with bounds (-inf, inf) (utils.py:2027-2041)."""
    if 'samples_batch' in res and 'batch_bounds' in res:
        return (np.asarray(res['samples_batch'], dtype=np.int64),
                np.array([tuple(b) for b in res['batch_bounds']], dtype=float).reshape(-1, 2))
    return np.zeros(len(res['logl']), dtype=np.int64), np.array([[-np.inf, np.inf]])


def merge_order(res_list):
    """merge_runs' grouping (utils.py:1842-1856): (order, nbase) -- the base runs (a sample in batch 0, or no batches
    at all) in their order, then the add-on runs in theirs; one base run and one add-on run are both merged as base
    runs, in the given order."""
    base = [i for i, r in enumerate(res_list) if 'samples_batch' not in r or np.any(np.asarray(r['samples_batch']) == 0)]
    add = [i for i in range(len(res_list)) if i not in set(base)]
    if not base:
        raise ValueError("merge_runs needs at least one run started from the prior (a sample in batch 0)")
    if len(base) == 1 and len(add) == 1:
        return [0, 1], 2
    return base + add, len(base)


def _strands_resolve(res):
    """True when the record's strand columns can be resolved inside it: it ends with its final live points and every
    samples_it > 0 names an earlier sample of the record's own batch with a logl not above the point's (a strand
    that unravel_run cut out of a larger record does not)."""
    if 'samples_id' not in res or 'samples_it' not in res:
        return False
    if 'samples_batch' not in res and len(res['logl']) <= int(res['niter']):
        return False
    logl = np.asarray(res['logl'], dtype=float)
    batch = _batches(res)[0]
    it = np.asarray(res['samples_it'], dtype=np.int64)
    later = np.nonzero(it > 0)[0]
    cnt = np.bincount(batch, minlength=int(batch.max()) + 1)
    k = it[later] - 1
    if np.any(k >= cnt[batch[later]]):
        return False
    prev = np.argsort(batch, kind='stable')[(np.cumsum(cnt) - cnt)[batch[later]] + k]
    return bool(np.all(prev < later) and np.all(logl[prev] <= logl[later]))


def check_result_static(res):
    """check_result_static (utils.py:1903-1929): a record whose counts are those of a static run -- constant, or
    constant with the final N, N-1, .., 1 tail -- gets nlive = that count and niter = its length - nlive."""
    n = samples_n_of(res)
    nlive, niter = int(n.max()), int(res['niter'])
    if n.size == niter and (np.all(n == nlive) or np.all(n == np.minimum(np.arange(niter, 0, -1), nlive))):
        res['nlive'], res['niter'] = nlive, niter - nlive
    return res


def merge_runs(res_list, ctx=None):
    """merge_runs (utils.py:1817-1929): the runs of `res_list` merged into one run, e.g. an ensemble of replicas
    into a run with the sum of their live points.  Base runs (started from the prior) merge as a pairwise tree,
    add-on runs (a dynamic batch's strands, as unravel_run makes them) merge onto the result one at a time; the
    order, the live counts, ln X (with the reference's plateau rule for equal logl) and the integrals are computed by
    ``b2n_merge_runs``.  Positions (samples_u / samples), ncall_per_it, samples_scale and blob are gathered here, and
    only when every run carries them (a run made with keep_samples=False: empty positions); ncall is the sum.

    Deliberate differences from the reference:
      * samples_id is offset per run, so that the strands of different runs stay distinct (the reference keeps
        the ids, and strand 0 of two static runs would collide);
      * every (run, batch) pair is a batch of its own, with its bounds in batch_bounds (the reference merges equal
        bounds, which would make samples_it meaningless across runs);
      * samples_id / samples_it are kept only when every run carries them, ends with its final live points and
        resolves them inside itself (see ``strand_plan``); otherwise they are dropped and resample_run raises
        NotImplementedError on the merged run.
    A single run is returned as it is (after check_result_static), as the reference does."""
    res_list = list(res_list)
    if any('logrwt' in r for r in res_list):
        raise ValueError("merge_runs: a run carries a log-reweight (reweight_run); the reweight is per sample, so "
                         "merge first, then reweight")
    order, nbase = merge_order(res_list)
    ndims = {np.shape(r[k])[1] for r in res_list for k in ('samples_u', 'samples') if k in r and np.ndim(r[k]) == 2}
    if len(ndims) > 1:
        raise ValueError("merge_runs: the runs differ in ndim (%s)" % sorted(ndims))
    if len(res_list) == 1:
        return check_result_static(Results(res_list[0]))
    runs = [res_list[i] for i in order]
    sizes = np.array([len(r['logl']) for r in runs], dtype=np.int64)
    run_ptr = np.r_[0, np.cumsum(sizes)]
    logl = np.concatenate([np.asarray(r['logl'], dtype=float) for r in runs])
    lowedge = []
    for r in runs:
        b, bounds = _batches(r)
        lowedge.append(float(np.min(bounds[b])))
    o = ops.merge_runs(logl, np.concatenate([samples_n_of(r) for r in runs]), run_ptr, nbase, lowedge, arrays=True,
                       ctx=ctx)
    perm = o['perm']
    N = len(perm)
    ncall = int(sum(int(r['ncall']) if 'ncall' in r else int(np.sum(r['ncall_per_it'])) for r in runs))
    new = Results(niter=N, ncall=ncall, eff=100. * N / max(ncall, 1), logl=logl[perm], samples_n=o['samples_n'],
                  logvol=o['logvol'], logwt=o['logwt'], logz=o['logz'],
                  logzerr=np.sqrt(np.maximum(o['logzvar'], 0)), information=o['h'])

    def gather(k):
        return np.concatenate([np.asarray(r[k]) for r in runs])[perm]

    def complete(k):
        return all(k in r and len(r[k]) == len(r['logl']) for r in runs)

    for k in ('ncall_per_it', 'samples_scale', 'blob'):
        if complete(k):
            new[k] = gather(k)
    if ndims:
        ndim = ndims.pop()
        for k in ('samples_u', 'samples'):
            new[k] = gather(k) if complete(k) else np.empty((0, ndim))
    batch, bounds, boff = [], [], 0
    for r in runs:
        b, bd = _batches(r)
        batch.append(b + boff)
        bounds.extend(tuple(float(x) for x in row) for row in bd)
        boff += len(bd)
    new.update(samples_batch=np.concatenate(batch)[perm], batch_bounds=bounds)
    if all(_strands_resolve(r) for r in runs):
        ids, off = [], 0
        for r in runs:
            i = np.asarray(r['samples_id'], dtype=np.int64)
            ids.append(i + off)
            off += int(i.max()) + 1
        new.update(samples_id=np.concatenate(ids)[perm], samples_it=gather('samples_it').astype(np.int64))
    return check_result_static(new)


# ---------------------------------------------------------------------------------------------- importance reweighting
def reweight_run(res, logp_new=None, logp_old=None, model=None, ctx=None):
    """reweight_run (utils.py:1663-1708): a copy of `res` whose weights are those of a new target, without rerunning.
    logrwt = logp_new - logp_old (logp_old: res['logl'] when not given), and compute_integrals(logl, logvol,
    reweight=logrwt) on the GPU (``b2n_compute_integrals``) gives logwt, logz and logzerr = sqrt(max(logzvar, 0)).
    Give exactly one of logp_new (N) and model: a ``DeviceModel`` whose likelihood is evaluated at every res['samples']
    in one launch (its likelihood-only twin, the model id ids()[1]).  logrwt may hold -inf (zero weight), not NaN or
    +inf, and not -inf everywhere.  The copy keeps logvol and records logrwt (N), which the realisations of this
    module carry from then on.  As in the reference, `information` is the input's: the reference hands h over under
    the key 'h', which its Results drops."""
    if (logp_new is None) == (model is None):
        raise ValueError("reweight_run needs exactly one of logp_new and model")
    logl = np.asarray(res['logl'], dtype=float)
    N = len(logl)
    if model is not None:
        x = np.asarray(res['samples']) if 'samples' in res else np.empty((0, 0))
        if x.ndim != 2 or len(x) != N or x.shape[1] < 1:
            raise ValueError("reweight_run(model=) needs the sample positions of every point (res['samples']); a run "
                             "made with keep_samples=False has none")
        if x.shape[1] != model.ndim:
            raise ValueError("the model has %d dimensions, the samples %d" % (model.ndim, x.shape[1]))
        logp_new = ops.model_eval(model.ids(ctx)[1], x, want_v=False, ctx=ctx)[1]
    logp_new = np.asarray(logp_new, dtype=float)
    logp_old = logl if logp_old is None else np.asarray(logp_old, dtype=float)
    if logp_new.shape != (N,) or logp_old.shape != (N,):
        raise ValueError("logp_new and logp_old must hold one value per sample (%d)" % N)
    with np.errstate(invalid='ignore'):
        logrwt = logp_new - logp_old
    if np.isnan(logrwt).any() or np.isposinf(logrwt).any():
        raise ValueError("logp_new - logp_old holds NaN or +inf")
    if np.all(logrwt == -np.inf):
        raise ValueError("logp_new - logp_old is -inf at every sample: the new target gives the run no weight")
    o = ops.compute_integrals(logl, res['logvol'], logrwt, ctx=ctx)
    new = Results(res)
    new.update(logwt=o['logwt'], logz=o['logz'], logzerr=np.sqrt(np.maximum(o['logzvar'], 0)), logrwt=logrwt)
    return new

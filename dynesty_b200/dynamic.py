"""Dynamic nested sampling with every run -- the baseline AND each batch -- as rounds on the device.

SURVEY.md 8(f) row 4.  What is mirrored (reference py/dynesty/dynamicsampler.py, same names / meaning):
  compute_weights / weight_function   :48-170     posterior / evidence importance -> (logl_min, logl_max)
  _configure_batch_sampler            :300-622    live points of a batch: saved samples above logl_min, picked with
                                                  weights X_i, a bound fitted to them, `nlive_batch` NEW points evolved
                                                  from them at the threshold logl_min
  sample_batch                        :1228-1466  the batch run: stop at logl_max, then its live points (n = N, N-1, ..)
  combine_runs                        :1467-1608  merge by logl; live count of a merged point = sum of the runs' counts
                                                  where they overlap; ln X recursion ln X -= ln((n+1)/n); integrals
  stopping_function                   :173-297    stop value from n_effective and the jitter scatter of ln Z
  run_nested / add_batch              :1610-2050  baseline, then batches until the stop value / maxbatch

B200 mapping: the baseline is ``NestedSampler.run_nested(loop='device')``; a batch is (i) ONE chain launch that
evolves the `nlive_batch` new live points from the selected saved samples (the reference loops `_new_point`
nlive_batch times, :553-577) and (ii) device rounds (``b2n_ns_run``) from those points with the ``logl_max`` stop
raised on the device; the merge is vectorised numpy on the host (sorting two records, a cumulative sum).  The
unmodified ``dynesty.DynamicNestedSampler`` also runs with the B200 bounds / samplers plugged in
(tests/test_gpu_dropin.py); this module is the path that keeps the batches' inner loops on the GPU.
"""
import math
import warnings

import numpy as np

from . import nested
from .nested import Results, _integrate

# chain ids of the stopping checks' jitter realisations: check k of a run uses STOP_CHAIN0 + k * 2^32 + r.  The block
# [3 * 2^61, 2^63) is disjoint from every id a run draws from (proposal chains count from 0, the initial live points
# are 2^61 + i, the round driver 2^62 + r), so a seeded dynamic run with a stopping check stays reproducible.
STOP_CHAIN0 = 3 << 61


def _logsumexp(a, b=None):
    a = np.asarray(a, dtype=float)
    m = np.max(a)
    if not np.isfinite(m):
        return m
    w = np.exp(a - m) if b is None else np.asarray(b) * np.exp(a - m)
    return m + math.log(np.sum(w))


def compute_weights(res):
    """dynamicsampler.py:48-81: (zweight, pweight) per sample."""
    logl, logz, logvol, logwt, n = res['logl'], res['logz'], res['logvol'], res['logwt'], res['samples_n']
    if np.ptp(logz) == 0:
        zweight = np.ones(len(logl)) / len(logl)
    else:
        logz_remain = logl[-1] + logvol[-1]
        logz_tot = np.logaddexp(logz[-1], logz_remain)
        # ln(remaining evidence) = ln(exp(logz_tot) - exp(logz))
        logzin = logz_tot + np.log1p(-np.exp(np.minimum(logz - logz_tot, -1e-300)))
        logzweight = logzin - np.log(n)
        logzweight -= _logsumexp(logzweight)
        zweight = np.exp(logzweight)
    pweight = np.exp(logwt - logz[-1])
    pweight /= pweight.sum()
    return zweight, pweight


def weight_function(res, args=None):
    """dynamicsampler.py:84-170: log-likelihood bounds of the next batch."""
    args = args or {}
    pfrac, maxfrac, lpad = args.get('pfrac', 0.8), args.get('maxfrac', 0.8), args.get('pad', 1)
    if not 0. <= pfrac <= 1. or not 0. <= maxfrac <= 1. or lpad < 0:
        raise ValueError("weight_function: need 0 <= pfrac, maxfrac <= 1 and pad >= 0")
    zweight, pweight = compute_weights(res)
    weight = (1. - pfrac) * zweight + pfrac * pweight
    nsamps = len(weight)
    b = np.nonzero(weight > maxfrac * weight.max())[0]
    b = [b[0] - lpad, b[-1] + lpad]
    logl = res['logl']
    if b[1] > nsamps - 1:
        b = [b[0] - (b[1] - (nsamps - 1)), nsamps - 1]
    if b[0] <= 0:
        logl_min, logl_max = -np.inf, logl[min(b[1] - b[0], nsamps - 1)]
    else:
        logl_min, logl_max = logl[b[0]], logl[b[1]]
    if b[1] == nsamps - 1:
        logl_max = np.inf
    return float(logl_min), float(logl_max)


def n_effective(logwt):
    """utils.py:1012-1030 get_neff_from_logwt (Kish)."""
    w = np.exp(logwt - np.max(logwt))
    return float(w.sum()**2 / (w * w).sum())


def stopping_function(results, args=None, seed=None, chain0=0, return_vals=False, ctx=None):
    """dynamicsampler.py:173-297: stop = pfrac * stop_post + (1 - pfrac) * stop_evid with
    stop_post = target_n_effective / n_effective and stop_evid = std(ln Z) / evid_thresh, the std over n_mc jitter
    realisations (``utils.jitter_realisations`` or, with error='resample', ``utils.resample_realisations``; streams
    (seed, chain0 + r)) or, with n_mc <= 1, logzerr[-1].
    args (defaults): pfrac 1.0, evid_thresh 0.1, target_n_effective 10000, n_mc 0, error 'jitter', approx True.
    Returns stop <= 1 [, (stop_post, stop_evid, stop)]."""
    from . import utils
    args = args or {}
    pfrac = args.get('pfrac', 1.0)
    if not 0. <= pfrac <= 1.:
        raise ValueError(f"The provided `pfrac` {pfrac} is not between 0. and 1.")
    evid_thresh = args.get('evid_thresh', 0.1)
    if pfrac < 1. and evid_thresh < 0.:
        raise ValueError(f"The provided `evid_thresh` {evid_thresh} is not non-negative even though `pfrac` is {pfrac}.")
    target_n_effective = args.get('target_n_effective', 10000)
    if pfrac > 0. and target_n_effective < 0.:
        raise ValueError(f"The provided `target_n_effective` {target_n_effective} is not non-negative even though "
                         f"`pfrac` is {pfrac}")
    n_mc = args.get('n_mc', 0)
    if n_mc < 0:
        raise ValueError(f"The number of realizations {n_mc} must be greater or equal to zero.")
    if 0 < n_mc < 20:
        warnings.warn("Using a small number of realizations might result in excessively noisy stopping value "
                      "estimates.")
    error = args.get('error', 'jitter')
    if error not in {'jitter', 'resample'}:
        raise ValueError(f"The chosen `'error'` option {error} is not valid.")
    approx = args.get('approx', True)
    if n_mc > 1:
        if error == 'resample':
            lnz = utils.resample_realisations(results, n_mc, utils._seed(seed), chain0=chain0, ctx=ctx)['logz']
        else:
            lnz = utils.jitter_realisations(results, n_mc, utils._seed(seed), chain0=chain0, approx=approx,
                                            ctx=ctx)['logz']
        lnz_std = np.std(lnz)
    else:
        lnz_std = results['logzerr'][-1]
    stop_evid = lnz_std / evid_thresh
    stop_post = target_n_effective / n_effective(results['logwt'])
    stop = pfrac * stop_post + (1. - pfrac) * stop_evid
    return (bool(stop <= 1.), (stop_post, stop_evid, stop)) if return_vals else bool(stop <= 1.)


def merge_two(saved, new, logl_min):
    """combine_runs (dynamicsampler.py:1467-1608) for two records dict(u, v, logl, n, nc, scale, batch[, id, it, blob]),
    every key one row per sample: both sorted
    by logl; ties go to the saved run; the live count of a merged point is its own run's plus -- above logl_min --
    the count the OTHER run has at that position."""
    ls, ln_ = saved['logl'], new['logl']
    ns_, nn = saved['n'], new['n']
    # position of the other run's pointer when a point is taken (the loop's idx_new / idx_saved)
    pos_new = np.searchsorted(ln_, ls, side='left')            # new points strictly below a saved point went first
    pos_sav = np.searchsorted(ls, ln_, side='right')           # saved points <= a new point went first
    n_new_at = np.where(pos_new < len(nn), nn[np.minimum(pos_new, len(nn) - 1)], 0)
    n_sav_at = np.where(pos_sav < len(ns_), ns_[np.minimum(pos_sav, len(ns_) - 1)], 0)
    n_saved = np.where(ls > logl_min, ns_ + n_new_at, ns_)
    head = np.where(pos_sav < len(ls), ls[np.minimum(pos_sav, len(ls) - 1)], np.inf)      # saved head when a new point is taken
    n_newpts = np.where(head > logl_min, n_sav_at + nn, n_sav_at)
    # merged order: saved point i lands at i + pos_new[i], new point j at j + pos_sav[j]
    tot = len(ls) + len(ln_)
    order_s = np.arange(len(ls)) + pos_new
    order_n = np.arange(len(ln_)) + pos_sav
    out = {}
    for k in saved:
        a, b = np.asarray(saved[k]), np.asarray(new[k])
        m = np.empty((tot,) + a.shape[1:], dtype=np.result_type(a, b))
        m[order_s] = a
        m[order_n] = b
        out[k] = m
    nm = np.empty(tot, dtype=np.int64)
    nm[order_s] = n_saved
    nm[order_n] = n_newpts
    out['n'] = nm
    return out


def integrate_record(rec, logvol_init=0.0):
    """ln X from the live counts (combine_runs :1560-1585, no plateau mode: continuous likelihoods), starting at
    `logvol_init`, the ln X of the base run's initial live points (``NestedSampler.initial_logvol``), then the
    trapezoid integrals (utils.compute_integrals)."""
    n = rec['n'].astype(float)
    logvol = logvol_init - np.cumsum(np.log((n + 1.) / n))
    logwt, logz, logzvar, h = _integrate(rec['logl'], logvol, logvol_init=logvol_init)
    return logvol, logwt, logz, logzvar, h


class DynamicNestedSampler:
    """Parameters follow dynesty.DynamicNestedSampler (dynesty.py:686-720) with `model` = a DeviceModel."""

    def __init__(self, model, nlive=500, bound='multi', sample='auto', seed=56432, ctx=None, **sampler_kwargs):
        self.model, self.nlive0, self.bound, self.sample = model, int(nlive), bound, sample
        self.seed, self.ctx, self.kw = int(seed), ctx, dict(sampler_kwargs)
        self.rstate = np.random.default_rng(seed)
        self.ndim = model.ndim
        self.saved = None
        self.batch = 0
        self.ncall = 0
        self.batch_bounds = []
        self.results = None
        self.logvol_init = 0.0            # ln X of the baseline's initial live points (sample_initial)
        self.strands = False              # record samples_id / samples_it (run_nested(strands=True))

    def _sampler(self, nlive, seed, live_points=None):
        return nested.NestedSampler(self.model, nlive=nlive, bound=self.bound, sample=self.sample, seed=seed, ctx=self.ctx,
                                    live_points=live_points, **self.kw)

    @staticmethod
    def _record(res, batch_id, id_offset=0):
        rec = dict(u=res['samples_u'], v=res['samples'], logl=res['logl'], n=np.asarray(res['samples_n'], dtype=np.int64),
                   nc=np.asarray(res['ncall_per_it'], dtype=np.int64), scale=np.asarray(res['samples_scale'], dtype=float),
                   batch=np.full(len(res['logl']), batch_id, dtype=np.int64))
        if 'blob' in res:
            rec['blob'] = np.asarray(res['blob'])
        if 'samples_id' in res:
            # a batch's strands are new strands: its slot ids follow the saved ones (dynamicsampler.py:1489)
            rec.update(id=np.asarray(res['samples_id'], dtype=np.int64) + id_offset,
                       it=np.asarray(res['samples_it'], dtype=np.int64))
        return rec

    def _results(self):
        rec = self.saved
        logvol, logwt, logz, logzvar, h = integrate_record(rec, self.logvol_init)
        self.results = Results(niter=len(rec['logl']), ncall=int(self.ncall), eff=100. * len(rec['logl']) / max(self.ncall, 1),
                               samples_u=rec['u'], samples=rec['v'], logl=rec['logl'], logvol=logvol, logwt=logwt, logz=logz,
                               logzerr=np.sqrt(logzvar), information=h, samples_n=rec['n'], samples_scale=rec['scale'],
                               ncall_per_it=rec['nc'], samples_batch=rec['batch'], batch_bounds=list(self.batch_bounds),
                               nbatch=self.batch)
        if 'id' in rec:
            self.results.update(samples_id=rec['id'], samples_it=rec['it'])
        if 'blob' in rec:
            self.results['blob'] = rec['blob']
        return self.results

    # ------------------------------------------------------------------ baseline (sample_initial, :927-1226)
    def sample_initial(self, nlive=None, dlogz=0.01, maxiter=None, maxcall=None, round_size=None):
        s = self._sampler(nlive or self.nlive0, self.seed)
        res = s.run_nested(dlogz=dlogz, maxiter=maxiter, maxcall=maxcall, add_live=True, loop='device', batch=round_size,
                           strands=self.strands)
        self.saved = self._record(res, 0)
        self.ncall = int(res['ncall'])
        self.base_sampler = s
        self.logvol_init = s.logvol_init
        self.batch_bounds = [(-np.inf, np.inf)]
        return self._results()

    # ------------------------------------------------------------------ one batch (sample_batch + combine_runs)
    def add_batch(self, nlive=None, wt_kwargs=None, logl_bounds=None, dlogz=0.01, maxiter=None, maxcall=None, round_size=None):
        nlive = int(nlive or self.nlive0)
        res = self.results
        logl_min, logl_max = logl_bounds if logl_bounds is not None else weight_function(res, wt_kwargs)
        sv = self.saved
        saved_logl, saved_logvol = sv['logl'], res['logvol']
        seed = self.seed + 1000003 * (self.batch + 1)
        if np.all(saved_logl > logl_min):
            # the batch starts from the prior (:413-461): a fresh run from the unit cube up to logl_max
            bs = self._sampler(nlive, seed)
            out = bs.run_nested(dlogz=dlogz, maxiter=maxiter, maxcall=maxcall, add_live=True, loop='device', batch=round_size,
                                logl_max=None if not np.isfinite(logl_max) else logl_max, strands=self.strands)
            logl_min = -np.inf
            ncall_new = int(out['ncall'])
        else:
            # live points of the batch (:463-577): saved samples above logl_min, chosen with weights X_i
            subset0 = np.nonzero(saved_logl > logl_min)[0]
            if len(subset0) == 0:
                raise RuntimeError('Could not find live points in the required logl interval.')
            if len(subset0) < nlive:
                if len(saved_logl) < nlive:
                    subset0 = np.arange(len(saved_logl))
                else:
                    subset0 = np.arange(subset0[-1] - nlive + 1, subset0[-1] + 1)
                logl_min = float(saved_logl[subset0[0] - 1]) if subset0[0] > 0 else -np.inf
            live_scale = float(sv['scale'][subset0[0]])
            lw = saved_logvol[subset0]
            w = np.exp(lw - lw.max())
            w /= w.sum()
            npos = int((w > 0).sum())
            subset = self.rstate.choice(subset0, size=min(nlive, npos), p=w, replace=False)
            if len(subset) == 1:
                raise RuntimeError('Only one live point is selected')
            pts = (sv['u'][subset].copy(), sv['v'][subset].copy(), saved_logl[subset].copy())
            bs = self._sampler(len(subset), seed, live_points=pts)
            # the bound of the batch is fitted to the selected samples (update_bound_if_needed(logl_min), :545)
            bs.unit_cube_sampling = False
            bs.bound, bs.internal_sampler = bs.bound_next, bs.internal_sampler_next
            bs.logl_first_update = logl_min
            if hasattr(bs.internal_sampler, 'scale'):
                bs.internal_sampler.scale = live_scale
            bs.update_bound()
            bs.nbound += 1
            # `nlive` NEW live points evolved at the threshold logl_min: one launch instead of nlive x _new_point
            bs.queue_size = nlive
            bs._fill_queue(logl_min)
            q = bs._q
            if not np.all(q['logl'] > logl_min):
                # (uniform draws always pass; a chain that never moved returns its start, which is above logl_min)
                raise RuntimeError('batch initialisation produced a point below logl_min')
            ncall0 = int(q['ncall'].sum())
            bs.nlive = nlive
            bs.live_u, bs.live_v, bs.live_logl = q['u'].copy(), q['v'].copy(), q['logl'].copy()
            bs._q = None
            bs.ncall = ncall0
            bs.ncall_at_last_update = 0
            bs.it = 1
            if self.strands:
                bs.live_it = np.zeros(nlive, dtype=np.int64)     # the batch's points start its strands
            # join the saved run where it crosses logl_min (:598-606): ln X and ln Z there start the batch's dlogz test
            vol_idx = 0 if not np.isfinite(logl_min) else int(np.argmin(np.abs(saved_logl - logl_min))) + 1
            lv0 = float(saved_logvol[vol_idx - 1]) if vol_idx > 0 else self.logvol_init
            lz0 = float(res['logz'][vol_idx - 1]) if vol_idx > 0 else nested.LOWL
            dev = bs._device_rounds(lz0, lv0, logl_min if np.isfinite(logl_min) else nested.LOWL, dlogz,
                                    maxiter if maxiter is not None else 1 << 62, maxcall, round_size,
                                    logl_max=None if not np.isfinite(logl_max) else logl_max)
            e = np.empty((0, self.ndim))
            out = bs._finalize(e, e, np.empty(0), np.empty(0), np.empty(0, dtype=np.int64), dev, True)
            ncall_new = int(bs.ncall)
        new = self._record(out, self.batch + 1, int(sv['id'].max()) + 1 if 'id' in sv else 0)
        self.saved = merge_two(self.saved, new, logl_min)
        self.ncall += ncall_new
        self.batch += 1
        self.batch_bounds.append((logl_min, logl_max))
        self.last_batch_sampler = bs
        return self._results()

    # ------------------------------------------------------------------ run_nested (:1610-1928)
    def run_nested(self, nlive_init=None, dlogz_init=0.01, nlive_batch=None, wt_kwargs=None, maxbatch=None,
                   n_effective=None, maxcall=None, round_size=None, stop_kwargs=None, strands=False):
        """Baseline run, then batches placed by ``weight_function`` until the Kish effective sample size of the merged
        run reaches `n_effective` (default max(ndim^2, 10000), :1782-1784) or `maxbatch` batches have been added.

        With `stop_kwargs` (the args of ``stopping_function``; its target_n_effective is `n_effective`, as in the
        reference, :1785-1794) the run instead stops once the stopping function's value is <= 1, evaluated before
        every batch (:1865-1880).  Check k draws its jitter realisations from the streams (seed, STOP_CHAIN0 +
        k * 2^32 + r); the values of every check are kept in ``self.stop_vals``.

        strands=True records every sample's strand (samples_id / samples_it, see NestedSampler.run_nested); a stop on
        error='resample' turns it on.  It applies from the baseline on: a sampler whose baseline ran without strands
        cannot add batches with them."""
        target = n_effective if n_effective is not None else max(self.ndim * self.ndim, 10000)
        maxbatch = maxbatch if maxbatch is not None else 1 << 30
        if stop_kwargs is not None:
            stop_kwargs = dict(stop_kwargs, target_n_effective=target)
            self.stop_vals = []
        if self.saved is None:
            self.strands = bool(strands or (stop_kwargs is not None and stop_kwargs.get('error') == 'resample'))
            self.sample_initial(nlive=nlive_init, dlogz=dlogz_init, maxcall=maxcall, round_size=round_size)
        for _ in range(self.batch, maxbatch):
            if maxcall is not None and self.ncall >= maxcall:
                break
            if stop_kwargs is None:
                if n_effective_of(self.results) >= target:
                    break
            else:
                stop, vals = stopping_function(self.results, stop_kwargs, seed=self.seed,
                                               chain0=self.stop_chain0(self.batch), return_vals=True, ctx=self.ctx)
                self.stop_vals.append(vals)
                if stop:
                    break
            self.add_batch(nlive=nlive_batch, wt_kwargs=wt_kwargs, round_size=round_size,
                           maxcall=None if maxcall is None else maxcall - self.ncall)
        return self.results

    @staticmethod
    def stop_chain0(batch):
        """first chain id of the stopping check made when `batch` batches have been added"""
        return STOP_CHAIN0 + (int(batch) << 32)


def n_effective_of(res):
    return n_effective(res['logwt'])

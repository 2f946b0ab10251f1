"""Prior-volume realisations of a dead-point record (the reference's jitter_run / kld_error), restated in numpy.

TEST INFRASTRUCTURE (see oracle/__init__.py).  What is restated (reference py/dynesty/utils.py):
  _find_decrease     :1273-1314   decreasing stretches of samples_n -- here without the loop
  jitter_run         :1317-1408   t per sample, logvol = cumsum(ln t)
  compute_integrals  :1411-1467   dynesty_b200.nested._integrate (same quadrature)
  kld_error          :1932-1997   cumulative KL divergence against the input run's weights

Random stream of realisation r (include/b200nest.h, b2n_jitter_runs): the B2N chain (seed, chain0 + r), events in the
reference's call order -- tick 0: one uniform vector event over the F flagged samples, ln t = ln(U_e) / n; tick s + 1:
stretch s draws nstart_s + 1 uniforms, y = -ln U.  ``ScriptedJitterGenerator(seed, chain0 + r)`` (below) drives the
unmodified reference with the same numbers (its beta() returns U^(1/n), whose log is ln(U)/n up to one rounding).
"""
import numpy as np

from . import philox


class ScriptedJitterGenerator(philox.ScriptedGenerator):
    """``philox.ScriptedGenerator`` plus the two draws jitter_run makes, each one uniform vector event of the B2N
    stream, so that the unmodified reference's jitter_run / kld_error consume the numbers b2n_jitter_runs consumes."""

    def beta(self, a, b=1.0, size=None):
        """utils.py:1368 ``rstate.beta(a=samples_n[flag], b=1)``: element e -> U_e^(1/a_e), the maximum of a_e
        uniforms."""
        assert b == 1 and size is None
        a = np.asarray(a, dtype=np.float64)
        return self.random(a.shape) ** (1.0 / a)

    def exponential(self, scale=1.0, size=None):
        """utils.py:1384 ``rstate.exponential(scale=1.0, size=nstart+1)``: -scale ln U."""
        return -scale * np.log(self.random(size))


def find_decrease(samples_n):
    """_find_decrease (utils.py:1273-1314): (nlive_flag, nlive_start, bounds) with bounds[s] = (b0, b1), the samples of
    stretch s, b0 = the sample before the first decrease."""
    n = np.asarray(samples_n)
    N = len(n)
    dec = np.zeros(N, dtype=bool)
    dec[1:] = np.diff(n) < 0
    prev = np.r_[False, dec[:-1]]
    nxt = np.r_[dec[1:], False]
    first = np.nonzero(dec & ~prev)[0]
    last = np.nonzero(dec & ~nxt)[0]
    bounds = np.stack([first - 1, last + 1], axis=1) if len(first) else np.empty((0, 2), dtype=np.int64)
    return ~dec, n[first - 1] if len(first) else np.empty(0, dtype=n.dtype), bounds


def segment_plan(samples_n, approx, tile):
    """(nseg, longest_scan) of b2n_jitter_runs' plan (jitter_plan in csrc/b2n_jitter.cu): every run of flagged samples
    outside the stretches and every stretch is cut into segments of at most `tile` samples; a piece of a stretch scans
    its exponentials 0..kprev (kprev = nstart for the first piece, else k of the sample before it).  longest_scan is
    the largest kprev + 1, the most exponentials one segment scans (0 without stretches)."""
    n = np.asarray(samples_n, dtype=np.int64)
    N = len(n)
    bounds = np.empty((0, 2), dtype=np.int64) if approx else find_decrease(n)[2]
    cover = np.zeros(N + 1, dtype=np.int64)
    np.add.at(cover, bounds[:, 0], 1)
    np.add.at(cover, bounds[:, 1], -1)
    edges = np.diff(np.r_[0, (np.cumsum(cover)[:N] == 0).astype(np.int64), 0])
    runs = np.nonzero(edges == -1)[0] - np.nonzero(edges == 1)[0]
    nseg, longest = int(np.sum(-(-runs // tile))), 0
    for b0, b1 in bounds:
        a = np.arange(b0, b1, tile)
        kprev = np.where(a == b0, n[b0], n[a - 1] - 1)
        nseg += len(a)
        longest = max(longest, int(kprev.max()) + 1)
    return nseg, longest


def integrate(logl, logvol):
    """compute_integrals (utils.py:1411-1467): logwt, logz, logzvar, h."""
    from dynesty_b200.nested import _integrate
    return _integrate(np.asarray(logl, dtype=float), logvol)


def log_t(samples_n, seed, chain, approx=False, plan=None, dtype=np.float64):
    """ln t per sample of one realisation (jitter_run, utils.py:1359-1393), computed in `dtype` from the float64
    uniforms."""
    n = np.asarray(samples_n)
    N = len(n)
    flag, nstart, bounds = plan if plan is not None else (
        (np.ones(N, dtype=bool), np.empty(0, dtype=int), np.empty((0, 2), dtype=int)) if approx else find_decrease(n))
    lt = np.zeros(N, dtype=dtype)
    lt[flag] = np.log(philox.event_uniforms(seed, chain, 0, int(flag.sum())).astype(dtype)) / n[flag]
    if len(nstart):
        # every stretch's exponentials at once: ticks 1..S, element e of stretch s at row s of a padded table
        m = nstart.astype(np.int64) + 1
        S, W = len(m), int(m.max())
        nb = (m + 1) // 2                                  # Philox blocks per event
        s_of = np.repeat(np.arange(S), nb)
        blk = np.arange(nb.sum()) - np.repeat(np.cumsum(nb) - nb, nb)
        ctr = np.empty((len(s_of), 4), dtype=np.uint64)
        ctr[:, 0] = blk
        ctr[:, 1] = s_of + 1
        ctr[:, 2] = int(chain) & 0xFFFFFFFF
        ctr[:, 3] = (int(chain) >> 32) & 0xFFFFFFFF
        key = np.array([int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF], dtype=np.uint64)
        r = philox.philox4x32_10(ctr, key)
        u = np.stack([philox.u53(r[:, 0], r[:, 1]), philox.u53(r[:, 2], r[:, 3])], axis=1)
        y = np.ones((S, 2 * int(nb.max())), dtype=dtype)
        y[s_of, 2 * blk] = u[:, 0]
        y[s_of, 2 * blk + 1] = u[:, 1]
        y = -np.log(y[:, :W])
        ycsum = np.cumsum(y, axis=1)                       # row s: the reference's y_arr.cumsum() (padding after m_s)
        ycsum /= ycsum[np.arange(S), m - 1][:, None]
        lens = bounds[:, 1] - bounds[:, 0]
        samp = np.arange(lens.sum()) - np.repeat(np.cumsum(lens) - lens, lens) + np.repeat(bounds[:, 0], lens)
        srow = np.repeat(np.arange(S), lens)
        k = n[samp] - 1
        first = np.r_[True, srow[1:] != srow[:-1]]
        kprev = np.where(first, nstart[srow], np.r_[0, k[:-1]])
        uorder_k, uorder_p = ycsum[srow, k], ycsum[srow, kprev]
        lt[samp] = np.log(uorder_k / uorder_p)
    return lt


def realisation(logl, samples_n, seed, chain, approx=False, logwt_ref=None, logz_ref=None, plan=None,
                dtype=np.float64):
    """One realisation: dict(logvol, logwt, logz, logzvar, h[, kld]), in `dtype` (np.longdouble: a reference for
    records so long that float64's running sums round at the bars the kernel is held to)."""
    lt = log_t(samples_n, seed, chain, approx, plan, dtype)
    logvol = np.cumsum(lt)
    logwt, logz, logzvar, h = integrate(logl, logvol)
    out = dict(logvol=logvol, logwt=logwt, logz=logz, logzvar=logzvar, h=h)
    if logwt_ref is not None:
        logp2 = np.asarray(logwt_ref) - logz_ref
        logp1 = logwt - logz[-1]
        out['kld'] = np.cumsum(np.exp(logp1) * (logp1 - logp2))
    return out


def jitter_runs(logl, samples_n, R, seed, chain0=0, approx=False, logwt_ref=None, logz_ref=None, arrays=False,
                dtype=np.float64):
    """Same contract as ``dynesty_b200.ops.jitter_runs``: the summaries (R each) and, with arrays, the R x N arrays
    (computed in `dtype`, returned in float64)."""
    n = np.asarray(samples_n)
    plan = (np.ones(len(n), dtype=bool), np.empty(0, dtype=int), np.empty((0, 2), dtype=int)) if approx \
        else find_decrease(n)
    rs = [realisation(logl, n, seed, chain0 + r, approx, logwt_ref, logz_ref, plan, dtype) for r in range(R)]
    out = dict(logz=np.array([o['logz'][-1] for o in rs]),
               logzerr=np.array([np.sqrt(max(o['logzvar'][-1], 0.)) for o in rs]),
               h=np.array([o['h'][-1] for o in rs]))
    if logwt_ref is not None:
        out['kld'] = np.array([o['kld'][-1] for o in rs])
    if arrays:
        for k in ('logvol', 'logwt', 'logz') + (('kld',) if logwt_ref is not None else ()):
            out[k + '_arr'] = np.array([o[k] for o in rs])
    return {k: v.astype(np.float64) for k, v in out.items()}


def expected_record(samples_n):
    """A record with the given samples_n at its expected volumes, ln X_i = sum_{j <= i} ln(n_j / (n_j + 1)), with a
    bounded logl whose posterior bulk sits halfway down in ln X: logl = -d/2 exp(2 ln X / d + 1), d = -ln X[-1]
    (at least 1).  Returns dict(logl, samples_n, logvol, logwt, logz)."""
    n = np.asarray(samples_n, dtype=np.int64)
    logvol = np.cumsum(np.log(n / (n + 1.)))
    d = max(-logvol[-1], 1.0)
    logl = -0.5 * d * np.exp(2.0 * logvol / d + 1.0)
    logwt, logz, _, _ = integrate(logl, logvol)
    return dict(logl=logl, samples_n=n, logvol=logvol, logwt=logwt, logz=logz)


def synthetic_record(nlive=2000, K=50, ndim=50, lnx_end=-25.0, seed=0):
    """A seeded dead-point record of the shape of a device-round run: rounds of K removals (samples_n = nlive,
    nlive-1, .., nlive-K+1) down to ln X = lnx_end, then the add_live tail (nlive, .., 1).  logl follows an isotropic
    ndim-D Gaussian's X(L): ln X = ndim ln(r / r0), logl = -r^2 / 2, r0^2 = ndim e^0.6 (the posterior bulk near
    ln X = -15), with the volumes jittered once by `seed` so that the record is not the expectation itself.
    Returns (logl, samples_n)."""
    rng = np.random.default_rng(seed)
    nrounds = int(np.ceil(-lnx_end * nlive / K))
    n = np.r_[np.tile(nlive - np.arange(K), nrounds), nlive - np.arange(nlive)].astype(np.int64)
    lnx = np.cumsum(np.log(rng.random(len(n))) / n)
    r2 = ndim * np.exp(0.6) * np.exp(2.0 * lnx / ndim)
    return np.sort(-0.5 * r2), n

"""Run uncertainties from simulated prior volumes, computed on the GPU.

What is mirrored (reference py/dynesty/utils.py, same names / meaning):
  jitter_run   :1317-1408   one realisation of the prior volumes of a run's dead points
  kld_error    :1932-1997   the KL divergence from the run to such a realisation
and ``jitter_realisations``, the batched form the dynamic sampler's stopping function needs: n_mc realisations in one
call (``b2n_jitter_runs``, a fixed number of kernel launches whatever n_mc, the record length or its number of
decreasing stretches).

Randomness: realisation r of a call is the B2N Philox stream (seed, chain0 + r) (include/b200nest.h,
b2n_jitter_runs), so a (seed, chain) pair names one realisation: it is the same whether it is computed alone or in a
batch of any size.  ``seed=None`` draws a fresh seed, like the reference's ``rstate=None``.

``resample_run`` (bootstrap over the threads of a run) is not provided: it needs, for every dead point, the live slot it
came from (the reference's samples_id / samples_it), and the device rounds do not record that.
"""
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


def jitter_realisations(res, n_mc, seed, chain0=0, approx=False, arrays=False, ctx=None):
    """n_mc realisations of `res` in one call.  Returns dict(logz, logzerr, h, kld): the last element of each
    realisation's logz / logzerr / information / cumulative KL divergence (n_mc values each); with arrays=True also
    logvol_arr, logwt_arr, logz_arr, kld_arr (n_mc x nsamps).  Realisation r uses the stream (seed, chain0 + r)."""
    logz = np.asarray(res['logz'])
    return ops.jitter_runs(res['logl'], samples_n_of(res), int(n_mc), int(seed), chain0=int(chain0),
                           approx=approx, logwt_ref=res['logwt'], logz_ref=float(logz[-1]), arrays=arrays, ctx=ctx)


def _realisation(res, seed, chain, approx, ctx):
    o = jitter_realisations(res, 1, _seed(seed), chain, approx, arrays=True, ctx=ctx)
    logvol = o['logvol_arr'][0]
    # logzerr and information as arrays: the quadrature of compute_integrals on the realisation's volumes (host,
    # O(nsamps) for the one realisation; their last elements are the kernel's)
    _, _, logzvar, h = _integrate(np.asarray(res['logl'], dtype=float), logvol)
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
    jitter_run; with return_new, also that realisation."""
    if error == 'resample':
        raise NotImplementedError(
            "error='resample' needs resample_run, which needs the live slot every dead point came from (samples_id / "
            "samples_it); the device rounds do not record it.  Use error='jitter'.")
    if error != 'jitter':
        raise ValueError("Input `'error'` option '{}' is not valid.".format(error))
    new, kld = _realisation(res, seed, chain, approx, ctx)
    return (kld, new) if return_new else kld

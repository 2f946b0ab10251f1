"""Per-chain restatement of dynesty's inner proposal samplers.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Citations are to
py/dynesty/internal_samplers.py unless noted.

Each function advances ONE chain and takes a ``stream`` with the
``oracle.philox.ChainStream`` interface (uniform / uniforms / normals /
permutation), i.e. the same draw events, in the same order, as the reference
makes on its ``numpy.random.Generator``.  Written as plain per-step Python
loops on purpose: that is what the reference's CPU path is, and it is the
thing ``bench.py``'s ``cpu_baseline`` times.
"""
import math
import numpy as np


def unitcheck(u, nonbounded=None):
    """utils.py:1036-1050 (strict inequalities)."""
    if nonbounded is None:
        return u.min() > 0 and u.max() < 1
    a, b = u[nonbounded], u[~nonbounded]
    ok = True
    if a.size:
        ok = a.min() > 0 and a.max() < 1
    if ok and b.size:
        ok = b.min() > -0.5 and b.max() < 1.5
    return bool(ok)


def reflect(u):
    """utils.py:1053-1078."""
    even = np.mod(u, 2) < 1
    out = np.empty_like(u)
    out[even] = np.mod(u[even], 1)
    out[~even] = 1 - np.mod(u[~even], 1)
    return out


def randsphere(n, stream):
    """bounding.py:1288-1297: uniform in the unit n-ball."""
    z = stream.normals(n)
    return z * (stream.uniform()**(1. / n) / math.sqrt(float(np.dot(z, z))))


def rwalk_chain(u0, loglstar, axes, scale, model, stream, walks,
                periodic=None, reflective=None, nonbounded=None):
    """generic_random_walk + propose_ball_point (:866-1035).

    axes is (ncdim, ncdim); dims >= ncdim get a fresh U(0,1) each proposal.
    Returns dict(u, v, logl, ncall, n_accept, n_reject)."""
    u = np.array(u0, dtype=float)
    n = u.shape[0]
    nc = axes.shape[0]
    n_acc = n_rej = ncall = 0
    v = logl = None
    while ncall < walks:                                          # :939
        up = np.zeros(n)
        up[nc:] = stream.uniforms(n - nc)                         # :1011-1013
        dr = randsphere(nc, stream)                               # :1016
        up[:nc] = u[:nc] + scale * np.dot(axes, dr)               # :1020-1021
        if periodic is not None:
            up[periodic] = np.mod(up[periodic], 1)                # :1024-1025
        if reflective is not None:
            up[reflective] = reflect(up[reflective])              # :1028-1029
        if not unitcheck(up, nonbounded):                         # :1032, :951-954
            n_rej += 1
            ncall += 1
            continue
        vp = model.prior_transform(up)                            # :957
        lp = float(model.loglike(vp))                             # :958
        ncall += 1
        if lp > loglstar:                                         # :963-969
            u, v, logl = up, vp, lp
            n_acc += 1
        else:
            n_rej += 1
    if n_acc == 0:                                                # :970-975
        v = model.prior_transform(u)
        logl = float(model.loglike(v))
    return dict(u=u, v=v, logl=logl, ncall=ncall, n_accept=n_acc,
                n_reject=n_rej, ticks=stream.tick)


class _SliceEval:
    def __init__(self, u, direction, model):
        self.u, self.d, self.model, self.nc = u, direction, model, 0

    def __call__(self, x):                                        # :1112-1123
        un = self.u + x * self.d
        self.nc += 1
        if unitcheck(un, None):
            return un, float(self.model.loglike(self.model.prior_transform(un)))
        return un, -np.inf


def _doubling_accept(x1, F, loglstar, L, R, fL, fR):
    """Neal (2003) alg. 6 as in :1038-1072."""
    lhat, rhat, fl, fr, D = L, R, fL, fR, False
    while rhat - lhat > 1.1:
        M = (lhat + rhat) / 2.
        if (0 < M <= x1) or (x1 < M <= 0):
            D = True
        if x1 < M:
            rhat = M
            fr = F(rhat)[1]
        else:
            lhat = M
            fl = F(lhat)[1]
        if D and loglstar >= fl and loglstar >= fr:
            return False
    return True


def slice_step(u, direction, loglstar, model, stream, doubling, stats=None):
    """generic_slice_step (:1075-1206).  Returns
    (u_new, logl_new, nc, n_expand, n_contract, expansion_warning).

    `stats`, if a dict, receives counts of the branches the step took (they change nothing it returns):
    'capped' (1 if the direction was shortened to sqrt(n)/2), 'doublings' (intervals doubled) and
    'doubling_rejects' (proposals inside the slice that _doubling_accept refused)."""
    n = len(u)
    n_expand = n_contract = 0
    rand0 = stream.uniform()                                      # :1099
    dirlen = math.sqrt(float(np.dot(direction, direction)))
    maxlen = math.sqrt(n) / 2.
    direction = direction / (dirlen / maxlen if dirlen > maxlen else 1)  # :1103-1108
    F = _SliceEval(u, direction, model)
    xl, xr = -rand0, 1 - rand0                                    # :1126-1127
    fl, fr = F(xl)[1], F(xr)[1]
    warn = False
    L = R = fL = fR = None
    ndbl = nrej = 0
    if not doubling:
        while fl > loglstar:                                      # :1134-1141
            xl -= 1
            fl = F(xl)[1]
            n_expand += 1
        while fr > loglstar:
            xr += 1
            fr = F(xr)[1]
            n_expand += 1
        warn = n_expand > 1000                                    # :1142
    else:
        K = 1
        while fl > loglstar or fr > loglstar:                     # :1150-1159
            if stream.uniform() < 0.5:
                xl -= (xr - xl)
                fl = F(xl)[1]
            else:
                xr += (xr - xl)
                fr = F(xr)[1]
            n_expand += K
            K *= 2
            ndbl += 1
        L, R, fL, fR = xl, xr, fl, fr
    while True:                                                   # :1168-1203
        xp = xl + stream.uniform() * (xr - xl)
        up, lp = F(xp)
        n_contract += 1
        if lp > loglstar:
            if not doubling or _doubling_accept(xp, F, loglstar, L, R, fL, fR):
                break
            nrej += 1
        if xp < 0:
            xl = xp
        elif xp > 0:
            xr = xp
        else:
            raise RuntimeError("Slice sampler has failed to find a valid point.")
    if stats is not None:
        stats.update(capped=int(dirlen > maxlen), doublings=ndbl, doubling_rejects=nrej)
    return up, lp, F.nc, n_expand, n_contract, warn


def _stats_init():
    """Per-chain branch counters of rslice_chain / slice_chain (see slice_step): doublings per step, steps with a
    capped direction, _doubling_accept rejections, and the slice / step index at which the expansion warning fired."""
    return dict(doublings=[], n_capped=0, n_doubling_rejects=0, warn_slice=None, warn_step=None)


def _stats_add(st, s, sl, step, w, doubling):
    st['doublings'].append(s['doublings'])
    st['n_capped'] += s['capped']
    st['n_doubling_rejects'] += s['doubling_rejects']
    if w and not doubling:
        st['warn_slice'], st['warn_step'] = sl, step


def rslice_chain(u0, loglstar, axes, scale, model, stream, slices,
                 doubling=False):
    """RSliceSampler.sample (:745-855).  The returned dict also carries the branch counters of _stats_init."""
    u = np.array(u0, dtype=float)
    n = u.shape[0]
    nc = nexp = ncon = 0
    warned = False
    logl = None
    st = _stats_init()
    for sl in range(slices):
        z = stream.normals(n)                                     # :820-821
        z = z / math.sqrt(float(np.dot(z, z)))
        direction = np.dot(axes, z) * scale                       # :824
        s = {}
        u, logl, c, e, k, w = slice_step(u, direction, loglstar, model, stream,
                                         doubling, s)
        nc, nexp, ncon = nc + c, nexp + e, ncon + k
        _stats_add(st, s, sl, sl, w, doubling)
        if w and not doubling:                                    # :836-838
            doubling = warned = True
    return dict(u=u, v=model.prior_transform(u), logl=logl, ncall=nc,
                n_expand=nexp, n_contract=ncon, expansion_warning_set=warned,
                ticks=stream.tick, **st)


def slice_chain(u0, loglstar, axes, scale, model, stream, slices,
                doubling=False):
    """SliceSampler.sample (:593-709): principal-axis Gibbs-like slices.  The returned dict also carries the branch
    counters of _stats_init (steps are counted over all slices: slice sl, axis j is step sl * n + j)."""
    u = np.array(u0, dtype=float)
    n = u.shape[0]
    ax = scale * axes.T                                           # :665
    nc = nexp = ncon = 0
    warned = False
    logl = None
    st = _stats_init()
    for sl in range(slices):
        for j, i in enumerate(stream.permutation(n)):             # :673-677
            s = {}
            u, logl, c, e, k, w = slice_step(u, ax[i], loglstar, model, stream,
                                             doubling, s)
            nc, nexp, ncon = nc + c, nexp + e, ncon + k
            _stats_add(st, s, sl, sl * n + j, w, doubling)
            if w and not doubling:
                doubling = warned = True
    return dict(u=u, v=model.prior_transform(u), logl=logl, ncall=nc,
                n_expand=nexp, n_contract=ncon, expansion_warning_set=warned,
                ticks=stream.tick, **st)


def unitcube_chain(loglstar, model, stream, ndim, max_tries=10**7):
    """UnitCubeSampler.sample (internal_samplers.py:420-441): u = rstate.uniform(size=ndim) until
    loglikelihood(prior_transform(u)) > loglstar; one uniform vector event per draw."""
    for nc in range(1, max_tries + 1):
        u = stream.uniforms(ndim)
        v = model.prior_transform(u)
        logl = float(model.loglike(v))
        if logl > loglstar:
            return dict(u=u, v=v, logl=logl, ncall=nc, ticks=stream.tick)
    raise RuntimeError("unitcube_chain: no point found")


def unif_chain(loglstar, multi, model, stream, ndim, nonbounded=None,
               max_tries=10**7):
    """UniformBoundSampler.sample (:243-340) with a MultiEll/Ell-like bound
    (bounding.py:525-590 for the draw).  `multi` is oracle.bounding.MultiEll."""
    nc = multi.ells[0].ndim
    K = multi.nells
    probs = np.exp(multi.logvol_ells - multi.logvol)
    cum = np.cumsum(probs)
    ncall = nprop = 0
    nb = None if nonbounded is None else nonbounded[:nc]
    for _ in range(max_tries):
        if K == 1:                                                # bounding.py:543-550
            x = multi.ells[0].ctr + np.dot(multi.ells[0].axes, randsphere(nc, stream))
        else:
            while True:                                           # bounding.py:553-590
                idx = min(int(np.searchsorted(cum, stream.uniform())), K - 1)
                x = multi.ells[idx].ctr + np.dot(multi.ells[idx].axes,
                                                 randsphere(nc, stream))
                q = int((multi.mahal2(x)[0] < 1).sum())
                if q == 0:
                    q = int((multi.mahal2(x)[0] <= 1 + 1e-3).sum())
                    if q == 0:
                        raise RuntimeError('Ellipsoid check failed q=0')
                if q == 1 or stream.uniform() < 1. / q:
                    break
        nprop += 1                                                # points the bound proposed
        if not unitcheck(x, nb):                                  # :314
            continue
        u = x if nc == ndim else np.concatenate((x, stream.uniforms(ndim - nc)))
        v = model.prior_transform(u)
        logl = float(model.loglike(v))
        ncall += 1
        if logl > loglstar:
            return dict(u=u, v=v, logl=logl, ncall=ncall, nprop=nprop, ticks=stream.tick)
    raise RuntimeError("unif_chain: no point found")

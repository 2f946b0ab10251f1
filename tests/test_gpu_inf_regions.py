"""GPU: likelihoods that are -inf on part of the prior.

Three things are checked, on the registry's diamond (the reference's tests/test_sampling.py region) and on two user
CUDA models with a numpy twin here: EDGES, a Gaussian truncated to -inf outside r0 = 5 in a box whose finite part is
volfrac = 1e-3 of the prior (the reference's tests/test_plateau.py EdgesInf, ln Z = 0), and HOLE, a Gaussian in a
+-10 box that is -inf outside r = 10 and in the strip |x0| < 0.1 (tests/test_misc.py loglike_inf).
  1. The init kernel (b2n_unitcube_batch at threshold -inf, which redraws every -inf draw) against the oracle on the
     same Philox streams: call counts exact, u / v / logl to rtol 1e-9; and the total draw count against f.
  2. The chain kernels with start points a few step lengths from a -inf edge, at loglstar = LOWL and at a finite
     threshold, against the oracle: the chain-kernel matrix's standard (counts exact, u / v / logl to rtol 1e-9).
  3. The evidence of whole runs -- static (host loop and device rounds), dynamic and a replica ensemble -- against
     the closed form or the quadrature, within 4 sigma of sqrt(logzerr^2 + (1 - f) / nlive); the second term is the
     variance of ln f-hat from the init draws.  Without the initial volume ln f-hat the diamond and EDGES runs are
     high by about -ln f (1.54 and 6.9)."""
import math

import numpy as np
import pytest
from scipy import integrate, special

from dynesty_b200 import dynamic as D, likelihoods as DL, nested, ops, replicas
from dynesty_b200.likelihoods import DeviceModel
from helpers import close
from oracle import bounding as OB, likelihoods as OL, philox, samplers as OS

pytestmark = pytest.mark.gpu

SEED = 56432
RTOL = 1e-9
LOWL = nested.LOWL

EDGES = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    double s = 0.0;
    for (int i = lane; i < n; i += 32) s = fma(v[i], v[i], s);
    s = b2n_warp_sum(s);
    return s > p[0] ? -INFINITY : -0.5 * s - p[1];
}
'''

HOLE = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    double s = 0.0;
    for (int i = lane; i < n; i += 32) s = fma(v[i], v[i], s);
    s = b2n_warp_sum(s);
    return (s > p[0] || fabs(v[0]) < p[1]) ? -INFINITY : -0.5 * s;
}
'''


class _Twin:
    """numpy twin of a user model with the registry's uniform prior v = lo + width * u."""

    def __init__(self, ndim, half, loglike, f, logz):
        self.ndim, self.half, self._loglike, self.f, self.logz = ndim, half, loglike, f, logz

    def prior_transform(self, u):
        return -self.half + 2. * self.half * np.asarray(u, dtype=float)

    def loglike(self, v):
        return self._loglike(np.asarray(v, dtype=float))


def edges(ndim, volfrac=1e-3, r0=5.0):
    """(DeviceModel, twin): the Gaussian of unit width truncated at r0, in a box of half-width `half` chosen so that
    the ball is `volfrac` of the box; normalised to Z = 1."""
    half = 0.5 * r0 * (math.pi ** (ndim / 2.) / (special.gamma(ndim / 2. + 1) * volfrac)) ** (1. / ndim)
    lnorm = 0.5 * ndim * math.log(math.pi / 2) - ndim * math.log(half) + math.log(special.gammainc(ndim / 2., 0.5 * r0 ** 2))

    def loglike(v):
        s = np.sum(v * v, axis=-1)
        return np.where(s > r0 * r0, -np.inf, -0.5 * s - lnorm)
    dm = DeviceModel.from_cuda(ndim, EDGES, params=np.array([r0 * r0, lnorm]), prior_kind=OL.PRIOR_UNIFORM,
                               prior_p0=np.full(ndim, -half), prior_p1=np.full(ndim, 2. * half), name='edges%d' % ndim)
    return dm, _Twin(ndim, half, loglike, volfrac, 0.0)


def hole():
    """(DeviceModel, twin): exp(-r^2 / 2) in the box +-10, -inf for r > 10 or |x0| < 0.1.
    ln Z = ln(2 pi erfc(0.1 / sqrt 2) / 400) (the mass beyond r = 10 is e^-50); f by quadrature."""
    def loglike(v):
        s = np.sum(v * v, axis=-1)
        return np.where((s > 100.) | (np.abs(v[..., 0]) < 0.1), -np.inf, -0.5 * s)
    strip = integrate.quad(lambda x: 2. * math.sqrt(100. - x * x), -0.1, 0.1)[0]
    f = (100. * math.pi - strip) / 400.
    logz = math.log(2. * math.pi * math.erfc(0.1 / math.sqrt(2.)) / 400.)
    dm = DeviceModel.from_cuda(2, HOLE, params=np.array([100., 0.1]), prior_kind=OL.PRIOR_UNIFORM,
                               prior_p0=np.full(2, -10.), prior_p1=np.full(2, 20.), name='hole')
    return dm, _Twin(2, 10., loglike, f, logz)


def diamond(ndim=2):
    """(DeviceModel, oracle model): the registry diamond on the first two coordinates; ln Z by quadrature."""
    def inner(x):
        y0 = math.sqrt(max(0.25 - x * x, 0.0))
        return integrate.quad(lambda y: math.exp(x * x + y * y - 0.25), y0, 0.5, epsabs=1e-14, epsrel=1e-13)[0]
    om = OL.region2d('diamond', ndim)
    om.f = 1. - math.pi / 4
    om.logz = math.log(4 * integrate.quad(inner, 0.0, 0.5, epsabs=1e-14, epsrel=1e-13, limit=200)[0])
    return DL.region2d('diamond', ndim), om


_CACHE = {}


def model(name):
    if name not in _CACHE:
        _CACHE[name] = {'diamond': diamond, 'diamond16': lambda: diamond(16), 'edges2': lambda: edges(2),
                        'edges5': lambda: edges(5), 'hole': hole}[name]()
    return _CACHE[name]


def test_truths():
    assert abs(model('diamond')[1].logz - (-1.4682353)) < 1e-6
    assert abs(model('hole')[1].logz - (-4.2365949)) < 1e-6
    # the EDGES normalisation: Z = 1 by quadrature over the ball, in 2-D
    dm, tw = model('edges2')
    z = integrate.quad(lambda r: 2 * math.pi * r * math.exp(float(tw.loglike(np.array([r, 0.])))), 0, 5)[0]
    assert abs(z / (2 * tw.half) ** 2 - 1.) < 1e-10


# ---- 1. the init kernel ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name,Q,check', [('diamond', 517, None), ('edges2', 300, 24), ('hole', 300, None)])
def test_init_kernel_matches_oracle(name, Q, check):
    """b2n_unitcube_batch at threshold -inf, slot q on the stream ChainStream(seed, chain0 + q), against
    oracle.samplers.unitcube_chain.  All slots, or (EDGES, ~10^3 draws a slot) the first, the last and a random
    sample.  The draws of all slots are negative-binomial with success probability f: their total is checked
    against Q / f within 5 sigma."""
    dm, om = model(name)
    chain0 = (1 << 61) + 5
    o = ops.unitcube_batch(dm.model_id(), Q, om.ndim, -np.inf, SEED, chain0=chain0)
    assert np.all(np.isfinite(o['logl'])) and np.all(o['ncall'] >= 1)
    rng = np.random.default_rng(Q)
    slots = range(Q) if check is None else sorted({0, Q - 1} | set(rng.choice(Q, size=check, replace=False).tolist()))
    for q in slots:
        r = OS.unitcube_chain(-np.inf, om, philox.ChainStream(SEED, chain0 + q), om.ndim)
        assert o['ncall'][q] == r['ncall'], q
        close(o['u'][q], r['u'], rtol=RTOL)
        close(o['v'][q], r['v'], rtol=RTOL)
        assert o['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL)
    d = float(o['ncall'].sum())
    sd = math.sqrt(Q * (1. - om.f)) / om.f
    assert abs(d - Q / om.f) < 5 * sd, (d, Q / om.f, sd)


# ---- 2. chain kernels next to a -inf edge ---------------------------------------------------------------------------
def _diamond_starts(n, Q, rng, dmin, dmax):
    """Points at distance dmin..dmax from a random corner of the unit square (the -inf quarter discs have radius
    1/2), free coordinates uniform in [0.2, 0.8]."""
    corner = rng.integers(2, size=(Q, 2)).astype(float)
    phi = rng.uniform(0.5, math.pi / 2 - 0.5, Q)          # (away from the two neighbouring discs)
    r = rng.uniform(dmin, dmax, Q)
    sgn = 1. - 2. * corner
    u = np.empty((Q, n))
    u[:, 0] = corner[:, 0] + sgn[:, 0] * r * np.cos(phi)
    u[:, 1] = corner[:, 1] + sgn[:, 1] * r * np.sin(phi)
    u[:, 2:] = rng.uniform(0.2, 0.8, (Q, n - 2))
    return u


def _edges_starts(tw, Q, rng, rmin, rmax):
    """Points at radius rmin..rmax (in v) of EDGES, in unit-cube coordinates."""
    z = rng.standard_normal((Q, tw.ndim))
    v = z / np.linalg.norm(z, axis=1)[:, None] * rng.uniform(rmin, rmax, (Q, 1))
    return (v + tw.half) / (2. * tw.half)


# (case, model, threshold, start radii, step length in u): the diamond's edge is at distance 0.5 from a corner and
# its logl there is 0, so logl > 0.01 needs distance > 0.51; EDGES is -inf beyond r = 5 (u step 0.005 = 1.4 in v)
EDGE_CASES = {
    'diamond-lowl': ('diamond', LOWL, (0.5, 0.56), 0.04),
    'diamond-finite': ('diamond', 0.01, (0.515, 0.57), 0.04),
    'diamond16-lowl': ('diamond16', LOWL, (0.5, 0.56), 0.04),
    'diamond16-finite': ('diamond16', 0.01, (0.515, 0.57), 0.04),
    'edges2-lowl': ('edges2', LOWL, (4.0, 5.0), 0.005),
    'edges2-finite': ('edges2', None, (4.0, 4.6), 0.005),
}


def _edge_queue(case, Q, seed):
    name, loglstar, (a, b), step = EDGE_CASES[case]
    dm, om = model(name)
    rng = np.random.default_rng(seed)
    if name.startswith('diamond'):
        u0 = _diamond_starts(om.ndim, Q, rng, a, b)
    else:
        u0 = _edges_starts(om, Q, rng, a, b)
        if loglstar is None:               # the threshold is the contour r = 4.7, between the starts and the edge
            loglstar = float(om.loglike(np.array([4.7] + [0.] * (om.ndim - 1))))
    l0 = om.loglike(om.prior_transform(u0))
    assert np.all(l0 > loglstar)
    axes = step * np.eye(om.ndim)[None]
    return dm, om, u0, float(loglstar), axes


def _compare(o, r, q):
    close(o['u'][q], r['u'], rtol=RTOL)
    close(o['v'][q], r['v'], rtol=RTOL)
    assert o['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL)


def _picks(Q, rng, extra):
    return sorted({0, Q - 1} | set(rng.choice(Q, size=extra, replace=False).tolist()))


RW_CASES = ['diamond-lowl', 'diamond-finite', 'diamond16-lowl', 'diamond16-finite', 'edges2-lowl', 'edges2-finite']


@pytest.mark.parametrize('case', RW_CASES)
def test_rwalk_next_to_inf_edge(case):
    """rwalk: the warp-per-chain kernel at n = 2 (diamond, user EDGES) and the lock-step kernel at n = 16 with 14 free
    dimensions (the diamond of the uniformity test).  Many proposals land where logl is -inf."""
    Q, walks, scale, chain0 = 2 * 132 + 5, 25, 1.0, 900
    dm, om, u0, loglstar, axes = _edge_queue(case, Q, 11)
    ops.bound_set(axes)
    ell = np.zeros(Q, dtype=np.int32)
    o = ops.rwalk_batch(dm.model_id(), u0, loglstar, scale, walks, SEED, chain0=chain0, ell=ell)
    assert np.all(o['logl'] > loglstar) and np.all(np.isfinite(o['logl']))
    assert (o['n_accept'] > 0).mean() > 0.3 and (o['n_reject'] > 0).mean() > 0.3
    rng = np.random.default_rng(1)
    for q in _picks(Q, rng, 24):
        r = OS.rwalk_chain(u0[q], loglstar, axes[0], scale, om, philox.ChainStream(SEED, chain0 + q), walks)
        assert (o['n_accept'][q], o['n_reject'][q], o['ncall'][q]) == (r['n_accept'], r['n_reject'], r['ncall']), q
        _compare(o, r, q)


SL_CASES = [(c, s, d) for c in ('diamond-lowl', 'diamond-finite', 'edges2-lowl', 'edges2-finite')
            for s in ('rslice', 'slice') for d in (False, True)]


@pytest.mark.parametrize('case,sampler,doubling', SL_CASES,
                         ids=['%s-%s-%s' % (c, s, 'dbl' if d else 'std') for c, s, d in SL_CASES])
def test_slice_next_to_inf_edge(case, sampler, doubling):
    """rslice / slice, stepping out and doubling: the interval ends and the shrinking proposals fall where logl is
    -inf (F(x) = -inf inside the cube, doubling_accept with -inf ends)."""
    Q, slices, chain0 = 132 + 5, 3, 1700
    dm, om, u0, loglstar, axes = _edge_queue(case, Q, 12)
    scale = 6.0 if doubling else 3.0
    fn, chain = (ops.rslice_batch, OS.rslice_chain) if sampler == 'rslice' else (ops.slice_batch, OS.slice_chain)
    ops.bound_set(axes)
    ell = np.zeros(Q, dtype=np.int32)
    o = fn(dm.model_id(), u0, loglstar, scale, slices, SEED, chain0=chain0, doubling=doubling, ell=ell)
    assert np.all(o['logl'] > loglstar) and np.all(np.isfinite(o['logl']))
    rng = np.random.default_rng(2)
    for q in _picks(Q, rng, 16):
        r = chain(u0[q], loglstar, axes[0], scale, om, philox.ChainStream(SEED, chain0 + q), slices,
                  doubling=doubling)
        assert (o['ncall'][q], o['n_expand'][q], o['n_contract'][q]) == (r['ncall'], r['n_expand'], r['n_contract']), q
        _compare(o, r, q)


@pytest.mark.parametrize('name,loglstar', [('diamond', LOWL), ('diamond', 0.01), ('hole', LOWL), ('hole', -2.0)])
def test_unif_over_inf_region(name, loglstar):
    """Uniform draws from an ellipsoid that covers the -inf region too: every draw there is rejected."""
    dm, om = model(name)
    n = om.ndim
    ell = OB.bounding_ellipsoid(np.random.default_rng(3).random((400, n)) * 0.9 + 0.05)
    me = OB.MultiEll([ell])
    ops.bound_set(me.axes, me.ctrs, me.ams, me.logvol_ells)
    Q, chain0 = 4 * 32 + 3, 2500
    o = ops.unif_batch(dm.model_id(), Q, n, loglstar, SEED, chain0=chain0)
    assert np.all(o['logl'] > loglstar) and np.all(np.isfinite(o['logl']))
    assert (o['ncall'] > 1).sum() > 10                   # draws were rejected
    for q in range(Q):
        r = OS.unif_chain(loglstar, me, om, philox.ChainStream(SEED, chain0 + q), n)
        assert (o['ncall'][q], o['nprop'][q]) == (r['ncall'], r['nprop']), q
        _compare(o, r, q)


# ---- 3. evidence against the truth ----------------------------------------------------------------------------------
def _tol(logzerr, f, nlive):
    return 4. * math.sqrt(logzerr ** 2 + (1. - f) / nlive)


RUNS = [(m, s, lp) for m in ('diamond', 'edges2', 'edges5', 'hole') for s in ('unif', 'rwalk', 'rslice')
        for lp in ('host', 'device')]


@pytest.mark.parametrize('name,sample,loop', RUNS, ids=['%s-%s-%s' % r for r in RUNS])
def test_static_evidence(name, sample, loop):
    nlive = 200
    dm, om = model(name)
    s = nested.NestedSampler(dm, nlive=nlive, bound='multi', sample=sample, seed=SEED + 1)
    res = s.run_nested(dlogz=0.05, loop=loop)
    err = res.logz[-1] - om.logz
    assert abs(err) < _tol(res.logzerr[-1], om.f, nlive), (res.logz[-1], om.logz, res.logzerr[-1])
    assert np.isfinite(res.logzerr[-1]) and np.isfinite(res.information[-1])
    assert res.logvol[0] == pytest.approx(s.logvol_init - math.log((nlive + 1.) / nlive), rel=1e-12)
    assert abs(s.logvol_init - math.log(om.f)) < 5 * math.sqrt((1. - om.f) / nlive)


def test_dynamic_evidence_edges():
    dm, om = model('edges2')
    d = D.DynamicNestedSampler(dm, nlive=200, bound='multi', sample='rwalk', seed=SEED + 2)
    res = d.run_nested(nlive_init=200, nlive_batch=100, maxbatch=2, n_effective=1e9, dlogz_init=0.05)
    assert d.batch == 2 and d.logvol_init == d.base_sampler.logvol_init < -5.0
    assert res.logvol[0] == d.logvol_init - math.log(201. / 200.)
    assert np.isfinite(res.logzerr[-1]) and np.isfinite(res.information[-1])
    assert abs(res.logz[-1] - om.logz) < _tol(res.logzerr[-1], om.f, 200), (res.logz[-1], res.logzerr[-1])


def test_replicas_evidence_edges_unbiased():
    """16 replicas of EDGES in 2-D: the mean ln Z is within 4 sigma / sqrt(16) of 0, sigma the per-run error."""
    dm, om = model('edges2')
    nlive = 100
    outs, _ = replicas.run_replicas(dm, list(range(100, 116)), nlive=nlive, bound='multi', sample='rwalk',
                                    max_in_flight=8, dlogz=0.05)
    lz = np.array([o['logz'] for o in outs])
    sig = math.sqrt(np.mean([o['logzerr'] ** 2 for o in outs]) + (1. - om.f) / nlive)
    assert np.all(np.isfinite([o['logzerr'] for o in outs]))
    assert abs(lz.mean() - om.logz) < 4 * sig / 4., (lz.mean(), lz.std(), sig)

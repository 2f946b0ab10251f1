"""GPU: user likelihoods (DeviceModel.from_cuda, B2N_LIKE_USER) run the same chain kernels as the registry.

Three registry formulas are restated as user CUDA code -- GAUSS_DIAG and SHELLS in the registry's operation order,
GAUSS_PREC with the precision matrix in the parameter array -- and every kernel slot of a user model is checked
against the registry model (forced onto the warp-per-chain rwalk kernel, B2N_RWALK_IMPL=warp) AND against the
float64 oracle on the same Philox streams: integer counts exact, u / v / logl to rtol 1e-9.  Whether a user output
is also bit-identical to the registry's is printed (``USER-BITWISE``), not required: NVRTC's libdevice need not be
nvcc's.  Then device-resident runs, a likelihood the registry does not have (a two-component mixture with an
analytic evidence), checkpoint / resume, replicas on a context pool and the error for the lock-step kernels."""
import math

import numpy as np
import pytest

from dynesty_b200 import _lib, nested, ops, replicas
from dynesty_b200.likelihoods import DeviceModel
from helpers import device_model
from oracle import bounding as OB, likelihoods as OL, philox, samplers as OS

pytestmark = pytest.mark.gpu

SEED = 56432
RTOL = 1e-9

DIAG = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    double s = 0.0;
    for (int i = lane; i < n; i += 32) {
        const double d = v[i] - p[i];
        s = fma(p[n + i] * d, d, s);
    }
    s = b2n_warp_sum(s);
    return fma(-0.5, s, p[2 * n]);
}
'''

SHELLS = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    double a = 0.0, b = 0.0;
    for (int i = lane; i < n; i += 32) {
        const double d1 = v[i] - p[i], d2 = v[i] - p[n + i];
        a = fma(d1, d1, a);
        b = fma(d2, d2, b);
    }
    a = sqrt(b2n_warp_sum(a));
    b = sqrt(b2n_warp_sum(b));
    const double r = p[2 * n], w = p[2 * n + 1];
    const double cst = log(1.0 / sqrt(2.0 * 3.14159265358979323846 * w * w));
    const double l1 = cst - (a - r) * (a - r) / (2.0 * w * w);
    const double l2 = cst - (b - r) * (b - r) / (2.0 * w * w);
    const double hi = fmax(l1, l2), lo = fmin(l1, l2);
    return hi + log1p(exp(lo - hi));
}
'''

# the precision matrix (column-major, n x n) follows the mean in p; the lane owns rows lane, lane + 32, ...
PREC = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    for (int i = lane; i < n; i += 32) work[i] = v[i] - p[i];
    __syncwarp();
    const double* P = p + n;
    double s = 0.0;
    for (int i = lane; i < n; i += 32) {
        double y = 0.0;
        for (int j = 0; j < n; j++) y = fma(P[(size_t)j * n + i], work[j], y);
        s = fma(work[i], y, s);
    }
    s = b2n_warp_sum(s);
    __syncwarp();
    return fma(-0.5, s, p[n + n * n]);
}
'''

# not in the registry: w1 N(m1, s1^2 I) + w2 N(m2, s2^2 I); the sums run over the lanes, the scalar tail on lane 0
MIXTURE = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    double q1 = 0.0, q2 = 0.0;
    for (int i = lane; i < n; i += 32) {
        const double d1 = v[i] - p[i], d2 = v[i] - p[n + i];
        q1 = fma(d1, d1, q1);
        q2 = fma(d2, d2, q2);
    }
    q1 = b2n_warp_sum(q1);
    q2 = b2n_warp_sum(q2);
    double l = 0.0;
    if (lane == 0) {
        const double s1 = p[2 * n], s2 = p[2 * n + 1], c = 0.5 * n * log(2.0 * 3.14159265358979323846);
        const double l1 = p[2 * n + 2] - 0.5 * q1 / (s1 * s1) - n * log(s1) - c;
        const double l2 = p[2 * n + 3] - 0.5 * q2 / (s2 * s2) - n * log(s2) - c;
        const double hi = fmax(l1, l2), lo = fmin(l1, l2);
        l = hi + log1p(exp(lo - hi));
    }
    return __shfl_sync(0xffffffffu, l, 0);
}
'''


def _prior_kw(m):
    p = m.p
    if m.prior_kind == OL.PRIOR_UNIFORM:
        return dict(prior_kind=m.prior_kind, prior_p0=p['lo'], prior_p1=p['width'])
    if m.prior_kind == OL.PRIOR_NORMAL_PPF:
        return dict(prior_kind=m.prior_kind, prior_p0=p['mu'], prior_p1=p['sigma'])
    return dict(prior_kind=m.prior_kind)


def _user_restatement(kind, m):
    p, n = m.p, m.ndim
    if kind == 'diag':
        src, prm = DIAG, np.concatenate([p['mean'] * np.ones(n), p['ivar'] * np.ones(n), [p['lnorm']]])
    elif kind == 'shell':
        src, prm = SHELLS, np.concatenate([p['c1'], p['c2'], [p['r'], p['w']]])
    else:
        src, prm = PREC, np.concatenate([p['mean'] * np.ones(n), np.asarray(p['prec']).T.ravel(), [p['lnorm']]])
    return DeviceModel.from_cuda(n, src, params=prm, name='user_' + kind, **_prior_kw(m))


_MODELS = {}


def _models(kind, n):
    """(oracle model, registry DeviceModel, user DeviceModel) -- the device models cached per test session."""
    if (kind, n) not in _MODELS:
        om = {'diag': lambda: OL.iid_normal_ppf(n), 'shell': lambda: OL.shells(n),
              'prec': lambda: OL.gauss_corr(n, 0.4, 5.)}[kind]()
        _MODELS[kind, n] = (om, device_model(om), _user_restatement(kind, om))
    return _MODELS[kind, n]


def close(a, b, rtol=RTOL):
    np.testing.assert_allclose(a, b, rtol=rtol, atol=rtol * max(np.abs(np.asarray(b)).max(), 1e-300))


def _same(case, ou, orr, ints):
    """user outputs == registry outputs: counts exact, floats to RTOL; report bit identity."""
    for k in ints:
        assert np.array_equal(ou[k], orr[k]), (case, k)
    for k in ('u', 'v', 'logl'):
        close(ou[k], orr[k])
    bit = all(np.array_equal(ou[k], orr[k]) for k in ('u', 'v', 'logl'))
    print('USER-BITWISE %s %s' % (case, bit))


def _cloud(kind, n, npts, rng):
    u = 0.5 + 0.03 * rng.standard_normal((npts, n))
    if kind == 'shell':     # on the first shell (centre -3.5, radius 2, prior U(-6, 6))
        u[:, 0] += (-1.5 / 12.0)
    return u


def _queue(kind, om, Q, rng, K=2):
    n = om.ndim
    pts = _cloud(kind, n, max(2000, 8 * K * n), rng)
    logl = om.loglike(om.prior_transform(pts))
    loglstar = float(np.quantile(logl, 0.3))
    good = pts[logl > loglstar]
    ells = [OB.bounding_ellipsoid(good[i::K]) for i in range(K)]
    u0 = np.ascontiguousarray(good[rng.integers(len(good), size=Q)])
    ell = rng.integers(K, size=Q).astype(np.int32)
    return u0, loglstar, ells, ell


def _oracle_rows(Q, rng, extra):
    return sorted({0, Q - 1} | {int(i) for i in rng.choice(Q, size=min(extra, Q), replace=False)})


KINDS = ['diag', 'shell', 'prec']


# ---- model evaluation ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('n', [10, 65])
def test_model_eval_restatement(kind, n):
    om, dm, um = _models(kind, n)
    rng = np.random.default_rng(n)
    u = _cloud(kind, n, 500, rng)
    vu, lu = um.evaluate(u)
    vr, lr = dm.evaluate(u)
    assert np.array_equal(vu, vr)                  # the prior is the registry's own code
    close(lu, lr)
    close(lu, om.loglike(om.prior_transform(u)))
    print('USER-BITWISE model_eval-%s%d %s' % (kind, n, np.array_equal(lu, lr)))


# ---- rwalk: axes in shared memory (n = 10) and in global memory (n = 200) ------------------------------------------
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('n', [10, 200])
def test_rwalk_restatement(monkeypatch, kind, n):
    om, dm, um = _models(kind, n)
    rng = np.random.default_rng(100 + n)
    Q = 301 if n == 10 else 40                     # n = 10: several chains per CTA
    u0, loglstar, ells, ell = _queue(kind, om, Q, rng)
    axes = np.array([e.axes for e in ells])
    ops.bound_set(axes)
    walks, scale, chain0 = 25, 0.6, 70 + n
    monkeypatch.setenv('B2N_RWALK_IMPL', 'warp')
    orr = ops.rwalk_batch(dm.model_id(), u0, loglstar, scale, walks, SEED, chain0=chain0, ell=ell)
    monkeypatch.delenv('B2N_RWALK_IMPL')
    ou = ops.rwalk_batch(um.model_id(), u0, loglstar, scale, walks, SEED, chain0=chain0, ell=ell)
    _same('rwalk-%s%d' % (kind, n), ou, orr, ('n_accept', 'n_reject', 'ncall'))
    assert ou['n_accept'].sum() > 0
    for q in _oracle_rows(Q, rng, 6 if n == 10 else 2):
        r = OS.rwalk_chain(u0[q], loglstar, axes[ell[q]], scale, om, philox.ChainStream(SEED, chain0 + q), walks)
        assert (ou['n_accept'][q], ou['n_reject'][q]) == (r['n_accept'], r['n_reject']), q
        close(ou['u'][q], r['u'])
        close(ou['v'][q], r['v'])
        assert ou['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL)


# ---- slice / rslice: all four RANDOM_DIR x AX_SMEM slots ----------------------------------------------------------
@pytest.mark.parametrize('sampler', ['slice', 'rslice'])
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('n', [10, 200])
def test_slice_restatement(sampler, kind, n):
    om, dm, um = _models(kind, n)
    rng = np.random.default_rng(200 + n)
    Q = 140 if n == 10 else 24
    u0, loglstar, ells, ell = _queue(kind, om, Q, rng)
    axes = np.array([e.axes for e in ells])
    ops.bound_set(axes)
    slices = 3 if sampler == 'rslice' else 1
    fn, chain = (ops.rslice_batch, OS.rslice_chain) if sampler == 'rslice' else (ops.slice_batch, OS.slice_chain)
    chain0 = 300 + n
    orr = fn(dm.model_id(), u0, loglstar, 1.0, slices, SEED, chain0=chain0, ell=ell)
    ou = fn(um.model_id(), u0, loglstar, 1.0, slices, SEED, chain0=chain0, ell=ell)
    _same('%s-%s%d' % (sampler, kind, n), ou, orr, ('n_expand', 'n_contract', 'ncall', 'flags'))
    assert np.all(ou['flags'] == 0) and np.all(ou['logl'] > loglstar)
    for q in _oracle_rows(Q, rng, 4 if n == 10 else 1):
        r = chain(u0[q], loglstar, axes[ell[q]], 1.0, om, philox.ChainStream(SEED, chain0 + q), slices)
        assert (ou['ncall'][q], ou['n_expand'][q], ou['n_contract'][q]) == (r['ncall'], r['n_expand'],
                                                                            r['n_contract']), q
        close(ou['u'][q], r['u'])
        close(ou['v'][q], r['v'])
        assert ou['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL)


# ---- unif / unitcube / friends-unif --------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', KINDS)
def test_unif_and_unitcube_restatement(kind):
    n = 10
    om, dm, um = _models(kind, n)
    rng = np.random.default_rng(7)
    u0, loglstar, ells, ell = _queue(kind, om, 8, rng)
    me = OB.MultiEll(ells)
    ops.bound_set(me.axes, me.ctrs, me.ams, me.logvol_ells)
    Q, chain0 = 4 * 32 + 3, 11
    orr = ops.unif_batch(dm.model_id(), Q, n, loglstar, SEED, chain0=chain0)
    ou = ops.unif_batch(um.model_id(), Q, n, loglstar, SEED, chain0=chain0)
    _same('unif-%s' % kind, ou, orr, ('ncall', 'nprop', 'flags'))
    for q in _oracle_rows(Q, rng, 8):
        r = OS.unif_chain(loglstar, me, om, philox.ChainStream(SEED, chain0 + q), n)
        assert (ou['ncall'][q], ou['nprop'][q]) == (r['ncall'], r['nprop']), q
        close(ou['u'][q], r['u'])
        assert ou['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL)
    # unit cube: a threshold low enough for prior draws to pass now and then
    thr = float(np.quantile(om.loglike(om.prior_transform(rng.random((4000, n)))), 0.9))
    orr = ops.unitcube_batch(dm.model_id(), Q, n, thr, SEED, chain0=chain0)
    ou = ops.unitcube_batch(um.model_id(), Q, n, thr, SEED, chain0=chain0)
    _same('unitcube-%s' % kind, ou, orr, ('ncall',))
    for q in _oracle_rows(Q, rng, 8):
        r = OS.unitcube_chain(thr, om, philox.ChainStream(SEED, chain0 + q), n)
        assert ou['ncall'][q] == r['ncall']
        close(ou['u'][q], r['u'])
        assert ou['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL)


@pytest.mark.parametrize('kind', KINDS)
def test_friends_unif_restatement(kind):
    """friends_unif_kernel: user == registry on the same resident RadFriends bound, and every returned point is the
    model (numpy) at its u."""
    n = 6
    om, dm, um = _models(kind, n)
    rng = np.random.default_rng(8)
    pts = _cloud(kind, n, 300, rng)
    f = ops.friends_update(pts, 'balls', use_clustering=False)
    ops.friends_set('balls', pts, f['axes'], f['axes_inv'])
    loglstar = float(np.quantile(om.loglike(om.prior_transform(pts)), 0.3))
    Q, chain0 = 97, 5
    orr = ops.friends_unif_batch(dm.model_id(), Q, n, loglstar, SEED, chain0=chain0)
    ou = ops.friends_unif_batch(um.model_id(), Q, n, loglstar, SEED, chain0=chain0)
    _same('friends-unif-%s' % kind, ou, orr, ('ncall', 'nprop', 'flags'))
    assert np.all(ou['logl'] > loglstar)
    close(ou['logl'], om.loglike(om.prior_transform(ou['u'])))


# ---- device-resident rounds ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('sample,kw', [('rwalk', dict(walks=20)), ('rslice', dict(slices=4))])
def test_device_rounds_restatement(monkeypatch, sample, kw):
    om, dm, um = _models('diag', 6)
    run = lambda m: nested.NestedSampler(m, nlive=300, bound='multi', sample=sample, seed=21, **kw).run_nested(
        loop='device', batch=10, dlogz=0.5)
    monkeypatch.setenv('B2N_RWALK_IMPL', 'warp')
    ref = run(dm)
    monkeypatch.delenv('B2N_RWALK_IMPL')
    res = run(um)
    assert (res.niter, res.ncall) == (ref.niter, ref.ncall)
    close(res.logl, ref.logl)
    assert res.logz[-1] == pytest.approx(ref.logz[-1], rel=RTOL, abs=RTOL)
    print('USER-BITWISE rounds-%s %s' % (sample, np.array_equal(res.logl, ref.logl)))


# ---- a likelihood the registry does not have ----------------------------------------------------------------------
class _NumpyMixture:
    def __init__(self, n, m1, m2, s1, s2, w1, lo, width):
        self.ndim, self.m1, self.m2, self.s1, self.s2, self.w1 = n, m1, m2, s1, s2, w1
        self.lo, self.width = lo, width

    def prior_transform(self, u):
        return self.lo + self.width * np.asarray(u, dtype=float)

    def loglike(self, v):
        v = np.asarray(v, dtype=float)
        n, c = self.ndim, 0.5 * self.ndim * math.log(2 * math.pi)
        l1 = math.log(self.w1) - 0.5 * np.sum((v - self.m1) ** 2, -1) / self.s1 ** 2 - n * math.log(self.s1) - c
        l2 = math.log(1 - self.w1) - 0.5 * np.sum((v - self.m2) ** 2, -1) / self.s2 ** 2 - n * math.log(self.s2) - c
        return np.logaddexp(l1, l2)


def _mixture():
    n, h = 10, 10.0
    m1, m2 = np.zeros(n), np.zeros(n)
    m1[:2], m2[:2] = -2.5, 2.5
    nm = _NumpyMixture(n, m1, m2, 1.0, 0.6, 0.3, -h, 2 * h)
    prm = np.concatenate([m1, m2, [1.0, 0.6, math.log(0.3), math.log(0.7)]])
    um = DeviceModel.from_cuda(n, MIXTURE, params=prm, prior_kind=_lib.PRIOR_UNIFORM, prior_p0=-h, prior_p1=2 * h,
                               name='mixture10')
    um.logz_truth = -n * math.log(2 * h)           # both components lie well inside the prior box
    return nm, um


def test_mixture_model_eval_matches_numpy():
    nm, um = _mixture()
    u = np.random.default_rng(3).random((2000, 10))
    u[:1000] = 0.5 + 0.08 * (u[:1000] - 0.5)       # near the modes as well as across the box
    v, l = um.evaluate(u)
    close(v, nm.prior_transform(u), rtol=1e-15)
    close(l, nm.loglike(v), rtol=1e-12)


def test_mixture_device_runs_land_on_the_analytic_evidence():
    nm, um = _mixture()
    outs, _ = replicas.run_replicas(um, range(4), nlive=500, bound='multi', sample='rslice', max_in_flight=4,
                                    sampler_kwargs=dict(slices=5))
    lz = np.array([o['logz'] for o in outs])
    err = np.mean([o['logzerr'] for o in outs])
    print('USER-MIXTURE logz %s truth %.4f logzerr %.3f' % (np.round(lz, 3), um.logz_truth, err))
    assert abs(lz.mean() - um.logz_truth) < 3 * err / np.sqrt(len(lz)) + 0.15, (lz.mean(), err)


# ---- plumbing -----------------------------------------------------------------------------------------------------
def _abort_at(k_stop):
    def cb(k):
        if k >= k_stop:
            raise KeyboardInterrupt('test: run aborted after checkpoint %d' % k)
    return cb


def test_checkpoint_resume_is_bit_identical(tmp_path):
    _, _, um = _models('prec', 10)
    mk = lambda: nested.NestedSampler(um, nlive=400, bound='multi', sample='rwalk', queue_size=40, seed=11, walks=30)
    ref = mk().run_nested(loop='device', batch=20)
    f = str(tmp_path / 'ckpt.pkl')
    s = mk()
    with pytest.raises(KeyboardInterrupt):
        s.run_nested(loop='device', batch=20, checkpoint_file=f, checkpoint_every=0., on_checkpoint=_abort_at(4))
    del s
    r = nested.NestedSampler.restore(f)
    res = r.run_nested(resume=True)
    assert res.niter == ref.niter and res.ncall == ref.ncall
    assert np.array_equal(res.logl, ref.logl) and np.array_equal(res.samples_u, ref.samples_u)
    assert res.logz[-1] == ref.logz[-1] and res.logzerr[-1] == ref.logzerr[-1]
    assert abs(res.logz[-1] - (-10 * math.log(10.0))) < 4 * res.logzerr[-1] + 0.1


def test_replicas_on_a_context_pool_equal_the_registry(monkeypatch):
    _, dm, um = _models('diag', 6)
    kw = dict(nlive=200, bound='multi', sample='rwalk', sampler_kwargs=dict(walks=20), dlogz=0.5, batch=10,
              max_in_flight=4)
    monkeypatch.setenv('B2N_RWALK_IMPL', 'warp')
    ref, _ = replicas.run_replicas(dm, [5, 6, 7, 8], **kw)
    monkeypatch.delenv('B2N_RWALK_IMPL')
    um._ids.clear()
    pool = replicas.ContextPool(0, 4)
    try:
        outs, _ = replicas.run_replicas(um, [5, 6, 7, 8], pool=pool, **kw)
        assert len(um._ids) >= 4                   # every context of the pool loaded the image
    finally:
        pool.close()
    for a, b in zip(outs, ref):
        assert (a['niter'], a['ncall']) == (b['niter'], b['ncall'])
        assert a['logz'] == pytest.approx(b['logz'], rel=RTOL, abs=RTOL)


def test_host_callables_match_numpy():
    om, _, um = _models('shell', 5)
    u = _cloud('shell', 5, 300, np.random.default_rng(4))
    v = um.prior_transform(u)
    close(v, om.prior_transform(u), rtol=1e-15)
    close(um.loglikelihood(v), om.loglike(v))
    assert um.loglikelihood(v[3]) == pytest.approx(float(om.loglike(v[3])), rel=RTOL)
    assert um.prior_transform(u[3]).shape == (5,)


def test_lockstep_rwalk_kernels_refuse_a_user_model(monkeypatch):
    om, _, um = _models('prec', 10)
    u0, loglstar, ells, ell = _queue('prec', om, 16, np.random.default_rng(1))
    ops.bound_set(np.array([e.axes for e in ells]))
    monkeypatch.setenv('B2N_RWALK_IMPL', 'mma')
    with pytest.raises(NotImplementedError, match='user-likelihood'):
        ops.rwalk_batch(um.model_id(), u0, loglstar, 0.5, 10, SEED, ell=ell)
    monkeypatch.delenv('B2N_RWALK_IMPL')
    o = ops.rwalk_batch(um.model_id(), u0, loglstar, 0.5, 10, SEED, ell=ell)     # the context still works
    assert np.all(o['ncall'] == 10)

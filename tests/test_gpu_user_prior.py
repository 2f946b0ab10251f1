"""GPU: user prior transforms (DeviceModel.from_cuda(..., prior_source=...), B2N_PRIOR_USER) in every kernel slot.

One prior program serves every test: ``PRIORS`` picks its transform from ``p[0]`` -- the registry's UNIFORM and
NORMAL_PPF restated, and three priors the registry lacks (a correlated Gaussian, ordered uniforms, log-uniform).
With the UNIFORM restatement (the registry's own fma) a user-prior model must reproduce the same likelihood with the
registry prior bit for bit in every slot; NORMAL_PPF to rtol 1e-9 (bit identity printed: NVRTC's normcdfinv is
libdevice's, but the two programs inline it differently).  The new priors run against numpy restatements through the
float64 oracle on the same Philox streams, and three whole runs land on analytic evidences.  Six programs are
compiled (three likelihoods, each with and without the prior), memoised for the session."""
import ctypes as C
import math

import numpy as np
import pytest
from scipy import special

from dynesty_b200 import _lib, dynamic, nested, ops, replicas
from dynesty_b200 import usermodel as UM
from dynesty_b200._lib import ModelDesc, ptr
from dynesty_b200.likelihoods import DeviceModel
from oracle import bounding as OB, likelihoods as OL, philox, samplers as OS

pytestmark = pytest.mark.gpu

SEED = 91173
RTOL = 1e-9

# p[0] selects the transform, its parameters follow at q = p + 1
PRIORS = r'''
__device__ void b2n_user_prior(const double* u, double* v, double* work, int n, const double* p, int lane) {
    const int kind = (int)p[0];
    const double* q = p + 1;
    if (kind == 0) {                    // the registry's UNIFORM: lo + width * u
        for (int i = lane; i < n; i += 32) v[i] = fma(q[n + i], u[i], q[i]);
    } else if (kind == 1) {             // the registry's NORMAL_PPF: mu + sigma * ndtri(u)
        for (int i = lane; i < n; i += 32) v[i] = fma(q[n + i], normcdfinv(u[i]), q[i]);
    } else if (kind == 2) {             // correlated Gaussian: mu + L ndtri(u), L lower-triangular, column-major
        for (int i = lane; i < n; i += 32) work[i] = normcdfinv(u[i]);
        __syncwarp();
        for (int i = lane; i < n; i += 32) {
            double s = q[i];
            for (int j = 0; j <= i; j++) s = fma(q[n + (size_t)j * n + i], work[j], s);
            v[i] = s;
        }
    } else if (kind == 3) {             // ordered uniforms 0 < v0 < ... < v(n-1) < 1: log v_i = sum_{k>=i} log(u_k)/(k+1)
        for (int i = lane; i < n; i += 32) work[i] = log(u[i]) / (double)(i + 1);
        __syncwarp();
        for (int i = lane; i < n; i += 32) {
            double s = 0.0;
            for (int k = n - 1; k >= i; k--) s += work[k];
            v[i] = exp(s);
        }
    } else {                            // log-uniform on [a_i, b_i]
        for (int i = lane; i < n; i += 32) v[i] = q[i] * exp(u[i] * log(q[n + i] / q[i]));
    }
}
'''

# Gaussian -0.5 sum ivar (x - mean)^2 + lnorm, x = v, or x = log v when p[2n + 1] != 0 (the registry's DIAG order)
DIAG = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    const bool lg = p[2 * n + 1] != 0.0;
    double s = 0.0;
    for (int i = lane; i < n; i += 32) {
        const double d = (lg ? log(v[i]) : v[i]) - p[i];
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


def close(a, b, rtol=RTOL):
    np.testing.assert_allclose(a, b, rtol=rtol, atol=rtol * max(np.abs(np.asarray(b)).max(), 1e-300))


# ---- 1. the registry's priors restated --------------------------------------------------------------------------
_MODELS = {}


def _restated(kind, n):
    """(oracle model, user likelihood + registry prior, same likelihood + the prior restated as user code)."""
    if (kind, n) not in _MODELS:
        if kind == 'shell':
            om = OL.shells(n)
            p = om.p
            src, prm = SHELLS, np.concatenate([p['c1'], p['c2'], [p['r'], p['w']]])
        elif kind == 'prec':
            om = OL.gauss_corr(n, 0.4, 5.)
            p = om.p
            src, prm = PREC, np.concatenate([p['mean'] * np.ones(n), np.asarray(p['prec']).T.ravel(), [p['lnorm']]])
        else:
            om = OL.iid_normal_ppf(n)
            p = om.p
            src, prm = DIAG, np.concatenate([p['mean'] * np.ones(n), p['ivar'] * np.ones(n), [p['lnorm'], 0.0]])
        if om.prior_kind == OL.PRIOR_UNIFORM:
            p0, p1, code = p['lo'], p['width'], 0
        else:
            p0, p1, code = p['mu'], p['sigma'], 1
        reg = DeviceModel.from_cuda(n, src, params=prm, prior_kind=om.prior_kind, prior_p0=p0, prior_p1=p1,
                                    name='reg_' + kind)
        pp = np.concatenate([[code], np.broadcast_to(p0, (n,)), np.broadcast_to(p1, (n,))])
        usr = DeviceModel.from_cuda(n, src, params=prm, prior_source=PRIORS, prior_params=pp, name='userprior_' + kind)
        _MODELS[kind, n] = (om, reg, usr)
    return _MODELS[kind, n]


def _same(kind, case, ou, orr, ints):
    """user prior == registry prior: counts exact; u / v / logl bit-identical for the UNIFORM restatement (shell,
    prec), to RTOL for NORMAL_PPF (diag)."""
    for k in ints:
        assert np.array_equal(ou[k], orr[k]), (case, k)
    bit = all(np.array_equal(ou[k], orr[k]) for k in ('u', 'v', 'logl'))
    print('PRIOR-BITWISE %s-%s %s' % (case, kind, bit))
    if kind == 'diag':
        for k in ('u', 'v', 'logl'):
            close(ou[k], orr[k])
    else:
        for k in ('u', 'v', 'logl'):
            assert np.array_equal(ou[k], orr[k]), (case, k)


def _cloud(kind, n, npts, rng):
    u = 0.5 + 0.03 * rng.standard_normal((npts, n))
    if kind == 'shell':     # on the first shell (centre -3.5, radius 2, prior U(-6, 6))
        u[:, 0] += (-1.5 / 12.0)
    return u


def _queue(model, cloud, Q, rng, K=2):
    """start points above a threshold, K ellipsoids around them, an ellipsoid per chain"""
    n = model.ndim
    pts = cloud(max(2000, 8 * K * n))
    logl = model.loglike(model.prior_transform(pts))
    loglstar = float(np.quantile(logl, 0.3))
    good = pts[logl > loglstar]
    ells = [OB.bounding_ellipsoid(good[i::K]) for i in range(K)]
    u0 = np.ascontiguousarray(good[rng.integers(len(good), size=Q)])
    ell = rng.integers(K, size=Q).astype(np.int32)
    return u0, loglstar, ells, ell


RKINDS = ['shell', 'prec', 'diag']


@pytest.mark.parametrize('kind', RKINDS)
@pytest.mark.parametrize('n', [10, 200])
def test_model_eval_restated_prior(kind, n):
    om, reg, usr = _restated(kind, n)
    u = _cloud(kind, n, 300, np.random.default_rng(n))
    vu, lu = usr.evaluate(u)
    vr, lr = reg.evaluate(u)
    _same(kind, 'eval%d' % n, dict(u=u, v=vu, logl=lu), dict(u=u, v=vr, logl=lr), ())
    close(vu, om.prior_transform(u))


@pytest.mark.parametrize('kind', RKINDS)
@pytest.mark.parametrize('n', [10, 200])
def test_rwalk_restated_prior(kind, n):
    om, reg, usr = _restated(kind, n)
    rng = np.random.default_rng(100 + n)
    Q = 301 if n == 10 else 40
    u0, loglstar, ells, ell = _queue(om, lambda k: _cloud(kind, n, k, rng), Q, rng)
    ops.bound_set(np.array([e.axes for e in ells]))
    args = (u0, loglstar, 0.6, 25, SEED)
    orr = ops.rwalk_batch(reg.model_id(), *args, chain0=70 + n, ell=ell)
    ou = ops.rwalk_batch(usr.model_id(), *args, chain0=70 + n, ell=ell)
    _same(kind, 'rwalk%d' % n, ou, orr, ('n_accept', 'n_reject', 'ncall'))
    assert ou['n_accept'].sum() > 0


@pytest.mark.parametrize('sampler', ['slice', 'rslice'])
@pytest.mark.parametrize('doubling', [False, True])
@pytest.mark.parametrize('kind', RKINDS)
@pytest.mark.parametrize('n', [10, 200])
def test_slice_restated_prior(sampler, doubling, kind, n):
    om, reg, usr = _restated(kind, n)
    rng = np.random.default_rng(200 + n)
    Q = 140 if n == 10 else 24
    u0, loglstar, ells, ell = _queue(om, lambda k: _cloud(kind, n, k, rng), Q, rng)
    ops.bound_set(np.array([e.axes for e in ells]))
    slices = 3 if sampler == 'rslice' else 1
    fn = ops.rslice_batch if sampler == 'rslice' else ops.slice_batch
    kw = dict(chain0=300 + n, ell=ell, doubling=doubling)
    orr = fn(reg.model_id(), u0, loglstar, 1.0, slices, SEED, **kw)
    ou = fn(usr.model_id(), u0, loglstar, 1.0, slices, SEED, **kw)
    _same(kind, '%s%d-doubling%d' % (sampler, n, doubling), ou, orr, ('n_expand', 'n_contract', 'ncall', 'flags'))
    assert np.all(ou['logl'] > loglstar)


@pytest.mark.parametrize('kind', RKINDS)
def test_unif_unitcube_friends_restated_prior(kind):
    n = 10
    om, reg, usr = _restated(kind, n)
    rng = np.random.default_rng(7)
    u0, loglstar, ells, ell = _queue(om, lambda k: _cloud(kind, n, k, rng), 8, rng)
    me = OB.MultiEll(ells)
    ops.bound_set(me.axes, me.ctrs, me.ams, me.logvol_ells)
    Q, chain0 = 4 * 32 + 3, 11
    orr = ops.unif_batch(reg.model_id(), Q, n, loglstar, SEED, chain0=chain0)
    ou = ops.unif_batch(usr.model_id(), Q, n, loglstar, SEED, chain0=chain0)
    _same(kind, 'unif', ou, orr, ('ncall', 'nprop', 'flags'))
    thr = float(np.quantile(om.loglike(om.prior_transform(rng.random((4000, n)))), 0.9))
    orr = ops.unitcube_batch(reg.model_id(), Q, n, thr, SEED, chain0=chain0)
    ou = ops.unitcube_batch(usr.model_id(), Q, n, thr, SEED, chain0=chain0)
    _same(kind, 'unitcube', ou, orr, ('ncall',))
    pts = _cloud(kind, n, 300, rng)
    f = ops.friends_update(pts, 'balls', use_clustering=False)
    ops.friends_set('balls', pts, f['axes'], f['axes_inv'])
    thr = float(np.quantile(om.loglike(om.prior_transform(pts)), 0.3))
    orr = ops.friends_unif_batch(reg.model_id(), 97, n, thr, SEED, chain0=5)
    ou = ops.friends_unif_batch(usr.model_id(), 97, n, thr, SEED, chain0=5)
    _same(kind, 'friends-unif', ou, orr, ('ncall', 'nprop', 'flags'))


# ---- 2. priors the registry lacks, against numpy through the float64 oracle --------------------------------------
class NumpyModel:
    """The PRIORS transform of `code` and the DIAG likelihood, in numpy (the oracle's model interface)."""

    def __init__(self, code, n, q, mean, ivar, lnorm, in_log):
        self.code, self.ndim, self.q = code, n, np.asarray(q, dtype=float)
        self.mean, self.ivar, self.lnorm, self.in_log = mean, ivar, lnorm, in_log

    def prior_transform(self, u):
        u = np.asarray(u, dtype=float)
        n, q = self.ndim, self.q
        if self.code == 2:
            L = q[n:].reshape(n, n).T                              # column-major in q
            return q[:n] + special.ndtri(u) @ L.T
        if self.code == 3:
            w = np.log(u) / np.arange(1, n + 1)
            return np.exp(np.cumsum(w[..., ::-1], axis=-1)[..., ::-1])
        a, b = q[:n], q[n:2 * n]
        return a * np.exp(u * np.log(b / a))

    def loglike(self, v):
        x = np.log(v) if self.in_log else np.asarray(v, dtype=float)
        return self.lnorm - 0.5 * np.sum(self.ivar * (x - self.mean) ** 2, axis=-1)

    def device(self):
        n = self.ndim
        prm = np.concatenate([self.mean, self.ivar, [self.lnorm, 1.0 if self.in_log else 0.0]])
        return DeviceModel.from_cuda(n, DIAG, params=prm, prior_source=PRIORS,
                                     prior_params=np.concatenate([[self.code], self.q]), name='prior%d' % self.code)


def _gauss_lnorm(sig):
    return -0.5 * float(np.sum(np.log(2 * math.pi * sig ** 2)))


def _corr_model(n, sig_like, mean_like=None):
    sd = np.linspace(1.0, 2.0, n)
    S0 = 0.5 * np.outer(sd, sd)
    np.fill_diagonal(S0, sd ** 2)
    L = np.linalg.cholesky(S0)
    mu0 = np.linspace(-0.5, 0.5, n)
    q = np.concatenate([mu0, L.T.ravel()])                         # L column-major
    mean = mu0 + 0.3 if mean_like is None else mean_like
    sig = np.full(n, sig_like)
    return NumpyModel(2, n, q, mean, 1 / sig ** 2, _gauss_lnorm(sig), False), mu0, S0


def _ordered_model(n, sig_like, mean_like=None):
    base = NumpyModel(3, n, [], 0, 0, 0, False)
    mean = base.prior_transform(np.full(n, 0.5)) if mean_like is None else mean_like
    sig = np.full(n, sig_like)
    return NumpyModel(3, n, [], mean, 1 / sig ** 2, _gauss_lnorm(sig), False)


def _logu_model(n, sig_like, mean_like=None, a=0.01, b=100.0):
    q = np.concatenate([np.full(n, a), np.full(n, b)])
    mean = np.zeros(n) if mean_like is None else mean_like
    sig = np.full(n, sig_like)
    return NumpyModel(4, n, q, mean, 1 / sig ** 2, _gauss_lnorm(sig), True)


_NEW = {}


def _new(name):
    if name not in _NEW:
        n = 8
        nm = {'corr': lambda: _corr_model(n, 1.0)[0], 'ordered': lambda: _ordered_model(n, 0.05),
              'logu': lambda: _logu_model(n, 1.0)}[name]()
        _NEW[name] = (nm, nm.device())
    return _NEW[name]


NEW = ['corr', 'ordered', 'logu']


def _bitwise_model_outputs(dm, o):
    """every chain output is the model at its u, bit for bit"""
    v, logl = dm.evaluate(o['u'])
    assert np.array_equal(o['v'], v)
    assert np.array_equal(o['logl'], logl)


@pytest.mark.parametrize('name', NEW)
def test_new_prior_evaluate_matches_numpy(name):
    nm, dm = _new(name)
    u = np.random.default_rng(5).random((1000, nm.ndim))
    v, logl = dm.evaluate(u)
    close(v, nm.prior_transform(u), rtol=1e-12)
    close(logl, nm.loglike(v), rtol=1e-12)
    if name == 'ordered':
        assert np.all(np.diff(v, axis=1) > 0) and np.all((v > 0) & (v < 1))


def _new_queue(nm, Q, seed):
    rng = np.random.default_rng(seed)
    return rng, _queue(nm, lambda k: 0.5 + 0.04 * rng.standard_normal((k, nm.ndim)), Q, rng)


@pytest.mark.parametrize('name', NEW)
def test_new_prior_rwalk_matches_oracle(name):
    nm, dm = _new(name)
    rng, (u0, loglstar, ells, ell) = _new_queue(nm, 150, 31)
    axes = np.array([e.axes for e in ells])
    ops.bound_set(axes)
    walks, scale, chain0 = 25, 0.6, 900
    o = ops.rwalk_batch(dm.model_id(), u0, loglstar, scale, walks, SEED, chain0=chain0, ell=ell)
    assert o['n_accept'].sum() > 0
    _bitwise_model_outputs(dm, o)
    for q in sorted({0, 149} | set(rng.choice(150, 6, replace=False).tolist())):
        r = OS.rwalk_chain(u0[q], loglstar, axes[ell[q]], scale, nm, philox.ChainStream(SEED, chain0 + q), walks)
        assert (o['n_accept'][q], o['n_reject'][q]) == (r['n_accept'], r['n_reject']), q
        close(o['u'][q], r['u'])
        close(o['v'][q], r['v'])
        assert o['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL)


@pytest.mark.parametrize('sampler', ['slice', 'rslice'])
@pytest.mark.parametrize('name', NEW)
def test_new_prior_slice_matches_oracle(sampler, name):
    nm, dm = _new(name)
    rng, (u0, loglstar, ells, ell) = _new_queue(nm, 90, 41)
    axes = np.array([e.axes for e in ells])
    ops.bound_set(axes)
    slices = 3 if sampler == 'rslice' else 1
    fn, chain = (ops.rslice_batch, OS.rslice_chain) if sampler == 'rslice' else (ops.slice_batch, OS.slice_chain)
    chain0 = 1300
    o = fn(dm.model_id(), u0, loglstar, 1.0, slices, SEED, chain0=chain0, ell=ell)
    assert np.all(o['flags'] == 0) and np.all(o['logl'] > loglstar)
    _bitwise_model_outputs(dm, o)
    for q in sorted({0, 89} | set(rng.choice(90, 4, replace=False).tolist())):
        r = chain(u0[q], loglstar, axes[ell[q]], 1.0, nm, philox.ChainStream(SEED, chain0 + q), slices)
        assert (o['ncall'][q], o['n_expand'][q], o['n_contract'][q]) == (r['ncall'], r['n_expand'],
                                                                         r['n_contract']), q
        close(o['u'][q], r['u'])
        close(o['v'][q], r['v'])
        assert o['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL)


@pytest.mark.parametrize('name', NEW)
def test_new_prior_unif_matches_oracle(name):
    nm, dm = _new(name)
    rng, (u0, loglstar, ells, ell) = _new_queue(nm, 8, 51)
    me = OB.MultiEll(ells)
    ops.bound_set(me.axes, me.ctrs, me.ams, me.logvol_ells)
    Q, chain0 = 2 * 32 + 5, 1700
    o = ops.unif_batch(dm.model_id(), Q, nm.ndim, loglstar, SEED, chain0=chain0)
    _bitwise_model_outputs(dm, o)
    for q in sorted({0, Q - 1} | set(rng.choice(Q, 6, replace=False).tolist())):
        r = OS.unif_chain(loglstar, me, nm, philox.ChainStream(SEED, chain0 + q), nm.ndim)
        assert (o['ncall'][q], o['nprop'][q]) == (r['ncall'], r['nprop']), q
        close(o['u'][q], r['u'])
        close(o['v'][q], r['v'])
        assert o['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL)


# ---- 3. whole runs against analytic evidences ---------------------------------------------------------------------
def _evidence_case(name):
    if name == 'gauss':
        # N(mu0, S0) prior x normalised N(m, s^2 I) likelihood: Z = N(m; mu0, S0 + s^2 I)
        n, s = 4, 0.5
        m = np.array([0.5, -0.3, 1.0, 0.2])
        nm, mu0, S0 = _corr_model(n, s, mean_like=m)
        S = S0 + s * s * np.eye(n)
        d = m - mu0
        truth = -0.5 * (n * math.log(2 * math.pi) + np.linalg.slogdet(S)[1] + d @ np.linalg.solve(S, d))
    elif name == 'logu':
        # log-uniform on [a, b]^n x normalised Gaussian in log v: Z = prod (Phi(hi) - Phi(lo)) / log(b / a)
        n, s, a, b = 3, 0.5, 0.01, 100.0
        m = np.array([0.0, 1.0, -4.0])                           # the last one straddles log a
        nm = _logu_model(n, s, mean_like=m, a=a, b=b)
        mass = special.ndtr((math.log(b) - m) / s) - special.ndtr((math.log(a) - m) / s)
        truth = -n * math.log(math.log(b / a)) + float(np.sum(np.log(mass)))
    else:
        # ordered uniforms (prior density 5! on 0 < v0 < ... < v4 < 1) x a narrow normalised Gaussian at
        # well-separated sorted means: Z = 5!
        n = 5
        nm = _ordered_model(n, 0.02, mean_like=np.array([0.15, 0.3, 0.5, 0.7, 0.85]))
        truth = math.log(120.0)
    return nm, truth


@pytest.mark.parametrize('name', ['gauss', 'logu', 'ordered'])
def test_user_prior_runs_land_on_the_analytic_evidence(name):
    nm, truth = _evidence_case(name)
    dm = nm.device()
    outs, _ = replicas.run_replicas(dm, range(4), nlive=500, bound='multi', sample='rslice', max_in_flight=4,
                                    sampler_kwargs=dict(slices=5))
    lz = np.array([o['logz'] for o in outs])
    err = np.mean([o['logzerr'] for o in outs])
    print('USER-PRIOR-EVIDENCE %s logz %s mean %.4f truth %.4f logzerr %.3f'
          % (name, np.round(lz, 3), lz.mean(), truth, err))
    assert abs(lz.mean() - truth) < 3 * err / np.sqrt(len(lz)) + 0.15, (lz.mean(), truth, err)


# ---- 4. plumbing -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('sample,kw', [('rwalk', dict(walks=20)), ('rslice', dict(slices=4))])
def test_device_rounds_restated_prior(sample, kw):
    _, reg, usr = _restated('prec', 6)
    run = lambda m: nested.NestedSampler(m, nlive=300, bound='multi', sample=sample, seed=21, **kw).run_nested(
        loop='device', batch=10, dlogz=0.5)
    ref, res = run(reg), run(usr)
    assert (res.niter, res.ncall) == (ref.niter, ref.ncall)
    close(res.logl, ref.logl)
    print('PRIOR-BITWISE rounds-%s %s' % (sample, np.array_equal(res.logl, ref.logl)))


def test_dynamic_sampler_restated_prior():
    _, reg, usr = _restated('prec', 6)

    def run(m):
        d = dynamic.DynamicNestedSampler(m, nlive=200, bound='multi', sample='rwalk', walks=20, seed=9)
        return d.run_nested(dlogz_init=0.5, nlive_batch=100, maxbatch=1, n_effective=1e9)

    ref, res = run(reg), run(usr)
    assert (res.niter, res.ncall) == (ref.niter, ref.ncall)
    close(res.logl, ref.logl)
    print('PRIOR-BITWISE dynamic %s' % np.array_equal(res.logl, ref.logl))


def _abort_at(k_stop):
    def cb(k):
        if k >= k_stop:
            raise KeyboardInterrupt('test: run aborted after checkpoint %d' % k)
    return cb


def test_checkpoint_resume_is_bit_identical(tmp_path):
    _, _, dm = _restated('prec', 10)
    mk = lambda: nested.NestedSampler(dm, nlive=400, bound='multi', sample='rwalk', queue_size=40, seed=11, walks=30)
    ref = mk().run_nested(loop='device', batch=20)
    f = str(tmp_path / 'ckpt.pkl')
    s = mk()
    with pytest.raises(KeyboardInterrupt):
        s.run_nested(loop='device', batch=20, checkpoint_file=f, checkpoint_every=0., on_checkpoint=_abort_at(4))
    del s
    r = nested.NestedSampler.restore(f)
    assert r.model.prior_source == PRIORS
    np.testing.assert_array_equal(r.model.prior_params, dm.prior_params)
    res = r.run_nested(resume=True)
    assert res.niter == ref.niter and res.ncall == ref.ncall
    assert np.array_equal(res.logl, ref.logl) and np.array_equal(res.samples_u, ref.samples_u)
    assert res.logz[-1] == ref.logz[-1] and res.logzerr[-1] == ref.logzerr[-1]


@pytest.mark.parametrize('name', NEW)
def test_host_callables_compose_to_evaluate(name):
    nm, dm = _new(name)
    u = np.random.default_rng(6).random((200, nm.ndim))
    v, logl = dm.evaluate(u)
    assert np.array_equal(dm.prior_transform(u), v)
    assert np.array_equal(dm.loglikelihood(dm.prior_transform(u)), logl)
    assert dm.loglikelihood(v[3]) == logl[3]


def _raw_create_user_ex(ctx, ndim, prior_kind, cm, prior_params=None):
    d = ModelDesc()
    d.ndim, d.prior_kind, d.like_kind = ndim, prior_kind, _lib.LIKE_USER
    prm = np.concatenate([np.zeros(ndim), np.ones(ndim), [0.0, 0.0]])
    names = (C.c_char_p * len(cm.lowered))(*[s.encode() for s in cm.lowered])
    mid = C.c_int32(-1)
    st = ctx.lib.b2n_model_create_user_ex(ctx.h, C.byref(d), ptr(prm), prm.size, ptr(prior_params),
                                          0 if prior_params is None else prior_params.size, cm.cubin, len(cm.cubin),
                                          names, C.byref(mid))
    return st, mid.value


def test_create_user_ex_refuses_an_image_without_a_prior():
    ctx = _lib.default_context()
    n = 4
    pp = np.concatenate([[0.0], np.zeros(n), np.ones(n)])
    st, _ = _raw_create_user_ex(ctx, n, _lib.PRIOR_USER, UM.compile_user(DIAG), pp)
    assert st == _lib.ERR_ARG
    assert 'without a prior' in ctx.lib.b2n_last_error(ctx.h).decode()
    # the context keeps working: the same image without a user prior, and the prior image, load and evaluate
    st, mid = _raw_create_user_ex(ctx, n, _lib.PRIOR_IDENTITY, UM.compile_user(DIAG))
    assert st == _lib.OK
    u = np.random.default_rng(2).random((64, n))
    v, logl = ops.model_eval(mid, u)
    assert np.array_equal(v, u) and np.all(np.isfinite(logl))
    st, mid = _raw_create_user_ex(ctx, n, _lib.PRIOR_USER, UM.compile_user(DIAG, PRIORS), pp)
    assert st == _lib.OK
    v2, logl2 = ops.model_eval(mid, u)
    assert np.array_equal(v2, u) and np.array_equal(logl2, logl)        # kind 0 with lo = 0, width = 1
    # a registry prior kind takes no prior parameters
    st, _ = _raw_create_user_ex(ctx, n, _lib.PRIOR_IDENTITY, UM.compile_user(DIAG), pp)
    assert st == _lib.ERR_ARG


def test_registry_entry_points_still_reject_the_user_prior_kind():
    ctx = _lib.default_context()
    n = 3
    d = ModelDesc()
    d.ndim, d.prior_kind, d.like_kind = n, _lib.PRIOR_USER, _lib.LIKE_GAUSS_DIAG
    vec = np.zeros(n)
    d.like_vec0 = d.like_vec1 = ptr(vec)
    mid = C.c_int32(-1)
    assert ctx.lib.b2n_model_create(ctx.h, C.byref(d), C.byref(mid)) == _lib.ERR_ARG
    cm = UM.compile_user(DIAG, PRIORS)
    d.like_kind = _lib.LIKE_USER
    names = (C.c_char_p * len(cm.lowered))(*[s.encode() for s in cm.lowered])
    prm = np.zeros(2 * n + 2)
    assert ctx.lib.b2n_model_create_user(ctx.h, C.byref(d), ptr(prm), prm.size, cm.cubin, len(cm.cubin), names,
                                         C.byref(mid)) == _lib.ERR_ARG

"""GPU tier of the posterior summaries: b2n_jitter_posterior / b2n_resample_posterior against the reference's own
mean_and_cov / quantile (tests/golden/posterior.npz), b2n_weighted_stats against the numpy restatement
(oracle/posterior.py) across its tile and chunk edges, consistency and bit-identity with the existing run-uncertainty
APIs, determinism, and a C2-shaped record at n = 50, R = 128."""
import numpy as np
import pytest

from oracle import posterior as OP, resample as ORS
from dynesty_b200 import likelihoods as DL, ops, replicas, utils as DU
from dynesty_b200.nested import Results
from test_posterior import GOLDEN, _records, golden_res

pytestmark = pytest.mark.gpu

PM_BK, PM_KCH, QC = 16, 2048, 1024


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLDEN))


def check(got, ref, x, rtol=1e-9, quant=True):
    """mean / cov / quantiles of R realisations: mean and quantiles to rtol times each coordinate's scale, cov against
    sqrt(cov_ii cov_jj)."""
    scale = np.abs(x).max(axis=0) + x.std(axis=0) + 1e-300
    np.testing.assert_allclose(got['mean'] / scale, ref['mean'] / scale, rtol=0, atol=rtol)
    d = np.sqrt(np.abs(np.einsum('rii->ri', ref['cov'])))
    dd = d[:, :, None] * d[:, None, :]
    np.testing.assert_allclose(got['cov'] / dd, ref['cov'] / dd, rtol=0, atol=rtol)
    if quant:
        np.testing.assert_allclose(got['quantiles'] / scale[None, :, None], ref['quantiles'] / scale[None, :, None],
                                   rtol=0, atol=rtol, equal_nan=True)


@pytest.mark.parametrize('error', ['jitter', 'resample'])
def test_realisations_match_the_reference(gold, error):
    seed, chain0, q = int(gold['post_seed']), int(gold['post_chain0']), gold['post_q']
    for name in _records(gold):
        res = golden_res(gold, name)
        x = np.asarray(res['samples'], dtype=float)
        for r in gold['post_r']:
            o = DU.posterior_realisations(res, 1, seed, chain0 + int(r), error=error, q=q)
            p = 'post_%s_%s%d_' % (name, {'jitter': 'j', 'resample': 's'}[error], r)
            assert abs(o['logz'][0] - gold[p + 'logz']) < 1e-9
            ref = dict(mean=gold[p + 'mean'][None], cov=gold[p + 'cov'][None], quantiles=gold[p + 'quant'][None])
            check(o, ref, x)


def _case(N, n, R, nq, seed=0):
    rng = np.random.default_rng(seed + 1000 * N + 10 * n + R)
    sig = 10.0 ** rng.uniform(-2, 1, n)
    x = 1e3 * sig + sig * rng.standard_normal((N, n))          # the posterior 10^3 sigma from the origin
    x[::3] = np.round(x[::3] / sig) * sig                       # ties
    w = rng.random((R, N)) * np.exp(rng.uniform(-30, 0, (R, N)))
    w[rng.random((R, N)) < 0.1] = 0.0                           # zero weights: nodes
    w[rng.random((R, N)) < 0.1] = -0.0                          # absent samples
    w[:, -1] = np.abs(w[:, -1]) + 1e-3
    if N > 1:
        w[:, 0] = 1e-3
    q = np.array([0.0, 0.025, 0.5, 0.975, 1.0])[:nq] if nq == 5 else np.array([0.3])
    return x, w, q


SWEEP = ([(N, 3, 9, 5) for N in (1, 2, PM_BK - 1, PM_BK + 1, QC - 1, QC + 1, PM_KCH - 1, PM_KCH + 1, 3 * PM_KCH + 5)]
         + [(300, n, 9, 5) for n in (1, 2, 3, 8, 9, 50, 64, 65)]
         + [(300, 4, R, 5) for R in (1, 7, 8, 9, 129)]
         + [(300, 4, 9, 1)])


@pytest.mark.parametrize('N,n,R,nq', SWEEP)
def test_weighted_stats_against_the_oracle(N, n, R, nq):
    x, w, q = _case(N, n, R, nq)
    shift = x.mean(axis=0)
    got = ops.weighted_stats(x, w, shift, q=q)
    with np.errstate(divide='ignore', invalid='ignore'):
        ref = OP.weighted_stats(x, w, q=q)
    if N == 1:                          # one node: every quantile NaN; cov's factor divides by wsum^2 - w2sum = 0
        assert np.isnan(got['quantiles']).all()
        np.testing.assert_allclose(got['mean'], ref['mean'], rtol=1e-12)
        return
    check(got, ref, x)


def test_moments_about_the_origin_would_fail():
    """The shift is what keeps the covariance: about 0 the second moments of a posterior 10^3 sigma out cancel."""
    x, w, _ = _case(5000, 4, 3, 5, seed=1)
    ref = OP.weighted_stats(x, w)
    check(ops.weighted_stats(x, w, x.mean(axis=0)), ref, x, quant=False)
    far = ops.weighted_stats(x, w, np.zeros(4))
    d = np.sqrt(np.einsum('rii->ri', ref['cov']))
    assert np.abs((far['cov'] - ref['cov']) / (d[:, :, None] * d[:, None, :])).max() > 1e-9


def test_consistency_with_the_existing_apis(gold):
    seed, q = 17, [0.1, 0.5, 0.9]
    for name in ('host', 'dyn', 'hd'):
        res = golden_res(gold, name)
        for chain in (0, 5):
            o = DU.posterior_realisations(res, 1, seed, chain, error='jitter')
            new = DU.jitter_run(res, seed, chain)
            m, c = DU.mean_and_cov(new['samples'], np.exp(new['logwt'] - new['logz'][-1]))
            np.testing.assert_allclose(o['mean'][0], m, rtol=1e-12, atol=1e-12 * np.abs(m).max())
            np.testing.assert_allclose(o['cov'][0], c, rtol=0, atol=1e-12 * np.abs(c).max())
            o = DU.posterior_realisations(res, 1, seed, chain, error='resample', q=q)
            new = DU.resample_run(res, seed, chain)
            m, c = DU.mean_and_cov(new['samples'], np.exp(new['logwt'] - new['logz'][-1]))
            np.testing.assert_allclose(o['mean'][0], m, rtol=1e-12, atol=1e-12 * np.abs(m).max())
            np.testing.assert_allclose(o['cov'][0], c, rtol=0, atol=1e-12 * np.abs(c).max())
        for error, fn in (('jitter', DU.jitter_realisations), ('resample', DU.resample_realisations)):
            o = DU.posterior_realisations(res, 9, seed, 3, error=error, q=q)
            ref = fn(res, 9, seed, 3)
            for k in ('logz', 'logzerr', 'h', 'kld'):
                assert np.array_equal(o[k], ref[k]), (name, error, k)


@pytest.mark.parametrize('error', ['jitter', 'resample'])
def test_deterministic_and_independent_of_R(gold, error):
    res = golden_res(gold, 'hd')
    q = [0.0, 0.16, 0.5, 0.84, 1.0]
    a = DU.posterior_realisations(res, 37, 23, 100, error=error, q=q)
    b = DU.posterior_realisations(res, 37, 23, 100, error=error, q=q)
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), k
    for r in (0, 1, 8, 31, 36):
        one = DU.posterior_realisations(res, 1, 23, 100 + r, error=error, q=q)
        for k in one:
            assert np.array_equal(one[k][0], a[k][r], equal_nan=True), (r, k)


def c2_record(n=50):
    rec = ORS.synthetic_strand_record(2000, 50, seed=0)
    rng = np.random.default_rng(7)
    u = rng.standard_normal((len(rec['logl']), n))
    u /= np.linalg.norm(u, axis=1)[:, None]
    rec['samples'] = 0.5 + 1e-3 * np.sqrt(-2.0 * rec['logl'])[:, None] * u
    return Results(rec)


def test_c2_shape_at_scale():
    res = c2_record()
    x = np.asarray(res['samples'])
    q = [0.025, 0.5, 0.975]
    for error in ('jitter', 'resample'):
        o = DU.posterior_realisations(res, 128, 3, 0, error=error, q=q)
        assert o['mean'].shape == (128, 50) and o['quantiles'].shape == (128, 50, 3)
        for r in (0, 127):
            if error == 'jitter':
                ref = OP.stats(x, OP.jitter_weights(res['logl'], res['samples_n'], 3, r), q)
            else:
                plan = DU.strand_plan(res)
                pptr, pstr = DU._piece_csr(np.asarray(res['logl']), plan)
                W, w2, pres = OP.resample_weights(res['logl'], plan['strand'], plan['base'], pptr, pstr, plan['end'],
                                                  3, r)
                ref = OP.stats(x, W, q, w2, pres)
            check({k: o[k][r:r + 1] for k in ('mean', 'cov', 'quantiles')},
                  {k: v[None] for k, v in ref.items()}, x)


def test_jitter_mean_scatter_matches_replica_scatter():
    """errors.rst's comparison: the scatter of the posterior means over jitter realisations of one run estimates the
    scatter of the means over independent runs (32 replicas) to within a factor of 2."""
    kw = dict(nlive=200, bound='multi', sample='unif', keep_results=True, dlogz=0.01)
    outs, _ = replicas.run_replicas(DL.gauss_test3d(), range(500, 532), **kw)
    means = np.array([OP.moments(o['results']['samples'], np.exp(o['results']['logwt'] - o['results']['logz'][-1]))[0]
                      for o in outs])
    res = outs[0]['results']
    o = DU.posterior_realisations(res, 256, 9, 0)
    ratio = np.mean(np.std(o['mean'], axis=0)) / np.mean(np.std(means, axis=0))
    assert 0.5 <= ratio <= 2.0, ratio

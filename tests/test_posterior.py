"""CPU tier of the posterior summaries: the numpy restatement (oracle/posterior.py) against the reference's own
mean_and_cov / quantile on its jitter_run / resample_run realisations (tests/golden/posterior.npz), the quantile
lookup rule on hand-made node sets, and the argument checks and return types of utils.mean_and_cov / quantile /
posterior_realisations with the GPU calls replaced by the oracle."""
import os

import numpy as np
import pytest

from oracle import posterior as OP
from dynesty_b200 import ops, utils as DU
from dynesty_b200.nested import Results

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'posterior.npz')
KEYS = ('logl', 'samples_id', 'samples_it', 'samples_n', 'logwt', 'logz', 'logvol', 'ncall_per_it', 'samples_batch',
        'samples')


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLDEN))


def golden_res(g, name):
    p = 'post_%s_' % name
    r = Results({k: g[p + k] for k in KEYS if p + k in g})
    r['niter'] = int(g[p + 'niter'])
    if p + 'batch_bounds' in g:
        r['batch_bounds'] = [tuple(b) for b in g[p + 'batch_bounds']]
    return r


def assert_stats(mean, cov, quant, g, q, rtol, x):
    """mean / cov / quantiles against the fixture's keys under prefix q: cov relative to sqrt(cov_ii cov_jj),
    quantiles to rtol times the coordinate's scale."""
    ref_c = g[q + 'cov']
    d = np.sqrt(np.diag(ref_c))
    scale = np.abs(x).max(axis=0) + x.std(axis=0)
    np.testing.assert_allclose(mean, g[q + 'mean'], rtol=0, atol=rtol * scale.max())
    np.testing.assert_allclose(cov / np.outer(d, d), ref_c / np.outer(d, d), rtol=0, atol=rtol)
    np.testing.assert_allclose(quant, g[q + 'quant'], rtol=0, atol=rtol * scale.max())


def _records(g):
    return [str(s) for s in g['post_names']]


def test_fixture_is_small_and_complete(gold):
    assert os.path.getsize(GOLDEN) < 1 << 20
    assert set(_records(gold)) == {'host', 'dev', 'devnolive', 'dyn', 'hd'}
    assert gold['post_hd_samples'].shape[1] == 12


@pytest.mark.parametrize('error', ['jitter', 'resample'])
def test_oracle_matches_the_reference(gold, error):
    seed, chain0, q = int(gold['post_seed']), int(gold['post_chain0']), gold['post_q']
    for name in _records(gold):
        res = golden_res(gold, name)
        x = np.asarray(res['samples'], dtype=float)
        logl = np.asarray(res['logl'], dtype=float)
        for r in gold['post_r']:
            if error == 'jitter':
                w = OP.jitter_weights(logl, DU.samples_n_of(res), seed, chain0 + int(r))
                o = OP.stats(x, w, q)
                p = 'post_%s_j%d_' % (name, r)
            else:
                plan = DU.strand_plan(res)
                pptr, pstr = DU._piece_csr(logl, plan)
                W, w2, present = OP.resample_weights(logl, plan['strand'], plan['base'], pptr, pstr, plan['end'],
                                                     seed, chain0 + int(r))
                idx = gold['post_%s_s%d_idx' % (name, r)]
                assert np.array_equal(present, np.bincount(idx, minlength=len(logl)) > 0)
                o = OP.stats(x, W, q, w2, present)
                p = 'post_%s_s%d_' % (name, r)
            assert_stats(o['mean'], o['cov'], o['quantiles'], gold, p, 1e-12, x)


# ---------------------------------------------------------------------------------------------- the lookup rule
def test_repeated_cdf_values_follow_np_interp():
    # cdf [0, 0, .25, .25, 1]: the weights of the first four nodes are 0, .25, 0, .75 (the last one's never counts)
    x = np.array([10., 11., 12., 13., 14.])
    w = np.array([0., .25, 0., .75, 5.])
    got = OP.quantile_nodes(x, [0, .1, .25], w)
    np.testing.assert_allclose(got, [11, 11.4, 13], rtol=0, atol=1e-15)
    np.testing.assert_allclose(got, np.interp([0, .1, .25], [0, 0, .25, .25, 1], x), rtol=0, atol=1e-15)


def test_zero_weight_nodes_stay_nodes_and_absent_samples_do_not():
    x = np.array([3., 1., 2., 4.])
    w = np.array([1., 0., 1., 2.])
    # sorted: 1 (w 0), 2 (1), 3 (1), 4 (2): cdf [0, 0, .5, 1]
    np.testing.assert_allclose(OP.quantile_nodes(x, [0., .25, .5, 1.], w), [2., 2.5, 3., 4.], rtol=0, atol=1e-15)
    present = np.array([True, False, True, True])
    # without node 1: 2 (1), 3 (1), 4 (2): cdf [0, .5, 1]
    np.testing.assert_allclose(OP.quantile_nodes(x, [0., .25, 1.], w, present), [2., 2.5, 4.], rtol=0, atol=1e-15)
    o = OP.weighted_stats(x[:, None], np.where(present, w, -0.0)[None], q=[0., .25, 1.], moments=False)
    np.testing.assert_allclose(o['quantiles'][0, 0], [2., 2.5, 4.], rtol=0, atol=1e-15)


def test_q_zero_and_one_and_two_nodes():
    x, w = np.array([5., -1.]), np.array([2., 7.])
    # sorted: -1 (w 7), 5: cdf [0, 1]
    np.testing.assert_allclose(OP.quantile_nodes(x, [0., .5, 1.], w), [-1., 2., 5.], rtol=0, atol=1e-15)
    assert np.isnan(OP.quantile_nodes(np.array([1.]), [0., 1.], np.array([1.]))).all()
    assert np.isnan(OP.quantile_nodes(np.array([1., 2.]), [.5], np.array([0., 1.]))).all()


def test_ties_keep_record_order():
    x = np.array([1., 0., 1., 1.])
    w = np.array([1., 1., 3., 2.])
    # sorted (value, index): 0 (1), 1@0 (1), 1@2 (3), 1@3: cdf [0, .2, .4, 1]; all ties share the value
    np.testing.assert_allclose(OP.quantile_nodes(x, [0., .1, .3, 1.], w), [0., .5, 1., 1.], rtol=0, atol=1e-15)
    # the reference's formula without ties in x
    rng = np.random.default_rng(0)
    x, w = rng.standard_normal(50), rng.random(50)
    idx = np.argsort(x)
    cdf = np.cumsum(w[idx])[:-1]
    cdf = np.append(0, cdf / cdf[-1])
    q = np.array([0., .025, .5, .975, 1.])
    np.testing.assert_allclose(OP.quantile_nodes(x, q, w), np.interp(q, cdf, x[idx]), rtol=0, atol=1e-14)


# ---------------------------------------------------------------------------------------------- the Python API
@pytest.fixture
def oracle_ops(monkeypatch):
    monkeypatch.setattr(ops, 'weighted_stats', lambda x, w, shift, q=None, moments=True, ctx=None:
                        OP.weighted_stats(x, w, shift, q, moments))
    monkeypatch.setattr(ops, 'jitter_posterior', lambda *a, ctx=None, **k: OP.jitter_posterior(*a, **k))
    monkeypatch.setattr(ops, 'resample_posterior', lambda *a, ctx=None, **k: OP.resample_posterior(*a, **k))


def test_mean_and_cov_shapes(oracle_ops):
    rng = np.random.default_rng(1)
    x, w = rng.standard_normal((40, 3)), rng.random((4, 40))
    m, c = DU.mean_and_cov(x, w[0])
    assert m.shape == (3,) and c.shape == (3, 3)
    mean = np.average(x, weights=w[0], axis=0)
    dx = x - mean
    ref = w[0].sum() / (w[0].sum() ** 2 - np.sum(w[0] ** 2)) * np.einsum('i,ij,ik', w[0], dx, dx)
    np.testing.assert_allclose(m, mean, rtol=1e-12)
    np.testing.assert_allclose(c, ref, rtol=1e-12)
    m, c = DU.mean_and_cov(x, w)
    assert m.shape == (4, 3) and c.shape == (4, 3, 3)
    with pytest.raises(ValueError):
        DU.mean_and_cov(x, w[0, :-1])
    with pytest.raises(ValueError):
        DU.mean_and_cov(x[:, 0], w[0])


def test_quantile_types_and_checks(oracle_ops):
    rng = np.random.default_rng(2)
    x, w = rng.standard_normal(30), rng.random(30)
    got = DU.quantile(x, [0.1, 0.5], weights=w)
    assert isinstance(got, list) and len(got) == 2
    un = DU.quantile(x, [0.1, 0.5])
    assert isinstance(un, np.ndarray)
    np.testing.assert_array_equal(un, np.percentile(x, [10., 50.]))
    with pytest.raises(ValueError, match='between 0. and 1.'):
        DU.quantile(x, [1.5], weights=w)
    with pytest.raises(ValueError, match='between 0. and 1.'):
        DU.quantile(x, -0.1)
    with pytest.raises(ValueError, match='Dimension mismatch'):
        DU.quantile(x, 0.5, weights=w[:-1])


def test_posterior_realisations_checks(oracle_ops, gold):
    res = golden_res(gold, 'host')
    with pytest.raises(ValueError, match='not valid'):
        DU.posterior_realisations(res, 2, 1, error='bootstrap')
    bare = Results({k: res[k] for k in res.keys() if k != 'samples'})
    with pytest.raises(ValueError, match='keep_samples'):
        DU.posterior_realisations(bare, 2, 1)
    empty = Results(res)
    empty['samples'] = np.empty((0, 3))
    with pytest.raises(ValueError, match='keep_samples'):
        DU.posterior_realisations(empty, 2, 1)
    nostrands = Results({k: res[k] for k in res.keys() if k not in ('samples_id', 'samples_it')})
    with pytest.raises(NotImplementedError):
        DU.posterior_realisations(nostrands, 2, 1, error='resample')
    q = [0.025, 0.5, 0.975]
    for error in ('jitter', 'resample'):
        o = DU.posterior_realisations(res, 3, 5, chain0=7, error=error, q=q)
        assert o['mean'].shape == (3, 3) and o['cov'].shape == (3, 3, 3) and o['quantiles'].shape == (3, 3, 3)
        assert set(o) >= {'logz', 'logzerr', 'h', 'kld'}
        assert 'quantiles' not in DU.posterior_realisations(res, 1, 5, error=error)

"""CPU tier of importance reweighting: the numpy restatement (oracle/reweight.py) against the reference's own
reweight_run and compute_integrals(reweight=) on its jitter_run / resample_run realisations (tests/golden/reweight.npz),
Results.importance_weights, and the argument checks and the logrwt bookkeeping of utils.reweight_run / jitter_run /
resample_run / unravel_run / merge_runs with the GPU calls replaced by the oracle."""
import os

import numpy as np
import pytest

from oracle import posterior as OP, reweight as OR
from dynesty_b200 import ops, utils as DU
from dynesty_b200.nested import Results, _integrate

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reweight.npz')
KEYS = ('logl', 'samples_id', 'samples_it', 'samples_n', 'logwt', 'logz', 'logvol', 'ncall_per_it', 'samples_batch',
        'samples')


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLDEN))


def golden_res(g, name):
    p = 'rw_%s_' % name
    r = Results({k: g[p + k] for k in KEYS if p + k in g})
    r['niter'] = int(g[p + 'niter'])
    r['information'] = np.zeros(len(r['logl']))
    if p + 'batch_bounds' in g:
        r['batch_bounds'] = [tuple(b) for b in g[p + 'batch_bounds']]
    return r


def _names(g):
    return [str(s) for s in g['rw_names']]


def assert_logwt(a, b, rtol):
    a, b = np.asarray(a), np.asarray(b)
    np.testing.assert_array_equal(np.isneginf(a), np.isneginf(b))
    f = np.isfinite(b)
    np.testing.assert_allclose(a[f], b[f], rtol=rtol, atol=0)


def test_fixture_is_small_and_complete(gold):
    assert os.path.getsize(GOLDEN) < 1 << 20
    assert set(_names(gold)) == {'host', 'dev', 'devnolive', 'dyn', 'hd', 'cut'}
    assert np.isneginf(gold['rw_cut_logp_new']).any() and np.isfinite(gold['rw_cut_logp_new']).any()


def test_oracle_reweight_run_matches_the_reference(gold):
    for name in _names(gold):
        p = 'rw_%s_' % name
        o = OR.reweight_run(gold[p + 'logl'], gold[p + 'logvol'], gold[p + 'logp_new'])
        assert_logwt(o['logwt'], gold[p + 'ref_logwt'], 1e-12)
        np.testing.assert_allclose(o['logz'], gold[p + 'ref_logz'], rtol=1e-12)
        np.testing.assert_allclose(o['logzerr'], gold[p + 'ref_logzerr'], rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(OR.importance_weights(o['logwt'], o['logz']), gold[p + 'ref_impw'], rtol=0,
                                   atol=1e-12)
        # the reference quirk: its reweighted run keeps the input's information, not the reweighted h
        assert np.array_equal(gold[p + 'ref_information'], gold[p + 'information'])


@pytest.mark.parametrize('error', ['jitter', 'resample'])
def test_oracle_realisations_match_the_reference(gold, error):
    seed, chain0, q = int(gold['rw_seed']), int(gold['rw_chain0']), gold['rw_q']
    for name in _names(gold):
        p = 'rw_%s_' % name
        res = golden_res(gold, name)
        logl = np.asarray(res['logl'], dtype=float)
        x = np.asarray(res['samples'], dtype=float)
        logrwt = gold[p + 'logp_new'] - logl
        wref, zref = gold[p + 'ref_logwt'], float(gold[p + 'ref_logz'][-1])
        rec = DU._strand_inputs(res)[1]
        for r in gold['rw_r']:
            k = p + ('j%d_' if error == 'jitter' else 's%d_') % r
            if error == 'jitter':
                o = OR.jitter_realisation(logl, DU.samples_n_of(res), seed, chain0 + r, logrwt, logwt_ref=wref,
                                          logz_ref=zref)
                w = np.exp(o["logwt"] - o["logz"][-1])
                s = OP.stats(x, w, q)
            else:
                o = OR.resample_realisation(*rec, seed, chain0 + r, logrwt, logwt_ref=wref, logz_ref=zref)
                np.testing.assert_array_equal(o['idx'], gold[k + 'idx'])
                W, w2, present = OR.resample_weights(*rec, seed, chain0 + r, logrwt)
                s = OP.stats(x, W, q, w2, present)
            assert_logwt(o['logwt'], gold[k + 'logwt'], 1e-12)
            last = [o['logz'][-1], np.sqrt(max(o['logzvar'][-1], 0.)), o['h'][-1], o['kld'][-1]]
            np.testing.assert_allclose(last, gold[k + 'last'], rtol=1e-10, atol=1e-12)
            assert np.isfinite(o['kld'][-1])
            d = np.sqrt(np.diag(gold[k + 'cov']))
            scale = (np.abs(x).max(axis=0) + x.std(axis=0)).max()
            np.testing.assert_allclose(s['mean'], gold[k + 'mean'], rtol=0, atol=1e-12 * scale)
            np.testing.assert_allclose(s['cov'] / np.outer(d, d), gold[k + 'cov'] / np.outer(d, d), rtol=0, atol=1e-10)
            np.testing.assert_allclose(s['quantiles'], gold[k + 'quant'], rtol=0, atol=1e-12 * scale)


def test_importance_weights_match_the_reference(gold):
    for name in _names(gold):
        p = 'rw_%s_' % name
        r = Results(logwt=gold[p + 'ref_logwt'], logz=gold[p + 'ref_logz'])
        np.testing.assert_allclose(r.importance_weights(), gold[p + 'ref_impw'], rtol=0, atol=1e-15)


def test_integrate_default_path_is_unchanged(gold):
    logl, logvol = gold['rw_host_logl'], gold['rw_host_logvol']
    a, b = _integrate(logl, logvol), _integrate(logl, logvol, reweight=None)
    for u, v in zip(a, b):
        assert np.array_equal(u, v)
    zero = _integrate(logl, logvol, reweight=np.zeros(len(logl)))
    for u, v in zip(a, zero):
        assert np.array_equal(u, v)


# ---- the Python API on the oracle backend
@pytest.fixture
def oracle_ops(monkeypatch):
    monkeypatch.setattr(ops, 'compute_integrals', lambda logl, logvol, logrwt=None, ctx=None:
                        OR.compute_integrals(logl, logvol, logrwt))
    for name in ('jitter_runs', 'resample_runs', 'jitter_posterior', 'resample_posterior'):
        monkeypatch.setattr(ops, name, (lambda f: lambda *a, ctx=None, **k: f(*a, **k))(getattr(OR, name)))


def test_reweight_run_matches_the_reference(oracle_ops, gold):
    for name in _names(gold):
        p = 'rw_%s_' % name
        res = golden_res(gold, name)
        new = DU.reweight_run(res, gold[p + 'logp_new'])
        assert_logwt(new['logwt'], gold[p + 'ref_logwt'], 1e-12)
        np.testing.assert_allclose(new['logzerr'], gold[p + 'ref_logzerr'], rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(new.importance_weights(), gold[p + 'ref_impw'], rtol=0, atol=1e-12)
        assert new['logvol'] is res['logvol'] and new['information'] is res['information']
        assert np.array_equal(new['logrwt'], gold[p + 'logp_new'] - res['logl'])
        assert 'logrwt' not in res


def test_reweight_run_checks(oracle_ops, gold):
    res = golden_res(gold, 'host')
    N = len(res['logl'])
    lp = gold['rw_host_logp_new']
    with pytest.raises(ValueError, match='exactly one'):
        DU.reweight_run(res)
    with pytest.raises(ValueError, match='exactly one'):
        DU.reweight_run(res, lp, model=object())
    with pytest.raises(ValueError, match='one value per sample'):
        DU.reweight_run(res, lp[:-1])
    with pytest.raises(ValueError, match='one value per sample'):
        DU.reweight_run(res, lp, logp_old=np.zeros(N + 1))
    for bad in (np.nan, np.inf):
        x = lp.copy()
        x[3] = bad
        with pytest.raises(ValueError, match='NaN or \\+inf'):
            DU.reweight_run(res, x)
    with pytest.raises(ValueError, match='-inf at every sample'):
        DU.reweight_run(res, np.full(N, -np.inf))
    nopos = Results(res)
    del nopos['samples']
    with pytest.raises(ValueError, match='keep_samples=False'):
        DU.reweight_run(nopos, model=object())
    # logp_old given: the reweight is logp_new - logp_old
    new = DU.reweight_run(res, lp + 1.0, logp_old=res['logl'] + 1.0)
    assert np.array_equal(new['logrwt'], (lp + 1.0) - (res['logl'] + 1.0))


def test_ops_refuse_a_bad_logrwt():
    with pytest.raises(ValueError, match='one value per sample'):
        ops._logrwt(np.zeros(3), 4)
    with pytest.raises(ValueError, match='NaN or \\+inf'):
        ops._logrwt(np.array([0.0, np.nan]), 2)
    assert ops._logrwt([0.0, -np.inf], 2).dtype == np.float64


def test_realisations_carry_the_reweight(oracle_ops, gold):
    res = golden_res(gold, 'host')
    new = DU.reweight_run(res, gold['rw_cut_logp_new'])
    logrwt = new['logrwt']
    j = DU.jitter_run(new, seed=5, chain=2)
    assert j['logrwt'] is logrwt
    o = OR.jitter_realisation(res['logl'], DU.samples_n_of(res), 5, 2, logrwt)
    assert_logwt(j['logwt'], o['logwt'], 0)
    np.testing.assert_array_equal(j['logzerr'], np.sqrt(np.maximum(o['logzvar'], 0)))
    np.testing.assert_array_equal(j['information'], o['h'])
    kj = DU.kld_error(new, seed=5, chain=2)
    assert np.all(np.isfinite(kj))
    s, idx = DU.resample_run(new, seed=5, chain=2, return_idx=True)
    assert np.array_equal(s['logrwt'], logrwt[idx])
    assert np.isneginf(s['logwt']).any()
    assert_logwt(s['logwt'], _integrate(res['logl'][idx], s['logvol'], reweight=logrwt[idx])[0], 0)
    kr = DU.kld_error(new, error='resample', seed=5, chain=2)
    assert np.all(np.isfinite(kr))
    # the summaries of the batched forms are those of the realisations
    jr = DU.jitter_realisations(new, 2, 5, chain0=1)
    np.testing.assert_array_equal(jr['logz'][1], j['logz'][-1])
    rr = DU.resample_realisations(new, 3, 5, chain0=0)
    np.testing.assert_allclose(rr['logz'][2], s['logz'][-1], rtol=1e-12)


def test_unravel_run_slices_and_integrates_the_reweight(gold):
    res = golden_res(gold, 'host')
    res['logrwt'] = gold['rw_host_logp_new'] - res['logl']
    ids = np.asarray(res['samples_id'])
    for strand in DU.unravel_run(res):
        sel = ids == strand['samples_id'][0]
        assert np.array_equal(strand['logrwt'], res['logrwt'][sel])
        assert np.array_equal(strand['logwt'], _integrate(strand['logl'], strand['logvol'],
                                                          reweight=res['logrwt'][sel])[0])


def test_merge_runs_refuses_reweighted_runs(oracle_ops, gold):
    a, b = golden_res(gold, 'dev'), golden_res(gold, 'devnolive')
    ra = DU.reweight_run(a, gold['rw_dev_logp_new'])
    with pytest.raises(ValueError, match='merge first, then reweight'):
        DU.merge_runs([ra, b])

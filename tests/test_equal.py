"""CPU tier of the equal-weight draws: the numpy restatement (oracle/equal.py) against the unmodified reference's
resample_equal (tests/golden/equal_ref.npz), what the scripted generator scripts, and the argument checks and the
renormalisation warning of utils.resample_equal / equal_realisations / Results.samples_equal with the GPU calls
replaced by the oracle."""
import os
import warnings

import numpy as np
import pytest

from oracle import equal as OE, philox, refshim
from dynesty_b200 import ops, utils as DU
from dynesty_b200.nested import Results

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'equal_ref.npz')


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLDEN))


def names(g):
    return [str(s) for s in g['eq_names']]


def test_fixture_covers_the_cases(gold):
    assert os.path.getsize(GOLDEN) < 1 << 20
    assert set(names(gold)) == {'doc', 'r1000', 'r70000', 'zeros', 'one', 'sum_hi', 'sum_lo'}
    assert [bool(gold[n + '_warned']) for n in ('sum_hi', 'sum_lo', 'doc', 'r70000')] == [True, True, False, False]
    np.testing.assert_array_equal(gold['doc_w'], [0.6, 0.2, 0.15, 0.05])


def test_oracle_reproduces_every_fixture(gold):
    seed = int(gold['eq_seed'])
    for n in names(gold):
        w = gold[n + '_w']
        o = OE.draw(w, len(w), seed, int(gold[n + '_chain']))
        np.testing.assert_array_equal(o['idx'], gold[n + '_idx'], err_msg=n)
        np.testing.assert_array_equal(o['counts'], np.bincount(gold[n + '_idx'], minlength=len(w)))
        assert o['wsum'] == np.cumsum(w)[-1]


def test_zero_weights_are_never_drawn_and_counts_round_m_w(gold):
    for n in ('zeros', 'one', 'r70000'):
        w = gold[n + '_w']
        cnt = np.bincount(gold[n + '_idx'], minlength=len(w))
        assert not cnt[w == 0].any()
        mw = len(w) * w / w.sum()
        assert np.all((cnt >= np.floor(mw) - 1e-9) & (cnt <= np.ceil(mw) + 1e-9)), n
    assert np.all(gold['one_idx'] == 137)


def test_scripted_generator_adds_only_permutation():
    own = {k for k in vars(OE.ScriptedEqualGenerator) if not k.startswith('__')}
    assert own == {'permutation'}
    g = OE.ScriptedEqualGenerator(5, 9)
    s = philox.ChainStream(5, 9)
    assert g.random() == s.uniform()
    x = np.arange(10) * 3
    np.testing.assert_array_equal(g.permutation(x), x[s.permutation(10)])
    assert g.tick == 2


@pytest.mark.skipif(not refshim.available(), reason='needs the reference copy (oracle/_ref)')
def test_reference_calls_only_random_and_permutation():
    U = refshim.import_reference().utils
    calls = []

    class Recording(OE.ScriptedEqualGenerator):
        def __getattribute__(self, name):
            if not name.startswith('_') and name != 'tick':
                calls.append(name)
            return super().__getattribute__(name)

    U.resample_equal(np.arange(7), np.full(7, 1 / 7), rstate=Recording(1, 2))
    assert calls == ['random', 'permutation']


@pytest.fixture
def oracle_ops(monkeypatch):
    def re(w, M, seed, chain0=0, x=None, counts=False, ctx=None):
        o = OE.resample_equal(w, M, seed, chain0)
        if x is not None:
            o['x'] = np.asarray(x)[o['idx']]
        return o

    def je(logl, samples_n, R, M, seed, chain0=0, approx=False, logwt_ref=None, logz_ref=None, x=None, counts=False,
           ctx=None):
        o = OE.jitter_equal(logl, samples_n, R, M, seed, chain0, approx, logwt_ref, logz_ref)
        if x is not None:
            o['x'] = np.asarray(x)[o['idx']]
        return o

    monkeypatch.setattr(ops, 'resample_equal', re)
    monkeypatch.setattr(ops, 'jitter_equal', je)


def test_resample_equal_matches_the_fixtures_and_warns(gold, oracle_ops):
    seed = int(gold['eq_seed'])
    for n in names(gold):
        w = gold[n + '_w']
        x = np.arange(len(w)) * 2.0
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter('always')
            got = DU.resample_equal(x, w, seed=seed, chain=int(gold[n + '_chain']))
        np.testing.assert_array_equal(got, 2.0 * gold[n + '_idx'])
        assert any('renormalized' in str(c.message) for c in caught) == bool(gold[n + '_warned']), n


def test_resample_equal_checks(oracle_ops):
    x = np.arange(4.0)
    for w in ([0.5, -0.1, 0.3, 0.3], [0.5, np.nan, 0.3, 0.2], [0.5, np.inf, 0.3, 0.2], [0.0] * 4):
        with pytest.raises(ValueError):
            DU.resample_equal(x, np.array(w), seed=1)
    with pytest.raises(ValueError):
        DU.resample_equal(x[:3], np.full(4, 0.25), seed=1)
    with pytest.raises(ValueError):
        DU.resample_equal(x, np.full((2, 2), 0.25), seed=1)


def test_rstate_gives_the_seed(oracle_ops):
    w = np.array([0.1, 0.2, 0.3, 0.4])
    a = DU.resample_equal(np.arange(4), w, rstate=np.random.default_rng(3))
    seed = int(np.random.default_rng(3).integers(1 << 63))
    np.testing.assert_array_equal(a, OE.draw(w, 4, seed, 0)['idx'])


def test_samples_equal_uses_importance_weights(oracle_ops):
    rng = np.random.default_rng(4)
    logwt = rng.normal(size=50)
    res = Results(dict(samples=rng.normal(size=(50, 3)), logwt=logwt, logz=np.r_[0.0, np.logaddexp.reduce(logwt)]))
    got = res.samples_equal(seed=11)
    idx = OE.draw(res.importance_weights(), 50, 11, 0)['idx']
    np.testing.assert_array_equal(got, res['samples'][idx])


def _record(n=40):
    rng = np.random.default_rng(8)
    logl = np.sort(rng.normal(size=n)) * 3
    samples_n = np.full(n, 10)
    logvol = -np.arange(1, n + 1) / 10.0
    wt = logl + logvol
    return Results(dict(logl=logl, samples_n=samples_n, logwt=wt, logz=np.logaddexp.accumulate(wt),
                        samples=rng.normal(size=(n, 2)), niter=n, nlive=10, logvol=logvol))


def test_equal_realisations_checks(oracle_ops):
    res = _record()
    with pytest.raises(ValueError):
        DU.equal_realisations(res, 2, 1, error='bootstrap')
    with pytest.raises(ValueError):
        DU.equal_realisations(res, 2, 1, of='logl')
    with pytest.raises(ValueError):
        DU.equal_realisations(res, 2, 1, of='blob')
    with pytest.raises(ValueError):
        DU.equal_realisations(res, 1 << 16, 1, nsamples=1 << 16)
    with pytest.raises(ValueError):
        DU.equal_realisations(res, 1000, 1, nsamples=1 << 20, of='samples')
    o = DU.equal_realisations(res, 3, 5, nsamples=17, of='samples')
    assert o['idx'].shape == (3, 17) and o['samples'].shape == (3, 17, 2)
    np.testing.assert_array_equal(o['samples'], res['samples'][o['idx']])
    ref = OE.jitter_equal(res['logl'], res['samples_n'], 3, 17, 5, 0, False, res['logwt'], res['logz'][-1])
    np.testing.assert_array_equal(o['idx'], ref['idx'])

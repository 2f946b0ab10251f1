"""GPU tier of the equal-weight draws: b2n_resample_equal against the unmodified reference's resample_equal
(tests/golden/equal_ref.npz) and against the numpy restatement (oracle/equal.py) across the kernels' block, unroll,
grid-stride and sort-segment edges; the counts property at N = 10^6; the realisation entries against
jitter_realisations / resample_realisations and the oracle on their weights; launch counts and refusals."""
import numpy as np
import pytest

from oracle import equal as OE, refshim
from dynesty_b200 import _lib, ops, utils as DU
from dynesty_b200.nested import Results
from test_equal import GOLDEN, names
from test_posterior import GOLDEN as POST_GOLDEN, golden_res

pytestmark = pytest.mark.gpu

EQ_CS_THREADS, EQ_THREADS, EQ_UNROLL, EQ_MAX_GRID = 128, 256, 8, 1 << 16


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope='module')
def post():
    return dict(np.load(POST_GOLDEN))


def test_reference_fixtures_exactly(gold):
    seed = int(gold['eq_seed'])
    for n in names(gold):
        w = gold[n + '_w']
        o = ops.resample_equal(w, len(w), seed, int(gold[n + '_chain']), counts=True)
        np.testing.assert_array_equal(o['idx'][0], gold[n + '_idx'], err_msg=n)
        np.testing.assert_array_equal(o['counts'][0], np.bincount(gold[n + '_idx'], minlength=len(w)))
        assert o['wsum'][0] == np.cumsum(w)[-1]


@pytest.mark.skipif(not refshim.available(), reason='needs the reference copy (oracle/_ref)')
def test_samples_equal_matches_the_reference(post):
    U = refshim.import_reference().utils
    res = golden_res(post, 'hd')
    for seed in (3, 41):
        ref = U.resample_equal(res['samples'], res.importance_weights(), rstate=OE.ScriptedEqualGenerator(seed, 0))
        np.testing.assert_array_equal(res.samples_equal(seed=seed), ref)


def weights(N, R, seed, kind='random'):
    rng = np.random.default_rng(seed)
    w = rng.exponential(size=(R, N)) * rng.random((R, N)) ** 2
    if kind == 'zeros':
        w[:, ::3] = 0.0
        w[:, -5:] = 0.0
        w[:, 0] = 0.0
    elif kind == 'dominant':
        w *= 1e-6
        w[:, N // 3] = 1.0
    return w


def check_oracle(w, M, seed, chain0, x=None):
    o = ops.resample_equal(w, M, seed, chain0, counts=True, x=x)
    ref = OE.resample_equal(w, M, seed, chain0)
    np.testing.assert_array_equal(o['idx'], ref['idx'])
    np.testing.assert_array_equal(o['counts'], ref['counts'])
    np.testing.assert_array_equal(o['wsum'], ref['wsum'])
    if x is not None:
        np.testing.assert_array_equal(o['x'], x[o['idx']])
    return o


@pytest.mark.parametrize('N', [1, 2, EQ_UNROLL - 1, EQ_UNROLL, EQ_UNROLL + 1, 255, 256, 257, 4099])
@pytest.mark.parametrize('mfac', [0.5, 1, 2.5])
def test_sizes_against_the_oracle(N, mfac):
    M = max(1, int(N * mfac))
    for kind in ('random', 'zeros', 'dominant'):
        if kind == 'zeros' and N < 3:
            continue
        w = weights(N, 3, N * 7 + M, kind)
        o = check_oracle(w, M, 5, 1000, x=np.arange(2.0 * N).reshape(N, 2))
        if kind == 'zeros':
            assert not o['counts'][w == 0].any()


@pytest.mark.parametrize('R', [1, 33, EQ_CS_THREADS - 1, EQ_CS_THREADS + 1, 1000])
def test_vectors_against_the_oracle(R):
    check_oracle(weights(777, R, R), 1001, 9, 1 << 40)


def test_sort_segments_and_grid_stride():
    for M in (EQ_THREADS - 1, EQ_THREADS, EQ_THREADS + 1, 4096, 70001):
        check_oracle(weights(300, 2, M), M, 12, 3)
    # counts: N x R threads beyond the grid of EQ_MAX_GRID CTAs (grid-stride); draws: R x M beyond it
    check_oracle(weights(EQ_MAX_GRID + 3, EQ_THREADS + 1, 1), 1000, 2, 0)
    check_oracle(weights(50, 3, 2), EQ_MAX_GRID * EQ_THREADS // 3 + 5, 2, 0)


def test_row_r_does_not_depend_on_R():
    w = weights(5000, 40, 3)
    a = ops.resample_equal(w, 3000, 7, 50, counts=True)
    for r in (0, 17, 39):
        one = ops.resample_equal(w[r], 3000, 7, 50 + r, counts=True)
        for k in ('idx', 'counts', 'wsum'):
            np.testing.assert_array_equal(one[k][0], a[k][r])


def test_counts_round_m_w_at_scale():
    N = 10 ** 6
    w = weights(N, 1, 11, 'dominant')[0]
    w[::7] = 0.0
    for M in (N, 3 * N + 1, N // 3):
        o = ops.resample_equal(w, M, 4, 0, counts=True)
        mw = M * w / w.sum()
        c = o['counts'][0]
        assert np.all((c >= np.floor(mw - 1e-6)) & (c <= np.ceil(mw + 1e-6)))
        assert c.sum() == M and not c[w == 0].any()
        assert np.array_equal(np.bincount(o['idx'][0], minlength=N), c)


def test_refusals():
    w = np.full((1, 10), 0.1)
    for bad in (-0.1, np.nan, np.inf):
        v = w.copy()
        v[0, 4] = bad
        with pytest.raises(ValueError):
            ops.resample_equal(v, 10, 1)
    with pytest.raises(ValueError):
        ops.resample_equal(np.zeros((1, 10)), 10, 1)
    with pytest.raises(ValueError):
        ops.resample_equal(w, 0, 1)
    ctx = _lib.default_context()
    idx = np.empty(16, dtype=np.int32)
    for N, M in ((10, 1 << 31), (1 << 31, 10)):         # refused before any output is written
        with pytest.raises(ValueError):
            ctx.check(ctx.lib.b2n_resample_equal(ctx.h, _lib.ptr(w), N, 1, M, 1, 0, None, 0, _lib.ptr(idx), None, None,
                                                 None))
    with pytest.raises(ValueError):
        ops.resample_equal(np.full((65536, 1), 1.0), 1, 1)
    # the context is usable after a refusal
    check_oracle(weights(10, 2, 0), 10, 1, 0)


def test_launch_count_is_fixed():
    ctx = _lib.default_context()
    counts = set()
    for N, R, M in ((1, 1, 1), (10, 3, 7), (200000, 64, 50000)):
        n0 = ctx.launch_count()
        ops.resample_equal(weights(N, R, 0), M, 1, 0, counts=True, ctx=ctx)
        counts.add(ctx.launch_count() - n0)
    assert len(counts) == 1, counts


def _near_boundary(pos, c, tol=1e-12):
    k = np.searchsorted(c, pos)
    d = np.full(len(pos), np.inf)
    for s in (k - 1, k):
        ok = (s >= 0) & (s < len(c))
        d[ok] = np.minimum(d[ok], np.abs(c[s[ok]] - pos[ok]))
    return d <= tol


def check_realisation(idx, W, M, seed, chain):
    """idx against the oracle's draw on the host-built weights W: exact except for draws whose position lies within
    1e-12 of a cumulative boundary (returns their count)."""
    ref = OE.draw(W, M, seed, OE.EQUAL_CHAIN0 + chain)
    near = _near_boundary(ref['pos'], ref['c'])[ref['perm']]
    np.testing.assert_array_equal(idx[~near], ref['idx'][~near])
    return int(near.sum())


@pytest.mark.parametrize('error', ['jitter', 'resample'])
def test_realisations(post, error):
    seed, chain0, R = 23, 100, 9
    nnear = 0
    for name in ('host', 'dyn', 'hd'):
        res = golden_res(post, name)
        N = len(res['logl'])
        fn = DU.jitter_realisations if error == 'jitter' else DU.resample_realisations
        o = DU.equal_realisations(res, R, seed, chain0, error=error, nsamples=N + 5)
        ref = fn(res, R, seed, chain0)
        for k in ('logz', 'logzerr', 'h', 'kld'):
            assert np.array_equal(o[k], ref[k]), (name, k)
        for r in (0, 4, R - 1):
            one = DU.equal_realisations(res, 1, seed, chain0 + r, error=error, nsamples=N + 5)
            for k in ('idx', 'wsum', 'logz', 'kld'):
                assert np.array_equal(one[k][0], o[k][r]), (name, r, k)
            if error == 'jitter':
                a = DU.jitter_realisations(res, 1, seed, chain0 + r, arrays=True)
                W = np.exp(a['logwt_arr'][0] - a['logz_arr'][0][-1])
            else:
                new, ix = DU.resample_run(res, seed, chain0 + r, return_idx=True)
                W = np.bincount(ix, weights=np.exp(new['logwt'] - new['logz'][-1]), minlength=N)
                assert not np.isin(o['idx'][r], np.setdiff1d(np.arange(N), ix)).any()
            nnear += check_realisation(o['idx'][r], W, N + 5, seed, chain0 + r)
    print('%s: draws within 1e-12 of a boundary: %d' % (error, nnear))


def test_reweighted_runs_carry_logrwt(post):
    res = golden_res(post, 'host')
    x = np.asarray(res['samples'])
    rw = Results(res)
    rw['logrwt'] = -0.5 * ((x - x.mean(axis=0)) ** 2).sum(axis=1)
    rw['logwt'] = np.asarray(res['logwt']) + rw['logrwt']
    rw['logz'] = np.logaddexp.accumulate(rw['logwt'])
    o = DU.equal_realisations(rw, 4, 6, 0)
    ref = DU.jitter_realisations(rw, 4, 6, 0, arrays=True)
    for k in ('logz', 'logzerr', 'h', 'kld'):
        assert np.array_equal(o[k], ref[k]), k
    plain = DU.equal_realisations(res, 4, 6, 0)
    assert not np.array_equal(plain['idx'], o['idx'])
    N = len(x)
    for r in range(4):
        check_realisation(o['idx'][r], np.exp(ref['logwt_arr'][r] - ref['logz_arr'][r][-1]), N, 6, r)


def test_gather_of_blob_and_samples(post):
    res = golden_res(post, 'dyn')
    N = len(res['logl'])
    res['blob'] = np.stack([np.arange(N) * 1.5, -np.arange(N) * 1.0], axis=1)
    for error in ('jitter', 'resample'):
        o = DU.equal_realisations(res, 3, 2, 0, error=error, of='blob', nsamples=700)
        np.testing.assert_array_equal(o['blob'], res['blob'][o['idx']])
        s = DU.equal_realisations(res, 3, 2, 0, error=error, of='samples', nsamples=700)
        np.testing.assert_array_equal(s['samples'], np.asarray(res['samples'])[s['idx']])
        np.testing.assert_array_equal(s['idx'], o['idx'])


def test_equal_mean_agrees_with_mean_and_cov(post):
    res = golden_res(post, 'hd')
    x = np.asarray(res['samples'])
    M = 200000
    for error in ('jitter', 'resample'):
        o = DU.equal_realisations(res, 4, 8, 0, error=error, nsamples=M, of='samples')
        p = DU.posterior_realisations(res, 4, 8, 0, error=error)
        for r in range(4):
            sd = np.sqrt(np.diag(p['cov'][r]) / M)
            assert np.all(np.abs(o['samples'][r].mean(axis=0) - p['mean'][r]) < 5 * sd + 1e-12), (error, r)

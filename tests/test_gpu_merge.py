"""GPU tier: b2n_merge_runs against the reference's own merge_runs (tests/golden/merge.npz) and against the numpy
restatement (oracle/merge.py) on records built to hit its boundaries -- totals around the quadrature's tile, a plateau
across a tile boundary, runs of one sample, base trees of 1 to 2000 runs with and without add-on runs -- its
reproducibility, and an ensemble of replicas merged into one run."""
import numpy as np
import pytest

from oracle import merge as OM
from dynesty_b200 import likelihoods as DL, ops, replicas, utils as DU
from test_jitter import JT_TILE
from test_merge import CASES, GOLDEN, check_against_reference, kernel_inputs

pytestmark = pytest.mark.gpu

ARRAYS = ('perm', 'samples_n', 'logvol', 'logwt', 'logz', 'logzvar', 'h')


@pytest.fixture(scope='module')
def gm():
    return dict(np.load(GOLDEN))


def build(sizes, nbase, seed, quant=None, edges=None):
    """Runs of the given sizes: ascending logl (rounded to multiples of `quant` when given: ties), counts of a device
    round's saw-tooth; add-on runs (index >= nbase) get low edges inside their range unless `edges` says otherwise."""
    rng = np.random.default_rng(seed)
    logl, n, le = [], [], []
    for r, m in enumerate(sizes):
        x = np.sort(rng.uniform(-30.0, 0.0, m))
        if quant:
            x = np.round(x / quant) * quant
        logl.append(x)
        K = int(rng.integers(1, 5))
        nl = int(rng.integers(max(K, 2), 60))
        n.append(nl - (np.arange(m) % K))
        le.append(-np.inf if r < nbase else float(x[0] - rng.uniform(0, 2)))
    if edges is not None:
        le = list(edges)
    return np.concatenate(logl), np.concatenate(n).astype(np.int64), np.r_[0, np.cumsum(sizes)], nbase, np.array(le)


def check_against_oracle(args):
    o = ops.merge_runs(*args)
    q = OM.merge_runs(*args)
    assert np.array_equal(o['perm'], q['perm'])
    assert np.array_equal(o['samples_n'], q['samples_n'])
    np.testing.assert_allclose(o['logvol'], q['logvol'], rtol=0, atol=1e-12)
    np.testing.assert_allclose(np.exp(o['logwt'] - o['logz'][-1]), np.exp(q['logwt'] - q['logz'][-1]), rtol=0,
                               atol=1e-12)
    np.testing.assert_allclose(o['logz'], q['logz'], rtol=0, atol=1e-10)
    np.testing.assert_allclose(o['h'], q['h'], rtol=0, atol=1e-10)
    np.testing.assert_allclose(o['logzvar'], q['logzvar'], rtol=1e-9, atol=1e-12)
    for k in ('logz', 'logzerr', 'h'):
        assert abs(o[k + '_end'] - q[k + '_end']) < 1e-10, k
    return o


@pytest.mark.parametrize('case', CASES)
def test_kernel_against_reference(gm, case):
    check_against_reference(gm, case, ops.merge_runs(*kernel_inputs(gm, case)))


def _boundary_records():
    T = JT_TILE
    out = {}
    for tag, N in (('Tm1', T - 1), ('T', T), ('Tp1', T + 1)):
        a = N // 3
        out['total_' + tag] = build([a, a, N - 2 * a], 3, 1)
    # a plateau of 80 equal logl at merged positions 960..1039, across the tile boundary at 1024
    A = np.r_[np.linspace(-20, -1, 480), np.zeros(40), np.linspace(1, 5, 80)]
    out['plateau'] = (np.r_[A, A], np.full(1200, 200, dtype=np.int64), np.array([0, 600, 1200]), 2, np.full(2, -np.inf))
    out['len1'] = build([1, 1, 5, 1, 1, 1, 7], 4, 2)
    out['ties'] = build([300, 200, 500, 100, 40], 3, 3, quant=0.5)
    for nbase in (1, 2, 3, 5, 64, 2000):
        for nadd in (0, 3):
            sizes = list(np.random.default_rng(nbase).integers(1, 12, nbase + nadd))
            out['nbase%d_add%d' % (nbase, nadd)] = build(sizes, nbase, 10 + nbase + nadd)
    return out


BOUNDARY = _boundary_records()


@pytest.mark.parametrize('name', sorted(BOUNDARY))
def test_kernel_against_oracle_at_boundaries(name):
    check_against_oracle(BOUNDARY[name])


def test_boundary_records_hit_the_boundaries():
    lp = BOUNDARY['plateau'][0]
    perm, _ = OM.merge_order_counts(*BOUNDARY['plateau'][:4])
    pl = np.nonzero(lp[perm] == 0.0)[0]
    assert pl[0] < JT_TILE <= pl[-1]
    assert len(BOUNDARY['total_T'][0]) == JT_TILE


def test_two_calls_are_bit_identical():
    args = build(list(np.random.default_rng(5).integers(1, 4000, 37)), 33, 6, quant=0.01)
    a, b = ops.merge_runs(*args), ops.merge_runs(*args)
    for k in ARRAYS:
        assert a[k].tobytes() == b[k].tobytes(), k
    assert (a['logz_end'], a['logzerr_end'], a['h_end']) == (b['logz_end'], b['logzerr_end'], b['h_end'])
    s = ops.merge_runs(*args, arrays=False)
    assert np.array_equal(s['perm'], a['perm']) and s['logz_end'] == a['logz_end'] and 'logvol' not in s


def test_merged_replicas():
    """8 device-round replicas with strands merged into one run: the evidence within 3 sigma of the truth, a smaller
    error than every replica's, and resample_realisations on the merged run."""
    m = DL.gauss_test3d()
    outs, _ = replicas.run_replicas(m, range(500, 508), nlive=200, bound='multi', sample='rwalk', keep_results=True,
                                    strands=True, dlogz=0.01)
    runs = [o['results'] for o in outs]
    res = DU.merge_runs(runs)
    assert len(res['logl']) == sum(len(r['logl']) for r in runs)
    assert abs(res['logz'][-1] - m.logz_truth) < 3 * res['logzerr'][-1]
    assert all(res['logzerr'][-1] < r['logzerr'][-1] for r in runs)
    # the strand rule with every strand once gives the merged counts
    plan = DU.strand_plan(res)
    start = DU._pieces(res['logl'], plan)[0]
    diff = np.bincount(start, minlength=len(res['logl'])).astype(np.int64)
    diff[1:] -= 1
    np.testing.assert_array_equal(np.cumsum(diff), res['samples_n'])
    z = DU.resample_realisations(res, 64, 3)['logz']
    assert np.all(np.isfinite(z)) and abs(z.mean() - res['logz'][-1]) < 5 * max(z.std(), 1e-12)

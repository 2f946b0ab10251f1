"""CPU tier: merging runs.  The numpy restatement (oracle/merge.py) against the reference's own merge_runs (recorded in
tests/golden/merge.npz by oracle/make_golden_merge.py), the flat rule the base tree reduces to, and
dynesty_b200.utils.merge_runs with ops.merge_runs answered by the restatement: the merged Results, the strand ids and
batches, the dropped columns, the error cases, the strand rule on a merged ensemble and the unravel -> merge round
trip."""
import os

import numpy as np
import pytest

from oracle import jitter as OJ, merge as OM
from dynesty_b200 import ops, utils as DU
from dynesty_b200.nested import Results

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'merge.npz')
CASES = ['static3', 'static5', 'hostnolive', 'dynstatic', 'unravel_host', 'unravel_dyn', 'ties', 'single']


@pytest.fixture(scope='module')
def gm():
    return dict(np.load(GOLDEN))


@pytest.fixture
def oracle_merge(monkeypatch):
    """ops.merge_runs answered by the numpy restatement (same arguments)."""
    monkeypatch.setattr(ops, 'merge_runs', lambda *a, ctx=None, **k: OM.merge_runs(*a, **k))


def kernel_inputs(gm, case):
    p = 'c_%s_' % case
    return (gm[p + 'logl'], gm[p + 'samples_n'], gm[p + 'run_ptr'], int(gm[p + 'nbase']), gm[p + 'lowedge'])


def check_against_reference(gm, case, o):
    """Permutation and counts exact; logvol and the importance weights to 1e-12; the final logz, logzerr and
    information to 1e-10."""
    p = 'c_%s_' % case
    assert np.array_equal(o['perm'], gm[p + 'ref_perm'])
    assert np.array_equal(o['samples_n'], gm[p + 'ref_samples_n'])
    np.testing.assert_allclose(o['logvol'], gm[p + 'ref_logvol'], rtol=0, atol=1e-12)
    w = np.exp(o['logwt'] - o['logz'][-1])
    np.testing.assert_allclose(w, np.exp(gm[p + 'ref_logwt'] - gm[p + 'ref_logz'][-1]), rtol=0, atol=1e-12)
    for mine, ref in ((o['logz'][-1], 'logz'), (np.sqrt(abs(o['logzvar'][-1])), 'logzerr'),
                      (o['h'][-1], 'information')):
        assert abs(mine - gm[p + 'ref_' + ref][-1]) < 1e-10, ref


def inputs(gm, case):
    """The case's input runs as our Results."""
    p = 'c_%s_' % case
    out = []
    for i in range(int(gm[p + 'nin'])):
        q = p + 'in%d_' % i
        r = Results({k[len(q):]: gm[k] for k in gm if k.startswith(q) and k != q + 'batch_bounds'})
        for k in ('niter', 'nlive'):
            if k in r:
                r[k] = int(r[k])
        if q + 'batch_bounds' in gm:
            r['batch_bounds'] = [tuple(b) for b in gm[q + 'batch_bounds']]
        r['ncall'] = int(np.sum(r['ncall_per_it']))
        out.append(r)
    return out


@pytest.mark.parametrize('case', CASES)
def test_oracle_reproduces_reference(gm, case):
    check_against_reference(gm, case, OM.merge_runs(*kernel_inputs(gm, case)))


@pytest.mark.parametrize('case', ['static3', 'static5', 'hostnolive', 'unravel_host', 'ties'])
def test_flat_rule_equals_base_tree(gm, case):
    """Every low edge -inf: the pairwise tree is a stable sort by logl, and the count the sum of every run's count at
    its pointer (DESIGN.md section 15.2)."""
    logl, n, rp, nbase, le = kernel_inputs(gm, case)
    assert nbase == len(rp) - 1 and np.all(le == -np.inf)
    perm, nf = OM.flat_order_counts(logl, n, rp)
    assert np.array_equal(perm, gm['c_%s_ref_perm' % case])
    assert np.array_equal(nf, gm['c_%s_ref_samples_n' % case])


def test_fixture_cases_cover_the_paths(gm):
    """Odd runs carried up the tree, add-on runs, plateaus across runs, a single run."""
    assert len(gm['c_static5_run_ptr']) - 1 == 5 and len(gm['c_static3_run_ptr']) - 1 == 3
    rp, nb = gm['c_unravel_dyn_run_ptr'], int(gm['c_unravel_dyn_nbase'])
    assert len(rp) - 1 > nb >= 2 and np.all(gm['c_unravel_dyn_lowedge'][nb:] > -np.inf)
    logl, rp = gm['c_ties_logl'], gm['c_ties_run_ptr']
    shared = np.intersect1d(logl[:rp[1]], logl[rp[1]:])
    assert len(shared) > 5 and len(np.unique(logl[:rp[1]])) < rp[1]
    assert len(gm['c_single_run_ptr']) == 2


@pytest.mark.parametrize('case', CASES)
def test_utils_merge_runs_against_reference(gm, case, oracle_merge):
    res = DU.merge_runs(inputs(gm, case))
    p = 'c_%s_' % case
    if case == 'single':                            # returned as it is, as the reference does
        np.testing.assert_array_equal(res['logvol'], inputs(gm, case)[0]['logvol'])
        return
    np.testing.assert_array_equal(res['logl'], gm[p + 'ref_logl'])
    check_against_reference(gm, case, dict(perm=gm[p + 'ref_perm'], samples_n=res['samples_n'], logvol=res['logvol'],
                                           logwt=res['logwt'], logz=res['logz'], logzvar=res['logzerr'] ** 2,
                                           h=res['information']))
    assert res['niter'] == gm[p + 'ref_niter']
    assert res.get('nlive', -1) == gm[p + 'ref_nlive']


def test_ids_batches_and_columns(gm, oracle_merge):
    runs = inputs(gm, 'dynstatic')                  # a dynamic record (3 batches) and a static run
    res = DU.merge_runs(runs)
    perm = gm['c_dynstatic_ref_perm']
    n0 = len(runs[0]['logl'])
    nb0 = len(runs[0]['batch_bounds'])
    assert res['batch_bounds'] == list(runs[0]['batch_bounds']) + [(-np.inf, np.inf)]
    cat_batch = np.r_[runs[0]['samples_batch'], np.full(len(runs[1]['logl']), nb0)]
    np.testing.assert_array_equal(res['samples_batch'], cat_batch[perm])
    off = int(runs[0]['samples_id'].max()) + 1
    np.testing.assert_array_equal(res['samples_id'], np.r_[runs[0]['samples_id'], runs[1]['samples_id'] + off][perm])
    np.testing.assert_array_equal(res['samples_it'], np.r_[runs[0]['samples_it'], runs[1]['samples_it']][perm])
    np.testing.assert_array_equal(res['ncall_per_it'], np.r_[runs[0]['ncall_per_it'], runs[1]['ncall_per_it']][perm])
    assert res['ncall'] == runs[0]['ncall'] + runs[1]['ncall']
    assert res['eff'] == pytest.approx(100. * len(perm) / res['ncall'])
    assert np.array_equal(np.unique(res['samples_id']).size,
                          np.unique(runs[0]['samples_id']).size + np.unique(runs[1]['samples_id']).size)


def test_positions_gathered_or_emptied(oracle_merge):
    rng = np.random.default_rng(0)
    runs = []
    for s in range(3):
        n = np.r_[np.full(30, 5), np.arange(5, 0, -1)]
        rec = OJ.expected_record(n)
        u = rng.random((35, 2))
        runs.append(Results(logl=rec['logl'] + 1e-3 * s, samples_n=n, niter=30, ncall=35, samples_u=u, samples=2 * u,
                            ncall_per_it=np.ones(35, dtype=np.int64)))
    res = DU.merge_runs(runs)
    perm = OM.merge_runs(np.concatenate([r['logl'] for r in runs]), np.concatenate([r['samples_n'] for r in runs]),
                         [0, 35, 70, 105], 3)['perm']
    np.testing.assert_array_equal(res['samples_u'], np.concatenate([r['samples_u'] for r in runs])[perm])
    np.testing.assert_array_equal(res['samples'], 2 * res['samples_u'])
    assert 'samples_id' not in res and 'samples_scale' not in res
    runs[1] = Results(runs[1], samples_u=np.empty((0, 2)), samples=np.empty((0, 2)))   # keep_samples=False
    res = DU.merge_runs(runs)
    assert res['samples_u'].shape == (0, 2) and res['samples'].shape == (0, 2)
    runs[2] = Results(runs[2], samples_u=np.zeros((35, 3)), samples=np.zeros((35, 3)))
    with pytest.raises(ValueError, match='ndim'):
        DU.merge_runs(runs)


def test_strands_dropped(gm, oracle_merge):
    res = DU.merge_runs(inputs(gm, 'hostnolive'))   # one run without its final live points
    assert 'samples_id' not in res and 'samples_it' not in res
    with pytest.raises(NotImplementedError):
        DU.resample_realisations(res, 2, 1)
    res = DU.merge_runs(inputs(gm, 'unravel_host'))  # strands of a larger record
    assert 'samples_id' not in res


def test_errors(gm):
    """No run started from the prior; a run whose logl is not ascending (both refused before any device work)."""
    runs = inputs(gm, 'unravel_dyn')
    add = [r for r in runs if not np.any(r['samples_batch'] == 0)]
    assert add
    with pytest.raises(ValueError, match='prior'):
        DU.merge_runs(add)
    bad = inputs(gm, 'static3')
    bad[1] = Results(bad[1], logl=bad[1]['logl'][::-1].copy())
    with pytest.raises(ValueError, match='ascending'):
        DU.merge_runs(bad)


def test_ops_argument_checks():
    with pytest.raises(ValueError):
        ops.merge_runs([0., 1.], [1, 1], [0, 1, 2], 3)
    with pytest.raises(ValueError):
        ops.merge_runs([0., 1.], [1, 1], [0, 2, 2], 1)
    with pytest.raises(ValueError):
        ops.merge_runs([0., np.nan], [1, 1], [0, 2], 1)
    with pytest.raises(ValueError):
        ops.merge_runs([0., 1.], [1, 0], [0, 2], 1)


def test_grouping_one_base_one_addon():
    """One base run and one add-on run are both merged as base runs, in the given order (utils.py:1855-1857)."""
    a = Results(logl=np.zeros(2), samples_batch=np.array([1, 1]))
    b = Results(logl=np.zeros(2))
    assert DU.merge_order([a, b]) == ([0, 1], 2)
    assert DU.merge_order([b, a, a]) == ([0, 1, 2], 1)


def test_strand_rule_reproduces_merged_counts(gm, oracle_merge):
    """Every strand drawn once: the strand rule's live counts of the merged ensemble are its merged samples_n."""
    res = DU.merge_runs(inputs(gm, 'static5'))
    assert 'samples_id' in res
    plan = DU.strand_plan(res)
    start, pstr = DU._pieces(res['logl'], plan)
    N = len(res['logl'])
    diff = np.bincount(start, minlength=N).astype(np.int64)
    diff[1:] -= 1
    np.testing.assert_array_equal(np.cumsum(diff), res['samples_n'])


def test_unravel_merge_round_trip(gm, oracle_merge):
    """unravel_run of a run with one removal per iteration, merged back: its own counts and evidence."""
    runs = inputs(gm, 'hostnolive')
    host = runs[0]
    res = DU.merge_runs(DU.unravel_run(host))
    np.testing.assert_array_equal(res['samples_n'], host['samples_n'])
    np.testing.assert_array_equal(res['logl'], host['logl'])
    logz = OJ.integrate(host['logl'], np.cumsum(np.log(host['samples_n'] / (host['samples_n'] + 1.))))[1]
    assert abs(res['logz'][-1] - logz[-1]) < 1e-10

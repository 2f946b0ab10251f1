"""CPU tier: strands and resample_run.  The numpy restatement of the strand rule (oracle/resample.py) against the
reference's own resample_run / kld_error(error='resample') on records with one removal per iteration (recorded in
tests/golden/resample.npz by oracle/make_golden_resample.py), the identity resample on records with batch > 1, the
strand records of the host loop and of the oracle-backed device rounds, checkpoints, and the error cases."""
import os

import numpy as np
import pytest

from oracle import jitter as OJ, nsstrands, resample as OR
from dynesty_b200 import dynamic as D, likelihoods as DL, nested as N, ops, utils as DU
from dynesty_b200.nested import Results
from test_jitter import csrc_constant

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'resample.npz')
NAMES = ['host', 'dev', 'devnolive', 'dyn']
KEYS = ('logl', 'samples_id', 'samples_it', 'samples_n', 'logwt', 'logz', 'logvol', 'ncall_per_it', 'samples_batch')
RS_TILE = csrc_constant('b2n_resample.cu', 'RS_TILE')    # samples per tile of resample_scan_kernel


def host_record(slots, nlive, logl=None):
    """A static record of a host loop (one removal per iteration): the dead points come from the live slots `slots`
    in order, then the nlive final live points (slots 0..nlive-1).  Every point is born right above the point its
    slot lost before it.  logl: rising along the record (default: oracle.jitter.expected_record's); logwt and logz
    are those of the expected volumes."""
    slots = np.asarray(slots, dtype=np.int64)
    ids = np.r_[slots, np.arange(nlive)]
    its = np.zeros(len(ids), dtype=np.int64)
    last = {}
    for i, s in enumerate(ids):
        its[i] = last.get(s, -1) + 1
        last[s] = i
    n = np.r_[np.full(len(slots), nlive), np.arange(nlive, 0, -1)]
    rec = OJ.expected_record(n)
    if logl is not None:
        rec['logl'] = np.asarray(logl, dtype=float)
        rec['logwt'], rec['logz'] = OJ.integrate(rec['logl'], rec['logvol'])[:2]
    return Results(dict(rec, samples_id=ids, samples_it=its, niter=len(slots)))


def _records():
    """Records at resample_scan_kernel's tile boundaries (R = RS_TILE):
      long_run  nlive 3: two slots die twice, then slot 0 more than 2R times in a row, then the final live points --
                a realisation that does not draw slot 0 has whole tiles without a present sample after present ones;
      N_*       N = R - 1, R, R + 1 (nlive 400: the tile boundary falls in the add_live tail, which carries weight);
      N1        one sample, one strand."""
    T = RS_TILE
    rng = np.random.default_rng(3)
    out = {}
    slots = np.r_[[1, 2, 1, 2], np.zeros(2 * T + 300, dtype=np.int64)]
    out['long_run'] = host_record(slots, 3, logl=np.linspace(-5.0, 0.0, len(slots) + 3))
    for tag, N in (('Tm1', T - 1), ('T', T), ('Tp1', T + 1)):
        out['N_' + tag] = host_record(rng.integers(0, 400, N - 400), 400)
    out['N1'] = host_record([], 1)
    return out


RECORDS = _records()


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLDEN))


@pytest.fixture
def strand_ops(fake_ops, monkeypatch):
    """The oracle backend plus the strand entry points answered by its round loop, and ops.resample_runs answered by
    the numpy restatement."""
    nsstrands.install(monkeypatch, fake_ops._state)
    monkeypatch.setattr(ops, 'resample_runs', lambda *a, ctx=None, **k: OR.resample_runs(*a, **k))
    return fake_ops


def golden_res(g, name):
    p = 'rs_%s_' % name
    r = Results({k: g[p + k] for k in KEYS if p + k in g})
    r['niter'] = int(g[p + 'niter'])
    if p + 'batch_bounds' in g:
        r['batch_bounds'] = [tuple(b) for b in g[p + 'batch_bounds']]
    return r


def restated(res, m):
    """One realisation of `res` with multiplicities m (per strand of the plan): the piece rule from the births."""
    plan = DU.strand_plan(res)
    c = OR.live_counts(plan['start'], plan['strand'], m, plan['open'])
    return OR.realisation(res['logl'], plan['strand'], m, c, plan['end'], res['logwt'], res['logz'][-1])


@pytest.mark.parametrize('name', NAMES)
def test_restatement_equals_reference(gold, name):
    res = golden_res(gold, name)
    plan = DU.strand_plan(res)
    seed, chain0 = int(gold['rs_seed']), int(gold['rs_chain0'])
    for r in gold['rs_r']:
        q = 'rs_%s_r%d_' % (name, r)
        m = OR.draw_multiplicities(plan['base'], seed, chain0 + r)
        assert int(gold[q + 'ticks']) == 1 + int((~plan['base']).any())
        o = restated(res, m)
        assert np.array_equal(o['idx'], gold[q + 'idx'])
        assert np.array_equal(o['samples_n'], gold[q + 'samples_n'])
        for k in ('logvol', 'logwt', 'logz', 'h'):
            np.testing.assert_allclose(o[k], gold[q + k], rtol=1e-12, atol=1e-12, err_msg=k)
        np.testing.assert_allclose(o['kld'], gold[q + 'kld'], rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize('name', NAMES)
def test_resample_run_equals_reference(gold, name, strand_ops):
    res = golden_res(gold, name)
    seed, chain0 = int(gold['rs_seed']), int(gold['rs_chain0'])
    for r in gold['rs_r']:
        q = 'rs_%s_r%d_' % (name, r)
        new, idx = DU.resample_run(res, seed, chain0 + r, return_idx=True)
        assert np.array_equal(idx, gold[q + 'idx'])
        assert np.array_equal(new.samples_n, gold[q + 'samples_n'])
        assert np.array_equal(new.samples_id, res.samples_id[idx])
        np.testing.assert_allclose(new.logz, gold[q + 'logz'], rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(new.logzerr, gold[q + 'logzerr'], rtol=1e-12, atol=1e-12)
        kld = DU.kld_error(res, error='resample', seed=seed, chain=chain0 + r)
        np.testing.assert_allclose(kld, gold[q + 'kld'], rtol=1e-12, atol=1e-13)
        o = DU.resample_realisations(res, 1, seed, chain0 + r)
        np.testing.assert_allclose(o['logz'][0], new.logz[-1], rtol=1e-12)
        np.testing.assert_allclose(o['kld'][0], kld[-1], rtol=1e-12, atol=1e-13)


# ---------------------------------------------------------------------------------------------- records with batch > 1
def _static(add_live=True, batch=5, loop='device', seed=11, **kw):
    s = N.NestedSampler(DL.gauss_test3d(), nlive=40, bound='multi', sample='rwalk', walks=10, seed=seed)
    return s, s.run_nested(dlogz=0.5, loop=loop, batch=batch, add_live=add_live, strands=True, **kw)


def _dynamic(round_size=5, **kw):
    d = D.DynamicNestedSampler(DL.gauss_test3d(), nlive=40, bound='multi', sample='rwalk', walks=10, seed=13)
    return d, d.run_nested(dlogz_init=0.5, nlive_batch=30, maxbatch=2, n_effective=1e9, round_size=round_size,
                           strands=True, **kw)


def _identity(res):
    plan = DU.strand_plan(res)
    return restated(res, np.ones(len(plan['ids']), dtype=np.int64))


@pytest.mark.parametrize('add_live', [True, False])
def test_identity_resample_reproduces_device_rounds(strand_ops, add_live):
    _, res = _static(add_live)
    o = _identity(res)
    assert np.array_equal(o['idx'], np.arange(len(res.logl)))
    assert np.array_equal(o['samples_n'], res.samples_n)
    assert np.ptp(res.samples_n[:-40 if add_live else None]) == 4          # the saw-tooth of rounds of 5
    np.testing.assert_allclose(o['logz'], res.logz, rtol=1e-12, atol=1e-12)


def test_identity_resample_reproduces_merged_dynamic_record(strand_ops):
    _, res = _dynamic()
    assert res.nbatch == 2 and len(np.unique(res.samples_batch)) == 3
    o = _identity(res)
    assert np.array_equal(o['samples_n'], res.samples_n)
    np.testing.assert_allclose(o['logz'], res.logz, rtol=1e-12, atol=1e-12)


def test_reference_rule_misses_device_round_counts(strand_ops):
    _, res = _static(add_live=False)
    plan = DU.strand_plan(res)
    m = np.ones(len(plan['ids']), dtype=np.int64)
    ref = OR.reference_counts(res.logl, plan['strand'], np.full(len(res.logl), -np.inf), m)
    h = int(res.niter) // 2
    # every slot counted as occupied: nlive everywhere instead of the saw-tooth nlive - j
    assert (ref[:h] == 40).all() and (res.samples_n[:h] < 40).sum() >= h * 3 // 5
    assert np.array_equal(_identity(res)['samples_n'], res.samples_n)


@pytest.mark.parametrize('name', list(RECORDS))
def test_tile_edge_records_are_consistent(name):
    """The hand-built records: the piece rule with every multiplicity 1 gives back samples_n, and they sit where their
    names say."""
    res = RECORDS[name]
    plan = _check_strands(res, int(res.samples_n[int(res.niter)]))           # the first final live point: nlive
    assert np.array_equal(_identity(res)['samples_n'], res.samples_n)
    pp, ps = DU._piece_csr(res.logl, plan)
    assert np.array_equal(OR.csr_counts(plan['strand'], pp, ps, np.ones(len(plan['ids']), dtype=np.int64)),
                          res.samples_n)
    N = len(res.logl)
    if name == 'long_run':
        ids = res.samples_id
        run = np.nonzero(ids == 0)[0][:-1]
        assert len(run) > 2 * RS_TILE and np.array_equal(run, np.arange(4, 4 + len(run)))
        assert set(ids[:4]) == {1, 2}
    else:
        assert N == {'N_Tm1': RS_TILE - 1, 'N_T': RS_TILE, 'N_Tp1': RS_TILE + 1, 'N1': 1}[name]


# ---------------------------------------------------------------------------------------------- strand records
def _check_strands(res, nlive, add_live=True, batch=None):
    ids, its, logl = res.samples_id, res.samples_it, res.logl
    assert ids.dtype == np.int64 and its.dtype == np.int64 and len(ids) == len(logl) == len(its)
    assert ids.min() >= 0 and ids.max() < nlive
    for s in np.unique(ids):
        assert (np.diff(logl[ids == s]) > 0).all()
    if add_live:
        assert sorted(ids[-nlive:].tolist()) == list(range(nlive))
    plan = DU.strand_plan(res)
    assert (plan['birth'] < logl).all()
    if batch and batch > 1:
        # a point born in a device round entered above the round threshold: the logl of the round's last removal
        ndead = int(res.niter)
        born = its > 0
        assert (its[born] % batch == 0).all()
        np.testing.assert_array_equal(plan['birth'][born], logl[its[born] - 1])
        assert (res.samples_n[its[born] - 1] == nlive - batch + 1).all()
        assert ndead % batch == 0
    return plan


def test_host_loop_records_strands(strand_ops):
    _, res = _static(loop='host', batch=None)
    plan = _check_strands(res, 40)
    # one removal per iteration: a point enters right above the point it replaced
    its = res.samples_it
    assert (res.samples_id[its[its > 0] - 1] == res.samples_id[its > 0]).all()
    assert plan['base'].all()


@pytest.mark.parametrize('add_live', [True, False])
def test_device_rounds_record_strands(strand_ops, add_live):
    _, res = _static(add_live)
    _check_strands(res, 40, add_live, batch=5)


def test_host_phase_hands_strands_to_the_device(strand_ops):
    _, res = _static(device_init=False)
    _check_strands(res, 40)
    assert len(res.logl) > 40 and (res.samples_n[:-40] == 40).any()
    o = _identity(res)
    assert np.array_equal(o['samples_n'], res.samples_n)


def test_dynamic_batches_offset_their_strands(strand_ops):
    _, res = _dynamic()
    ids, b = res.samples_id, res.samples_batch
    for k in range(1, 3):
        assert ids[b == k].min() > ids[b < k].max()
    assert set(np.unique(ids[b == 0])) == set(range(40))
    for s in np.unique(ids):
        assert (np.diff(res.logl[ids == s]) > 0).all()
        assert len(np.unique(b[ids == s])) == 1
    plan = DU.strand_plan(res)
    assert (plan['birth'] < res.logl).all()
    lo = np.array([x[0] for x in res.batch_bounds])
    first = res.samples_it == 0
    np.testing.assert_array_equal(plan['birth'][first], lo[b[first]])
    assert plan['base'][plan['strand'][b == 0]].all()


def test_strands_off_by_default(strand_ops):
    s = N.NestedSampler(DL.gauss_test3d(), nlive=40, bound='multi', sample='rwalk', walks=10, seed=11)
    res = s.run_nested(dlogz=0.5, loop='device', batch=5)
    assert 'samples_id' not in res and 'samples_it' not in res


def test_checkpoint_resume_is_bit_identical_with_strands(strand_ops, tmp_path):
    ck = str(tmp_path / 'run.pkl')
    _, full = _static(seed=21)
    s = N.NestedSampler(DL.gauss_test3d(), nlive=40, bound='multi', sample='rwalk', walks=10, seed=21)
    with pytest.raises(KeyboardInterrupt):
        def stop(k):
            raise KeyboardInterrupt
        s.run_nested(dlogz=0.5, loop='device', batch=5, strands=True, checkpoint_file=ck, checkpoint_every=0.,
                     on_checkpoint=stop)
    assert 'strands' in N.NestedSampler.restore(ck)._dev_snap
    res = N.NestedSampler.restore(ck).run_nested(resume=True, checkpoint_file=ck)
    for k in ('logl', 'logz', 'samples_n', 'samples_id', 'samples_it'):
        assert np.array_equal(res[k], full[k]), k


# ---------------------------------------------------------------------------------------------- errors and wiring
def test_errors(strand_ops):
    _, res = _static()
    plain = Results({k: v for k, v in res.items() if k not in ('samples_id', 'samples_it')})
    for f in (lambda: DU.resample_run(plain), lambda: DU.kld_error(plain, error='resample'),
              lambda: D.stopping_function(plain, dict(n_mc=30, error='resample'))):
        with pytest.raises(NotImplementedError, match='strands=True'):
            f()
    nobase = Results(res, samples_batch=np.ones(len(res.logl), dtype=np.int64),
                     batch_bounds=[(-np.inf, np.inf), (-1e3, np.inf)])
    with pytest.raises(ValueError, match='initially sampled from the prior'):
        DU.resample_run(nobase)
    with pytest.raises(ValueError):
        DU.kld_error(res, error='bootstrap')


def test_unravel_run(strand_ops):
    _, res = _static(loop='host', batch=None)
    strands = DU.unravel_run(res)
    assert len(strands) == 40 and sum(len(s.logl) for s in strands) == len(res.logl)
    for s in strands:
        assert s.nlive == 1 and s.niter == len(s.logl) - 1 and (np.diff(s.logl) > 0).all()
        np.testing.assert_allclose(s.logvol[:-1], -np.log(2) * (1. + np.arange(s.niter)))


def test_dynamic_run_stops_on_the_resample_error(strand_ops):
    d = D.DynamicNestedSampler(DL.gauss_test3d(), nlive=40, bound='multi', sample='rwalk', walks=10, seed=4)
    res = d.run_nested(dlogz_init=0.5, nlive_batch=30, maxbatch=4, round_size=5,
                       stop_kwargs=dict(error='resample', pfrac=0., evid_thresh=0.5, n_mc=32))
    assert 'samples_id' in res and d.strands
    stops = [v[2] for v in d.stop_vals]
    assert stops[-1] <= 1 or d.batch == 4
    again = D.stopping_function(res, dict(error='resample', pfrac=0., evid_thresh=0.5, n_mc=32), seed=4,
                                chain0=d.stop_chain0(d.batch), return_vals=True)[1]
    assert again[2] == stops[-1]

"""GPU tier: strands recorded by the device rounds against the oracle's round loop, strand hand-over and checkpoints,
b2n_resample_runs against the numpy restatement (oracle/resample.py) and the reference's own realisations
(tests/golden/resample.npz), the resample scatter against the scatter of real replicas, and the dynamic sampler's
stop on the resample error."""
import os

import numpy as np
import pytest

from oracle import nsstrands, resample as OR
from dynesty_b200 import _lib, dynamic as D, likelihoods as DL, nested as N, ops, replicas, utils as DU
from dynesty_b200.nested import Results
from test_gpu_nsloop import _bound, _live, _models
from test_resample import RECORDS as TILE_RECORDS, RS_TILE, host_record

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'resample.npz')
SEED, CHAIN0 = 56432, 9000
KEYS = ('logl', 'samples_id', 'samples_it', 'samples_n', 'logwt', 'logz', 'logvol', 'ncall_per_it', 'samples_batch')


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLDEN))


def golden_res(g, name):
    p = 'rs_%s_' % name
    r = Results({k: g[p + k] for k in KEYS if p + k in g})
    r['niter'] = int(g[p + 'niter'])
    if p + 'batch_bounds' in g:
        r['batch_bounds'] = [tuple(b) for b in g[p + 'batch_bounds']]
    return r


# ---------------------------------------------------------------------------------------------- device strand records
@pytest.mark.parametrize('sampler,n,Nl,K,steps,rounds', [
    ('rwalk', 6, 64, 16, 30, 3), ('rwalk', 6, 64, 1, 30, 12), ('rslice', 5, 64, 8, 4, 3), ('slice', 4, 48, 12, 1, 2),
    ('unif', 4, 64, 16, 1, 3), ('unif', 4, 64, 1, 1, 10)])
def test_device_strands_match_oracle(sampler, n, Nl, K, steps, rounds):
    dm, om = _models('gauss', n)
    rng = np.random.default_rng(200 + n + K)
    u, v, l, groups = _live(om, n, Nl, rng)
    seed, chain0 = 56432, 1000
    o = nsstrands.StrandBatchNS(om, u, v, l, K, sampler, steps, seed, chain0=chain0, scale=0.7, logvol=-2.5, logz=-40.0,
                       loglstar=float(l.min()) - 0.5, ncall=500, dlogz=1e-6)
    ops.ns_create(dm.model_id(), Nl, n, K, ('rwalk', 'rslice', 'slice', 'unif').index(sampler), steps, seed,
                  chain0=chain0, dlogz=1e-6, dead_capacity=rounds * K + 5)
    try:
        ops.ns_set_state(u, v, l, -2.5, -40.0, float(l.min()) - 0.5, 500, 0.7)
        for r in range(rounds):
            b = _bound([o.live_u])
            o.bound = b
            ops.bound_set(b['axes'], b['ctrs'], b['ams'], b['logvols'])
            assert o.step()
            st = ops.ns_run(1, 0)
        assert st['it'] == rounds * K
        slot, it = ops.ns_get_strands(0, st['it'])
        oslot, oit = o.strand_arrays()
        assert slot.dtype == np.int32 and it.dtype == np.int64
        assert np.array_equal(slot, oslot) and np.array_equal(it, oit)
        assert np.array_equal(ops.ns_get_live_it(Nl), o.live_it)
        assert (it % K == 0).all()                                   # births at round ends only
    finally:
        ops.ns_destroy()


def test_unitcube_phase_strands_match_oracle():
    dm, om = _models('gauss', 4)
    rng = np.random.default_rng(8)
    Nl, K, n = 60, 6, 4
    u = rng.random((Nl, n))
    v = om.prior_transform(u)
    l = np.array([float(om.loglike(x)) for x in v])
    kw = dict(unit_cube_phase=True, first_min_ncall=2 * Nl, first_min_eff=25.0, it0=1)
    o = nsstrands.StrandBatchNS(om, u, v, l, K, 'rwalk', 9, 5, chain0=0, ncall=Nl, dlogz=1e-6, **kw)
    ops.ns_create(dm.model_id(), Nl, n, K, 0, 9, 5, chain0=0, dlogz=1e-6, **kw)
    try:
        ops.ns_set_state(u, v, l, 0.0, -1e300, -1e300, Nl, 1.0)
        # a hand-over: counts from a phase before the device, in the device's numbering
        start = -np.arange(Nl, dtype=np.int64)
        ops.ns_set_live_it(start)
        o.live_it = start.copy()
        nr = 0
        while o.step():
            nr += 1
        st = ops.ns_run(nr + 5, 0)
        assert st['rounds'] == nr >= 3
        slot, it = ops.ns_get_strands(0, st['it'])
        oslot, oit = o.strand_arrays()
        assert np.array_equal(slot, oslot) and np.array_equal(it, oit) and (it < 0).any()
        assert np.array_equal(ops.ns_get_live_it(Nl), o.live_it)
    finally:
        ops.ns_destroy()


def _static(seed=11, **kw):
    s = N.NestedSampler(DL.gauss_corr(6, 0.4, 5.0), nlive=200, bound='multi', sample='rwalk', walks=30,
                        queue_size=20, seed=seed)
    return s.run_nested(loop='device', batch=10, strands=True, **kw)


def _check_identity(res):
    plan = DU.strand_plan(res)
    m = np.ones(len(plan['ids']), dtype=np.int64)
    pp, ps = DU._piece_csr(res.logl, plan)
    assert np.array_equal(OR.csr_counts(plan['strand'], pp, ps, m), res.samples_n)


def test_host_phase_hands_strands_to_the_device():
    res = _static(device_init=False)
    nlive = 200
    assert (res.samples_n[:-nlive] == nlive).sum() > nlive                      # a host phase, then rounds
    ids, its = res.samples_id, res.samples_it
    assert sorted(ids[-nlive:].tolist()) == list(range(nlive))
    for s in np.unique(ids):
        assert (np.diff(res.logl[ids == s]) > 0).all()
    assert (DU.strand_plan(res)['birth'] < res.logl).all()
    _check_identity(res)


def test_checkpoint_resume_is_bit_identical_with_strands(tmp_path):
    ref = _static(seed=12)
    f = str(tmp_path / 'ckpt.pkl')
    s = N.NestedSampler(DL.gauss_corr(6, 0.4, 5.0), nlive=200, bound='multi', sample='rwalk', walks=30,
                        queue_size=20, seed=12)

    def stop(k):
        if k >= 3:
            raise KeyboardInterrupt

    with pytest.raises(KeyboardInterrupt):
        s.run_nested(loop='device', batch=10, strands=True, checkpoint_file=f, checkpoint_every=0., on_checkpoint=stop)
    r = N.NestedSampler.restore(f)
    assert len(r._dev_snap['strands'][0]) > 0
    res = r.run_nested(resume=True)
    for k in ('logl', 'logz', 'samples_u', 'samples_n', 'samples_id', 'samples_it'):
        assert np.array_equal(res[k], ref[k]), k
    _check_identity(res)


def test_strands_off_records_nothing():
    s = N.NestedSampler(DL.gauss_corr(6, 0.4, 5.0), nlive=200, bound='multi', sample='rwalk', walks=30,
                        queue_size=20, seed=11)
    res = s.run_nested(loop='device', batch=10)
    ref = _static()
    assert 'samples_id' not in res
    for k in ('logl', 'logz', 'samples_u', 'samples_n', 'logzerr'):
        assert np.array_equal(res[k], ref[k]), k


# ---------------------------------------------------------------------------------------------- the kernel
@pytest.fixture(scope='module')
def dyn_record():
    d = D.DynamicNestedSampler(DL.gauss_test3d(), nlive=200, bound='multi', sample='rwalk', walks=20, seed=11)
    return d.run_nested(dlogz_init=0.5, nlive_batch=150, maxbatch=2, n_effective=1e9, round_size=10, strands=True)


@pytest.fixture(scope='module')
def records(gold, dyn_record):
    out = {name: golden_res(gold, name) for name in ('host', 'dev', 'devnolive', 'dyn')}
    out['c2'] = Results(OR.synthetic_strand_record())
    out['dynrun'] = dyn_record
    return out


def _oracle(res, R, chain0=CHAIN0, seed=SEED, dtype=np.float64):
    plan = DU.strand_plan(res)
    pp, ps = DU._piece_csr(res['logl'], plan)
    return OR.resample_runs(res['logl'], plan['strand'], plan['base'], pp, ps, plan['end'], R, seed, chain0,
                            res['logwt'], res['logz'][-1], multiplicities=True, dtype=dtype)


def _compare(o, ref, rows=slice(None)):
    """Realisations `rows` of the kernel's output o against the oracle's ref (the same realisations, in order)."""
    assert np.array_equal(o['mult'][rows], ref['mult'])
    for k in ('logz', 'logzerr', 'h', 'kld'):
        np.testing.assert_allclose(o[k][rows], ref[k], rtol=1e-9, atol=1e-12, err_msg=k)


_cache = {}


@pytest.mark.parametrize('R', [1, 7, 128])
@pytest.mark.parametrize('name', ['host', 'dev', 'devnolive', 'dyn', 'c2', 'dynrun'])
def test_kernel_matches_oracle(records, name, R):
    res = records[name]
    if name not in _cache:
        _cache[name] = _oracle(res, 128)
    ref = _cache[name]
    o = DU.resample_realisations(res, R, SEED, CHAIN0, multiplicities=True)
    _compare(o, {k: v[:R] for k, v in ref.items()})


@pytest.mark.parametrize('name', list(TILE_RECORDS))
def test_kernel_matches_oracle_at_tile_edges(name):
    """Records at resample_scan_kernel's tile boundaries (tests/test_resample.py)."""
    res = TILE_RECORDS[name]
    _check_identity(res)
    ref = _oracle(res, 16)
    if name == 'long_run':
        # realisations without slot 0: whole tiles with no present sample between present ones; and without slot 1:
        # the first sample is absent
        assert (ref['mult'][:, 0] == 0).any() and (ref['mult'][:, 1] == 0).any()
    _compare(DU.resample_realisations(res, 16, SEED, CHAIN0, multiplicities=True), ref)


def test_kernel_matches_oracle_without_the_final_live_points():
    """The C2-shaped record cut before its add_live tail: the live points' open pieces run to the end of the record,
    across tiles."""
    full = OR.synthetic_strand_record()
    nd = int(full['niter'])
    res = Results({k: v[:nd] if isinstance(v, np.ndarray) else v for k, v in full.items()})
    plan = DU.strand_plan(res)
    assert plan['end'] is None and (plan['open'] < nd - RS_TILE).any()
    _compare(DU.resample_realisations(res, 4, SEED, CHAIN0, multiplicities=True), _oracle(res, 4))


def test_kernel_matches_oracle_on_c4_sized_record():
    """nlive 8000, K 400, ln X -> -100 (808k samples): numpy's float64 running sums are off by 2.7e-11 in kld (3.6e-4)
    against the same oracle in long double, the whole gap to the kernel; the long double oracle keeps the bars."""
    res = Results(OR.synthetic_strand_record(8000, 400, lnx_end=-100.))
    _compare(DU.resample_realisations(res, 2, SEED, CHAIN0, multiplicities=True), _oracle(res, 2, dtype=np.longdouble))


def test_kernel_matches_oracle_at_stream_limits():
    """Chain ids crossing into their high word, a seed with bits above 32 set, and the largest R on a one-tile record;
    R = 65536 is refused before anything is launched."""
    res = host_record(np.random.default_rng(5).integers(0, 20, 200), 20)
    _compare(DU.resample_realisations(res, 4, SEED, 2 ** 32 - 2, multiplicities=True), _oracle(res, 4, 2 ** 32 - 2))
    seed = (0x9E3779B9 << 32) | 12345
    _compare(DU.resample_realisations(res, 3, seed, CHAIN0, multiplicities=True), _oracle(res, 3, CHAIN0, seed))
    o = DU.resample_realisations(res, 65535, SEED, CHAIN0, multiplicities=True)
    for r in (0, 65534):
        _compare(o, _oracle(res, 1, CHAIN0 + r), slice(r, r + 1))
    ctx = _lib.default_context()
    launches = ctx.launch_count()
    with pytest.raises(ValueError):
        DU.resample_realisations(res, 65536, SEED, CHAIN0)
    assert ctx.launch_count() == launches


def test_kernel_matches_reference_fixture(gold, records):
    for name in ('host', 'dev', 'devnolive', 'dyn'):
        o = DU.resample_realisations(records[name], int(gold['rs_r'].max()) + 1, SEED, CHAIN0)
        for r in gold['rs_r']:
            q = 'rs_%s_r%d_' % (name, r)
            np.testing.assert_allclose(o['logz'][r], gold[q + 'logz'][-1], rtol=1e-9)
            np.testing.assert_allclose(o['logzerr'][r], gold[q + 'logzerr'][-1], rtol=1e-9)
            np.testing.assert_allclose(o['h'][r], gold[q + 'h'][-1], rtol=1e-9)
            np.testing.assert_allclose(o['kld'][r], gold[q + 'kld'][-1], rtol=1e-9, atol=1e-12)


def test_realisation_does_not_depend_on_the_batch(records):
    res = records['c2']
    a = DU.resample_realisations(res, 8, 99, 5, multiplicities=True)
    b = DU.resample_realisations(res, 128, 99, 5, multiplicities=True)
    c = DU.resample_realisations(res, 8, 99, 5, multiplicities=True)
    d = DU.resample_realisations(res, 4, 99, 9, multiplicities=True)
    for k in a:
        assert np.array_equal(a[k], b[k][:8]) and np.array_equal(a[k], c[k]), k
        assert np.array_equal(d[k], a[k][4:]), k


def test_resample_run_is_realisation_zero(records):
    for name in ('dynrun', 'c2'):
        res = records[name]
        o = DU.resample_realisations(res, 3, 17, 40)
        new = DU.resample_run(res, seed=17, chain=40)
        np.testing.assert_allclose(new.logz[-1], o['logz'][0], rtol=1e-12)
        np.testing.assert_allclose(new.logzerr[-1], o['logzerr'][0], rtol=1e-9)
        kld = DU.kld_error(res, error='resample', seed=17, chain=40)
        np.testing.assert_allclose(kld[-1], o['kld'][0], rtol=1e-9, atol=1e-12)


def test_resample_scatter_matches_replica_scatter():
    """16 independent runs (unif, gauss_test3d) give the scatter of ln Z; device-round runs of the same configuration
    with strands give the resample std of ln Z (n_mc = 256), which estimates the same error."""
    outs, _ = replicas.run_replicas(DL.gauss_test3d(), range(300, 316), nlive=200, bound='multi', sample='unif',
                                    keep_results=True, dlogz=0.01)
    lnz = np.array([o['logz'] for o in outs])
    stds, errs = [], []
    for seed in range(400, 404):
        s = N.NestedSampler(DL.gauss_test3d(), nlive=200, bound='multi', sample='unif', seed=seed)
        res = s.run_nested(loop='device', dlogz=0.01, strands=True)
        z = DU.resample_realisations(res, 256, 5, 0)['logz']
        assert abs(z.mean() - res.logz[-1]) < 3 * z.std() / np.sqrt(len(z))
        stds.append(np.std(z))
    ratio = np.mean(stds) / np.std(lnz)
    assert 0.5 <= ratio <= 2.0, (ratio, np.mean(stds), np.std(lnz))


def test_dynamic_sampler_stops_on_the_resample_error():
    run = dict(dlogz_init=0.5, nlive_batch=100, round_size=5, maxbatch=4)
    mk = lambda: D.DynamicNestedSampler(DL.gauss_test3d(), nlive=100, bound='multi', sample='rwalk', walks=20, seed=21)
    # the ln Z scatter of this run's checks when it never stops: a threshold just above the smallest one
    probe = mk()
    probe.run_nested(stop_kwargs=dict(error='resample', pfrac=0., evid_thresh=1e-12, n_mc=32), **run)
    std = np.array([v[1] * 1e-12 for v in probe.stop_vals])
    thresh = std.min() * (1 + 1e-9)
    j = int(np.argmax(std <= thresh))
    kw = dict(error='resample', pfrac=0., evid_thresh=thresh, n_mc=32)
    d = mk()
    res = d.run_nested(stop_kwargs=kw, **run)
    assert d.strands and 'samples_id' in res and d.batch == j
    stops = [v[2] for v in d.stop_vals]
    assert stops[-1] <= 1 and all(s > 1 for s in stops[:-1])
    again = D.stopping_function(res, kw, seed=d.seed, chain0=d.stop_chain0(d.batch), return_vals=True)[1]
    assert again[2] == stops[-1]

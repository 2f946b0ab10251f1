"""GPU tier: b2n_jitter_runs against the numpy restatement (oracle/jitter.py) and the reference's own realisations
(tests/golden/jitter.npz), the stream layout's properties, the jitter scatter against the scatter of real replicas, and
the dynamic sampler's evidence stop."""
import os

import numpy as np
import pytest

from oracle import jitter as OJ
from dynesty_b200 import _lib, dynamic as D, likelihoods as DL, ops, replicas, utils as DU
from test_jitter import EDGES, JT_CHUNK, JT_TILE

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'jitter.npz')
SEED, CHAIN0 = 56432, 7000


@pytest.fixture(scope='module')
def jit():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope='module')
def dyn_record():
    """a merged record of a real dynamic run: baseline and two batches as device rounds"""
    d = D.DynamicNestedSampler(DL.gauss_test3d(), nlive=200, bound='multi', sample='rwalk', walks=20, seed=11)
    r = d.run_nested(dlogz_init=0.5, nlive_batch=150, maxbatch=2, n_effective=1e9, round_size=10)
    return r.logl, r.samples_n, r.logwt, r.logz[-1]


@pytest.fixture(scope='module')
def records(jit, dyn_record):
    logl, n = OJ.synthetic_record()
    logwt = -np.log(len(logl)) * np.ones(len(logl))
    return {'golden': (jit['jit_golden_logl'], jit['jit_golden_samples_n'], jit['jit_golden_logwt'],
                       jit['jit_golden_logz'][-1]),
            'c2': (logl, n, logwt, 0.0),
            'dyn': dyn_record}


_oracle_cache = {}


def _oracle(records, name, approx):
    if (name, approx) not in _oracle_cache:
        logl, n, wt, z = records[name]
        _oracle_cache[name, approx] = OJ.jitter_runs(logl, n, 128, SEED, CHAIN0, approx, wt, z, arrays=True)
    return _oracle_cache[name, approx]


def _compare(o, ref, rows=slice(None)):
    """Realisations `rows` of the kernel's output o against the oracle's ref (the same realisations, in order)."""
    for k in ('logz', 'logzerr', 'h', 'kld'):
        np.testing.assert_allclose(o[k][rows], ref[k], rtol=1e-9, atol=0, err_msg=k)
    for k in ('logvol', 'logz'):
        np.testing.assert_allclose(o[k + '_arr'][rows], ref[k + '_arr'], rtol=0, atol=1e-9, err_msg=k)
    # logwt is compared through the importance weights it defines: where ln t is within a few ulps of 0 (U next to 1),
    # numpy's dlogvol = diff(cumsum(ln t)) inside log1p(-exp(dlogvol)) has a large relative rounding error, which the
    # kernel (it uses ln t itself) does not; those samples carry no weight
    np.testing.assert_allclose(np.exp(o['logwt_arr'][rows] - o['logz'][rows, None]),
                               np.exp(ref['logwt_arr'] - ref['logz'][:, None]), rtol=0, atol=1e-12)
    np.testing.assert_allclose(o['kld_arr'][rows], ref['kld_arr'], rtol=0, atol=1e-9)


@pytest.mark.parametrize('R', [1, 7, 128])
@pytest.mark.parametrize('approx', [False, True])
@pytest.mark.parametrize('name', ['golden', 'c2', 'dyn'])
def test_kernel_matches_oracle(records, name, approx, R):
    logl, n, wt, z = records[name]
    o = ops.jitter_runs(logl, n, R, SEED, chain0=CHAIN0, approx=approx, logwt_ref=wt, logz_ref=z, arrays=True)
    ref = _oracle(records, name, approx)
    _compare(o, {k: v[:R] for k, v in ref.items()})
    # the summary-only path computes the same numbers
    s = ops.jitter_runs(logl, n, R, SEED, chain0=CHAIN0, approx=approx, logwt_ref=wt, logz_ref=z)
    for k in ('logz', 'logzerr', 'h', 'kld'):
        assert np.array_equal(s[k], o[k]), k


def _run_both(rec, R, approx, seed=SEED, chain0=CHAIN0, dtype=np.float64):
    """The kernel's R realisations (full arrays) and the oracle's (computed in dtype)."""
    args = (rec['logl'], rec['samples_n'], R, seed)
    kw = dict(chain0=chain0, approx=approx, logwt_ref=rec['logwt'], logz_ref=rec['logz'][-1], arrays=True)
    return ops.jitter_runs(*args, **kw), OJ.jitter_runs(*args, dtype=dtype, **kw)


@pytest.mark.parametrize('approx', [False, True])
@pytest.mark.parametrize('name', list(EDGES))
def test_kernel_matches_oracle_at_plan_edges(name, approx):
    """Records at the segment tiles of the scan kernels, the chunks of a stretch piece's scan and the tiles of flagged
    samples (tests/test_jitter.py): every carry from one piece to the next is used."""
    n, plan = EDGES[name]
    assert OJ.segment_plan(n, approx, JT_TILE) == plan[approx]
    # flat: numpy's float64 running sums over its 2^20 + 1 samples are off by 6.5e-10 in kld (0.44) against the same
    # oracle in long double, the whole gap to the kernel; the long double oracle keeps the bars
    o, ref = _run_both(OJ.expected_record(n), 2, approx, dtype=np.longdouble if name == 'flat' else np.float64)
    _compare(o, ref)


@pytest.mark.parametrize('approx', [False, True])
@pytest.mark.parametrize('shape', ['c2', 'c4'])
def test_kernel_matches_oracle_on_real_run_sizes(shape, approx):
    """A C2-shaped record run to ln X = -30 (more segments than a scan tile) and a C4-shaped one (nlive 8000, K 400,
    ln X -> -100: more segments than a tile and an add_live tail scanning several chunks); the oracle on two of 16
    realisations."""
    nlive, K, lnx = {'c2': (2000, 50, -30.), 'c4': (8000, 400, -100.)}[shape]
    logl, n = OJ.synthetic_record(nlive, K, lnx_end=lnx)
    nseg, scan = OJ.segment_plan(n, approx, JT_TILE)
    if not approx:
        assert nseg > JT_TILE and (shape == 'c2' or scan > JT_CHUNK)
    wt, lz = OJ.integrate(logl, np.cumsum(np.log(n / (n + 1.))))[:2]
    z = lz[-1]
    o = ops.jitter_runs(logl, n, 16, SEED, chain0=CHAIN0, approx=approx, logwt_ref=wt, logz_ref=z, arrays=True)
    for r in (0, 15):
        ref = OJ.jitter_runs(logl, n, 1, SEED, CHAIN0 + r, approx, wt, z, arrays=True)
        _compare(o, ref, slice(r, r + 1))


@pytest.mark.parametrize('approx', [False, True])
def test_kernel_matches_oracle_at_stream_limits(approx):
    """Chain ids crossing into their high word, a seed with bits above 32 set, and the largest R on a one-segment
    record; R = 65536 is refused before anything is launched."""
    rec = OJ.expected_record(np.r_[np.full(40, 30), np.arange(50, 0, -1)])
    _compare(*_run_both(rec, 4, approx, chain0=2 ** 32 - 2))
    _compare(*_run_both(rec, 3, approx, seed=(0x9E3779B9 << 32) | 12345))
    one = OJ.expected_record([6, 5, 4, 3, 2, 1])
    assert OJ.segment_plan(one['samples_n'], approx, JT_TILE)[0] == 1
    args = (one['logl'], one['samples_n'])
    kw = dict(approx=approx, logwt_ref=one['logwt'], logz_ref=one['logz'][-1], arrays=True)
    o = ops.jitter_runs(*args, 65535, SEED, chain0=CHAIN0, **kw)
    for r in (0, 65534):
        _compare(o, OJ.jitter_runs(*args, 1, SEED, chain0=CHAIN0 + r, **kw), slice(r, r + 1))
    ctx = _lib.default_context()
    launches = ctx.launch_count()
    with pytest.raises(ValueError):
        ops.jitter_runs(*args, 65536, SEED, chain0=CHAIN0, **kw)
    assert ctx.launch_count() == launches


@pytest.mark.parametrize('approx', [False, True])
def test_kernel_matches_reference_fixture(jit, approx):
    q = 'jit_golden_a%d_' % approx
    rs = jit['jit_r']
    o = ops.jitter_runs(jit['jit_golden_logl'], jit['jit_golden_samples_n'], int(rs.max()) + 1, int(jit['jit_seed']),
                        chain0=int(jit['jit_chain0']), approx=approx, logwt_ref=jit['jit_golden_logwt'],
                        logz_ref=jit['jit_golden_logz'][-1], arrays=True)
    for i, r in enumerate(rs):
        for k in ('logz', 'logzerr', 'h', 'kld'):
            np.testing.assert_allclose(o[k][r], jit[q + k][i][-1], rtol=1e-9, err_msg=k)
        for k in ('logvol', 'logz'):
            np.testing.assert_allclose(o[k + '_arr'][r], jit[q + k][i], rtol=0, atol=1e-9, err_msg=k)


def test_realisation_does_not_depend_on_the_batch(records):
    logl, n, wt, z = records['c2']
    a = ops.jitter_runs(logl, n, 8, 99, chain0=5, logwt_ref=wt, logz_ref=z, arrays=True)
    b = ops.jitter_runs(logl, n, 128, 99, chain0=5, logwt_ref=wt, logz_ref=z, arrays=True)
    c = ops.jitter_runs(logl, n, 8, 99, chain0=5, logwt_ref=wt, logz_ref=z, arrays=True)
    d = ops.jitter_runs(logl, n, 4, 99, chain0=9, logwt_ref=wt, logz_ref=z)
    for k in a:
        assert np.array_equal(a[k], b[k][:8]), k
        assert np.array_equal(a[k], c[k]), k
    for k in d:
        assert np.array_equal(d[k], a[k][4:]), k


def test_jitter_run_is_realisation_zero(records):
    logl, n, wt, z = records['dyn']
    from dynesty_b200.nested import Results
    res = Results(logl=logl, samples_n=n, logwt=wt, logz=np.full(len(logl), z), logzerr=np.zeros(len(logl)),
                  information=np.zeros(len(logl)))
    o = DU.jitter_realisations(res, 3, 17, chain0=40, arrays=True)
    new = DU.jitter_run(res, seed=17, chain=40)
    for k in ('logvol', 'logwt', 'logz'):
        assert np.array_equal(new[k], o[k + '_arr'][0]), k
    np.testing.assert_allclose(new.logzerr[-1], o['logzerr'][0], rtol=1e-9)
    np.testing.assert_allclose(new.information[-1], o['h'][0], rtol=1e-9)
    kld, new2 = DU.kld_error(res, seed=17, chain=40, return_new=True)
    assert np.array_equal(kld, o['kld_arr'][0]) and np.array_equal(new2.logz, new.logz)


def test_jitter_scatter_matches_replica_scatter():
    """16 independent runs (unif, gauss_test3d): the jitter std of ln Z of each run (n_mc = 256) against the scatter of
    the 16 ln Z values.  Both estimate the same statistical error, so their ratio is near 1."""
    outs, _ = replicas.run_replicas(DL.gauss_test3d(), range(300, 316), nlive=200, bound='multi', sample='unif',
                                    keep_results=True, dlogz=0.01)
    lnz = np.array([o['logz'] for o in outs])
    stds = [np.std(DU.jitter_realisations(o['results'], 256, 5, chain0=0)['logz']) for o in outs]
    ratio = np.mean(stds) / np.std(lnz)
    assert 0.5 <= ratio <= 2.0, (ratio, np.mean(stds), np.std(lnz))


def _dyn(seed=21):
    return D.DynamicNestedSampler(DL.gauss_test3d(), nlive=100, bound='multi', sample='rwalk', walks=20, seed=seed)


RUN = dict(dlogz_init=0.5, nlive_batch=100, round_size=5)


def test_dynamic_sampler_stops_on_the_evidence_error():
    # the ln Z scatter of this run's checks when it never stops: pick a threshold the scatter first falls below
    probe = _dyn()
    probe.run_nested(maxbatch=4, stop_kwargs=dict(pfrac=0., evid_thresh=1e-12, n_mc=64), **RUN)
    std = [v[1] * 1e-12 for v in probe.stop_vals]
    j = next(i for i in range(1, len(std)) if std[i] < min(std[:i]))
    thresh = 0.5 * (std[j] + min(std[:j]))
    kw = dict(pfrac=0., evid_thresh=thresh, n_mc=64)
    d = _dyn()
    res = d.run_nested(maxbatch=4, stop_kwargs=kw, **RUN)
    assert d.batch == j
    final = D.stopping_function(res, kw, seed=d.seed, chain0=d.stop_chain0(d.batch), return_vals=True)[1][2]
    assert final <= 1 and final == d.stop_vals[-1][2]
    before = _dyn()
    prev = before.run_nested(maxbatch=j - 1, n_effective=1e12, **RUN)
    val = D.stopping_function(prev, kw, seed=d.seed, chain0=d.stop_chain0(j - 1), return_vals=True)[1][2]
    assert val > 1 and val == d.stop_vals[-2][2]


def test_default_stop_is_unchanged():
    a = _dyn(seed=33)
    r0 = a.sample_initial(dlogz=RUN['dlogz_init'], round_size=RUN['round_size'])
    target = 1.6 * D.n_effective_of(r0)
    ra = a.run_nested(n_effective=target, maxbatch=5, **RUN)
    b = _dyn(seed=33)
    b.sample_initial(dlogz=RUN['dlogz_init'], round_size=RUN['round_size'])
    rb = b.run_nested(n_effective=target, maxbatch=5, stop_kwargs={'pfrac': 1.0, 'n_mc': 0}, **RUN)
    assert a.batch == b.batch
    for k in ('logl', 'logvol', 'logwt', 'logz', 'logzerr', 'samples_n', 'samples'):
        assert np.array_equal(ra[k], rb[k]), k

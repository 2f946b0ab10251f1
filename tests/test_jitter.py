"""CPU tier: run uncertainties from simulated prior volumes.  The numpy restatement (oracle/jitter.py) against the
reference's own jitter_run / kld_error / _find_decrease (recorded in tests/golden/jitter.npz by oracle/make_golden_jitter.py,
driven by ScriptedJitterGenerator on the same B2N streams; tests/golden/jitter_edges.npz for records at the kernel's piece
boundaries), the kernel's segment plan on those records, the stopping function's argument handling, and a dynamic run on
the oracle backend that stops on the evidence error."""
import os
import re
import warnings

import numpy as np
import pytest

from oracle import jitter as OJ, philox
from dynesty_b200 import dynamic as D, likelihoods as DL, ops, utils as DU
from dynesty_b200.nested import Results

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'golden', 'jitter.npz')
GOLDEN_EDGES = os.path.join(HERE, 'golden', 'jitter_edges.npz')
CSRC = os.path.join(os.path.dirname(HERE), 'dynesty_b200', 'csrc')


def csrc_constant(fname, name):
    """`constexpr int name = value;` of a kernel source: the records below are built from the kernels' own tile sizes,
    so that they keep straddling the boundaries when a size changes."""
    with open(os.path.join(CSRC, fname)) as f:
        m = re.search(r'constexpr\s+int\s+%s\s*=\s*(\d+)\s*;' % name, f.read())
    assert m, '%s not found in %s' % (name, fname)
    return int(m.group(1))


JT_TILE = csrc_constant('b2n_jitter.cu', 'JT_TILE')      # samples per segment, segments per scan tile
JT_CHUNK = csrc_constant('b2n_jitter.cu', 'JT_CHUNK')    # exponentials per step of a stretch piece's scan


def _cdiv(a, b):
    return -(-a // b)


def _edges():
    """Records at b2n_jitter_runs' piece boundaries: name -> (samples_n, {approx: segment_plan}).  T = JT_TILE,
    C = JT_CHUNK.
      pairs_*    [2, 1] repeated: that many two-sample stretches, one segment each (the scan kernels' tiles of T);
      flat       T^2 + 1 flagged samples: T + 1 segments in both modes;
      stretch_*  one stretch nstart, .., 1: a scan of nstart + 1 exponentials (chunks of C), pieces of T samples;
      run_*      a run of flagged samples (tiles of T) right before a stretch;
      n1, n2*    the smallest records."""
    T, C = JT_TILE, JT_CHUNK
    out = {}
    for tag, k in (('Tm1', T - 1), ('T', T), ('Tp1', T + 1), ('2Tp1', 2 * T + 1)):
        out['pairs_' + tag] = (np.tile([2, 1], k), {False: (k, 3), True: (_cdiv(2 * k, T), 0)})
    out['flat'] = (np.full(T * T + 1, 500), {False: (T + 1, 0), True: (T + 1, 0)})
    for tag, s in (('Cm1', C - 1), ('C', C), ('Cp1', C + 1), ('2C', 2 * C), ('8000', 8000)):
        out['stretch_' + tag] = (np.arange(s, 0, -1), {False: (_cdiv(s, T), s + 1), True: (_cdiv(s, T), 0)})
    for tag, L in (('Tm1', T - 1), ('T', T), ('Tp1', T + 1)):
        out['run_' + tag] = (np.r_[np.full(L, 100), np.arange(200, 0, -1)],
                             {False: (_cdiv(L, T) + 1, 201), True: (_cdiv(L + 200, T), 0)})
    out['n1'] = (np.array([7]), {False: (1, 0), True: (1, 0)})
    out['n2'] = (np.array([2, 1]), {False: (1, 3), True: (1, 0)})
    out['n2flat'] = (np.array([4, 4]), {False: (1, 0), True: (1, 0)})
    return out


EDGES = _edges()


@pytest.fixture(scope='module')
def jit():
    return dict(np.load(GOLDEN))


@pytest.fixture
def oracle_jitter(monkeypatch):
    """ops.jitter_runs answered by the numpy restatement (same arguments, same streams)."""
    monkeypatch.setattr(ops, 'jitter_runs', lambda *a, ctx=None, **k: OJ.jitter_runs(*a, **k))


def test_find_decrease_docstring_example():
    flag, nstart, bounds = OJ.find_decrease(np.array([3, 2, 1, 13, 13, 12, 23, 22]))
    assert flag.tolist() == [True, False, False, True, True, False, True, False]
    assert nstart.tolist() == [3, 13, 23]
    assert bounds.tolist() == [[0, 3], [4, 6], [6, 8]]


@pytest.mark.parametrize('name', ['golden', 'dyn'])
def test_stretch_plan_equals_reference(jit, name):
    p = 'jit_%s_' % name
    flag, nstart, bounds = OJ.find_decrease(jit[p + 'samples_n'])
    assert np.array_equal(flag, jit[p + 'flag'])
    assert np.array_equal(nstart, jit[p + 'nstart'])
    assert np.array_equal(bounds, jit[p + 'bounds'])
    # one tick-0 event plus one event per stretch; approx: the tick-0 event only
    assert np.all(jit[p + 'a0_ticks'] == 1 + len(nstart)) and np.all(jit[p + 'a1_ticks'] == 1)


@pytest.mark.parametrize('approx', [False, True])
@pytest.mark.parametrize('name', ['golden', 'dyn'])
def test_oracle_realisations_equal_reference(jit, name, approx):
    p = 'jit_%s_' % name
    q = p + 'a%d_' % approx
    rs = jit['jit_r']
    o = OJ.jitter_runs(jit[p + 'logl'], jit[p + 'samples_n'], int(rs.max()) + 1, int(jit['jit_seed']),
                       int(jit['jit_chain0']), approx, jit[p + 'logwt'], jit[p + 'logz'][-1], arrays=True)
    for i, r in enumerate(rs):
        for k in ('logz', 'logzerr', 'h', 'kld'):
            np.testing.assert_allclose(o[k][r], jit[q + k][i][-1], rtol=1e-12, atol=0, err_msg=k)
        for k in ('logvol', 'logwt', 'logz'):
            np.testing.assert_allclose(o[k + '_arr'][r], jit[q + k][i], rtol=1e-12, atol=1e-12, err_msg=k)
        np.testing.assert_allclose(o['kld_arr'][r], jit[q + 'kld'][i], rtol=0, atol=1e-13)


@pytest.mark.parametrize('name', list(EDGES))
def test_segment_plan_of_edge_records(name):
    n, plan = EDGES[name]
    for approx in (False, True):
        assert OJ.segment_plan(n, approx, JT_TILE) == plan[approx], approx


def test_segment_plan_of_synthetic_records():
    T = JT_TILE
    # [3, 2, 1 | 13 | 13, 12 | 23, 22]: stretches of 3, 2, 2 samples around one flagged sample
    assert OJ.segment_plan([3, 2, 1, 13, 13, 12, 23, 22], False, 2) == (5, 24)
    assert OJ.segment_plan([3, 2, 1, 13, 13, 12, 23, 22], True, 2) == (4, 0)
    # rounds of K (one stretch each, K < T), then the add_live tail nlive, .., 1 in pieces of T
    for (nlive, K, lnx), nrounds in (((2000, 50, -25.), 1000), ((2000, 50, -30.), 1200), ((8000, 400, -100.), 2000)):
        n = OJ.synthetic_record(nlive, K, lnx_end=lnx)[1]
        assert len(n) == nrounds * K + nlive
        assert OJ.segment_plan(n, False, T) == (nrounds + _cdiv(nlive, T), nlive + 1)
        assert OJ.segment_plan(n, True, T) == (_cdiv(len(n), T), 0)
    # the sizes a real run reaches straddle both boundaries: more than T segments, more than C exponentials
    assert OJ.segment_plan(OJ.synthetic_record(2000, 50, lnx_end=-30.)[1], False, T)[0] > T
    assert OJ.segment_plan(OJ.synthetic_record(8000, 400, lnx_end=-100.)[1], False, T)[1] > JT_CHUNK


def test_oracle_realisations_equal_reference_at_plan_edges():
    """The reference's own jitter_run / kld_error on two records at the kernel's piece boundaries (recorded by
    oracle/make_golden_jitter.py): more stretches than a scan tile holds, and a stretch scanning one exponential
    more than a chunk."""
    g = dict(np.load(GOLDEN_EDGES))
    for name in g['names']:
        p = 'edge_%s_' % name
        q = p + 'new_'
        o = OJ.jitter_runs(g[p + 'logl'], g[p + 'samples_n'], len(g['r']), int(g['seed']), int(g['chain0']), False,
                           g[p + 'logwt'], g[p + 'logz'][-1], arrays=True)
        for i in range(len(g['r'])):
            for k in ('logz', 'kld'):
                np.testing.assert_allclose(o[k][i], g[q + k][i][-1], rtol=1e-12, atol=0, err_msg=k)
            for k in ('logzerr', 'h'):
                np.testing.assert_allclose(o[k][i], g[q + k][i], rtol=1e-12, atol=0, err_msg=k)
            for k in ('logvol', 'logwt', 'logz'):
                np.testing.assert_allclose(o[k + '_arr'][i], g[q + k][i], rtol=1e-12, atol=1e-12, err_msg=k)
            np.testing.assert_allclose(o['kld_arr'][i], g[q + 'kld'][i], rtol=0, atol=1e-13)


def test_scripted_generator_beta_and_exponential_are_single_events():
    g = OJ.ScriptedJitterGenerator(7, 11)
    a = np.array([5, 3, 9])
    t = g.beta(a=a, b=1)
    assert g.tick == 1
    np.testing.assert_array_equal(t, philox.event_uniforms(7, 11, 0, 3) ** (1.0 / a))
    y = g.exponential(scale=1.0, size=4)
    assert g.tick == 2
    np.testing.assert_array_equal(y, -np.log(philox.event_uniforms(7, 11, 1, 4)))


def _res(jit, name='golden'):
    p = 'jit_%s_' % name
    logl, logwt, logz = jit[p + 'logl'], jit[p + 'logwt'], jit[p + 'logz']
    return Results(logl=logl, logwt=logwt, logz=logz, logzerr=np.full(len(logl), 0.25), samples_n=jit[p + 'samples_n'])


@pytest.mark.parametrize('args', [dict(pfrac=1.5), dict(pfrac=-0.1), dict(pfrac=0.5, evid_thresh=-1.),
                                  dict(pfrac=0.5, target_n_effective=-1), dict(n_mc=-1), dict(error='bogus')])
def test_stopping_function_argument_errors(jit, args):
    with pytest.raises(ValueError):
        D.stopping_function(_res(jit), args)


def test_stopping_function_without_realisations_uses_logzerr(jit, monkeypatch):
    def boom(*a, **k):
        raise AssertionError('no realisations for n_mc <= 1')
    monkeypatch.setattr(ops, 'jitter_runs', boom)
    res = _res(jit)
    neff = D.n_effective(res.logwt)
    for n_mc in (0, 1):
        stop, (sp, se, s) = D.stopping_function(res, dict(pfrac=0.3, evid_thresh=0.5, target_n_effective=200,
                                                          n_mc=n_mc, error='resample'), return_vals=True)
        assert se == 0.25 / 0.5 and sp == 200 / neff and s == 0.3 * sp + 0.7 * se and stop == (s <= 1.)
    # pfrac = 1 is the Kish criterion alone
    assert D.stopping_function(res, dict(target_n_effective=neff * 0.99)) is True
    assert D.stopping_function(res, dict(target_n_effective=neff * 1.01)) is False


def test_stopping_function_realisations(jit, oracle_jitter):
    res = _res(jit)
    with pytest.warns(UserWarning, match='small number of realizations'):
        _, (_, se, _) = D.stopping_function(res, dict(pfrac=0., evid_thresh=0.1, n_mc=8), seed=3, chain0=40,
                                            return_vals=True)
    lnz = OJ.jitter_runs(res.logl, res.samples_n, 8, 3, 40, True, res.logwt, res.logz[-1])['logz']
    assert se == np.std(lnz) / 0.1
    with pytest.raises(NotImplementedError):
        D.stopping_function(res, dict(n_mc=30, error='resample'))


def test_kld_error_error_argument(jit, oracle_jitter):
    res = _res(jit)
    with pytest.raises(NotImplementedError, match='samples_id'):
        DU.kld_error(res, error='resample')
    with pytest.raises(ValueError):
        DU.kld_error(res, error='bootstrap')
    kld, new = DU.kld_error(res, seed=int(jit['jit_seed']), chain=int(jit['jit_chain0']), return_new=True)
    np.testing.assert_allclose(kld, jit['jit_golden_a0_kld'][0], rtol=0, atol=1e-13)
    np.testing.assert_allclose(new.logz, jit['jit_golden_a0_logz'][0], rtol=1e-12)
    np.testing.assert_allclose(new.logzerr, jit['jit_golden_a0_logzerr'][0], rtol=1e-12)
    assert new.logl is res.logl


def test_dynamic_run_stops_on_the_evidence_error(fake_ops, oracle_jitter):
    """ln Z scatter of this run's checks: ~0.32, 0.31, 0.26, 0.25 -- a threshold of 0.28 stops before batch 3."""
    d = D.DynamicNestedSampler(DL.gauss_test3d(), nlive=80, bound='multi', sample='rwalk', walks=10, seed=4)
    with warnings.catch_warnings():
        warnings.simplefilter('error')
        res = d.run_nested(dlogz_init=0.5, nlive_batch=60, maxbatch=6, round_size=6,
                           stop_kwargs=dict(pfrac=0., evid_thresh=0.28, n_mc=32))
    stops = [v[2] for v in d.stop_vals]
    assert len(stops) == d.batch + 1 and d.batch >= 1
    assert all(s > 1 for s in stops[:-1]) and stops[-1] <= 1
    # the last check is reproducible from the recorded chain ids
    again = D.stopping_function(res, dict(pfrac=0., evid_thresh=0.28, n_mc=32), seed=4,
                                chain0=d.stop_chain0(d.batch), return_vals=True)[1]
    assert again[2] == stops[-1]

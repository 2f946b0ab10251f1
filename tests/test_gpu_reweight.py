"""GPU tier of importance reweighting: b2n_compute_integrals against the reference's reweight_run
(tests/golden/reweight.npz) and the numpy restatement (oracle/reweight.py) across its tile edges; the four realisation
entry points with a log-reweight (b2n_set_reweight) against the fixture and the oracle; bit identity with a zero
reweight, R independence and posterior / summary identity; -inf reweights; the pending-reweight rules; reweight_run
with a device model; and a seeded end-to-end run reweighted to another target."""
import math

import numpy as np
import pytest

from oracle import jitter as OJ, reweight as OR
from dynesty_b200 import _lib, likelihoods as DL, nested, ops, utils as DU
from dynesty_b200.likelihoods import DeviceModel
from test_reweight import GOLDEN, _names, assert_logwt, golden_res

pytestmark = pytest.mark.gpu

SUMMARY = ('logz', 'logzerr', 'h', 'kld')
RTOL = 1e-9


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLDEN))


def _reweighted(g, name):
    res = golden_res(g, name)
    return DU.reweight_run(res, g['rw_%s_logp_new' % name])


def test_compute_integrals_matches_the_reference(gold):
    for name in _names(gold):
        p = 'rw_%s_' % name
        new = _reweighted(gold, name)
        np.testing.assert_allclose(new.importance_weights(), gold[p + 'ref_impw'], rtol=0, atol=1e-12)
        np.testing.assert_allclose(new['logz'][-1], gold[p + 'ref_logz'][-1], rtol=1e-10)
        np.testing.assert_allclose(new['logzerr'][-1], gold[p + 'ref_logzerr'][-1], rtol=1e-10)
        assert_logwt(new['logwt'], gold[p + 'ref_logwt'], 1e-10)


@pytest.mark.parametrize('N', [1, 1023, 1024, 1025, 5000])
def test_compute_integrals_tile_edges(N):
    rng = np.random.default_rng(N)
    rec = OJ.expected_record(np.full(N, 50, dtype=np.int64))
    rw = rng.normal(0.0, 0.5, N)
    if N > 1:
        rw[rng.random(N) < 0.1] = -np.inf
        rw[-1] = 0.0
    for logrwt in (None, rw):
        got = ops.compute_integrals(rec['logl'], rec['logvol'], logrwt)
        ref = OR.compute_integrals(rec['logl'], rec['logvol'], logrwt)
        assert_logwt(got['logwt'], ref['logwt'], 1e-10)
        for k in ('logz', 'logzvar', 'h'):
            np.testing.assert_allclose(got[k], ref[k], rtol=1e-10, atol=1e-12, err_msg=k)


def _entry(error, res, R, chain0, seed, approx=False, posterior=False, logrwt='record'):
    """The realisation entry point of (error, posterior) on the record res, the reweight from the record or given."""
    rw = DU._logrwt(res) if isinstance(logrwt, str) else logrwt
    logl = np.asarray(res['logl'], dtype=float)
    zref = float(np.asarray(res['logz'])[-1])
    kw = dict(chain0=chain0, logwt_ref=res['logwt'], logz_ref=zref, logrwt=rw)
    if error == 'jitter':
        if posterior:
            return ops.jitter_posterior(logl, DU.samples_n_of(res), res['samples'], R, seed, approx=approx,
                                        q=[0.1, 0.5, 0.9], **kw)
        return ops.jitter_runs(logl, DU.samples_n_of(res), R, seed, approx=approx, **kw)
    rec = DU._strand_inputs(res)[1]
    if posterior:
        return ops.resample_posterior(*rec, res['samples'], R, seed, q=[0.1, 0.5, 0.9], **kw)
    return ops.resample_runs(*rec, R, seed, **kw)


@pytest.mark.parametrize('R', [1, 7, 128])
@pytest.mark.parametrize('error', ['jitter', 'resample'])
def test_realisations_match_the_fixture(gold, error, R):
    seed, chain0, q = int(gold['rw_seed']), int(gold['rw_chain0']), gold['rw_q']
    for name in _names(gold):
        new = _reweighted(gold, name)
        o = _entry(error, new, R, chain0, seed)
        post = DU.posterior_realisations(new, R, seed, chain0=chain0, error=error, q=q)
        x = np.asarray(new['samples'], dtype=float)
        scale = (np.abs(x).max(axis=0) + x.std(axis=0)).max()
        for r in gold['rw_r']:
            if r >= R:
                continue
            k = 'rw_%s_%s%d_' % (name, 'j' if error == 'jitter' else 's', r)
            got = [o[s][r] for s in SUMMARY]
            np.testing.assert_allclose(got, gold[k + 'last'], rtol=RTOL, atol=1e-11)
            np.testing.assert_allclose(post['mean'][r], gold[k + 'mean'], rtol=0, atol=RTOL * scale)
            d = np.sqrt(np.diag(gold[k + 'cov']))
            np.testing.assert_allclose(post['cov'][r] / np.outer(d, d), gold[k + 'cov'] / np.outer(d, d), rtol=0,
                                       atol=RTOL)
            np.testing.assert_allclose(post['quantiles'][r], gold[k + 'quant'], rtol=0, atol=RTOL * scale)


@pytest.mark.parametrize('R', [1, 7, 128])
def test_jitter_approx_matches_the_oracle(gold, R):
    new = _reweighted(gold, 'dyn')
    got = _entry('jitter', new, R, 40, 77, approx=True)
    ref = OR.jitter_runs(new['logl'], DU.samples_n_of(new), R, 77, 40, True, new['logwt'], float(new['logz'][-1]),
                         logrwt=new['logrwt'])
    for s in SUMMARY:
        np.testing.assert_allclose(got[s], ref[s], rtol=RTOL, atol=1e-11, err_msg=s)


@pytest.mark.parametrize('posterior', [False, True])
@pytest.mark.parametrize('error', ['jitter', 'resample'])
def test_zero_reweight_is_bit_identical(gold, error, posterior):
    res = golden_res(gold, 'hd')
    a = _entry(error, res, 9, 5, 123, posterior=posterior, logrwt=None)
    b = _entry(error, res, 9, 5, 123, posterior=posterior, logrwt=np.zeros(len(res['logl'])))
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), k


@pytest.mark.parametrize('error', ['jitter', 'resample'])
def test_r_independence_and_posterior_identity(gold, error):
    new = _reweighted(gold, 'dev')
    many = _entry(error, new, 16, 100, 9)
    one = _entry(error, new, 1, 111, 9)
    for s in SUMMARY:
        assert many[s][11] == one[s][0], s
    post = DU.posterior_realisations(new, 16, 9, chain0=100, error=error)
    summ = (DU.jitter_realisations if error == 'jitter' else DU.resample_realisations)(new, 16, 9, chain0=100)
    for s in SUMMARY:
        assert np.array_equal(post[s], summ[s]) and np.array_equal(summ[s], many[s]), s


def test_neg_inf_reweight_gives_zero_weights(gold):
    new = _reweighted(gold, 'cut')
    cut = np.isneginf(new['logrwt'])
    o = ops.jitter_runs(new['logl'], DU.samples_n_of(new), 8, 3, logwt_ref=new['logwt'],
                        logz_ref=float(new['logz'][-1]), arrays=True, logrwt=new['logrwt'])
    assert np.all(np.isneginf(o['logwt_arr'][:, cut])) and np.all(np.isfinite(o['logwt_arr'][:, ~cut]))
    assert np.all(np.isfinite(o['kld_arr'])) and np.all(np.isfinite(o['kld']))
    for error in ('jitter', 'resample'):
        p = _entry(error, new, 8, 3, 3, posterior=True)
        for s in SUMMARY + ('mean', 'cov'):
            assert np.all(np.isfinite(p[s])), (error, s)


def test_pending_reweight_rules(gold):
    ctx = _lib.default_context()
    res = golden_res(gold, 'host')
    logl, n = np.asarray(res['logl'], dtype=float), DU.samples_n_of(res)
    N = len(logl)
    rw = gold['rw_host_logp_new'] - logl
    plain = ops.jitter_runs(logl, n, 4, 1)
    given = ops.jitter_runs(logl, n, 4, 1, logrwt=rw)
    # consumed by the next realisation call, once
    ctx.set_reweight(_lib.ptr(rw), N)
    pending = ops.jitter_runs(logl, n, 4, 1)
    assert all(np.array_equal(pending[k], given[k]) for k in given)
    after = ops.jitter_runs(logl, n, 4, 1)
    assert all(np.array_equal(after[k], plain[k]) for k in plain)
    # refused and cleared by the three entry points that do not read it
    calls = (lambda: ops.merge_runs(logl, n, [0, N], 1),
             lambda: ops.weighted_stats(res['samples'], np.ones((1, N)), np.zeros(res['samples'].shape[1])),
             lambda: ops.compute_integrals(logl, res['logvol']))
    for call in calls:
        ctx.set_reweight(_lib.ptr(rw), N)
        with pytest.raises(NotImplementedError, match='log-reweight'):
            call()
        call()
        assert all(np.array_equal(a, b) for a, b in zip(ops.jitter_runs(logl, n, 4, 1).values(), plain.values()))
    # another N: refused, and cleared all the same
    ctx.set_reweight(_lib.ptr(rw), N - 1)
    with pytest.raises(ValueError):
        ops.jitter_runs(logl, n, 4, 1)
    assert all(np.array_equal(a, b) for a, b in zip(ops.jitter_runs(logl, n, 4, 1).values(), plain.values()))
    with pytest.raises(ValueError):
        ctx.set_reweight(_lib.ptr(np.array([0.0, np.nan])), 2)
    assert all(np.array_equal(a, b) for a, b in zip(ops.jitter_runs(logl, n, 4, 1).values(), plain.values()))


DIAG = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    double s = 0.0;
    for (int i = lane; i < n; i += 32) {
        const double d = v[i] - p[i];
        s = fma(p[n + i] * d, d, s);
    }
    s = b2n_warp_sum(s);
    return fma(-0.5, s, p[2 * n]);
}
'''


def test_reweight_run_with_a_device_model(gold):
    res = golden_res(gold, 'host')
    n = res['samples'].shape[1]
    user = DeviceModel.from_cuda(n, DIAG, params=np.r_[0.1 * np.ones(n), 0.8 * np.ones(n), -2.0], name='rw_diag',
                                 prior_kind=_lib.PRIOR_UNIFORM, prior_p0=-5.0, prior_p1=10.0)
    for m in (DL.gauss_corr(n, 0.2), user):
        a = DU.reweight_run(res, model=m)
        b = DU.reweight_run(res, logp_new=m.loglikelihood(res['samples']))
        for k in ('logwt', 'logz', 'logzerr', 'logrwt'):
            assert np.array_equal(a[k], b[k]), k


def test_end_to_end_reweight_to_another_target():
    old, target = DL.gauss_corr(3, rho=0.5), DL.gauss_corr(3, rho=0.0)
    assert old.logz_truth == target.logz_truth == pytest.approx(-3 * math.log(10))
    res = nested.NestedSampler(old, nlive=500, bound='multi', sample='rwalk', seed=4242).run_nested(
        dlogz=0.1, loop='device', batch=10)
    new = DU.reweight_run(res, model=target)
    sig = float(np.std(DU.jitter_realisations(new, 128, 99)['logz']))
    assert 0 < sig < 1
    assert abs(new['logz'][-1] - target.logz_truth) < 4 * sig, (new['logz'][-1], target.logz_truth, sig)

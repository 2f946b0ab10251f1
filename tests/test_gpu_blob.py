"""GPU: blobs of user models -- derived quantities saved with every sample (NestedSampler(..., blob=True)).

``b2n_model_blob`` is checked against numpy bit for bit (the blob formulas below are exact in float64) over the shapes
where its staging changes: ndim across one and two warps, blob rows shorter and longer than a warp, point counts of
0, 1 and one that is not a multiple of the warps per block, host and device pointers.  Then every run path that
saves samples: the identity blob (blob = v, the reference's tests/test_blob.py) must equal the samples exactly, a
derived blob must equal model.blob of the samples, and a run with blob=True must give the bits of the same run
without it in every other key."""
import math

import numpy as np
import pytest

from dynesty_b200 import _lib, dynamic, nested, replicas, utils
from dynesty_b200 import likelihoods as DL
from dynesty_b200.likelihoods import DeviceModel

pytestmark = pytest.mark.gpu

LIKE = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    double s = 0.0;
    for (int i = lane; i < n; i += 32) {
        const double d = v[i] - p[i];
        s = fma(d, d, s);
    }
    return -2.0 * b2n_warp_sum(s);
}
'''

# blob = v
IDENT = LIKE + r'''
__device__ void b2n_user_blob(const double* v, double* work, int n, const double* p, int lane, double* blob,
                              int nblob) {
    for (int i = lane; i < n; i += 32) blob[i] = v[i];
}
'''

# blob = (v[i] * v[(i + 1) % n] for i < n, logl)
DERIVED = LIKE + r'''
__device__ void b2n_user_blob(const double* v, double* work, int n, const double* p, int lane, double* blob,
                              int nblob) {
    const double l = b2n_user_loglike(v, work, n, p, lane);
    for (int i = lane; i < n; i += 32) blob[i] = v[i] * v[(i + 1) % n];
    if (lane == 0) blob[n] = l;
}
'''

# any nblob: column 0 = logl, column j % 5 == 4 left unwritten (NaN), else v[j % n] * (j + 1)
GENERIC = LIKE + r'''
__device__ void b2n_user_blob(const double* v, double* work, int n, const double* p, int lane, double* blob,
                              int nblob) {
    const double l = b2n_user_loglike(v, work, n, p, lane);
    for (int j = lane; j < nblob; j += 32) {
        if (j == 0) blob[0] = l;
        else if (j % 5 != 4) blob[j] = v[j % n] * (double)(j + 1);
    }
}
'''

# the registry's UNIFORM prior restated, lo = p[0, n), width = p[n, 2n)
PRIOR = r'''
__device__ void b2n_user_prior(const double* u, double* v, double* work, int n, const double* p, int lane) {
    for (int i = lane; i < n; i += 32) v[i] = fma(p[n + i], u[i], p[i]);
}
'''

H = 5.0


def _model(src, n, nblob, **kw):
    if 'prior_source' not in kw:
        kw.update(prior_kind=_lib.PRIOR_UNIFORM, prior_p0=-H, prior_p1=2 * H)
    return DeviceModel.from_cuda(n, src, params=np.linspace(-0.5, 0.5, n), nblob=nblob, **kw)


def _generic_ref(v, l, nblob):
    n = v.shape[1]
    out = np.full((len(v), nblob), np.nan)
    for j in range(nblob):
        if j == 0:
            out[:, 0] = l
        elif j % 5 != 4:
            out[:, j] = v[:, j % n] * float(j + 1)
    return out


def _same(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b, equal_nan=a.dtype.kind == 'f')
    return a == b


def _device_blob(model, v, nblob):
    """b2n_model_blob with device pointers (torch tensors on the context's device)."""
    import torch
    ctx = _lib.default_context()
    dev = 'cuda:%d' % ctx.device
    tv = torch.as_tensor(np.ascontiguousarray(v)).to(dev)
    tb = torch.full((len(v), nblob), -7.0, dtype=torch.float64, device=dev)
    ctx.set_pointer_mode(_lib.PTR_DEVICE)
    try:
        ctx.check(ctx.lib.b2n_model_blob(ctx.h, model.model_id(), _lib.ptr(tv), len(v), nblob, _lib.ptr(tb)))
    finally:
        ctx.set_pointer_mode(_lib.PTR_HOST)
    ctx.synchronize()
    return tb.cpu().numpy()


# ---- b2n_model_blob against numpy ---------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [3, 33, 64])
def test_model_blob_matches_numpy(n):
    rng = np.random.default_rng(n)
    for nblob in (1, 5, 40, 3 * n):
        m = _model(GENERIC, n, nblob)
        for M in (0, 1, 1001):
            v = rng.uniform(-H, H, (M, n))
            got = m.blob(v)
            assert got.shape == (M, nblob) and got.dtype == np.float64
            l = m.loglikelihood(v) if M else np.empty(0)
            ref = _generic_ref(v, l, nblob)
            np.testing.assert_array_equal(got, ref)               # bit for bit, NaN where left unwritten
            if M:
                assert np.array_equal(got[:, 0], l)                # b2n_user_loglike inside the blob: its own bits
                assert np.isnan(got[:, 4::5]).all()
                assert not np.isnan(np.delete(got, np.s_[4::5], axis=1)).any()
            np.testing.assert_array_equal(_device_blob(m, v, nblob), got)


def test_user_prior_blob_sees_v():
    n = 5
    pp = np.concatenate([np.full(n, -H), np.full(n, 2 * H)])
    m = _model(IDENT, n, n, prior_source=PRIOR, prior_params=pp)
    u = np.random.default_rng(2).random((300, n))
    v, _ = m.evaluate(u)
    assert np.array_equal(m.blob(v), v)
    res = nested.NestedSampler(m, nlive=100, sample='rwalk', seed=3, walks=20, blob=True).run_nested(
        loop='device', dlogz=0.5)
    assert np.array_equal(res['blob'], res['samples'])
    assert not np.array_equal(res['blob'], res['samples_u'])


# ---- static runs ----------------------------------------------------------------------------------------------------
_models_cache = {}


def _ident_derived(n=4):
    if n not in _models_cache:
        _models_cache[n] = (_model(IDENT, n, n), _model(DERIVED, n, n + 1))
    return _models_cache[n]


@pytest.mark.parametrize('loop', ['host', 'device'])
@pytest.mark.parametrize('sample', ['rwalk', 'rslice', 'slice', 'unif'])
def test_static_runs_save_the_blob(sample, loop):
    ident, derived = _ident_derived()
    kw = dict(nlive=100, bound='multi', sample=sample, seed=17)
    run = lambda m, blob: nested.NestedSampler(m, blob=blob, **kw).run_nested(loop=loop, dlogz=0.5)
    plain = run(ident, False)
    res = run(ident, True)
    assert 'blob' not in plain
    assert set(res) == set(plain) | {'blob'}
    for k in plain:
        assert _same(res[k], plain[k]), k
    assert res['blob'].shape == res['samples'].shape and res['blob'].dtype == np.float64
    assert np.array_equal(res['blob'], res['samples'])
    d = run(derived, True)
    assert d['blob'].shape == (len(d['samples']), 5)
    assert np.array_equal(d['blob'], derived.blob(d['samples']))
    assert np.array_equal(d['blob'][:, 4], d['logl'])


# ---- other run paths ------------------------------------------------------------------------------------------------
def test_dynamic_run_with_two_batches():
    ident, _ = _ident_derived()
    run = lambda blob: dynamic.DynamicNestedSampler(ident, nlive=100, sample='rwalk', seed=5, walks=20,
                                                    blob=blob).run_nested(maxbatch=2, nlive_batch=60, dlogz_init=0.5)
    plain, res = run(False), run(True)
    assert res['nbatch'] == 2
    assert np.array_equal(res['blob'], res['samples'])
    assert set(res) == set(plain) | {'blob'}
    for k in plain:
        assert _same(res[k], plain[k]), k


def _abort_at(k):
    def cb(i):
        if i >= k:
            raise KeyboardInterrupt
    return cb


def test_checkpoint_resume_is_bit_identical(tmp_path):
    _, derived = _ident_derived(6)
    mk = lambda: nested.NestedSampler(derived, nlive=400, bound='multi', sample='rwalk', queue_size=40, seed=11,
                                      walks=30, blob=True)
    ref = mk().run_nested(loop='device', batch=20)
    f = str(tmp_path / 'ckpt.pkl')
    s = mk()
    with pytest.raises(KeyboardInterrupt):
        s.run_nested(loop='device', batch=20, checkpoint_file=f, checkpoint_every=0., on_checkpoint=_abort_at(2))
    del s
    r = nested.NestedSampler.restore(f)
    assert r.blob and r.model.nblob == 7
    res = r.run_nested(resume=True)
    assert res.niter == ref.niter and res.ncall == ref.ncall
    for k in ('logl', 'samples', 'samples_u', 'logz', 'logzerr', 'blob'):
        assert np.array_equal(res[k], ref[k]), k
    assert np.array_equal(res['blob'], derived.blob(res['samples']))


@pytest.fixture(scope='module')
def replica_results():
    ident, _ = _ident_derived()
    outs, _ = replicas.run_replicas(ident, [1, 2, 3], nlive=100, sample='rwalk', max_in_flight=3, keep_results=True,
                                    sampler_kwargs=dict(blob=True, walks=20), dlogz=0.5, strands=True)
    return [o['results'] for o in outs]


def test_run_utilities_keep_the_blob(replica_results):
    res = replica_results[0]
    assert np.array_equal(res['blob'], res['samples'])
    new = utils.resample_run(res, seed=9, chain=2)
    assert len(new['blob']) == len(new['logl']) and np.array_equal(new['blob'], new['samples'])
    strands = utils.unravel_run(res)
    assert sum(len(s['blob']) for s in strands) == len(res['blob'])
    for s in strands:
        assert np.array_equal(s['blob'], s['samples'])
    merged = utils.merge_runs(replica_results)
    assert len(merged['blob']) == sum(len(r['logl']) for r in replica_results)
    assert np.array_equal(merged['blob'], merged['samples'])
    for new in (utils.jitter_run(res, seed=9, chain=2), utils.reweight_run(res, logp_new=0.5 * res['logl'])):
        assert np.array_equal(new['blob'], new['samples'])
    # a run without a blob merges without one
    no_blob = {k: v for k, v in replica_results[1].items() if k != 'blob'}
    assert 'blob' not in utils.merge_runs([replica_results[0], no_blob])


@pytest.mark.parametrize('error', ['jitter', 'resample'])
def test_posterior_of_the_identity_blob_is_that_of_the_samples(replica_results, error):
    res = replica_results[0]
    a = utils.posterior_realisations(res, 16, 123, chain0=40, error=error, q=[0.1, 0.5, 0.9])
    b = utils.posterior_realisations(res, 16, 123, chain0=40, error=error, q=[0.1, 0.5, 0.9], of='blob')
    assert set(a) == set(b)
    for k in a:
        assert _same(a[k], b[k]), k


def test_posterior_of_a_derived_blob_matches_jitter_run():
    _, derived = _ident_derived()
    res = nested.NestedSampler(derived, nlive=100, sample='rwalk', seed=29, walks=20, blob=True).run_nested(
        loop='device', dlogz=0.5)
    seed, c0, R = 77, 1000, 6
    o = utils.posterior_realisations(res, R, seed, chain0=c0, of='blob')
    assert o['mean'].shape == (R, 5) and o['cov'].shape == (R, 5, 5)
    for r in range(R):
        new = utils.jitter_run(res, seed, c0 + r)
        m, c = utils.mean_and_cov(res['blob'], np.exp(new['logwt'] - new['logz'][-1]))
        np.testing.assert_allclose(o['mean'][r], m, rtol=1e-12, atol=1e-12 * np.abs(m).max())
        np.testing.assert_allclose(o['cov'][r], c, rtol=0, atol=1e-12 * np.abs(c).max())


# ---- refusals -------------------------------------------------------------------------------------------------------
def test_refusals():
    ident, _ = _ident_derived()
    with pytest.raises(ValueError, match='model with blobs'):
        nested.NestedSampler(DL.gauss_corr(4), nlive=50, blob=True)
    plain = _model(LIKE, 4, 0)
    with pytest.raises(ValueError, match='model with blobs'):
        nested.NestedSampler(plain, nlive=50, blob=True)
    with pytest.raises(ValueError, match='keep_samples'):
        nested.NestedSampler(ident, nlive=50, blob=True).run_nested(loop='device', keep_samples=False)
    ctx = _lib.default_context()
    v = np.zeros((3, 4))
    out = np.empty((3, 4))

    def call(mid, M=3, nblob=4):
        ctx.check(ctx.lib.b2n_model_blob(ctx.h, mid, _lib.ptr(v), M, nblob, _lib.ptr(out)))

    with pytest.raises(ValueError, match='registry model'):
        call(DL.gauss_corr(4).model_id())
    with pytest.raises(ValueError, match='b2n_user_blob_kernel'):
        call(plain.model_id())
    with pytest.raises(ValueError, match='nblob >= 1'):
        call(ident.model_id(), nblob=0)
    with pytest.raises(ValueError, match='M >= 0'):
        call(ident.model_id(), M=-1)
    with pytest.raises(ValueError, match='shared memory'):
        call(ident.model_id(), nblob=1 << 20)
    call(ident.model_id(), M=0)                           # nothing to do
    call(ident.model_id())
    assert np.array_equal(out, v)

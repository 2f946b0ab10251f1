"""CPU tier: blobs of user models (DeviceModel.from_cuda(..., nblob=k), NestedSampler(..., blob=True)).

A program with blobs is the user translation unit compiled with B2N_USER_BLOB: it holds the extern "C" kernel
b2n_user_blob_kernel beside the 10 slot kernels, whose mangled names and SASS are those of the same source compiled
without it.  A source without b2n_user_blob is refused with a message naming it.  The argument rules, pickling and the
dynamic sampler's merge of two records are checked without a GPU."""
import os
import pickle
import shutil
import subprocess

import numpy as np
import pytest

from dynesty_b200 import _lib, build, dynamic, nested, utils
from dynesty_b200 import likelihoods as DL
from dynesty_b200 import usermodel as UM
from dynesty_b200.likelihoods import DeviceModel

DIAG = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    double s = 0.0;
    for (int i = lane; i < n; i += 32) {
        const double d = v[i] - p[i];
        s = fma(d, d, s);
    }
    return -0.5 * b2n_warp_sum(s);
}
'''

# blob = (logl, |v|^2)
BLOB = DIAG + r'''
__device__ void b2n_user_blob(const double* v, double* work, int n, const double* p, int lane, double* blob,
                              int nblob) {
    const double l = b2n_user_loglike(v, work, n, p, lane);
    double s = 0.0;
    for (int i = lane; i < n; i += 32) s = fma(v[i], v[i], s);
    s = b2n_warp_sum(s);
    if (lane == 0) {
        blob[0] = l;
        blob[1] = s;
    }
}
'''


@pytest.fixture(scope='module', autouse=True)
def lib():
    if not os.path.exists(_lib.LIBPATH):
        build.build()
    return _lib.load()


def _nvrtc_or_skip():
    try:
        return UM.nvrtc()
    except UM.UserModelCompileError as e:
        pytest.skip(str(e))


def _sass(cubin, tmp_path):
    """{kernel name: its SASS} of a cubin (cuobjdump)."""
    tool = os.path.join(UM.CUDA_HOME, 'bin', 'cuobjdump')
    if not os.path.exists(tool):
        tool = shutil.which('cuobjdump')
    if not tool:
        pytest.skip('cuobjdump not found')
    f = tmp_path / 'image.cubin'
    f.write_bytes(cubin)
    out = subprocess.run([tool, '-sass', str(f)], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in out.split('Function : ')[1:]:
        name, body = part.split('\n', 1)
        funcs[name.strip()] = body.strip()
    return funcs


def test_program_source_defines_the_switch():
    assert UM.program_source(DIAG, blob=False) == UM.program_source(DIAG)
    src = UM.program_source(BLOB, blob=True)
    assert src.startswith('#define B2N_USER_BLOB\n#include "b2n_user_kernels.cuh"\n#line 1 "user_likelihood.cu"\n')
    prior = '__device__ void b2n_user_prior(const double* u, double* v, double* w, int n, const double* p, int l) {}'
    src = UM.program_source(BLOB, prior, blob=True)
    assert src.startswith('#define B2N_USER_PRIOR\n#define B2N_USER_BLOB\n#include "b2n_user_kernels.cuh"\n')


def test_blob_program_has_the_kernel_and_the_same_slots(tmp_path):
    _nvrtc_or_skip()
    plain = UM.compile_user(BLOB)
    with_blob = UM.compile_user(BLOB, blob=True)
    assert with_blob is not plain and UM.compile_user(BLOB, blob=True) is with_blob     # memoised apart
    assert with_blob.exprs == plain.exprs == UM.kernel_exprs() and len(with_blob.exprs) == 10
    assert with_blob.lowered == plain.lowered
    assert b'b2n_user_blob_kernel' in with_blob.cubin
    assert b'b2n_user_blob_kernel' not in plain.cubin
    sp, sb = _sass(plain.cubin, tmp_path), _sass(with_blob.cubin, tmp_path)
    assert set(sb) - set(sp) == {'b2n_user_blob_kernel'}
    for low in plain.lowered:
        assert sb[low] == sp[low], low                  # the slot kernels do not change with B2N_USER_BLOB


def test_program_without_b2n_user_blob_is_refused_by_name():
    _nvrtc_or_skip()
    with pytest.raises(UM.UserModelCompileError, match='b2n_user_blob'):
        UM.compile_user(DIAG, blob=True)
    UM.compile_user(DIAG)                                # the same source without blobs compiles


def test_from_cuda_nblob_rules_and_pickling():
    for bad in (-1, 1.5, True):
        with pytest.raises(ValueError):
            DeviceModel.from_cuda(3, BLOB, nblob=bad)
    assert DeviceModel.from_cuda(3, DIAG).nblob == 0
    assert DL.gauss_corr(3).nblob == 0
    with pytest.raises(ValueError, match='no blob'):
        DeviceModel.from_cuda(3, DIAG).blob(np.zeros((2, 3)))
    m = DeviceModel.from_cuda(4, BLOB, params=np.arange(4.0), nblob=2, name='blob4')
    m._ids[12345] = (0, 1)
    r = pickle.loads(pickle.dumps(m))
    assert r._ids == {} and r.nblob == 2 and r.source == BLOB and r.name == 'blob4'
    np.testing.assert_array_equal(r.params, np.arange(4.0))


def _live(n, k=12):
    rng = np.random.default_rng(1)
    return rng.random((k, n)), rng.random((k, n)), rng.random(k)


def test_sampler_blob_refusals():
    with pytest.raises(ValueError, match='model with blobs'):
        nested.NestedSampler(DL.gauss_corr(3), nlive=12, live_points=_live(3), blob=True)
    with pytest.raises(ValueError, match='model with blobs'):
        nested.NestedSampler(DeviceModel.from_cuda(3, DIAG), nlive=12, live_points=_live(3), blob=True)
    m = DeviceModel.from_cuda(3, BLOB, nblob=2)
    s = nested.NestedSampler(m, nlive=12, sample='rwalk', live_points=_live(3), blob=True)
    with pytest.raises(ValueError, match='keep_samples'):
        s.run_nested(loop='device', keep_samples=False)
    assert pickle.loads(pickle.dumps(s)).blob is True   # a checkpoint keeps the flag


def test_live_points_may_carry_the_reference_blobs():
    m = DeviceModel.from_cuda(3, BLOB, nblob=2)
    u, v, l = _live(3)
    s = nested.NestedSampler(m, nlive=12, sample='rwalk', live_points=(u, v, l, np.zeros((12, 2))), blob=True)
    np.testing.assert_array_equal(s.live_u, u)
    np.testing.assert_array_equal(s.live_v, v)
    np.testing.assert_array_equal(s.live_logl, l)


def test_posterior_realisations_of_argument():
    res = dict(logl=np.arange(3.0), samples=np.zeros((3, 2)), logwt=np.zeros(3), logz=np.zeros(3))
    with pytest.raises(ValueError, match='of must be'):
        utils.posterior_realisations(res, 4, 1, of='samples_u')
    with pytest.raises(ValueError, match='blob=True'):
        utils.posterior_realisations(res, 4, 1, of='blob')


def test_merge_two_keeps_each_blob_row_with_its_sample():
    rng = np.random.default_rng(7)
    f = lambda v: np.stack([v.sum(1), (v * v).sum(1), v[:, 0]], 1)

    def rec(k, batch):
        logl = np.sort(rng.standard_normal(k))
        v = rng.standard_normal((k, 4))
        return dict(u=rng.random((k, 4)), v=v, logl=logl, n=np.full(k, 10, dtype=np.int64),
                    nc=np.ones(k, dtype=np.int64), scale=np.ones(k), batch=np.full(k, batch, dtype=np.int64),
                    blob=f(v))

    saved, new = rec(40, 0), rec(25, 1)
    out = dynamic.merge_two(saved, new, float(new['logl'][0]))
    assert out['blob'].shape == (65, 3)
    np.testing.assert_array_equal(out['blob'], f(out['v']))
    assert np.all(np.diff(out['logl']) >= 0)

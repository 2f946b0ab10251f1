"""CPU tier: user likelihoods (DeviceModel.from_cuda) compile for sm_90a without a GPU.

NVRTC runs on the CPU: the user translation unit (b2n_user_kernels.cuh + the user's source) must compile and
yield a mangled name for every kernel slot the library lists (b2n_user_kernel_exprs); a broken source must raise
with NVRTC's own message; a model with parameters must survive pickling (the device handles do not)."""
import os
import pickle

import numpy as np
import pytest

from dynesty_b200 import _lib, build
from dynesty_b200 import usermodel as UM
from dynesty_b200.likelihoods import DeviceModel

GAUSS_DIAG = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    double s = 0.0;
    for (int i = lane; i < n; i += 32) {
        const double d = v[i] - p[i];
        s = fma(p[n + i] * d, d, s);
    }
    return fma(-0.5, b2n_warp_sum(s), p[2 * n]);
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


def test_slots_are_the_library_list():
    exprs = UM.kernel_exprs()
    assert len(exprs) == 10 and len(set(exprs)) == 10
    assert exprs[0] == 'model_eval_kernel<5>' and exprs[-1] == 'friends_unif_kernel<5>'
    for e in exprs:
        assert '<5' in e          # B2N_LIKE_USER


def test_user_translation_unit_compiles_every_slot():
    nv = _nvrtc_or_skip()
    cm = UM.compile_user(GAUSS_DIAG)
    assert cm.exprs == UM.kernel_exprs()
    assert len(cm.lowered) == len(cm.exprs)
    for e, low in zip(cm.exprs, cm.lowered):
        assert low.startswith('_Z'), (e, low)
        assert e.split('<')[0] in low
    assert cm.cubin[:4] == b'\x7fELF'            # an sm_90a cubin, not PTX
    assert UM.compile_user(GAUSS_DIAG) is cm      # memoised per process
    print('NVRTC %d.%d compiled the user translation unit (%d kernels, %.0f KB cubin) in %.1f s on the CPU'
          % (nv.version() + (len(cm.lowered), len(cm.cubin) / 1024, cm.seconds)))


def test_syntax_error_raises_with_the_nvrtc_log():
    _nvrtc_or_skip()
    bad = GAUSS_DIAG.replace('s = fma(p[n + i] * d, d, s);', 's = fma(p[n + i] * d, d, s)')
    with pytest.raises(UM.UserModelCompileError) as ei:
        UM.compile_user(bad)
    msg = str(ei.value)
    assert 'user_likelihood.cu' in msg and 'error' in msg
    assert 'expected a ";"' in msg


def test_undefined_identifier_is_reported():
    _nvrtc_or_skip()
    with pytest.raises(UM.UserModelCompileError, match='identifier "nope" is undefined'):
        UM.compile_user(GAUSS_DIAG.replace('p[2 * n]', 'nope'))


def test_user_model_pickles_with_its_parameters():
    n = 7
    params = np.concatenate([np.linspace(-1, 1, n), np.full(n, 2.0), [-3.5]])
    m = DeviceModel.from_cuda(n, GAUSS_DIAG, params=params, prior_kind=_lib.PRIOR_UNIFORM, prior_p0=-5.0,
                              prior_p1=10.0, name='diag7')
    m._ids[12345] = (0, 1)                        # device handles are per process
    r = pickle.loads(pickle.dumps(m))
    assert r._ids == {}
    assert r.like_kind == _lib.LIKE_USER and r.ndim == n and r.name == 'diag7'
    assert r.source == GAUSS_DIAG
    np.testing.assert_array_equal(r.params, params)
    np.testing.assert_array_equal(r.prior_p0, np.full(n, -5.0))
    np.testing.assert_array_equal(r.prior_p1, np.full(n, 10.0))


def test_user_model_without_parameters():
    m = DeviceModel.from_cuda(3, GAUSS_DIAG.replace('p[', 'v['))
    assert m.params is None and m.prior_kind == _lib.PRIOR_IDENTITY

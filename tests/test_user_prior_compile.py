"""CPU tier: user priors (DeviceModel.from_cuda(..., prior_source=...)) compile for sm_90a without a GPU.

A program with a prior is the user translation unit compiled with B2N_USER_PRIOR: every kernel slot the library
lists must still resolve to a mangled sm_90a kernel, and the image must carry the marker b2n_user_prior_abi that
b2n_model_create_user_ex checks.  A program without a prior is the same text as before.  NVRTC messages about the
prior name user_prior.cu and its line; the argument rules of from_cuda and pickling are checked without compiling."""
import os
import pickle

import numpy as np
import pytest

from dynesty_b200 import _lib, build
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

# the registry's UNIFORM prior restated: v = lo + width * u, lo = p[0, n), width = p[n, 2n)
UNIFORM = r'''
__device__ void b2n_user_prior(const double* u, double* v, double* work, int n, const double* p, int lane) {
    for (int i = lane; i < n; i += 32) {
        v[i] = fma(p[n + i], u[i], p[i]);
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


def test_prior_kind_constant_matches_the_header():
    hdr = open(os.path.join(UM.INCLUDE, 'b200nest.h')).read()
    assert '#define B2N_PRIOR_USER       3' in hdr
    assert _lib.PRIOR_USER == 3


def test_likelihood_and_prior_compile_every_slot_with_the_marker():
    nv = _nvrtc_or_skip()
    cm = UM.compile_user(DIAG, UNIFORM)
    assert cm.exprs == UM.kernel_exprs() and len(cm.exprs) == 10
    assert len(cm.lowered) == len(cm.exprs)
    for e, low in zip(cm.exprs, cm.lowered):
        assert low.startswith('_Z'), (e, low)
        assert e.split('<')[0] in low
    assert cm.cubin[:4] == b'\x7fELF'                       # an sm_90a cubin, not PTX
    assert b'b2n_user_prior_abi' in cm.cubin
    assert UM.compile_user(DIAG, UNIFORM) is cm              # memoised per process
    print('NVRTC %d.%d compiled the user translation unit with a prior (%d kernels, %.0f KB cubin) in %.1f s '
          'on the CPU' % (nv.version() + (len(cm.lowered), len(cm.cubin) / 1024, cm.seconds)))


def test_program_without_a_prior_is_unchanged_and_memoised_apart():
    assert UM.program_source(DIAG) == '#include "b2n_user_kernels.cuh"\n#line 1 "user_likelihood.cu"\n' + DIAG + '\n'
    assert UM.program_source(DIAG, None) == UM.program_source(DIAG)
    src = UM.program_source(DIAG, UNIFORM)
    assert src.startswith('#define B2N_USER_PRIOR\n#include "b2n_user_kernels.cuh"\n#line 1 "user_prior.cu"\n')
    assert src.index(UNIFORM) < src.index('#line 1 "user_likelihood.cu"') < src.index(DIAG)
    _nvrtc_or_skip()
    plain = UM.compile_user(DIAG)
    with_prior = UM.compile_user(DIAG, UNIFORM)
    assert plain is not with_prior
    assert b'b2n_user_prior_abi' not in plain.cubin
    assert b'b2n_user_prior_abi' in with_prior.cubin
    assert UM.compile_user(DIAG) is plain


def test_syntax_error_in_the_prior_names_its_file_and_line():
    _nvrtc_or_skip()
    bad = UNIFORM.replace('v[i] = fma(p[n + i], u[i], p[i]);', 'v[i] = fma(p[n + i], u[i], p[i])')
    line = bad.split('\n').index('        v[i] = fma(p[n + i], u[i], p[i])') + 1
    with pytest.raises(UM.UserModelCompileError) as ei:
        UM.compile_user(DIAG, bad)
    msg = str(ei.value)
    assert 'expected a ";"' in msg
    # NVRTC reports the missing ';' at the token after the statement (the closing brace on the next line)
    assert any('user_prior.cu(%d)' % k in msg for k in (line, line + 1)), msg
    assert 'user_likelihood.cu' not in msg


def test_from_cuda_argument_errors():
    with pytest.raises(ValueError):
        DeviceModel.from_cuda(3, DIAG, prior_source=UNIFORM, prior_kind=_lib.PRIOR_UNIFORM)
    with pytest.raises(ValueError):
        DeviceModel.from_cuda(3, DIAG, prior_source=UNIFORM, prior_p0=0.0)
    with pytest.raises(ValueError):
        DeviceModel.from_cuda(3, DIAG, prior_source=UNIFORM, prior_p1=1.0)
    with pytest.raises(ValueError):
        DeviceModel.from_cuda(3, DIAG, prior_params=[1.0, 2.0])
    with pytest.raises(ValueError):
        DeviceModel.from_cuda(3, DIAG, prior_kind=_lib.PRIOR_USER)
    m = DeviceModel.from_cuda(3, DIAG, prior_source=UNIFORM)
    assert m.prior_kind == _lib.PRIOR_USER and m.prior_params is None
    assert m.prior_p0 is None and m.prior_p1 is None
    r = DeviceModel.from_cuda(3, DIAG)
    assert r.prior_kind == _lib.PRIOR_IDENTITY and r.prior_source is None and r.prior_params is None


def test_user_prior_model_pickles_with_its_prior():
    n = 5
    pp = np.concatenate([np.full(n, -5.0), np.full(n, 10.0)])
    m = DeviceModel.from_cuda(n, DIAG, prior_source=UNIFORM, prior_params=pp, name='diag5_userprior')
    m._ids[12345] = (0, 1)                                   # device handles are per process
    r = pickle.loads(pickle.dumps(m))
    assert r._ids == {}
    assert r.prior_kind == _lib.PRIOR_USER and r.like_kind == _lib.LIKE_USER and r.name == 'diag5_userprior'
    assert r.source == DIAG and r.prior_source == UNIFORM
    np.testing.assert_array_equal(r.prior_params, pp)
    assert r.params is None

"""Run-time compilation of user likelihoods (B2N_LIKE_USER) and user priors (B2N_PRIOR_USER) with NVRTC.

The user writes one warp-cooperative CUDA device function ``b2n_user_loglike``, and optionally a second one,
``b2n_user_prior``, and a third, ``b2n_user_blob`` (contract: ``include/b200nest.h``, ``DeviceModel.from_cuda``).
``compile_user`` compiles the library's chain-kernel templates with them -- the program is ``b2n_user_kernels.cuh``
followed by the user's source -- for sm_90a, asking NVRTC for every instantiation the library lists
(``b2n_user_kernel_exprs``), and returns the cubin and the mangled kernel names that ``b2n_model_create_user(_ex)``
loads.  No GPU is needed to compile.

A compile is done once per process for a given (source, prior, blob switch, options) and kept in memory only:
nothing is cached on disk, like the library build itself (build.py).
"""
import ctypes as C
import glob
import os
import threading

from . import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
INCLUDE = os.path.join(os.path.dirname(HERE), 'include')
CUDA_HOME = os.environ.get('CUDA_HOME', '/usr/local/cuda')

# the library's own code-generation flags (build.py), plus the switch that compiles the user branch of the
# likelihood; -default-device: NVRTC has no host code, so the C declarations of include/b200nest.h are read as
# (never defined, never called) device declarations
OPTIONS = ('--gpu-architecture=sm_90a', '-std=c++17', '-fmad=true', '-lineinfo', '-DB2N_USER_MODEL',
           '-default-device')


class UserModelCompileError(RuntimeError):
    """NVRTC rejected the program; the message carries NVRTC's log."""


def _wheel_dirs(sub):
    """Directories `sub` of the CUDA wheels torch depends on (the `nvidia` namespace package)."""
    try:
        import nvidia
    except ImportError:
        return []
    return [os.path.join(p, sub) for p in getattr(nvidia, '__path__', [])]


def _find_nvrtc():
    cands = []
    for d in _wheel_dirs(os.path.join('cuda_nvrtc', 'lib')):
        cands += sorted(glob.glob(os.path.join(d, 'libnvrtc.so*')))
    cands += [os.path.join(CUDA_HOME, 'lib64', 'libnvrtc.so.12'), os.path.join(CUDA_HOME, 'lib64', 'libnvrtc.so')]
    for c in cands:
        if os.path.exists(c) and 'builtins' not in os.path.basename(c):
            return c
    raise UserModelCompileError('NVRTC not found (looked in the nvidia-cuda-nvrtc wheel and %s/lib64)' % CUDA_HOME)


def cuda_include_dirs():
    """CUDA headers for the program (curand's Philox, the vector types, <cuda/std/cstdint>)."""
    inc = os.path.join(CUDA_HOME, 'include')
    if os.path.exists(os.path.join(inc, 'curand_philox4x32_x.h')):
        return [inc]
    dirs = []
    for sub in ('curand', 'cuda_runtime', 'cuda_cccl'):
        dirs += [d for d in _wheel_dirs(os.path.join(sub, 'include')) if os.path.isdir(d)]
    return dirs


class _Nvrtc:
    """The few NVRTC calls the compile needs (ctypes)."""

    def __init__(self, path):
        self.path = path
        lib = self.lib = C.CDLL(path)
        P, S = C.c_void_p, C.c_size_t
        sig = {
            'nvrtcVersion': [C.POINTER(C.c_int), C.POINTER(C.c_int)],
            'nvrtcGetErrorString': [C.c_int],
            'nvrtcCreateProgram': [C.POINTER(P), C.c_char_p, C.c_char_p, C.c_int, P, P],
            'nvrtcDestroyProgram': [C.POINTER(P)],
            'nvrtcAddNameExpression': [P, C.c_char_p],
            'nvrtcCompileProgram': [P, C.c_int, C.POINTER(C.c_char_p)],
            'nvrtcGetProgramLogSize': [P, C.POINTER(S)],
            'nvrtcGetProgramLog': [P, C.c_char_p],
            'nvrtcGetLoweredName': [P, C.c_char_p, C.POINTER(C.c_char_p)],
            'nvrtcGetCUBINSize': [P, C.POINTER(S)],
            'nvrtcGetCUBIN': [P, C.c_char_p],
        }
        for name, args in sig.items():
            f = getattr(lib, name)
            f.argtypes = args
            f.restype = C.c_char_p if name == 'nvrtcGetErrorString' else C.c_int

    def version(self):
        a, b = C.c_int(), C.c_int()
        self.check(self.lib.nvrtcVersion(C.byref(a), C.byref(b)), 'nvrtcVersion')
        return a.value, b.value

    def check(self, rc, what, log=''):
        if rc != 0:
            msg = '%s: %s' % (what, self.lib.nvrtcGetErrorString(rc).decode())
            raise UserModelCompileError(msg + ('\n' + log if log else ''))

    def compile(self, source, name, exprs, options):
        prog = C.c_void_p()
        self.check(self.lib.nvrtcCreateProgram(C.byref(prog), source.encode(), name.encode(), 0, None, None),
                   'nvrtcCreateProgram')
        try:
            for e in exprs:
                self.check(self.lib.nvrtcAddNameExpression(prog, e.encode()), 'nvrtcAddNameExpression')
            opts = (C.c_char_p * len(options))(*[o.encode() for o in options])
            rc = self.lib.nvrtcCompileProgram(prog, len(options), opts)
            n = C.c_size_t()
            self.lib.nvrtcGetProgramLogSize(prog, C.byref(n))
            buf = C.create_string_buffer(n.value)
            self.lib.nvrtcGetProgramLog(prog, buf)
            log = buf.value.decode(errors='replace')
            self.check(rc, 'NVRTC compile of the user likelihood failed', log)
            lowered = []
            for e in exprs:
                s = C.c_char_p()
                self.check(self.lib.nvrtcGetLoweredName(prog, e.encode(), C.byref(s)), 'nvrtcGetLoweredName ' + e)
                lowered.append(s.value.decode())
            self.check(self.lib.nvrtcGetCUBINSize(prog, C.byref(n)), 'nvrtcGetCUBINSize')
            cubin = C.create_string_buffer(n.value)
            self.check(self.lib.nvrtcGetCUBIN(prog, cubin), 'nvrtcGetCUBIN')
            return cubin.raw, lowered, log
        finally:
            self.lib.nvrtcDestroyProgram(C.byref(prog))


_nvrtc = None
_cache = {}
_mu = threading.Lock()


def nvrtc():
    global _nvrtc
    if _nvrtc is None:
        _nvrtc = _Nvrtc(_find_nvrtc())
    return _nvrtc


def kernel_exprs():
    """The name expressions of the user-likelihood kernels, in the library's slot order."""
    lib = _lib.load()
    arr, cnt = C.POINTER(C.c_char_p)(), C.c_int32()
    st = lib.b2n_user_kernel_exprs(C.byref(arr), C.byref(cnt))
    if st != _lib.OK:
        raise RuntimeError('b2n_user_kernel_exprs: %s' % lib.b2n_strerror(st).decode())
    return [arr[i].decode() for i in range(cnt.value)]


def program_source(source, prior_source=None, blob=False):
    """The NVRTC program of a user likelihood: the kernel templates, then the user's code (line numbers of NVRTC
    messages refer to the user's source).  With a user prior (``prior_source`` defines b2n_user_prior) the
    templates are compiled with B2N_USER_PRIOR, and the prior precedes the likelihood under its own file name.  With
    blob=True (``source`` also defines b2n_user_blob) the program is compiled with B2N_USER_BLOB, which adds the
    kernel b2n_user_blob_kernel."""
    head = '#define B2N_USER_BLOB\n' if blob else ''
    if prior_source is None:
        return head + '#include "b2n_user_kernels.cuh"\n#line 1 "user_likelihood.cu"\n' + source + '\n'
    return ('#define B2N_USER_PRIOR\n' + head + '#include "b2n_user_kernels.cuh"\n#line 1 "user_prior.cu"\n' +
            prior_source + '\n#line 1 "user_likelihood.cu"\n' + source + '\n')


class CompiledUserModel:
    def __init__(self, cubin, exprs, lowered, log, seconds):
        self.cubin, self.exprs, self.lowered, self.log, self.seconds = cubin, exprs, lowered, log, seconds


def compile_user(source, prior_source=None, blob=False):
    """Compile `source` (defines b2n_user_loglike, and with blob=True b2n_user_blob) and, if given, `prior_source`
    (defines b2n_user_prior) into every user-kernel slot; memoised per process."""
    import time
    options = OPTIONS + tuple('-I' + d for d in [CSRC, INCLUDE] + cuda_include_dirs())
    blob = bool(blob)
    key = (source, options, prior_source, blob)
    with _mu:
        hit = _cache.get(key)
        if hit is None:
            exprs = kernel_exprs()
            t0 = time.perf_counter()
            try:
                cubin, lowered, log = nvrtc().compile(program_source(source, prior_source, blob), 'b2n_user_model.cu',
                                                      exprs, list(options))
            except UserModelCompileError as e:
                if blob and 'b2n_user_blob' in str(e):
                    raise UserModelCompileError(
                        'a model with blobs (nblob > 0) needs its source to define __device__ void b2n_user_blob('
                        'const double* v, double* work, int n, const double* p, int lane, double* blob, int nblob)'
                        '\n' + str(e)) from None
                raise
            hit = _cache[key] = CompiledUserModel(cubin, exprs, lowered, log, time.perf_counter() - t0)
        return hit

"""CPU tier: the drop-in boundary itself.  libb200nest.so (built for sm_90a by
dynesty_b200/build.py) must load without a GPU, export every function include/b200nest.h
declares, and the ctypes table the host side binds must be exactly that set.  No compute entry
point is called here; the product path must FAIL LOUDLY without a CUDA device (no CPU
fallback)."""
import ctypes as C
import os
import re

import pytest

from dynesty_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'b200nest.h')


def _declared():
    src = open(HEADER).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)          # comments mention functions too
    return set(re.findall(r'\b(b2n_[a-z0-9_]+)\s*\(', src))


@pytest.fixture(scope='module')
def lib():
    if not os.path.exists(_lib.LIBPATH):
        build.build()
    return C.CDLL(_lib.LIBPATH)


def test_header_declares_the_path():
    d = _declared()
    for must in ('b2n_init', 'b2n_bounding_ellipsoid', 'b2n_multi_decompose', 'b2n_multi_tree', 'b2n_membership',
                 'b2n_scale_to_logvol', 'b2n_bootstrap_expand', 'b2n_bound_set', 'b2n_rwalk_batch',
                 'b2n_rslice_batch', 'b2n_slice_batch', 'b2n_unif_batch', 'b2n_peer_export', 'b2n_peer_import'):
        assert must in d
    assert len(d) >= 30


def test_library_exports_every_declared_symbol(lib):
    missing = [name for name in sorted(_declared()) if not hasattr(lib, name)]
    assert not missing, missing


def test_ctypes_table_matches_header():
    assert set(_lib.SYMBOLS) == _declared()


def test_no_torch_types_in_signatures():
    src = re.sub(r'/\*.*?\*/', '', open(HEADER).read(), flags=re.S)
    assert 'torch' not in src.lower() and 'at::' not in src and 'extern "C"' in src
    assert '#include <torch' not in open(HEADER).read()


def test_pure_host_entry_points(lib):
    l = _lib.load()
    assert b'sm_90a' in l.b2n_version()
    assert l.b2n_strerror(_lib.OK) == b'ok'
    for code in range(1, 13):
        assert l.b2n_strerror(code) != b'unknown status'
    al = lambda b: (b + 255) // 256 * 256
    assert l.b2n_peer_window_bytes(2000, 50) == 256 + 2 * (2 * al(2000 * 50 * 8) + al(2000 * 8) + 4 * al(2000 * 4))


CHAIN_ENTRY_POINTS = ['b2n_rwalk_batch', 'b2n_rslice_batch', 'b2n_slice_batch', 'b2n_unif_batch',
                      'b2n_unitcube_batch', 'b2n_friends_unif_batch']


@pytest.mark.parametrize('name', CHAIN_ENTRY_POINTS)
def test_chain_entry_points_refuse_a_null_ctx(name):
    """A chain entry point answers a NULL ctx with B2N_ERR_ARG before it touches CUDA, whether or not it is given
    its arguments (the NULL-args case with a live ctx is in tests/test_gpu_chain_entry.py)."""
    l = _lib.load()
    argtypes = _lib.SYMBOLS[name][1]
    rest = [0 if t is _lib._I else None for t in argtypes[2:]]
    a = _lib.ChainArgs()
    assert getattr(l, name)(None, C.byref(a), *rest) == _lib.ERR_ARG
    assert getattr(l, name)(None, None, *rest) == _lib.ERR_ARG


def test_product_path_fails_loudly_without_a_gpu():
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip('a GPU is present')
    except ImportError:
        pass
    with pytest.raises(_lib.B200Unavailable, match='no CPU fallback'):
        _lib.Context(0)
    from dynesty_b200 import ops
    import numpy as np
    with pytest.raises(_lib.B200Unavailable):
        ops.bounding_ellipsoid(np.random.default_rng(0).random((20, 3)))


def test_header_is_plain_c_and_the_library_links(lib, tmp_path):
    """The drop-in boundary is a C ABI: include/b200nest.h must compile as strict C99 (no C++, no torch) and a C
    program must link against libb200nest.so and reach its host-only entry points without a GPU -- what a cgo / JNI /
    ctypes binding on the reference's side relies on."""
    import shutil
    import subprocess
    cc = shutil.which('gcc') or shutil.which('cc')
    if cc is None:
        pytest.skip('no C compiler')
    libdir = os.path.dirname(_lib.LIBPATH)
    src = tmp_path / 'abi.c'
    src.write_text('#include "b200nest.h"\n#include <stddef.h>\n#include <string.h>\n'
                   'int main(void) {\n'
                   '    b2n_chain_args a; memset(&a, 0, sizeof a);\n'
                   '    if (strcmp(b2n_strerror(B2N_OK), "ok") != 0) return 1;\n'
                   '    if (b2n_set_start_rows(NULL, NULL, 0) != B2N_ERR_ARG) return 2;\n'
                   '    if (b2n_rwalk_batch(NULL, &a, 1, NULL, NULL, NULL, NULL, NULL, NULL) != B2N_ERR_ARG) return 3;\n'
                   '    return 0;\n}\n')
    exe = tmp_path / 'abi'
    cmd = [cc, '-std=c99', '-Wall', '-Wextra', '-pedantic', '-Werror', '-I', os.path.dirname(HEADER), str(src),
           '-L', libdir, '-lb200nest', '-Wl,-rpath,' + os.path.abspath(libdir), '-o', str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([str(exe)]).returncode == 0

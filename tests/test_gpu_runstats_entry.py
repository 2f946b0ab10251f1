"""GPU: the host side the run-statistics entry points share (b2n_jitter_runs, b2n_resample_runs, b2n_weighted_stats,
b2n_jitter_posterior, b2n_resample_posterior, b2n_merge_runs).  Host and device pointers give the same bits, with every
output given and with some passed as NULL; an output passed as NULL, and the bytes past the end of every output, keep
their fill; every call makes a fixed number of launches."""
import ctypes as C

import numpy as np
import pytest

from dynesty_b200 import _lib, utils as DU
from dynesty_b200._lib import ptr
from oracle import jitter as OJ, resample as ORS

pytestmark = pytest.mark.gpu

SEED, CHAIN0, R, NDIM = 11, 3, 5, 3
GUARD = 37                                  # elements past the end of every output buffer
FILL = {np.float64: -12345.0, np.int32: -7, np.int64: -7}
Q = np.array([0.1, 0.5, 0.9])


def _jitter_record():
    logl, n = OJ.synthetic_record(nlive=200, K=10, ndim=NDIM, lnx_end=-5.0, seed=4)
    logwt, logz, _, _ = OJ.integrate(logl, np.cumsum(np.log(n / (n + 1.))))
    return logl, n, logwt, float(logz[-1])


def _strand_record():
    res = ORS.synthetic_strand_record(nlive=200, K=10, lnx_end=-5.0, seed=4)
    plan = DU.strand_plan(res)
    logl = np.asarray(res['logl'], dtype=float)
    pptr, pstr = DU._piece_csr(logl, plan)
    host = [np.ascontiguousarray(plan['strand'], dtype=np.int32), len(plan['ids']),
            np.ascontiguousarray(plan['base'], dtype=np.uint8), pptr, np.ascontiguousarray(pstr, dtype=np.int32),
            None if plan['end'] is None else np.ascontiguousarray(plan['end'], dtype=np.uint8)]
    return logl, host, np.asarray(res['logwt'], dtype=float), float(np.asarray(res['logz'])[-1])


def _x(N):
    return np.random.default_rng(N).standard_normal((N, NDIM))


# An entry point's arguments after ctx, in order: ('dev', array) follows the pointer mode, ('host', array) is a host
# pointer in both modes, anything else is passed as it is.  Then its outputs: (name, shape, dtype), in argument order.
def _jitter_runs():
    logl, n, wref, zref = _jitter_record()
    N = len(logl)
    args = [('dev', logl), ('host', n), N, ('dev', wref), zref, 0, R, SEED, CHAIN0]
    outs = [(k, (R,), np.float64) for k in ('logz', 'logzerr', 'h', 'kld')] + \
           [(k, (R, N), np.float64) for k in ('logvol_full', 'logwt_full', 'logz_full', 'kld_full')]
    return 'b2n_jitter_runs', args, outs


def _resample_runs():
    logl, (strand, S, base, pptr, pstr, end), wref, zref = _strand_record()
    N = len(logl)
    args = [('dev', logl), ('host', strand), N, S, ('host', base), ('host', pptr), ('host', pstr), ('host', end),
            ('dev', wref), zref, R, SEED, CHAIN0]
    outs = [(k, (R,), np.float64) for k in ('logz', 'logzerr', 'h', 'kld')] + [('mult', (R, S), np.int32)]
    return 'b2n_resample_runs', args, outs


def _post_outs():
    return [('mean', (R, NDIM), np.float64), ('cov', (R, NDIM, NDIM), np.float64),
            ('quant', (R, NDIM, len(Q)), np.float64)]


def _weighted_stats():
    N = 3000
    x = _x(N)
    rng = np.random.default_rng(2)
    w = rng.random((R, N)) * np.exp(rng.uniform(-10, 0, (R, N)))
    args = [('dev', x), N, NDIM, ('dev', w), R, ('dev', x.mean(axis=0)), ('dev', Q), len(Q)]
    return 'b2n_weighted_stats', args, _post_outs()


def _jitter_posterior():
    fn, args, outs = _jitter_runs()
    N = args[2]
    return 'b2n_jitter_posterior', args + [('dev', _x(N)), NDIM, ('dev', Q), len(Q)], outs[:4] + _post_outs()


def _resample_posterior():
    fn, args, outs = _resample_runs()
    N = args[2]
    return 'b2n_resample_posterior', args + [('dev', _x(N)), NDIM, ('dev', Q), len(Q)], outs[:4] + _post_outs()


def _merge_runs():
    recs = [OJ.synthetic_record(nlive=50, K=5, ndim=NDIM, lnx_end=-3.0, seed=s) for s in range(3)]
    logl = np.concatenate([r[0] for r in recs])
    n = np.concatenate([r[1] for r in recs])
    run_ptr = np.r_[0, np.cumsum([len(r[0]) for r in recs])].astype(np.int64)
    N = len(logl)
    args = [('dev', logl), ('dev', n), ('host', run_ptr), 3, 2, ('host', np.array([-np.inf, -np.inf, -4.0]))]
    outs = [('perm', (N,), np.int64), ('samples_n', (N,), np.int64), ('last3', (3,), np.float64)] + \
           [(k, (N,), np.float64) for k in ('logvol', 'logwt', 'logz', 'logzvar', 'h')]
    return 'b2n_merge_runs', args, outs


ENTRY = {'jitter_runs': _jitter_runs, 'resample_runs': _resample_runs, 'weighted_stats': _weighted_stats,
         'jitter_posterior': _jitter_posterior, 'resample_posterior': _resample_posterior, 'merge_runs': _merge_runs}
# the outputs passed as NULL in the 'some' calls
NULLED = {'jitter_runs': ('logzerr', 'kld', 'logwt_full', 'kld_full'), 'resample_runs': ('logz', 'h', 'mult'),
          'weighted_stats': ('mean', 'quant'), 'jitter_posterior': ('logzerr', 'h', 'mean', 'cov'),
          'resample_posterior': ('logz', 'kld', 'mean', 'cov'), 'merge_runs': ('perm', 'logwt', 'logzvar', 'h')}
# kernel launches per call (CUB's segmented sort counts as one), with every output given and in the 'some' calls
LAUNCHES = {'jitter_runs': (5, 4), 'resample_runs': (2, 2), 'weighted_stats': (8, 4), 'jitter_posterior': (11, 9),
            'resample_posterior': (9, 7), 'merge_runs': (9, 8)}


def _call(ctx, kind, mode, nulled=()):
    """One direct call in pointer mode `mode` ('host' or 'device'); returns the outputs with their guard tails (every
    output buffer, the NULL ones included, as numpy) and the launches the call made."""
    import torch
    fn, args, outs = ENTRY[kind]()
    dev = 'cuda:%d' % ctx.device

    def mem(a):
        t = torch.as_tensor(np.ascontiguousarray(a))
        return t.to(dev) if mode == 'device' else t

    keep = []
    cargs = []
    for a in args:
        if isinstance(a, tuple):
            where, v = a
            v = None if v is None else (mem(v) if where == 'dev' else np.ascontiguousarray(v))
            keep.append(v)
            cargs.append(ptr(v))
        else:
            cargs.append(a)
    bufs = {k: mem(np.full(int(np.prod(shape)) + GUARD, FILL[dt], dtype=dt)) for k, shape, dt in outs}
    cargs += [None if k in nulled else ptr(bufs[k]) for k, _, _ in outs]
    before = ctx.launch_count()
    if mode == 'device':
        ctx.set_pointer_mode(_lib.PTR_DEVICE)
    try:
        ctx.check(getattr(ctx.lib, fn)(ctx.h, *cargs))
    finally:
        ctx.set_pointer_mode(_lib.PTR_HOST)
    ctx.synchronize()
    return {k: b.cpu().numpy() for k, b in bufs.items()}, ctx.launch_count() - before, outs


def _same_bits(a, b):
    return a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize('kind', list(ENTRY))
def test_pointer_modes_and_null_outputs(kind):
    """Host and device pointers, all outputs and some NULL: the same bits in every output given; the NULL outputs and
    the guard tails keep their fill; the written parts do not."""
    ctx = _lib.Context(0)
    ref, _, outs = _call(ctx, kind, 'host')
    for mode in ('host', 'device'):
        for nulled in ((), NULLED[kind]):
            got, _, _ = _call(ctx, kind, mode, nulled)
            for k, shape, dt in outs:
                size = int(np.prod(shape))
                fill = np.full(size + GUARD, FILL[dt], dtype=dt)
                assert _same_bits(got[k][size:], fill[size:]), (mode, nulled, k, 'guard')
                if k in nulled:
                    assert _same_bits(got[k], fill), (mode, k, 'NULL output written')
                else:
                    assert _same_bits(got[k], ref[k]), (mode, nulled, k)
                    assert not np.any(got[k][:size] == FILL[dt]), (mode, nulled, k, 'left unwritten')
    ctx.close()


@pytest.mark.parametrize('kind', list(ENTRY))
@pytest.mark.parametrize('mode', ['host', 'device'])
def test_launches_per_call(kind, mode):
    ctx = _lib.Context(0)
    assert _call(ctx, kind, mode)[1] == LAUNCHES[kind][0]
    assert _call(ctx, kind, mode, NULLED[kind])[1] == LAUNCHES[kind][1]
    ctx.close()


def test_null_args():
    ctx = _lib.Context(0)
    for kind in ENTRY:
        fn, args, outs = ENTRY[kind]()
        assert getattr(ctx.lib, fn)(None, *[None if isinstance(a, tuple) else a for a in args],
                                    *[None] * len(outs)) == _lib.ERR_ARG, kind
    ctx.close()

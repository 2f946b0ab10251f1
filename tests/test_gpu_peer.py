"""GPU: the fused multi-GPU gather (include/b200nest.h "peer" section, csrc/b2n_peer.cu) on ONE
device.  (a) world = 1: the chain kernels write into the exchange window and run the
arrive/wait against themselves -- layout, row offsets, double buffering, error paths.
(b) two contexts on the same device play ranks 0 and 1 (windows exchanged as raw device
pointers instead of CUDA IPC handles): each kernel stores its rows into BOTH windows and waits
in-kernel for the other -- the real protocol, minus NVLink.  The IPC transport itself is
covered by tests/test_gpu_dist.py on a >= 2-GPU box.  Gathered rows must be bit-identical to a
plain single-context call (same chain ids -> same Philox streams)."""
import numpy as np
import pytest

from dynesty_b200 import _lib, ops
from helpers import MODELS, device_model
from oracle import bounding as OB

pytestmark = pytest.mark.gpu


def _setup(name, npts=300, seed=5, ctx=None):
    m = MODELS[name]
    dm = device_model(m)
    n = m.ndim
    rng = np.random.default_rng(seed)
    C = np.full((n, n), 0.3)
    np.fill_diagonal(C, 1.0)
    pts = 0.5 + 0.04 * rng.standard_normal((npts, n)) @ np.linalg.cholesky(C).T
    e = OB.bounding_ellipsoid(pts)
    logl = m.loglike(m.prior_transform(pts))
    loglstar = float(np.quantile(logl, 0.3))
    u0 = np.ascontiguousarray(pts[logl > loglstar][:128])
    return m, dm, e, u0, loglstar


def _bound(e, ctx):
    ops.bound_set(e.axes[None], ctrs=e.ctr[None], ams=e.am[None], logvols=np.array([e.logvol]), ctx=ctx)


def _self_ctx(total, n):
    ctx = _lib.Context(0)
    h = ctx.peer_export(ctx.peer_window_bytes(total, n))
    ctx.peer_import(0, 1, [h])
    return ctx


@pytest.mark.parametrize('name', ['g6', 'g50', 'n200'])
def test_peer_world1_rwalk_rows(name):
    m, dm, e, u0, loglstar = _setup(name)
    Q, n = u0.shape
    total, row0 = Q + 40, 25
    ctx = _self_ctx(total, n)
    _bound(e, ctx)
    mid = dm.model_id(ctx)
    ref = ops.rwalk_batch(mid, u0, loglstar, 0.7, 15, 3, chain0=900, ctx=ctx)
    for rep in range(3):            # three calls: both window slots, monotonic arrive counter
        o = ops.rwalk_batch(mid, u0, loglstar, 0.7, 15, 3, chain0=900, ctx=ctx, peer=(row0, total))
        for k in ref:
            assert o[k].shape[0] == total
            assert np.array_equal(o[k][row0:row0 + Q], ref[k]), k
    ctx.peer_check()
    g = ctx.peer_gathered(total, n, ['n_accept', 'n_reject', 'ncall'])
    for k in ref:
        assert np.array_equal(g[k][row0:row0 + Q], ref[k]), k
    # gather mode off again: plain call, Q rows
    o = ops.rwalk_batch(mid, u0, loglstar, 0.7, 15, 3, chain0=900, ctx=ctx)
    assert o['u'].shape[0] == Q and np.array_equal(o['u'], ref['u'])
    ctx.close()


@pytest.mark.parametrize('kind', ['rslice', 'slice', 'unif', 'unitcube'])
def test_peer_world1_slice_unif(kind):
    m, dm, e, u0, loglstar = _setup('g6')
    Q, n = u0.shape
    total, row0 = Q + 8, 8
    ctx = _self_ctx(total, n)
    _bound(e, ctx)
    mid = dm.model_id(ctx)
    if kind == 'unif':
        run = lambda **kw: ops.unif_batch(mid, Q, n, loglstar, 3, chain0=70, ctx=ctx, **kw)
    elif kind == 'unitcube':          # prior draws: a threshold half of them pass
        prior = np.random.default_rng(1).random((1000, n))
        lcube = float(np.median(m.loglike(m.prior_transform(prior))))
        run = lambda **kw: ops.unitcube_batch(mid, Q, n, lcube, 3, chain0=70, ctx=ctx, **kw)
    else:
        fn = ops.rslice_batch if kind == 'rslice' else ops.slice_batch
        run = lambda **kw: fn(mid, u0, loglstar, 0.8, 4, 3, chain0=70, ctx=ctx, **kw)
    ref = run()
    o = run(peer=(row0, total))
    assert o.keys() == ref.keys()
    for k in ref:
        assert np.array_equal(o[k][row0:row0 + Q], ref[k]), k
    ctx.close()


def test_peer_errors():
    m, dm, e, u0, loglstar = _setup('g6')
    Q, n = u0.shape
    ctx = _lib.Context(0)
    with pytest.raises(RuntimeError):                     # windows not set up
        ctx.peer_rows(0, Q)
    h = ctx.peer_export(ctx.peer_window_bytes(Q // 2, n))
    ctx.peer_import(0, 1, [h])
    _bound(e, ctx)
    with pytest.raises(RuntimeError, match='window too small'):
        ops.rwalk_batch(dm.model_id(ctx), u0, loglstar, 0.7, 5, 3, ctx=ctx, peer=(0, Q))
    ctx.close()
    ctx = _self_ctx(Q, n)
    _bound(e, ctx)
    with pytest.raises(ValueError):                       # rows [8, 8+Q) exceed total
        ops.rwalk_batch(dm.model_id(ctx), u0, loglstar, 0.7, 5, 3, ctx=ctx, peer=(8, Q))
    ctx.close()


@pytest.mark.parametrize('name,walks', [('g6', 12), ('g50', 30)])
def test_peer_two_ranks_on_one_device(name, walks):
    """Rank 0 runs rows [0, Q/2), rank 1 rows [Q/2, Q); asynchronous device-pointer calls so
    that the two kernels can wait for each other; afterwards BOTH windows hold all Q rows."""
    import torch
    m, dm, e, u0, loglstar = _setup(name)
    Q, n = u0.shape
    half = Q // 2
    ref_ctx = _lib.Context(0)
    _bound(e, ref_ctx)
    ref = ops.rwalk_batch(dm.model_id(ref_ctx), u0, loglstar, 0.7, walks, 3, chain0=40, ctx=ref_ctx)
    ref_ctx.close()
    ctxs = [_lib.Context(0), _lib.Context(0)]
    wins = []
    for c in ctxs:
        c.peer_export(c.peer_window_bytes(Q, n))
        wins.append(c.peer_result()[0])
    d_u0 = torch.from_numpy(u0).cuda()
    mids = []
    for r, c in enumerate(ctxs):
        c.peer_import_raw(r, 2, wins)
        _bound(e, c)
        mids.append(dm.model_id(c))
    torch.cuda.synchronize()
    for rep in range(3):
        for r, c in enumerate(ctxs):
            c.set_pointer_mode(_lib.PTR_DEVICE)
            lo = r * half
            ops.rwalk_batch(mids[r], d_u0[lo:lo + half], loglstar, 0.7, walks, 3, chain0=40 + lo, ctx=c,
                            out=ops.NO_OUT, peer=(lo, Q))
            c.set_pointer_mode(_lib.PTR_HOST)
        for c in ctxs:
            c.peer_check()                               # synchronises; raises if a rank never arrived
            g = c.peer_gathered(Q, n, ['n_accept', 'n_reject', 'ncall'])
            for k in ref:
                assert np.array_equal(g[k], ref[k]), (rep, k)
    for c in ctxs:
        c.close()


def test_peer_window_bytes_formula():
    ctx = _lib.Context(0)
    al = lambda b: (b + 255) // 256 * 256
    R, n = 2000, 50
    assert ctx.peer_window_bytes(R, n) == 256 + 2 * (2 * al(R * n * 8) + al(R * 8) + 4 * al(R * 4))
    ctx.close()

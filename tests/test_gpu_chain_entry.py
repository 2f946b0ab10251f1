"""GPU: the host side every chain entry point shares (b2n_rwalk_batch, b2n_rslice_batch, b2n_slice_batch,
b2n_unif_batch, b2n_unitcube_batch, b2n_friends_unif_batch).  Pageable, pinned (zero-copy) and device pointers give
the same bits; Q == 0 launches nothing; a pending b2n_set_start_rows is for the next rwalk call only; the chain flags
map to the documented status codes; every call makes a fixed number of launches."""
import ctypes as C

import numpy as np
import pytest

from dynesty_b200 import _lib, ops
from dynesty_b200._lib import ptr
from helpers import MODELS, SEED, device_model
from oracle import bounding as OB

pytestmark = pytest.mark.gpu

# entry point, its int arguments, its outputs after (u, v, logl) in argument order (None: passed as NULL, as ops
# passes unitcube's flags), whether it reads u0, a->reserved
ENTRY = {
    'rwalk': ('b2n_rwalk_batch', (12,), ('n_accept', 'n_reject', 'ncall'), True, 0),
    'rslice': ('b2n_rslice_batch', (3, 0), ('n_expand', 'n_contract', 'ncall', 'flags'), True, 0),
    'slice': ('b2n_slice_batch', (3, 0), ('n_expand', 'n_contract', 'ncall', 'flags'), True, 0),
    'unif': ('b2n_unif_batch', (), ('ncall', 'nprop', 'flags'), False, 0),
    'unif_draw': ('b2n_unif_batch', (), ('ncall', 'nprop', 'flags'), False, 1),
    'unif_mixture': ('b2n_unif_batch', (), ('ncall', 'nprop', 'flags'), False, 3),
    'unitcube': ('b2n_unitcube_batch', (), ('ncall', None), False, 0),
    'unitcube_flags': ('b2n_unitcube_batch', (), ('ncall', 'flags'), False, 0),
    'friends_unif': ('b2n_friends_unif_batch', (), ('ncall', 'nprop', 'flags'), False, 0),
}
ENTRY_POINTS = ['rwalk', 'rslice', 'slice', 'unif', 'unitcube', 'friends_unif']
FILL = {'pageable': 0, 'pinned': 7, 'device': -3}      # different in every mode: an output left unwritten shows


class _World:
    """A fresh context with the g6 registry Gaussian, `nell` resident ellipsoids around a point cloud, a friends bound
    on the same points and, with `total`, a world = 1 exchange window of `total` rows."""

    def __init__(self, nell=1, total=None, npts=300):
        self.m = m = MODELS['g6']
        self.n = n = m.ndim
        rng = np.random.default_rng(5)
        cov = np.full((n, n), 0.3)
        np.fill_diagonal(cov, 1.0)
        pts = 0.5 + 0.04 * rng.standard_normal((npts, n)) @ np.linalg.cholesky(cov).T
        logl = m.loglike(m.prior_transform(pts))
        lstar = float(np.quantile(logl, 0.3))
        self.ctx = ctx = _lib.Context(0)
        if total is not None:
            ctx.peer_import(0, 1, [ctx.peer_export(ctx.peer_window_bytes(total, n))])
        side = pts[:, 0] > np.median(pts[:, 0])
        parts = [pts] if nell == 1 else [pts[~side], pts[side]]
        es = [OB.bounding_ellipsoid(p) for p in parts]
        ops.bound_set(np.array([e.axes for e in es]), ctrs=np.array([e.ctr for e in es]),
                      ams=np.array([e.am for e in es]), logvols=np.array([e.logvol for e in es]), ctx=ctx)
        fr = ops.friends_update(pts, 'balls', use_clustering=False, ctx=ctx)
        ops.friends_set('balls', pts, fr['axes'], fr['axes_inv'], ctx=ctx)
        keep = logl > lstar
        self.u0 = np.ascontiguousarray(pts[keep][:40])
        self.ell = None if nell == 1 else side[keep][:40].astype(np.int32)
        prior = np.random.default_rng(1).random((1000, n))
        lcube = float(np.median(m.loglike(m.prior_transform(prior))))        # half the prior draws pass
        self.loglstar = {k: (lcube if k.startswith('unitcube') else lstar) for k in ENTRY}
        self.mid = device_model(m).model_id(ctx)

    def close(self):
        self.ctx.close()


def _mem(a, mode, dtype, device):
    import torch
    t = torch.as_tensor(a, dtype=dtype)
    if mode == 'pinned':
        return t.pin_memory()
    return t.to('cuda:%d' % device) if mode == 'device' else t


def _call(w, kind, mode='pageable', Q=None, nchain=None, loglstar=None, peer=None):
    """One direct call of the entry point of `kind` in pointer mode `mode`; outputs as numpy arrays.  Q rows of
    u0 and outputs (total rows with `peer`), a->nchain = `nchain` if given."""
    import torch
    fn, ints, names, reads_u0, opt = ENTRY[kind]
    Q = len(w.u0) if Q is None else Q
    R = Q if peer is None else peer[1]
    u0 = _mem(w.u0[:Q], mode, torch.float64, w.ctx.device) if reads_u0 else None
    ell = w.ell[:Q] if (reads_u0 and w.ell is not None) else None
    a, keep, _, _ = ops._chain_args(w.mid, u0, None, w.loglstar[kind] if loglstar is None else loglstar, 0.7, SEED,
                                    90, ell, None, Q=Q, ndim=w.n)
    a.reserved = opt
    if nchain is not None:
        a.nchain = nchain
    shape = {'u': (R, w.n), 'v': (R, w.n), 'logl': (R,)}
    o = {nm: _mem(np.full(shape.get(nm, (R,)), FILL[mode]), mode, torch.float64 if nm in shape else torch.int32,
                  w.ctx.device) for nm in ('u', 'v', 'logl') + names if nm}
    args = [ptr(o.get(nm)) for nm in ('u', 'v', 'logl') + names]
    if mode == 'device':
        w.ctx.set_pointer_mode(_lib.PTR_DEVICE)
    if peer is not None:
        w.ctx.peer_rows(*peer)
    try:
        w.ctx.check(getattr(w.ctx.lib, fn)(w.ctx.h, C.byref(a), *ints, *args))
    finally:
        w.ctx.set_pointer_mode(_lib.PTR_HOST)
        w.ctx.peer_rows(0, 0)
    w.ctx.synchronize()
    o = {k: t.cpu().numpy() for k, t in o.items()}
    if 'flags' in o:
        o['flags'] = o['flags'].view(np.uint32)
    return o


@pytest.mark.parametrize('kind,nell', [(k, 1) for k in ENTRY] +
                         [(k, 2) for k in ('rwalk', 'rslice', 'slice', 'unif', 'unif_draw', 'unif_mixture')])
def test_pointer_modes_agree(kind, nell):
    """Pageable numpy, pinned host buffers written in place and device pointers: bit-identical outputs."""
    w = _World(nell)
    ref = _call(w, kind, 'pageable')
    for mode in ('pinned', 'device'):
        o = _call(w, kind, mode)
        assert o.keys() == ref.keys()
        for k in ref:
            assert np.array_equal(o[k], ref[k]), (mode, k)
    w.close()


@pytest.mark.parametrize('kind', ENTRY_POINTS)
def test_no_chains_launch_nothing(kind):
    """Q == 0 returns OK and launches nothing; in gather mode every rank must run a chain (friends sampling has no
    gather mode at all)."""
    w = _World(1, total=8)
    before = w.ctx.launch_count()
    o = _call(w, kind, Q=1, nchain=0)
    assert w.ctx.launch_count() == before
    assert np.all(o['logl'] == FILL['pageable'])
    exc, msg = (NotImplementedError, 'no gather mode') if kind == 'friends_unif' else \
        (ValueError, 'every rank must run at least one chain')
    with pytest.raises(exc, match=msg):
        _call(w, kind, Q=1, nchain=0, peer=(0, 8))
    assert w.ctx.launch_count() == before
    w.close()


@pytest.mark.parametrize('kind', ENTRY_POINTS)
def test_null_args(kind):
    w = _World(1)
    fn, ints, names, _, _ = ENTRY[kind]
    rest = [None] * (3 + len(names))
    assert getattr(w.ctx.lib, fn)(w.ctx.h, None, *ints, *rest) == _lib.ERR_ARG
    w.close()


@pytest.mark.parametrize('kind', ['slice', 'unif', 'unitcube', 'friends_unif'])
def test_pending_start_rows_are_for_rwalk_only(kind):
    """b2n_set_start_rows is for the next rwalk call: another entry point refuses it and clears it, so that the
    rwalk call after it runs on u0 as given."""
    w = _World(1)
    ref = _call(w, 'rwalk')
    starts = np.arange(len(w.u0), dtype=np.int32)[::-1].copy()
    w.ctx.set_start_rows(ptr(starts), len(w.u0))
    with pytest.raises(NotImplementedError, match='start rows'):
        _call(w, kind)
    o = _call(w, 'rwalk')
    for k in ref:
        assert np.array_equal(o[k], ref[k]), k
    w.close()


@pytest.mark.parametrize('kind', ['slice', 'rslice'])
@pytest.mark.parametrize('gather', [False, True])
def test_collapsed_slice_is_slice_fail(kind, gather):
    """loglstar = +inf: every shrink loop collapses onto the start point, B2N_ERR_SLICE_FAIL."""
    w = _World(1, total=40)
    with pytest.raises(RuntimeError, match='Slice sampler has failed to find a valid point'):
        _call(w, kind, loglstar=np.inf, peer=(0, 40) if gather else None)
    w.close()


# kernel launches of one call (the chain kernel, then the flag summary of slice, unif and unitcube)
LAUNCHES = {'rwalk': 1, 'rslice': 2, 'slice': 2, 'unif': 2, 'unitcube': 2, 'friends_unif': 1}


@pytest.mark.parametrize('kind', ENTRY_POINTS)
@pytest.mark.parametrize('gather', [False, True])
def test_launches_per_call(kind, gather):
    if gather and kind == 'friends_unif':
        pytest.skip('friends sampling has no gather mode')
    w = _World(1, total=40)
    before = w.ctx.launch_count()
    _call(w, kind, peer=(0, 40) if gather else None)
    assert w.ctx.launch_count() - before == LAUNCHES[kind]
    w.close()

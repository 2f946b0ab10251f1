"""numpy-level wrappers of the C ABI (host-pointer mode).  Every function here is a
single C call; array-in/array-out, the reference's exceptions on failure."""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import ChainArgs, ptr, f64


def _ctx(ctx):
    return ctx if ctx is not None else _lib.default_context()


def model_eval(model, u, want_v=True, ctx=None):
    """(v, logl) for the rows of u (M, ndim)."""
    ctx = _ctx(ctx)
    u = f64(np.atleast_2d(u))
    M, n = u.shape
    v = np.empty((M, n)) if want_v else None
    logl = np.empty(M)
    ctx.check(ctx.lib.b2n_model_eval(ctx.h, model, ptr(u), M, ptr(v), ptr(logl)))
    return v, logl


def model_blob(model, v, nblob, ctx=None):
    """The blob (M, nblob) of the physical points v (M, ndim) of a user model with blobs (b2n_model_blob)."""
    ctx = _ctx(ctx)
    v = f64(np.atleast_2d(v))
    M = len(v)
    blob = np.empty((M, int(nblob)))
    ctx.check(ctx.lib.b2n_model_blob(ctx.h, model, ptr(v), M, int(nblob), ptr(blob)))
    return blob


def membership(x, ctrs, ams, strict=True, want_d2=False, ctx=None):
    """mask (M, K) bool, q (M,) int32 [, d2 (M, K)]  (bounding.py:502-523)."""
    ctx = _ctx(ctx)
    x = f64(np.atleast_2d(x))
    ctrs = f64(np.atleast_2d(ctrs))
    ams = f64(ams).reshape(ctrs.shape[0], ctrs.shape[1], ctrs.shape[1])
    M, n = x.shape
    K = ctrs.shape[0]
    mask = np.empty((M, K), dtype=np.uint8)
    q = np.empty(M, dtype=np.int32)
    d2 = np.empty((M, K)) if want_d2 else None
    ctx.check(ctx.lib.b2n_membership(ctx.h, ptr(x), M, n, ptr(ctrs), ptr(ams), K, int(bool(strict)),
                                     ptr(mask), ptr(q), ptr(d2)))
    out = (mask.astype(bool), q)
    return out + (d2,) if want_d2 else out


def bounding_ellipsoid(points, ctx=None):
    """dict(ctr, cov, am, axes, axlens, logvol, warn)  (bounding.py:1387-1461)."""
    ctx = _ctx(ctx)
    points = f64(points)
    N, n = points.shape
    o = dict(ctr=np.empty(n), cov=np.empty((n, n)), am=np.empty((n, n)), axes=np.empty((n, n)),
             axlens=np.empty(n))
    lv = np.empty(1)
    warn = C.c_uint32(0)
    ctx.check(ctx.lib.b2n_bounding_ellipsoid(ctx.h, ptr(points), N, n, ptr(o['ctr']), ptr(o['cov']),
                                             ptr(o['am']), ptr(o['axes']), ptr(o['axlens']), ptr(lv),
                                             C.addressof(warn)))
    o['logvol'] = float(lv[0])
    o['warn'] = warn.value
    return o


def multi_decompose(points, max_ells=None, ctx=None):
    """dict(nells, labels, ctrs, covs, ams, axes, axlens, logvols, warn)  (bounding.py:665-686)."""
    ctx = _ctx(ctx)
    points = f64(points)
    N, n = points.shape
    if max_ells is None:
        max_ells = max(1, N // max(2 * n, 1))
    K = int(max_ells)
    o = dict(labels=np.empty(N, dtype=np.int32), ctrs=np.empty((K, n)), covs=np.empty((K, n, n)),
             ams=np.empty((K, n, n)), axes=np.empty((K, n, n)), axlens=np.empty((K, n)),
             logvols=np.empty(K))
    nells = C.c_int32(0)
    warn = C.c_uint32(0)
    ctx.check(ctx.lib.b2n_multi_decompose(ctx.h, ptr(points), N, n, K, C.addressof(nells),
                                          ptr(o['labels']), ptr(o['ctrs']), ptr(o['covs']), ptr(o['ams']),
                                          ptr(o['axes']), ptr(o['axlens']), ptr(o['logvols']),
                                          C.addressof(warn)))
    k = nells.value
    for key in ('ctrs', 'covs', 'ams', 'axes', 'axlens', 'logvols'):
        o[key] = o[key][:k].copy()
    o['nells'] = k
    o['warn'] = warn.value
    return o


def multi_tree(points, ctx=None):
    """Diagnostic: the candidate tree b2n_multi_decompose builds on `points`.  dict(start, count, children (T, 2),
    split (T, 2), logvol, leaf (bool), perm (N,), path 'cholesky' | 'eigen'); node i's points are
    perm[start[i]:start[i] + count[i]] as a set, -1 marks no child / no split attempted."""
    ctx = _ctx(ctx)
    points = f64(points)
    N, n = points.shape
    cap = max(3, N // n + 3)
    nodes = np.empty((cap, 7), dtype=np.int32)
    logvols = np.empty(cap)
    perm = np.empty(N, dtype=np.int32)
    T, path = C.c_int32(0), C.c_int32(0)
    ctx.check(ctx.lib.b2n_multi_tree(ctx.h, ptr(points), N, n, cap, C.addressof(T), ptr(nodes), ptr(logvols),
                                     ptr(perm), C.addressof(path)))
    t = nodes[:T.value]
    return dict(start=t[:, 0].copy(), count=t[:, 1].copy(), children=t[:, 2:4].copy(), split=t[:, 4:6].copy(),
                leaf=t[:, 6] == 1, logvol=logvols[:T.value].copy(), perm=perm,
                path='cholesky' if path.value else 'eigen')


def moments(points, ctx=None):
    """(mean, cov) = (np.mean(points, 0), np.cov(points, rowvar=False)) of one shard of the live set."""
    ctx = _ctx(ctx)
    points = f64(points)
    N, n = points.shape
    mean, cov = np.empty(n), np.empty((n, n))
    ctx.check(ctx.lib.b2n_moments(ctx.h, ptr(points), N, n, ptr(mean), ptr(cov)))
    return mean, cov


def improve_covar(covar, ctx=None):
    """(good, cov, am, axes, warn) = improve_covar_mat(covar)  (bounding.py:1311-1384)."""
    ctx = _ctx(ctx)
    covar = f64(covar)
    n = covar.shape[0]
    cov, am, axes = np.empty((n, n)), np.empty((n, n)), np.empty((n, n))
    good, warn = C.c_int32(0), C.c_uint32(0)
    ctx.check(ctx.lib.b2n_improve_covar(ctx.h, ptr(covar), n, ptr(cov), ptr(am), ptr(axes), C.addressof(good),
                                        C.addressof(warn)))
    return bool(good.value), cov, am, axes, warn.value


FP64_KINDS = {'fma': 0, 'mma': 1, 'mma16x8x4': 2, 'mma16x8x8': 3, 'mma16x8x16': 4}


def fp64_peak(kind, iters=20000, ctx=None):
    """Measured FP64 ceiling in TFLOP/s: kind 'fma' (vector pipe), 'mma' (m8n8k4 tensor pipe) or one of the
    m16n8 shapes 'mma16x8x4', 'mma16x8x8', 'mma16x8x16'."""
    ctx = _ctx(ctx)
    t, ms = C.c_double(0.0), C.c_double(0.0)
    ctx.check(ctx.lib.b2n_fp64_peak(ctx.h, FP64_KINDS[kind], int(iters), C.byref(t), C.byref(ms)))
    return t.value, ms.value


def fp64_latency(kind, iters=4096, ctx=None):
    """Dependent-issue latency of fp64_peak's instruction `kind`, in SM clocks: one warp, one dependency chain."""
    ctx = _ctx(ctx)
    cyc = C.c_double(0.0)
    ctx.check(ctx.lib.b2n_fp64_latency(ctx.h, FP64_KINDS[kind], int(iters), C.byref(cyc)))
    return cyc.value


def dmma_probe(a, b, c, ctx=None):
    """The FP64 MMA shapes on tiles a (T, 16, 8), b (T, 8, 8) (k x n), c (T, 16, 8): a dict of (T, 16, 8) results
    'k4' (one m16n8k4 on k 0..3), 'k4x2rows' (two m8n8k4, rows 0..7 and 8..15), 'k8' (one m16n8k8) and
    'k4x2steps' (two chained m16n8k4, k 0..3 then 4..7), each plus c (b2n_dmma_probe)."""
    ctx = _ctx(ctx)
    a, b, c = (np.ascontiguousarray(x, dtype=np.float64) for x in (a, b, c))
    T = a.shape[0]
    if a.shape != (T, 16, 8) or b.shape != (T, 8, 8) or c.shape != (T, 16, 8):
        raise ValueError('dmma_probe: tiles must be (T, 16, 8), (T, 8, 8), (T, 16, 8)')
    out = np.empty((4, T, 16, 8))
    ctx.check(ctx.lib.b2n_dmma_probe(ctx.h, T, ptr(a), ptr(b), ptr(c), ptr(out)))
    return dict(zip(('k4', 'k4x2rows', 'k8', 'k4x2steps'), out))


def scale_to_logvol(covs, ams, axes, axlens, logvols, targets, ctx=None):
    """In-place Ellipsoid.scale_to_logvol on K stacked ellipsoids (bounding.py:242-276)."""
    ctx = _ctx(ctx)
    K, n = axlens.shape
    targets = f64(targets)
    for a in (covs, ams, axes, axlens, logvols):
        assert a.dtype == np.float64 and a.flags['C_CONTIGUOUS']
    ctx.check(ctx.lib.b2n_scale_to_logvol(ctx.h, K, n, ptr(covs), ptr(ams), ptr(axes), ptr(axlens),
                                          ptr(logvols), ptr(targets)))


def bootstrap_expand(points, multi, nboot, seed, chain0, ctx=None):
    ctx = _ctx(ctx)
    points = f64(points)
    N, n = points.shape
    out = np.empty(nboot)
    ctx.check(ctx.lib.b2n_bootstrap_expand(ctx.h, ptr(points), N, n, int(bool(multi)), nboot, seed,
                                           chain0, ptr(out)))
    return out


# ---- RadFriends / SupFriends (include/b200nest.h, b2n_friends_*) ---------------------------------
def friends_update(points, kind, am_prev=None, use_clustering=True, nboot=0, seed=0, chain0=0, ctx=None):
    """RadFriends.update / SupFriends.update (bounding.py:874-958 / 1142-1226).  kind: 'balls' | 'cubes'.
    Returns dict(cov, am, axes, axes_inv, logvol, radius, nclusters)."""
    ctx = _ctx(ctx)
    points = f64(points)
    N, n = points.shape
    o = dict(cov=np.empty((n, n)), am=np.empty((n, n)), axes=np.empty((n, n)), axes_inv=np.empty((n, n)))
    lv, rad, ncl = C.c_double(0.0), C.c_double(0.0), C.c_int32(0)
    amp = f64(am_prev) if (use_clustering and am_prev is not None) else None
    ctx.check(ctx.lib.b2n_friends_update(ctx.h, ptr(points), N, n, {'balls': 0, 'cubes': 1}[kind],
                                         int(bool(use_clustering and amp is not None)), ptr(amp), int(nboot), int(seed),
                                         int(chain0), ptr(o['cov']), ptr(o['am']), ptr(o['axes']), ptr(o['axes_inv']),
                                         C.addressof(lv), C.addressof(rad), C.addressof(ncl)))
    o.update(logvol=lv.value, radius=rad.value, nclusters=ncl.value)
    return o


def friends_set(kind, ctrs, axes, axes_inv, ctx=None, key=None):
    """Make (ctrs, axes, axes_inv) the resident friends bound of the ctx."""
    ctx = _ctx(ctx)
    ctrs, axes, axes_inv = f64(ctrs), f64(axes), f64(axes_inv)
    N, n = ctrs.shape
    ctx.friends_key = None
    ctx.check(ctx.lib.b2n_friends_set(ctx.h, {'balls': 0, 'cubes': 1}[kind], ptr(ctrs), N, n, ptr(axes), ptr(axes_inv)))
    ctx.friends_key = key


def friends_overlap(x, ctx=None):
    """q (M,) int32: number of balls / cubes of the resident friends bound containing each row of x."""
    ctx = _ctx(ctx)
    x = f64(np.atleast_2d(x))
    q = np.empty(len(x), dtype=np.int32)
    ctx.check(ctx.lib.b2n_friends_overlap(ctx.h, ptr(x), len(x), x.shape[1], ptr(q)))
    return q


def friends_unif_batch(model, nchain, ndim, loglstar, seed, chain0=0, dimflags=None, ctx=None, draw_only=False,
                       mixture=False):
    """UniformBoundSampler.sample x nchain on the resident friends bound; draw_only: Bound.samples(nchain)."""
    ctx = _ctx(ctx)
    a, keep, Q, n = _chain_args(model, None, ndim, loglstar, 1.0, seed, chain0, None, dimflags, Q=int(nchain), ndim=int(ndim))
    if draw_only:
        a.reserved = 3 if mixture else 1
    o = _chain_outputs('unif', Q, n)
    ctx.check(ctx.lib.b2n_friends_unif_batch(ctx.h, C.byref(a), *_chain_ptrs(o, 'unif')))
    if not draw_only and (o['flags'] & 0x80000000).any():
        raise NotImplementedError("uniform sampling did not find a point (bound draw limit)")
    return o


def bound_set(axes, ctrs=None, ams=None, logvols=None, ctx=None, key=None):
    """Make K ellipsoids resident for the proposal kernels (axes: (K, nc, nc)).
    A ctx holds ONE resident bound; `key` (the uploading bound's version token, None = anonymous) is
    recorded on the Context so that every user of the ctx can tell whether its bound is still the
    resident one (``ensure_resident``)."""
    ctx = _ctx(ctx)
    ctx.resident_key = None
    axes = f64(axes)
    if axes.ndim == 2:
        axes = axes[None]
    K, nc, _ = axes.shape
    if ctrs is not None:
        ctrs, ams, logvols = f64(ctrs).reshape(K, nc), f64(ams).reshape(K, nc, nc), f64(logvols).reshape(K)
    ctx.check(ctx.lib.b2n_bound_set(ctx.h, K, nc, ptr(ctrs), ptr(ams), ptr(axes), ptr(logvols)))
    ctx.resident_key = key


def ensure_resident(bound, ctx=None):
    """Upload `bound` (a B200 bound) unless it already is the resident bound of the ctx."""
    ctx = _ctx(ctx if ctx is not None else getattr(bound, 'ctx', None))
    if ctx.resident_key is None or ctx.resident_key != bound.version:
        bound.make_resident()


def _chain_args(model, u0, ncdim, loglstar, scale, seed, chain0, ell, dimflags, Q=None, ndim=None):
    a = ChainArgs()
    keep = []
    if u0 is not None:
        if not hasattr(u0, 'data_ptr'):          # numpy (host mode); torch tensors pass through
            u0 = f64(np.atleast_2d(u0))
        Q, ndim = int(u0.shape[0]), int(u0.shape[1])
        keep.append(u0)
    a.nchain, a.ndim, a.ncdim, a.model_id = Q, ndim, (ncdim or ndim), model
    a.u0 = ptr(u0)
    if ell is not None:
        ell = np.ascontiguousarray(ell, dtype=np.int32)
        keep.append(ell)
    a.ell = ptr(ell)
    if dimflags is not None:
        dimflags = np.ascontiguousarray(dimflags, dtype=np.uint8)
        keep.append(dimflags)
    a.dimflags = ptr(dimflags)
    a.loglstar, a.scale, a.seed, a.chain0 = float(loglstar), float(scale), int(seed), int(chain0)
    return a, keep, Q, ndim


def dimflags_from(ndim, periodic=None, reflective=None):
    """B2N_DIM_* flags from dynesty's periodic / reflective index lists."""
    if periodic is None and reflective is None:
        return None
    f = np.zeros(ndim, dtype=np.uint8)
    if periodic is not None:
        f[np.asarray(periodic, dtype=int)] |= _lib.DIM_PERIODIC
    if reflective is not None:
        f[np.asarray(reflective, dtype=int)] |= _lib.DIM_REFLECTIVE
    return f


def _chain_outputs(sampler, R, n):
    """Fresh output arrays of R chains of `sampler` (_lib.CHAIN_OUTPUTS), keyed as the sampler returns them."""
    o = dict(u=np.empty((R, n)), v=np.empty((R, n)), logl=np.empty(R))
    for nm in _lib.CHAIN_OUTPUTS[sampler]:
        if nm is not None:
            o[nm] = np.empty(R, dtype=np.uint32 if nm == 'flags' else np.int32)
    return o


# the output arguments of each sampler's entry point, in order (names built once: rwalk_batch is on the timed path)
_CHAIN_ARGS = {s: ('u', 'v', 'logl') + tuple(nm for nm in names if nm is not None)
               for s, names in _lib.CHAIN_OUTPUTS.items()}


def _chain_ptrs(o, sampler):
    """The output arguments of the sampler's entry point: addresses of o's arrays (NULL where o has none)."""
    g = o.get
    return [ptr(g(nm)) for nm in _CHAIN_ARGS[sampler]]


class _gather:
    """Context manager for the fused multi-GPU gather (include/b200nest.h, peer section):
    `peer = (row0, total_rows)` makes the chains of the call rows [row0, row0 + Q) of a
    total_rows-chain fill whose outputs come back COMPLETE (all ranks' rows)."""

    def __init__(self, ctx, peer):
        self.ctx, self.peer = ctx, peer

    def __enter__(self):
        if self.peer is not None:
            self.ctx.peer_rows(self.peer[0], self.peer[1])

    def __exit__(self, *exc):
        if self.peer is not None:
            self.ctx.peer_rows(0, 0)
        return False


_NO_OUT = {}          # out=ops.NO_OUT: gather mode, device-pointer callers that read the window
NO_OUT = _NO_OUT


def rwalk_batch(model, u0, loglstar, scale, walks, seed, chain0=0, ncdim=None, ell=None,
                dimflags=None, ctx=None, out=None, peer=None, start_rows=None):
    """RWalkSampler.sample for every row of u0 (internal_samplers.py:505-561).
    `out`: optional dict of preallocated buffers (numpy, or torch tensors on the ctx device
    when the ctx is in device-pointer mode) with keys u, v, logl, n_accept, n_reject, ncall.
    `peer=(row0, total)`: fused multi-GPU gather, outputs have `total` rows.
    `start_rows`: int32 indices -- `u0` is then the whole live set and chain q starts from row start_rows[q]
    (b2n_set_start_rows: the gather of Sampler._fill_queue done by the kernel)."""
    ctx = _ctx(ctx)
    a, keep, Q, n = _chain_args(model, u0, ncdim, loglstar, scale, seed, chain0, ell, dimflags)
    if start_rows is not None:
        if not hasattr(start_rows, 'data_ptr'):
            start_rows = np.ascontiguousarray(start_rows, dtype=np.int32)
        keep.append(start_rows)
        a.nchain = int(start_rows.shape[0])
        ctx.set_start_rows(ptr(start_rows), Q)          # Q rows of u0 = the live set
        Q = a.nchain
    R = Q if peer is None else int(peer[1])
    o = out if out is not None else _chain_outputs('rwalk', R, n)
    with _gather(ctx, peer):
        ctx.check(ctx.lib.b2n_rwalk_batch(ctx.h, C.byref(a), int(walks), *_chain_ptrs(o, 'rwalk')))
    return o


# ---- stepped random walk of a TorchModel (include/b200nest.h, b2n_rwalk_step / b2n_ns_rwalk_step) ---------------
class _torch_stream:
    """Context manager: the library works on torch's current stream of `device`, in device-pointer mode, and the
    previous stream and pointer mode come back however the block ends.  (torch's default stream, handle 0, is the
    legacy default stream: passed as cudaStreamLegacy, 1, since a NULL stream means the context's own.)"""

    def __init__(self, ctx, device):
        import torch
        self.ctx = ctx
        self.stream = torch.cuda.current_stream(device).cuda_stream or 1

    def __enter__(self):
        c = self.ctx
        self.prev_stream, self.prev_mode = c.stream, c.mode
        if self.stream != c.stream:
            c.set_stream(self.stream)
        c.set_pointer_mode(_lib.PTR_DEVICE)

    def __exit__(self, *exc):
        c = self.ctx
        try:
            c.set_pointer_mode(self.prev_mode)
        finally:
            if c.stream != self.prev_stream:
                c.set_stream(self.prev_stream)
        return False


def _step_state(Q, n, device, dimflags, worklist):
    """A b2n_rwalk_state over fresh device buffers for Q chains; returns (state, buffers)."""
    import torch
    b = dict(u_prop=torch.full((Q, n), 0.5, dtype=torch.float64, device=device),
             tick=torch.zeros(Q, dtype=torch.int32, device=device),
             in_cube=torch.zeros(Q, dtype=torch.int32, device=device))
    if dimflags is not None:
        b['dimflags'] = torch.as_tensor(np.asarray(dimflags, dtype=np.int32), device=device)
    if worklist:
        b['order'] = torch.empty(Q, dtype=torch.int32, device=device)
        b['cta'] = torch.empty(3 * Q, dtype=torch.int32, device=device)
    else:
        b['u_start'] = torch.full((Q, n), 0.5, dtype=torch.float64, device=device)
    st = _lib.RwalkState()
    for k, t in b.items():
        setattr(st, k, t.data_ptr())
    return st, b


def _step_through(model, walks, launch, st, u_start, u_prop):
    """walks + 1 stepped launches with the model's calls between them, all enqueued on the current stream: launch(s)
    enqueues step s; the start rows u_start are evaluated after step 0 (which writes them in a device round), the
    proposals u_prop after every step but the last."""
    for s in range(walks + 1):
        launch(s)
        if s == 0:
            v_start, l_start = model._eval(u_start)     # (kept alive until the last launch has been enqueued)
            st.v_start, st.logl_start = v_start.data_ptr(), l_start.data_ptr()
        if s < walks:
            v_prop, l_prop = model._eval(u_prop)
            st.v_prop, st.logl_prop = v_prop.data_ptr(), l_prop.data_ptr()


def rwalk_stepped(model, u0, loglstar, scale, walks, seed, chain0=0, ell=None, dimflags=None, ncdim=None, ctx=None):
    """rwalk_batch for a TorchModel: the same chains (same random streams, same proposals) with the likelihood
    evaluated by the model's torch callables between walks + 1 launches of the stepped kernel, on torch's current
    stream and with no host synchronisation until the outputs are read.  u0: numpy or a CUDA tensor (Q, ndim).
    Returns rwalk_batch's dict of numpy arrays."""
    import torch
    ctx = _ctx(ctx)
    dev = model.device(ctx)
    u0 = torch.as_tensor(u0, dtype=torch.float64, device=dev).contiguous()
    a, keep, Q, n = _chain_args(-1, u0, ncdim, loglstar, scale, seed, chain0, ell, None)
    st, bufs = _step_state(Q, n, dev, dimflags, worklist=True)
    o = dict(u=torch.empty((Q, n), dtype=torch.float64, device=dev), v=torch.empty((Q, n), dtype=torch.float64, device=dev),
             logl=torch.empty(Q, dtype=torch.float64, device=dev))
    for k in _lib.CHAIN_OUTPUTS['rwalk'][:3]:
        o[k] = torch.empty(Q, dtype=torch.int32, device=dev)
    args = _chain_ptrs(o, 'rwalk')
    with _torch_stream(ctx, dev):
        _step_through(model, int(walks),
                      lambda s: ctx.check(ctx.lib.b2n_rwalk_step(ctx.h, C.byref(a), int(walks), s, C.byref(st), *args)),
                      st, u0, bufs['u_prop'])
        return {k: t.cpu().numpy() for k, t in o.items()}


def _slice_batch(fn, model, u0, loglstar, scale, slices, seed, chain0, doubling, ell, ctx, peer=None):
    ctx = _ctx(ctx)
    a, keep, Q, n = _chain_args(model, u0, None, loglstar, scale, seed, chain0, ell, None)
    R = Q if peer is None else int(peer[1])
    o = _chain_outputs('slice', R, n)
    with _gather(ctx, peer):
        ctx.check(getattr(ctx.lib, fn)(ctx.h, C.byref(a), int(slices), int(bool(doubling)), *_chain_ptrs(o, 'slice')))
    return o


def rslice_batch(model, u0, loglstar, scale, slices, seed, chain0=0, doubling=False, ell=None, ctx=None,
                 peer=None):
    """RSliceSampler.sample per row of u0 (internal_samplers.py:745-855)."""
    return _slice_batch('b2n_rslice_batch', model, u0, loglstar, scale, slices, seed, chain0, doubling, ell, ctx,
                        peer)


def slice_batch(model, u0, loglstar, scale, slices, seed, chain0=0, doubling=False, ell=None, ctx=None,
                peer=None):
    """SliceSampler.sample per row of u0 (internal_samplers.py:593-709)."""
    return _slice_batch('b2n_slice_batch', model, u0, loglstar, scale, slices, seed, chain0, doubling, ell, ctx,
                        peer)


def unif_batch(model, nchain, ndim, loglstar, seed, chain0=0, ncdim=None, dimflags=None, ctx=None,
               draw_only=False, mixture=False, peer=None):
    """UniformBoundSampler.sample x nchain on the resident bound (internal_samplers.py:243-340).
    draw_only=True: just Bound.samples(nchain) (no cube test / likelihood)."""
    ctx = _ctx(ctx)
    a, keep, Q, n = _chain_args(model, None, ncdim, loglstar, 1.0, seed, chain0, None, dimflags,
                                Q=int(nchain), ndim=int(ndim))
    if draw_only:
        a.reserved = 3 if mixture else 1      # mixture: no 1/q test, q returned in 'ncall'
    R = Q if peer is None else int(peer[1])
    o = _chain_outputs('unif', R, n)
    with _gather(ctx, peer):
        ctx.check(ctx.lib.b2n_unif_batch(ctx.h, C.byref(a), *_chain_ptrs(o, 'unif')))
    return o


def unitcube_batch(model, nchain, ndim, loglstar, seed, chain0=0, ctx=None, peer=None):
    """UnitCubeSampler.sample x nchain (internal_samplers.py:343-441): prior draws until logl > loglstar."""
    ctx = _ctx(ctx)
    a, keep, Q, n = _chain_args(model, None, None, loglstar, 1.0, seed, chain0, None, None, Q=int(nchain), ndim=int(ndim))
    R = Q if peer is None else int(peer[1])
    o = _chain_outputs('unitcube', R, n)
    with _gather(ctx, peer):
        ctx.check(ctx.lib.b2n_unitcube_batch(ctx.h, C.byref(a), *_chain_ptrs(o, 'unitcube'), None))
    return o


# ---- device-resident nested-sampling rounds (include/b200nest.h, b2n_ns_*) ----------------------
def ns_create(model, nlive, ndim, batch, sampler, steps, seed, chain0=0, ncdim=None, strict_contains=True,
              facc=0.5, dlogz=0.01, maxiter=None, maxcall=None, update_interval=1 << 62, dimflags=None,
              dead_capacity=None, ctx=None, unit_cube_phase=False, first_min_ncall=0, first_min_eff=100., it0=0,
              logl_max=None):
    """Allocate the device state of a batched-replacement run (sampler: 0 rwalk, 1 rslice, 2 slice, 3 unif).
    model = -1: no in-kernel model, the rwalk chains are stepped with a TorchModel (ns_run_stepped).
    unit_cube_phase: start with rounds that draw from the prior until the first bound is due
    (need_bound = 4 once ncall >= first_min_ncall and 100 (it0 + it) / ncall < first_min_eff)."""
    ctx = _ctx(ctx)
    c = _lib.NsConfig()
    c.nlive, c.ndim, c.ncdim, c.batch = int(nlive), int(ndim), int(ncdim or ndim), int(batch)
    c.sampler, c.steps, c.model_id, c.strict_contains = int(sampler), int(steps), int(model), int(bool(strict_contains))
    c.facc, c.dlogz = float(facc), float(dlogz)
    big = (1 << 62)
    c.maxiter = int(maxiter) if maxiter is not None else big
    c.maxcall = int(maxcall) if maxcall is not None else big
    c.update_interval, c.seed, c.chain0 = int(update_interval), int(seed), int(chain0)
    if dimflags is not None:
        dimflags = np.ascontiguousarray(dimflags, dtype=np.uint8)
    c.dimflags = ptr(dimflags)
    c.unit_cube_phase, c.first_min_ncall, c.first_min_eff, c.it0 = int(bool(unit_cube_phase)), int(first_min_ncall), \
        float(first_min_eff), int(it0)
    c.use_logl_max, c.logl_max = (0, 0.0) if logl_max is None else (1, float(logl_max))
    cap = int(dead_capacity) if dead_capacity is not None else 64 * int(nlive)
    ctx.ns_stepped = None
    ctx.check(ctx.lib.b2n_ns_create(ctx.h, C.byref(c), cap))
    if int(model) == -1:         # no in-kernel model: the chains are stepped (ns_run_stepped)
        ctx.ns_stepped = (int(batch), int(ndim), int(steps), dimflags)


def ns_set_state(live_u, live_v, live_logl, logvol, logz, loglstar, ncall, scale, ctx=None):
    ctx = _ctx(ctx)
    live_u, live_v, live_logl = f64(live_u), f64(live_v), f64(live_logl)
    ctx.check(ctx.lib.b2n_ns_set_state(ctx.h, ptr(live_u), ptr(live_v), ptr(live_logl), float(logvol), float(logz),
                                       float(loglstar), 0, int(ncall), float(scale)))


def _ns_status(st):
    return {k: getattr(st, k) for k, _ in st._fields_}


def ns_run(max_rounds, check_every=0, ctx=None):
    """Enqueue up to max_rounds rounds; returns the status dict (it, ncall, rounds, logz, logvol, loglstar,
    lmax, delta_logz, scale, done, need_bound, doubling, error)."""
    ctx = _ctx(ctx)
    st = _lib.NsStatus()
    ctx.check(ctx.lib.b2n_ns_run(ctx.h, int(max_rounds), int(check_every), C.byref(st)))
    return _ns_status(st)


def ns_run_stepped(model, max_rounds, ctx=None):
    """ns_run for a run created with a TorchModel (ns_create(model_id=-1)): enqueue max_rounds rounds, each
    b2n_ns_step(3) then walks + 1 x (b2n_ns_rwalk_step, torch call), and the closing commit b2n_ns_step(1), on torch's
    current stream; read the status once at the end.  Returns ns_run's status dict."""
    ctx = _ctx(ctx)
    if ctx.ns_stepped is None:
        raise ValueError("ns_run_stepped needs a run created with a TorchModel (ns_create(model_id=-1))")
    K, n, walks, dimflags = ctx.ns_stepped
    dev = model.device(ctx)
    st, bufs = _step_state(K, n, dev, dimflags, worklist=False)
    with _torch_stream(ctx, dev):
        for _ in range(int(max_rounds)):
            ctx.check(ctx.lib.b2n_ns_step(ctx.h, 3))
            _step_through(model, walks, lambda s: ctx.check(ctx.lib.b2n_ns_rwalk_step(ctx.h, s, C.byref(st))), st,
                          bufs['u_start'], bufs['u_prop'])
        if max_rounds > 0:
            ctx.check(ctx.lib.b2n_ns_step(ctx.h, 1))
        s = ns_status(ctx)
    if s['error']:
        raise _lib._EXC.get(s['error'], RuntimeError)(
            "device rounds stopped with status %d after round %d (it %d, ncall %d)"
            % (s['error'], s['rounds'], s['it'], s['ncall']))
    return s


def ns_status(ctx=None):
    ctx = _ctx(ctx)
    st = _lib.NsStatus()
    ctx.check(ctx.lib.b2n_ns_status_get(ctx.h, C.byref(st)))
    return _ns_status(st)


def ns_set_counters(rounds, ncall_last_update, doubling, ctx=None):
    """Counters of a restored run (round index, calls at the last bound update, slice-doubling switch)."""
    ctx = _ctx(ctx)
    ctx.check(ctx.lib.b2n_ns_set_counters(ctx.h, int(rounds), int(ncall_last_update), int(bool(doubling))))


def ns_bound_updated(ctx=None):
    ctx = _ctx(ctx)
    ctx.check(ctx.lib.b2n_ns_bound_updated(ctx.h))


_ns_bound_serial = [0]


def ns_update_bound(multi, enlarge=1.0, ctx=None):
    """Sampler.update_bound on the device (b2n_ns_update_bound): fit the bound to the run's live points in HBM,
    enlarge, make resident.  Returns (nells, logvol, warn)."""
    ctx = _ctx(ctx)
    nells, warn, lv = C.c_int32(0), C.c_uint32(0), C.c_double(0.0)
    ctx.resident_key = None
    ctx.check(ctx.lib.b2n_ns_update_bound(ctx.h, int(bool(multi)), float(enlarge), C.addressof(nells), C.addressof(lv),
                                          C.addressof(warn)))
    _ns_bound_serial[0] += 1
    ctx.resident_key = ('ns', ctx.serial, _ns_bound_serial[0])     # no host bound object owns these ellipsoids
    return nells.value, lv.value, warn.value


def ns_get_bound(nells, ncdim, ctx=None):
    """The bound the last ns_update_bound built: dict(ctrs, covs, ams, axes, axlens, logvols)."""
    ctx = _ctx(ctx)
    K, n = int(nells), int(ncdim)
    o = dict(ctrs=np.empty((K, n)), covs=np.empty((K, n, n)), ams=np.empty((K, n, n)), axes=np.empty((K, n, n)),
             axlens=np.empty((K, n)), logvols=np.empty(K))
    ctx.check(ctx.lib.b2n_ns_get_bound(ctx.h, K, ptr(o['ctrs']), ptr(o['covs']), ptr(o['ams']), ptr(o['axes']),
                                       ptr(o['axlens']), ptr(o['logvols'])))
    return o


def ns_reserve_dead(capacity, ctx=None):
    ctx = _ctx(ctx)
    ctx.check(ctx.lib.b2n_ns_reserve_dead(ctx.h, int(capacity)))


def ns_get_live(nlive, ndim, ctx=None, only_u=False):
    ctx = _ctx(ctx)
    u = np.empty((nlive, ndim))
    if only_u:          # what a bound update needs
        ctx.check(ctx.lib.b2n_ns_get_live(ctx.h, ptr(u), None, None))
        return u
    v, l = np.empty((nlive, ndim)), np.empty(nlive)
    ctx.check(ctx.lib.b2n_ns_get_live(ctx.h, ptr(u), ptr(v), ptr(l)))
    return u, v, l


def ns_get_dead(first, count, ndim, ctx=None, positions=True):
    """(u, v, logl, logvol, ncall) of dead points [first, first + count); positions=False skips the two
    (count, ndim) position arrays (zero-row placeholders) -- the evidence needs only the scalars."""
    ctx = _ctx(ctx)
    u, v = (np.empty((count, ndim)), np.empty((count, ndim))) if positions else (None, None)
    l, lv, nc = np.empty(count), np.empty(count), np.empty(count, dtype=np.int32)
    ctx.check(ctx.lib.b2n_ns_get_dead(ctx.h, int(first), int(count), ptr(u), ptr(v), ptr(l), ptr(lv), ptr(nc)))
    if not positions:
        u, v = np.empty((0, ndim)), np.empty((0, ndim))
    return u, v, l, lv, nc


def ns_get_strands(first, count, ctx=None):
    """(slot, it) of dead points [first, first + count): the live slot each occupied (int32) and the dead rows of the
    device buffer recorded before it entered the live set (int64)."""
    ctx = _ctx(ctx)
    slot, it = np.empty(count, dtype=np.int32), np.empty(count, dtype=np.int64)
    ctx.check(ctx.lib.b2n_ns_get_strands(ctx.h, int(first), int(count), ptr(slot), ptr(it)))
    return slot, it


def ns_set_live_it(live_it, ctx=None):
    """Per live slot: the dead rows of the device buffer recorded before its occupant entered (negative: before the
    first row).  Follows ns_set_state, which sets them all to 0."""
    ctx = _ctx(ctx)
    a = np.ascontiguousarray(live_it, dtype=np.int64)
    ctx.check(ctx.lib.b2n_ns_set_live_it(ctx.h, ptr(a)))


def ns_get_live_it(nlive, ctx=None):
    ctx = _ctx(ctx)
    a = np.empty(int(nlive), dtype=np.int64)
    ctx.check(ctx.lib.b2n_ns_get_live_it(ctx.h, ptr(a)))
    return a


def ns_destroy(ctx=None):
    ctx = _ctx(ctx)
    ctx.check(ctx.lib.b2n_ns_destroy(ctx.h))


# ---- run uncertainties (include/b200nest.h, b2n_jitter_runs) ----------------------------------------------
def _logwt_ref(logwt_ref, N):
    wref = f64(logwt_ref)
    if len(wref) != N:
        raise ValueError("logwt_ref and logl differ in length")
    return wref


def _jitter_record(logl, samples_n, logwt_ref, kl):
    """(logl, samples_n, logwt_ref) of a jitter call as the C API takes them; logwt_ref is None when kl is False."""
    logl = f64(logl)
    n = np.ascontiguousarray(samples_n, dtype=np.int64)
    if len(n) != len(logl):
        raise ValueError("logl and samples_n differ in length")
    return logl, n, _logwt_ref(logwt_ref, len(logl)) if kl else None


def _strand_record(N, strand, base, piece_ptr, piece_strand, end):
    """(strand, base, piece_ptr, piece_strand, end) of a resample call over N samples as the C API takes them."""
    strand = np.ascontiguousarray(strand, dtype=np.int32)
    base = np.ascontiguousarray(base, dtype=np.uint8)
    pp = np.ascontiguousarray(piece_ptr, dtype=np.int64)
    ps = np.ascontiguousarray(piece_strand, dtype=np.int32)
    if len(strand) != N or len(pp) != N + 1:
        raise ValueError("logl, strand and piece_ptr differ in length")
    if end is not None:
        end = np.ascontiguousarray(end, dtype=np.uint8)
        if len(end) != N:
            raise ValueError("logl and end differ in length")
    return strand, base, pp, ps, end


def _logrwt(logrwt, N):
    """A log-reweight as the C API takes it: N float64 values, none NaN or +inf (-inf: zero weight)."""
    rw = f64(logrwt)
    if rw.shape != (N,):
        raise ValueError("logrwt must hold one value per sample (%d)" % N)
    if np.isnan(rw).any() or np.isposinf(rw).any():
        raise ValueError("logrwt holds NaN or +inf")
    return rw


def _set_reweight(ctx, rw):
    """b2n_set_reweight for the C call that follows at once (None: nothing pending)."""
    if rw is not None:
        ctx.set_reweight(ptr(rw), len(rw))


def _summaries(R, kl):
    """The per-realisation outputs logz, logzerr, h and, with kl, kld (R each)."""
    o = dict(logz=np.empty(R), logzerr=np.empty(R), h=np.empty(R))
    if kl:
        o['kld'] = np.empty(R)
    return o


def jitter_runs(logl, samples_n, R, seed, chain0=0, approx=False, logwt_ref=None, logz_ref=None, arrays=False,
                logrwt=None, ctx=None):
    """R prior-volume realisations of one record (jitter_run / kld_error, utils.py:1317-1408, 1932-1997); realisation
    r draws from the B2N stream (seed, chain0 + r).  Returns dict(logz, logzerr, h[, kld]) with R values each (the
    last elements of the realisations' arrays) and, with arrays=True, logvol_arr, logwt_arr, logz_arr[, kld_arr]
    (R x N).  kld needs the input run's weights: logwt_ref (N) and logz_ref (its logz[-1]).  logrwt (N): a log-reweight
    added to every logwt of every realisation (b2n_set_reweight)."""
    ctx = _ctx(ctx)
    kl = logwt_ref is not None
    logl, n, wref = _jitter_record(logl, samples_n, logwt_ref, kl)
    N, R = len(logl), int(R)
    rw = None if logrwt is None else _logrwt(logrwt, N)
    o = _summaries(R, kl)
    if arrays:
        for k in ('logvol', 'logwt', 'logz') + (('kld',) if kl else ()):
            o[k + '_arr'] = np.empty((R, N))
    _set_reweight(ctx, rw)
    ctx.check(ctx.lib.b2n_jitter_runs(ctx.h, ptr(logl), ptr(n), N, ptr(wref), float(logz_ref) if kl else 0.0,
                                      int(bool(approx)), R, int(seed), int(chain0), ptr(o['logz']),
                                      ptr(o['logzerr']), ptr(o['h']), ptr(o.get('kld')), ptr(o.get('logvol_arr')),
                                      ptr(o.get('logwt_arr')), ptr(o.get('logz_arr')), ptr(o.get('kld_arr'))))
    return o


def resample_runs(logl, strand, base, piece_ptr, piece_strand, end, R, seed, chain0=0, logwt_ref=None, logz_ref=None,
                  multiplicities=False, logrwt=None, ctx=None):
    """R bootstrap realisations of one strand-labelled record (resample_run / kld_error(error='resample'),
    utils.py:1495-1660, 1932-1997); realisation r draws from the B2N stream (seed, chain0 + r).  strand: compacted
    strand index per sample (0..S-1); base: per strand, drawn in the base event; piece_ptr / piece_strand: CSR of
    the pieces whose first covered sample is i; end: per sample, the copies of a final live point share out its live
    count (or None).  Returns dict(logz, logzerr, h[, kld]) with R values each and, with multiplicities=True, mult
    (R x S, int64): the times every strand is drawn.  logrwt (N): a log-reweight added to the logwt of every copy of
    every sample (b2n_set_reweight)."""
    ctx = _ctx(ctx)
    logl = f64(logl)
    N = len(logl)
    strand, base, pp, ps, end = _strand_record(N, strand, base, piece_ptr, piece_strand, end)
    S, R = len(base), int(R)
    kl = logwt_ref is not None
    wref = _logwt_ref(logwt_ref, N) if kl else None
    rw = None if logrwt is None else _logrwt(logrwt, N)
    o = _summaries(R, kl)
    m = np.empty((R, S), dtype=np.int32) if multiplicities else None
    _set_reweight(ctx, rw)
    ctx.check(ctx.lib.b2n_resample_runs(ctx.h, ptr(logl), ptr(strand), N, S, ptr(base), ptr(pp), ptr(ps), ptr(end),
                                        ptr(wref), float(logz_ref) if kl else 0.0, R, int(seed), int(chain0),
                                        ptr(o['logz']), ptr(o['logzerr']), ptr(o['h']), ptr(o.get('kld')), ptr(m)))
    if multiplicities:
        o['mult'] = m.astype(np.int64)
    return o


# ---- posterior summaries (include/b200nest.h, b2n_weighted_stats / b2n_jitter_posterior / b2n_resample_posterior) --
def _post_outputs(R, n, q, moments):
    o = dict(mean=np.empty((R, n)), cov=np.empty((R, n, n))) if moments else {}
    if q is not None:
        o['quantiles'] = np.empty((R, n, len(q)))
    return o


def _post_q(q):
    if q is None:
        return None
    q = f64(np.atleast_1d(q))
    if q.ndim != 1 or len(q) < 1:
        raise ValueError("q must be a non-empty list of quantiles")
    if np.any(q < 0.0) or np.any(q > 1.0) or np.isnan(q).any():
        raise ValueError("Quantiles must be between 0. and 1.")
    return q


def _post_x(x, N):
    x = f64(x)
    if x.ndim != 2 or len(x) != N or x.shape[1] < 1:
        raise ValueError("the sample positions must be an array of shape (%d, ndim)" % N)
    return x


def weighted_stats(x, w, shift, q=None, moments=True, ctx=None):
    """Weighted means, covariances and quantiles of the samples x (N x n) under R weight vectors w (R x N, >= 0),
    second moments about `shift` (n).  Returns dict(mean (R x n), cov (R x n x n)) with moments=True and
    quantiles (R x n x nq) with q."""
    ctx = _ctx(ctx)
    w = f64(np.atleast_2d(w))
    R, N = w.shape
    x = _post_x(x, N)
    n = x.shape[1]
    shift = f64(shift)
    if shift.shape != (n,):
        raise ValueError("shift must hold one number per dimension")
    q = _post_q(q)
    o = _post_outputs(R, n, q, moments)
    ctx.check(ctx.lib.b2n_weighted_stats(ctx.h, ptr(x), N, n, ptr(w), R, ptr(shift), ptr(q),
                                         0 if q is None else len(q), ptr(o.get('mean')), ptr(o.get('cov')),
                                         ptr(o.get('quantiles'))))
    return o


def jitter_posterior(logl, samples_n, x, R, seed, chain0=0, approx=False, logwt_ref=None, logz_ref=None, q=None,
                     logrwt=None, ctx=None):
    """jitter_runs plus, per realisation, the weighted mean (R x n), covariance (R x n x n) and, with q, quantiles
    (R x n x nq) of the sample positions x (N x n).  logwt_ref / logz_ref (the record's own) are required.  logrwt:
    as in jitter_runs."""
    ctx = _ctx(ctx)
    logl, n_, wref = _jitter_record(logl, samples_n, logwt_ref, True)
    N, R = len(logl), int(R)
    x = _post_x(x, N)
    q = _post_q(q)
    rw = None if logrwt is None else _logrwt(logrwt, N)
    o = _summaries(R, True)
    o.update(_post_outputs(R, x.shape[1], q, True))
    _set_reweight(ctx, rw)
    ctx.check(ctx.lib.b2n_jitter_posterior(ctx.h, ptr(logl), ptr(n_), N, ptr(wref), float(logz_ref),
                                           int(bool(approx)), R, int(seed), int(chain0), ptr(x), x.shape[1], ptr(q),
                                           0 if q is None else len(q), ptr(o['logz']), ptr(o['logzerr']), ptr(o['h']),
                                           ptr(o['kld']), ptr(o['mean']), ptr(o['cov']), ptr(o.get('quantiles'))))
    return o


def resample_posterior(logl, strand, base, piece_ptr, piece_strand, end, x, R, seed, chain0=0, logwt_ref=None,
                       logz_ref=None, q=None, logrwt=None, ctx=None):
    """resample_runs plus, per realisation, the weighted mean, covariance and, with q, quantiles of the sample
    positions x (N x n) over the realisation's copies.  logwt_ref / logz_ref (the record's own) are required.  logrwt:
    as in resample_runs."""
    ctx = _ctx(ctx)
    logl = f64(logl)
    N = len(logl)
    strand, base, pp, ps, end = _strand_record(N, strand, base, piece_ptr, piece_strand, end)
    S, R = len(base), int(R)
    wref = _logwt_ref(logwt_ref, N)
    x = _post_x(x, N)
    q = _post_q(q)
    rw = None if logrwt is None else _logrwt(logrwt, N)
    o = _summaries(R, True)
    o.update(_post_outputs(R, x.shape[1], q, True))
    _set_reweight(ctx, rw)
    ctx.check(ctx.lib.b2n_resample_posterior(ctx.h, ptr(logl), ptr(strand), N, S, ptr(base), ptr(pp), ptr(ps),
                                             ptr(end), ptr(wref), float(logz_ref), R, int(seed), int(chain0), ptr(x),
                                             x.shape[1], ptr(q), 0 if q is None else len(q), ptr(o['logz']),
                                             ptr(o['logzerr']), ptr(o['h']), ptr(o['kld']), ptr(o['mean']),
                                             ptr(o['cov']), ptr(o.get('quantiles'))))
    return o


# ---- equal-weight draws (include/b200nest.h, b2n_resample_equal / b2n_jitter_equal / b2n_resample_equal_runs) ------
EQUAL_CHAIN0 = 1 << 62          # B2N_EQUAL_CHAIN0: the draws of realisation r use the stream (seed, this + chain0 + r)


def _equal_outputs(R, N, M, x, counts):
    """The outputs of an equal-weight call: idx (R x M), wsum (R), counts (R x N) with counts, x (R x M x k) with x."""
    o = dict(idx=np.empty((R, M), dtype=np.int32), wsum=np.empty(R))
    if counts:
        o['counts'] = np.empty((R, N), dtype=np.int32)
    if x is not None:
        o['x'] = np.empty((R, M, x.shape[1]))
    return o


def _equal_x(x, N):
    """The rows to gather as the C API takes them (N x k float64), or None."""
    if x is None:
        return None
    x = f64(x)
    if x.ndim != 2 or len(x) != N or x.shape[1] < 1:
        raise ValueError("the rows to gather must be an array of shape (%d, k)" % N)
    return x


def _equal_done(o):
    o['idx'] = o['idx'].astype(np.int64)
    if 'counts' in o:
        o['counts'] = o['counts'].astype(np.int64)
    return o


def resample_equal(w, M, seed, chain0=0, x=None, counts=False, ctx=None):
    """M equal-weight draws from each of R weight vectors w (R x N; finite, >= 0, positive sum) by the reference's
    systematic resampling, with its rounding (resample_equal, utils.py:1120-1187); vector r uses the B2N stream (seed,
    chain0 + r).  Returns dict(idx (R x M, int64): the drawn samples in random order, wsum (R): the sequential sum of
    each vector) and, with counts=True, counts (R x N, int64): the times each sample is drawn; with x (N x k), x (R x M
    x k): its rows x[idx]."""
    ctx = _ctx(ctx)
    w = f64(np.atleast_2d(w))
    R, N = w.shape
    x = _equal_x(x, N)
    o = _equal_outputs(R, N, int(M), x, counts)
    ctx.check(ctx.lib.b2n_resample_equal(ctx.h, ptr(w), N, R, int(M), int(seed), int(chain0), ptr(x),
                                         0 if x is None else x.shape[1], ptr(o['idx']), ptr(o.get('counts')),
                                         ptr(o['wsum']), ptr(o.get('x'))))
    return _equal_done(o)


def jitter_equal(logl, samples_n, R, M, seed, chain0=0, approx=False, logwt_ref=None, logz_ref=None, x=None,
                 counts=False, logrwt=None, ctx=None):
    """jitter_runs plus, per realisation, M equal-weight draws over the record's samples under its weights
    exp(logwt - logz[-1]) (resample_equal's outputs above).  The draws of realisation r use the stream (seed,
    EQUAL_CHAIN0 + chain0 + r).  logwt_ref / logz_ref (the record's own) are required.  logrwt: as in jitter_runs."""
    ctx = _ctx(ctx)
    logl, n_, wref = _jitter_record(logl, samples_n, logwt_ref, True)
    N, R = len(logl), int(R)
    x = _equal_x(x, N)
    rw = None if logrwt is None else _logrwt(logrwt, N)
    o = _summaries(R, True)
    o.update(_equal_outputs(R, N, int(M), x, counts))
    _set_reweight(ctx, rw)
    ctx.check(ctx.lib.b2n_jitter_equal(ctx.h, ptr(logl), ptr(n_), N, ptr(wref), float(logz_ref), int(bool(approx)), R,
                                       int(seed), int(chain0), int(M), ptr(x), 0 if x is None else x.shape[1],
                                       ptr(o['logz']), ptr(o['logzerr']), ptr(o['h']), ptr(o['kld']), ptr(o['idx']),
                                       ptr(o.get('counts')), ptr(o['wsum']), ptr(o.get('x'))))
    return _equal_done(o)


def resample_equal_runs(logl, strand, base, piece_ptr, piece_strand, end, R, M, seed, chain0=0, logwt_ref=None,
                        logz_ref=None, x=None, counts=False, logrwt=None, ctx=None):
    """resample_runs plus, per realisation, M equal-weight draws over the record's samples, each weighted by the sum
    of its copies' exp(logwt - logz[-1]) (a sample drawn 0 times is never drawn).  The draws of realisation r use the
    stream (seed, EQUAL_CHAIN0 + chain0 + r).  logwt_ref / logz_ref (the record's own) are required.  logrwt: as in
    resample_runs."""
    ctx = _ctx(ctx)
    logl = f64(logl)
    N = len(logl)
    strand, base, pp, ps, end = _strand_record(N, strand, base, piece_ptr, piece_strand, end)
    S, R = len(base), int(R)
    wref = _logwt_ref(logwt_ref, N)
    x = _equal_x(x, N)
    rw = None if logrwt is None else _logrwt(logrwt, N)
    o = _summaries(R, True)
    o.update(_equal_outputs(R, N, int(M), x, counts))
    _set_reweight(ctx, rw)
    ctx.check(ctx.lib.b2n_resample_equal_runs(ctx.h, ptr(logl), ptr(strand), N, S, ptr(base), ptr(pp), ptr(ps),
                                              ptr(end), ptr(wref), float(logz_ref), R, int(seed), int(chain0), int(M),
                                              ptr(x), 0 if x is None else x.shape[1], ptr(o['logz']),
                                              ptr(o['logzerr']), ptr(o['h']), ptr(o['kld']), ptr(o['idx']),
                                              ptr(o.get('counts')), ptr(o['wsum']), ptr(o.get('x'))))
    return _equal_done(o)


def merge_runs(logl, samples_n, run_ptr, nbase, lowedge=None, arrays=True, ctx=None):
    """R records merged into one (merge_runs / _merge_two, utils.py:1817-1900, 2045-2225; include/b200nest.h,
    b2n_merge_runs).  logl / samples_n: the records concatenated, run r = [run_ptr[r], run_ptr[r + 1]), each run's
    logl ascending; the first nbase runs are the base group (pairwise tree), the others add-on runs merged in order;
    lowedge (R): each run's low edge (None: -inf for all).  Returns dict(perm, samples_n, logz_end, logzerr_end, h_end):
    the index in the concatenation of every merged sample, the merged live counts and the last elements of logz,
    logzerr and information; with arrays=True also logvol, logwt, logz, logzvar, h (N each)."""
    logl = f64(logl)
    n = np.ascontiguousarray(samples_n, dtype=np.int64)
    rp = np.ascontiguousarray(run_ptr, dtype=np.int64)
    N, R = len(logl), len(rp) - 1
    if len(n) != N:
        raise ValueError("logl and samples_n differ in length")
    if R < 1 or rp[0] != 0 or rp[-1] != N or np.any(np.diff(rp) < 1):
        raise ValueError("run_ptr must run from 0 to len(logl) through non-empty runs")
    if not 1 <= int(nbase) <= R:
        raise ValueError("nbase must lie in 1..%d" % R)
    if np.isnan(logl).any():
        raise ValueError("logl holds NaN")
    inner = np.ones(max(N - 1, 0), dtype=bool)
    inner[rp[1:-1] - 1] = False                   # pairs that straddle two runs
    if np.any(np.diff(logl)[inner] < 0):
        raise ValueError("the logl of every run must be ascending")
    if np.any(n < 1):
        raise ValueError("samples_n must be >= 1")
    le = None
    if lowedge is not None:
        le = f64(lowedge)
        if len(le) != R or np.isnan(le).any():
            raise ValueError("lowedge must hold one number per run")
    o = dict(perm=np.empty(N, dtype=np.int64), samples_n=np.empty(N, dtype=np.int64))
    last = np.empty(3)
    if arrays:
        for k in ('logvol', 'logwt', 'logz', 'logzvar', 'h'):
            o[k] = np.empty(N)
    ctx = _ctx(ctx)
    ctx.check(ctx.lib.b2n_merge_runs(ctx.h, ptr(logl), ptr(n), ptr(rp), R, int(nbase), ptr(le), ptr(o['perm']),
                                     ptr(o['samples_n']), ptr(last), ptr(o.get('logvol')), ptr(o.get('logwt')),
                                     ptr(o.get('logz')), ptr(o.get('logzvar')), ptr(o.get('h'))))
    o.update(logz_end=float(last[0]), logzerr_end=float(last[1]), h_end=float(last[2]))
    return o


def compute_integrals(logl, logvol, logrwt=None, ctx=None):
    """compute_integrals(logl, logvol, reweight=logrwt) (utils.py:1411-1467; include/b200nest.h,
    b2n_compute_integrals) on the GPU.  Returns dict(logwt, logz, logzvar, h) (N each)."""
    logl = f64(logl)
    N = len(logl)
    logvol = f64(logvol)
    if logl.ndim != 1 or N < 1 or logvol.shape != (N,):
        raise ValueError("logl and logvol must be 1-D arrays of the same, non-zero length")
    rw = None if logrwt is None else _logrwt(logrwt, N)
    o = {k: np.empty(N) for k in ('logwt', 'logz', 'logzvar', 'h')}
    ctx = _ctx(ctx)
    ctx.check(ctx.lib.b2n_compute_integrals(ctx.h, ptr(logl), ptr(logvol), ptr(rw), N, None, ptr(o['logwt']),
                                            ptr(o['logz']), ptr(o['logzvar']), ptr(o['h'])))
    return o

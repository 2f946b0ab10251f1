"""GPU: batched rwalk chains vs (a) fixtures produced by the UNMODIFIED reference
driven with the scripted Philox stream, (b) the oracle on fresh seeded inputs,
(c) size-independent properties at the BASELINE C2 size.

float64 tolerance: device libm (log, sincospi, pow) and FMA contraction differ
from numpy/glibc in the last bits, so chain end points are compared at
rtol 1e-9; accept/reject COUNTS must agree exactly for all but a vanishing
fraction of chains (a proposal whose logl is within ~1e-13 of loglstar can flip).
"""
import numpy as np
import pytest

from dynesty_b200 import ops
from helpers import MODELS, device_model, close, SEED
from oracle import samplers as OS, philox, bounding as OB

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('name', ['g6', 'g6nc', 'wall', 'g50', 'n200'])
def test_rwalk_golden(golden, name):
    g = golden['chains']
    p = 'rwalk_%s_' % name
    m = MODELS[name]
    dm = device_model(m)
    per, ref = g[p + 'periodic'], g[p + 'reflective']
    flags = ops.dimflags_from(m.ndim, per if len(per) else None, ref if len(ref) else None)
    ops.bound_set(g[p + 'axes'])
    o = ops.rwalk_batch(dm.model_id(), g[p + 'u0'], float(g[p + 'loglstar']), float(g[p + 'scale']),
                        int(g[p + 'walks']), SEED, chain0=int(g[p + 'chain0']),
                        ncdim=int(g[p + 'ncdim']), dimflags=flags)
    assert np.array_equal(o['n_accept'], g[p + 'accept'])
    assert np.array_equal(o['n_reject'], g[p + 'reject'])
    assert np.array_equal(o['ncall'], g[p + 'ncall'])
    close(o['u'], g[p + 'u'], rtol=1e-9)
    close(o['v'], g[p + 'v'], rtol=1e-9)
    np.testing.assert_allclose(o['logl'], g[p + 'logl'], rtol=1e-9, atol=1e-9)


def _cloud(rng, npts, n, spread):
    C = np.full((n, n), 0.4)
    np.fill_diagonal(C, 1.0)
    return 0.5 + spread * rng.standard_normal((npts, n)) @ np.linalg.cholesky(C).T


def test_rwalk_vs_oracle_multi_ellipsoid():
    """Chains spread over K=3 ellipsoids (grouping by ellipsoid must not change results)."""
    m = MODELS['g6']
    dm = device_model(m)
    rng = np.random.default_rng(11)
    pts = _cloud(rng, 400, 6, 0.06)
    ells = [OB.bounding_ellipsoid(pts[i::3]) for i in range(3)]
    axes = np.array([e.axes for e in ells])
    logl = m.loglike(m.prior_transform(pts))
    loglstar = float(np.quantile(logl, 0.4))
    u0 = pts[logl > loglstar][:100]
    ell = rng.integers(3, size=len(u0)).astype(np.int32)
    ops.bound_set(axes)
    o = ops.rwalk_batch(dm.model_id(), u0, loglstar, 0.9, 20, 777, chain0=5000, ell=ell)
    bad = 0
    for i in range(len(u0)):
        r = OS.rwalk_chain(u0[i], loglstar, axes[ell[i]], 0.9, m, philox.ChainStream(777, 5000 + i), 20)
        if r['n_accept'] != o['n_accept'][i]:
            bad += 1
            continue
        close(o['u'][i], r['u'], rtol=1e-9)
        assert abs(o['logl'][i] - r['logl']) < 1e-9 * max(1, abs(r['logl']))
    assert bad == 0


def test_rwalk_c2_properties():
    """BASELINE C2 size (50-D, 2000 chains x 70 walks): size-independent properties."""
    m = MODELS['g50']
    dm = device_model(m)
    rng = np.random.default_rng(5)
    pts = _cloud(rng, 2000, 50, 0.02)
    e = OB.bounding_ellipsoid(pts)
    logl = m.loglike(m.prior_transform(pts))
    loglstar = float(np.quantile(logl, 0.2))
    u0 = pts[logl > loglstar]
    u0 = u0[rng.integers(len(u0), size=2000)]
    ops.bound_set(e.axes)
    o = ops.rwalk_batch(dm.model_id(), u0, loglstar, 0.3, 70, SEED, chain0=0)
    assert np.all(o['ncall'] == 70)
    assert np.all(o['n_accept'] + o['n_reject'] == 70)
    assert np.all((o['u'] > 0) & (o['u'] < 1))
    # every returned point satisfies the constraint and (v, logl) are consistent with u
    assert np.all(o['logl'] > loglstar)
    v0 = m.prior_transform(o['u'])
    close(o['v'], v0, rtol=1e-13)
    np.testing.assert_allclose(o['logl'], m.loglike(v0), rtol=1e-10)
    # chains that never accepted stay at their start
    stay = o['n_accept'] == 0
    assert np.array_equal(o['u'][stay], u0[stay])
    assert 0.05 < o['n_accept'].mean() / 70 < 0.95
    # determinism + independence of the batch composition (counter-based RNG)
    o2 = ops.rwalk_batch(dm.model_id(), u0[100:200], loglstar, 0.3, 70, SEED, chain0=100)
    assert np.array_equal(o2['u'], o['u'][100:200])
    # spot-check 8 chains against the oracle
    for i in (0, 1, 500, 999, 1000, 1500, 1998, 1999):
        r = OS.rwalk_chain(u0[i], loglstar, e.axes, 0.3, m, philox.ChainStream(SEED, i), 70)
        assert r['n_accept'] == o['n_accept'][i]
        close(o['u'][i], r['u'], rtol=1e-9)


def test_rwalk_edge_cases():
    m = MODELS['g6']
    dm = device_model(m)
    ops.bound_set(np.eye(6) * 0.01)
    # empty batch
    o = ops.rwalk_batch(dm.model_id(), np.empty((0, 6)), -1e300, 1.0, 5, 1)
    assert o['u'].shape == (0, 6)
    # impossible constraint: nothing accepted, start returned with its own logl
    u0 = np.full((3, 6), 0.5)
    o = ops.rwalk_batch(dm.model_id(), u0, 1e300, 1.0, 9, 1)
    assert np.all(o['n_accept'] == 0) and np.all(o['n_reject'] == 9)
    assert np.array_equal(o['u'], u0)
    np.testing.assert_allclose(o['logl'], m.loglike(m.prior_transform(u0)), rtol=1e-12)
    # huge scale: every proposal leaves the cube -> rejects without likelihood calls
    o = ops.rwalk_batch(dm.model_id(), u0, -1e300, 1e6, 9, 1)
    assert np.all(o['n_reject'] >= 8)
    # wrong resident bound dimension is an argument error, not a silent fallback
    ops.bound_set(np.eye(4))
    with pytest.raises(ValueError):
        ops.rwalk_batch(dm.model_id(), u0, 0.0, 1.0, 5, 1)


def test_rwalk_c4_properties():
    """BASELINE C4 shape (200-D iid normal, normal-ppf prior, single ellipsoid, walks=220):
    the axes matrix (320 KB) does not fit in shared memory -> global/L2 path."""
    m = MODELS['n200']
    dm = device_model(m)
    rng = np.random.default_rng(8)
    pts = 0.5 + 0.04 * rng.standard_normal((4000, 200))
    e = OB.bounding_ellipsoid(pts)
    logl = m.loglike(m.prior_transform(pts))
    loglstar = float(np.quantile(logl, 0.3))
    u0 = pts[logl > loglstar][:600]
    ops.bound_set(e.axes)
    o = ops.rwalk_batch(dm.model_id(), u0, loglstar, 0.12, 220, SEED, chain0=77)
    assert np.all(o['ncall'] == 220) and np.all(o['n_accept'] + o['n_reject'] == 220)
    assert np.all(o['logl'] > loglstar)
    v0 = m.prior_transform(o['u'])
    close(o['v'], v0, rtol=1e-12)
    np.testing.assert_allclose(o['logl'], m.loglike(v0), rtol=1e-10)
    assert 0.05 < o['n_accept'].mean() / 220 < 0.95
    for i in (0, 599):
        r = OS.rwalk_chain(u0[i], loglstar, e.axes, 0.12, m, philox.ChainStream(SEED, 77 + i), 220)
        assert r['n_accept'] == o['n_accept'][i]
        close(o['u'][i], r['u'], rtol=1e-9)


def test_rwalk_large_queue_many_ellipsoids():
    """Queue much larger than 16 x SMs (warps loop over chains) spread over K=5 ellipsoids."""
    m = MODELS['g6']
    dm = device_model(m)
    rng = np.random.default_rng(21)
    pts = _cloud(rng, 600, 6, 0.06)
    ells = [OB.bounding_ellipsoid(pts[i::5]) for i in range(5)]
    axes = np.array([e.axes for e in ells])
    logl = m.loglike(m.prior_transform(pts))
    loglstar = float(np.quantile(logl, 0.4))
    good = pts[logl > loglstar]
    Q = 20000
    u0 = good[rng.integers(len(good), size=Q)]
    ell = rng.integers(5, size=Q).astype(np.int32)
    ops.bound_set(axes)
    o = ops.rwalk_batch(dm.model_id(), u0, loglstar, 0.9, 10, 99, chain0=0, ell=ell)
    assert np.all(o['logl'] > loglstar) and np.all(o['ncall'] == 10)
    for i in (0, 1, 7777, 19999):
        r = OS.rwalk_chain(u0[i], loglstar, axes[ell[i]], 0.9, m, philox.ChainStream(99, i), 10)
        assert r['n_accept'] == o['n_accept'][i]
        close(o['u'][i], r['u'], rtol=1e-9)


class _Impl:
    """Force one of the two rwalk kernels (b2n_rwalk.cu reads B2N_RWALK_IMPL per call)."""

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        import os
        self.old = os.environ.get('B2N_RWALK_IMPL')
        os.environ['B2N_RWALK_IMPL'] = self.name

    def __exit__(self, *a):
        import os
        if self.old is None:
            os.environ.pop('B2N_RWALK_IMPL', None)
        else:
            os.environ['B2N_RWALK_IMPL'] = self.old


@pytest.mark.parametrize('name', ['g6', 'wall', 'g50'])
def test_rwalk_mma_kernel_golden(golden, name):
    """The lock-step DMMA kernel against the reference-generated fixtures (ncdim == ndim cases)."""
    g = golden['chains']
    p = 'rwalk_%s_' % name
    m = MODELS[name]
    dm = device_model(m)
    per, ref = g[p + 'periodic'], g[p + 'reflective']
    flags = ops.dimflags_from(m.ndim, per if len(per) else None, ref if len(ref) else None)
    ops.bound_set(g[p + 'axes'])
    with _Impl('mma'):
        o = ops.rwalk_batch(dm.model_id(), g[p + 'u0'], float(g[p + 'loglstar']), float(g[p + 'scale']),
                            int(g[p + 'walks']), SEED, chain0=int(g[p + 'chain0']), dimflags=flags)
    assert np.array_equal(o['n_accept'], g[p + 'accept'])
    assert np.array_equal(o['n_reject'], g[p + 'reject'])
    close(o['u'], g[p + 'u'], rtol=1e-9)
    close(o['v'], g[p + 'v'], rtol=1e-9)
    np.testing.assert_allclose(o['logl'], g[p + 'logl'], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize('like', ['g50', 'n40diag', 'egg32', 'shell20', 'g100', 'n130diag'])
def test_rwalk_mma_matches_warp_kernel(like):
    """Both kernels on the same queue (K = 3 ellipsoids, 5000 chains > 16 per CTA): identical
    accept counts, end points equal to round-off, for every likelihood kind."""
    from oracle import likelihoods as OL
    m = {'g50': MODELS['g50'], 'n40diag': OL.iid_normal_ppf(40), 'egg32': OL.eggbox(32),
         'shell20': OL.shells(20), 'g100': OL.gauss_corr(100, 0.4, 5.), 'n130diag': OL.iid_normal_ppf(130)}[like]
    n = m.ndim
    dm = device_model(m)
    rng = np.random.default_rng(n)
    pts = (0.5 + 0.03 * rng.standard_normal((3000, n))) if like != 'egg32' else rng.random((3000, n))
    logl = m.loglike(m.prior_transform(pts))
    loglstar = float(np.quantile(logl, 0.3))
    good = pts[logl > loglstar]
    ells = [OB.bounding_ellipsoid(good[i::3]) for i in range(3)]
    axes = np.array([e.axes for e in ells])
    Q = 5000
    u0 = good[rng.integers(len(good), size=Q)]
    ell = rng.integers(3, size=Q).astype(np.int32)
    ops.bound_set(axes)
    out = {}
    # n <= 64: register-fragment DMMA kernel (forced); n > 64: 'auto' picks the streamed-fragment one
    for impl in ('warp', 'mma'):
        with _Impl(impl if (impl == 'warp' or n <= 64) else 'auto'):
            out[impl] = ops.rwalk_batch(dm.model_id(), u0, loglstar, 0.4, 30, 4242, chain0=9, ell=ell)
    a, b = out['warp'], out['mma']
    same = a['n_accept'] == b['n_accept']
    assert same.mean() > 0.999            # a proposal within round-off of loglstar may flip
    close(b['u'][same], a['u'][same], rtol=1e-9)
    np.testing.assert_allclose(b['logl'][same], a['logl'][same], rtol=1e-9, atol=1e-9)
    assert np.all(b['logl'] > loglstar) and np.all(b['n_accept'] + b['n_reject'] == 30)
    assert 0.002 < b['n_accept'].mean() / 30 < 0.98      # (eggbox at 32-D accepts ~1 %)


@pytest.mark.parametrize('n,walks', [(50, 30), (62, 17), (64, 17), (32, 8), (52, 70)])
def test_rwalk_lockstep_variants_agree(n, walks):
    """The lock-step kernels for the precision-matrix Gaussian -- rwalk_mma_kernel (B2N_RWALK_IMPL=mma) and the default,
    which is the warp-specialised kernel at 32, 50, 52, 62 (symmetric quadratic form, static tile schedule: n at the
    largest slab count of each KT) -- on one queue with 3 ellipsoids, several groups of chains per CTA and a ring that is
    not a multiple of 8 steps: same draws, so the same accept counts (up to proposals within round-off of the threshold)
    and end points equal to round-off."""
    from oracle import likelihoods as OL
    m = OL.gauss_corr(n, 0.4, 5.)
    dm = device_model(m)
    rng = np.random.default_rng(100 + n)
    pts = 0.5 + 0.03 * rng.standard_normal((3000, n))
    logl = m.loglike(m.prior_transform(pts))
    loglstar = float(np.quantile(logl, 0.3))
    good = pts[logl > loglstar]
    ells = [OB.bounding_ellipsoid(good[i::3]) for i in range(3)]
    ops.bound_set(np.array([e.axes for e in ells]))
    Q = 5003
    u0 = good[rng.integers(len(good), size=Q)]
    ell = rng.integers(3, size=Q).astype(np.int32)
    impls = ('mma', 'auto')
    out = {}
    for impl in impls:
        with _Impl(impl):
            out[impl] = ops.rwalk_batch(dm.model_id(), u0, loglstar, 0.4, walks, 777, chain0=11, ell=ell)
    a, b = out['mma'], out['auto']
    assert np.all(a['n_accept'] + a['n_reject'] == walks) and a['n_accept'].mean() > 0.05 * walks
    same = a['n_accept'] == b['n_accept']
    assert same.mean() > 0.999
    close(b['u'][same], a['u'][same], rtol=1e-9)
    close(b['v'][same], a['v'][same], rtol=1e-9)
    np.testing.assert_allclose(b['logl'][same], a['logl'][same], rtol=1e-9, atol=1e-9)
    assert np.all(b['logl'] > loglstar) and np.all(b['n_accept'] + b['n_reject'] == walks)
    # wrapped dimensions: the generic (not straight-line) chain phase of the warp-specialised kernel
    flags = ops.dimflags_from(n, [0, 3, n - 1], [5, 6])
    fo = {}
    for impl in impls:
        with _Impl(impl):
            fo[impl] = ops.rwalk_batch(dm.model_id(), u0[:777], loglstar, 0.4, walks, 778, chain0=3, ell=ell[:777],
                                       dimflags=flags)
    same = fo['mma']['n_accept'] == fo['auto']['n_accept']
    assert same.mean() > 0.995
    close(fo['auto']['u'][same], fo['mma']['u'][same], rtol=1e-9)
    np.testing.assert_allclose(fo['auto']['logl'][same], fo['mma']['logl'][same], rtol=1e-9, atol=1e-9)
    # a start point that never moves keeps its (recomputed) v and logl in every kernel
    hi = 1e300
    for impl in impls:
        with _Impl(impl):
            o = ops.rwalk_batch(dm.model_id(), u0[:64], hi, 0.4, 9, 5, chain0=0, ell=ell[:64])
        assert np.all(o['n_accept'] == 0)
        np.testing.assert_array_equal(o['u'], u0[:64])
        np.testing.assert_allclose(o['logl'], m.loglike(m.prior_transform(u0[:64])), rtol=1e-10)


@pytest.mark.parametrize('sampler', ['rwalk', 'rslice'])
def test_pinned_buffers_are_used_in_place(sampler):
    """Host-pointer mode with PINNED caller buffers: the chain kernels read the start points and write the
    finished chains straight through the buffers' device alias (no staging copy, csrc/b2n_common.cuh
    b2n_zc_ok); results must be identical to the staged path used for pageable numpy arrays."""
    import torch
    m = MODELS['g50']
    dm = device_model(m)
    rng = np.random.default_rng(11)
    pts = _cloud(rng, 600, 50, 0.02)
    e = OB.bounding_ellipsoid(pts)
    logl = m.loglike(m.prior_transform(pts))
    loglstar = float(np.quantile(logl, 0.2))
    u0 = pts[logl > loglstar][:256]
    Q, n = u0.shape
    ops.bound_set(e.axes)
    pin = lambda *s, dt=torch.float64: torch.empty(*s, dtype=dt).pin_memory()
    h_u0 = pin(Q, n)
    h_u0.numpy()[:] = u0
    if sampler == 'rwalk':
        ref = ops.rwalk_batch(dm.model_id(), u0, loglstar, 0.3, 30, SEED, chain0=7)
        out = dict(u=pin(Q, n), v=pin(Q, n), logl=pin(Q), n_accept=pin(Q, dt=torch.int32),
                   n_reject=pin(Q, dt=torch.int32), ncall=pin(Q, dt=torch.int32))
        for t in out.values():
            t.zero_()
        o = ops.rwalk_batch(dm.model_id(), h_u0.numpy(), loglstar, 0.3, 30, SEED, chain0=7,
                            out={k: t.numpy() for k, t in out.items()})
    else:
        ref = ops.rslice_batch(dm.model_id(), u0, loglstar, 0.3, 4, SEED, chain0=7)
        o = ops.rslice_batch(dm.model_id(), h_u0.numpy(), loglstar, 0.3, 4, SEED, chain0=7)   # pinned input only
    for k in ref:
        assert np.array_equal(np.asarray(o[k]), ref[k]), k


@pytest.mark.parametrize('name,ncdim', [('g6', 4), ('g6', None), ('g50', None), ('n200', None)])
@pytest.mark.parametrize('pinned', [False, True])
def test_start_points_by_index(name, ncdim, pinned):
    """b2n_set_start_rows: the chain kernels read their start points as rows idx[q] of the whole live set (the
    gather of Sampler.propose_live / _fill_queue, sampler.py:469-491, 708-717, done by the kernel).  Every rwalk
    kernel (warp per chain, lock-step DMMA, warp-specialised, streamed) must give exactly the chains it gives for
    the gathered rows; pageable and pinned (zero-copy) live sets; the setting lasts for one call; a bad index is an
    argument error."""
    import torch
    m = MODELS[name]
    dm = device_model(m)
    n = m.ndim
    rng = np.random.default_rng(3)
    pts = 0.5 + (0.02 if n > 6 else 0.06) * rng.standard_normal((500, n))
    nc = ncdim or n
    e = OB.bounding_ellipsoid(pts[:, :nc])
    logl = m.loglike(m.prior_transform(pts))
    loglstar = float(np.quantile(logl, 0.3))
    ok = np.flatnonzero(logl > loglstar)
    starts = rng.choice(ok, size=300).astype(np.int32)
    ops.bound_set(e.axes)
    ref = ops.rwalk_batch(dm.model_id(), pts[starts], loglstar, 0.4, 12, SEED, chain0=40, ncdim=ncdim)
    live = pts
    if pinned:
        t = torch.empty(pts.shape, dtype=torch.float64).pin_memory()
        t.numpy()[:] = pts
        live = t.numpy()
    o = ops.rwalk_batch(dm.model_id(), live, loglstar, 0.4, 12, SEED, chain0=40, ncdim=ncdim, start_rows=starts)
    for k in ref:
        assert o[k].shape == ref[k].shape and np.array_equal(o[k], ref[k]), k
    again = ops.rwalk_batch(dm.model_id(), pts[starts], loglstar, 0.4, 12, SEED, chain0=40, ncdim=ncdim)   # plain call: not sticky
    assert np.array_equal(again['u'], ref['u'])
    bad = starts.copy()
    bad[5] = len(pts)
    with pytest.raises(Exception):
        ops.rwalk_batch(dm.model_id(), live, loglstar, 0.4, 12, SEED, chain0=40, ncdim=ncdim, start_rows=bad)
    after = ops.rwalk_batch(dm.model_id(), pts[starts], loglstar, 0.4, 12, SEED, chain0=40, ncdim=ncdim)   # and the failed call left nothing behind
    assert np.array_equal(after['u'], ref['u'])
    if ncdim is None and n == 6:
        # a pending setting is for the next rwalk call only: another chain entry point refuses it and clears it
        from dynesty_b200 import _lib
        ctx = _lib.default_context()
        ctx.set_start_rows(_lib.ptr(starts), len(pts))
        with pytest.raises(Exception):
            ops.rslice_batch(dm.model_id(), pts[starts], loglstar, 0.4, 2, SEED)
        again = ops.rwalk_batch(dm.model_id(), pts[starts], loglstar, 0.4, 12, SEED, chain0=40)
        assert np.array_equal(again['u'], ref['u'])

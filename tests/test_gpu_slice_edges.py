"""GPU: the slice samplers (slice_kernel, csrc/b2n_slice_kernel.cuh) against the float64 oracle (oracle/samplers.py) on
the same Philox streams, where a step leaves the well-scaled path that the kernel matrix covers.

  * the expansion warning at exactly 1000 / 1001 stepping-out expansions, and the switch to doubling it causes in
    the first and in the last slice of a chain (internal_samplers.py:689-693, 836-838, 1142);
  * the direction-length cap |d| <= sqrt(n) / 2 (:1103-1108), exactly at its edge and far past it;
  * proposals inside the slice that the doubling acceptance test refuses (:1038-1072), on lines that cross a
    likelihood more than once (eggbox, shells);
  * long doublings: D doublings count 2^D - 1 expansions, D = 28 ... 54; the kernel returns n_expand saturated at
    INT32_MAX (include/b200nest.h), where the reference's Python int grows on;
  * the stepping-out guard B2N_MAX_EXPAND, in a host fill and in a device round;
  * the same edges in the device-resident rounds (the doubling switch, the tune after long doublings), in the host
    loop, across the hand-back from the rounds and a checkpoint / resume, and through a user CUDA model.

Standard of comparison (that of tests/test_gpu_kernel_matrix.py::test_slice_matrix): ncall, n_expand, n_contract and
the B2N_WARN_DOUBLING bit equal; u, v, logl to rtol 1e-9.  Every case also asserts, from the oracle's branch
counters, that it reached the edge it is named after.
"""
import ctypes as C
import math

import numpy as np
import pytest

from dynesty_b200 import ops, _lib, nested, likelihoods as DL
from helpers import device_model, close
from oracle import samplers as OS, philox, likelihoods as OL, nsloop

pytestmark = pytest.mark.gpu

SEED = 4242
RTOL = 1e-9
INT32_MAX = 2**31 - 1
FAIL_BIT = 0x80000000


def _g(n):
    return OL.gauss_corr(n, 0.4, 5.)


def _run(sampler, om, u0, loglstar, axes, scale, slices, doubling=False, chain0=0, dm=None):
    """One fill of Q = len(u0) chains on one ellipsoid; returns the kernel's outputs and the oracle's chain dicts."""
    dm = dm or device_model(om)
    ops.bound_set(axes[None])
    fn, chain = (ops.rslice_batch, OS.rslice_chain) if sampler == 'rslice' else (ops.slice_batch, OS.slice_chain)
    o = fn(dm.model_id(), u0, loglstar, scale, slices, SEED, chain0=chain0, doubling=doubling)
    refs = [chain(u0[q], loglstar, axes, scale, om, philox.ChainStream(SEED, chain0 + q), slices, doubling=doubling)
            for q in range(len(u0))]
    return o, refs


def _check(o, refs, rows=None):
    """Kernel chain q == oracle chain q for q in rows (all by default)."""
    for q in (range(len(refs)) if rows is None else rows):
        r = refs[q]
        assert (o['ncall'][q], o['n_expand'][q], o['n_contract'][q]) == \
            (r['ncall'], min(r['n_expand'], INT32_MAX), r['n_contract']), q
        assert bool(o['flags'][q] & _lib.WARN_DOUBLING) == r['expansion_warning_set'], q
        assert not o['flags'][q] & FAIL_BIT, q
        close(o['u'][q], r['u'], rtol=RTOL)
        close(o['v'][q], r['v'], rtol=RTOL)
        assert o['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL), q


def _centre(om, n, Q, dl=2.0):
    """Q copies of the prior centre and a threshold dl below its log-likelihood."""
    u0 = np.full((Q, n), 0.5)
    return u0, float(om.loglike(om.prior_transform(u0[0]))) - dl


# ---- the expansion warning -----------------------------------------------------------------------------------------
# n = 1 Gaussian (sigma = 0.1 in u) started at its mean, threshold 2 below the peak: the slice is a chord of length
# 0.4 (u), and a step of length chord / 1000.5 takes 1000 or 1001 unit expansions depending on rand0.  Chains found by
# scanning the oracle (the test re-checks them): (chain with 1000, chain with 1001).
THRESHOLD = {'rslice': (6, 0), 'slice': (0, 1)}


@pytest.mark.parametrize('sampler', ['rslice', 'slice'])
def test_expansion_warning_threshold(sampler):
    om = _g(1)
    u0, loglstar = _centre(om, 1, 8)
    scale = 2 * 0.1 * math.sqrt(2 * 2.0) / 1000.5
    o, refs = _run(sampler, om, u0, loglstar, np.eye(1), scale, 1)
    q1000, q1001 = THRESHOLD[sampler]
    assert refs[q1000]['n_expand'] == 1000 and not refs[q1000]['expansion_warning_set']
    assert refs[q1001]['n_expand'] == 1001 and refs[q1001]['warn_slice'] == 0
    _check(o, refs)
    assert not o['flags'][q1000] & _lib.WARN_DOUBLING and o['flags'][q1001] & _lib.WARN_DOUBLING


# ---- the switch to doubling inside a chain --------------------------------------------------------------------------
def test_switch_in_first_and_last_rslice():
    """rslice, n = 2, slices = 3: chain 1 warns in slice 0 and doubles in slices 1-2; chain 24 warns in slice 2."""
    om = _g(2)
    u0, loglstar = _centre(om, 2, 25)
    dm = device_model(om)
    ops.bound_set(np.eye(2)[None])
    o = ops.rslice_batch(dm.model_id(), u0, loglstar, 3.5e-4, 3, SEED)
    refs = {q: OS.rslice_chain(u0[q], loglstar, np.eye(2), 3.5e-4, om, philox.ChainStream(SEED, q), 3)
            for q in (0, 1, 13, 24)}
    assert refs[1]['warn_slice'] == 0 and refs[1]['doublings'][1] > 0 and refs[1]['doublings'][2] > 0
    assert refs[24]['warn_slice'] == 2 and refs[24]['doublings'] == [0, 0, 0]
    _check(o, refs, refs)


def test_switch_inside_a_33d_slice():
    """slice, n = 33: the permutation spans two lane passes; the warning fires at an axis inside the slice and the
    remaining axes of the same slice double."""
    om = _g(33)
    rng = np.random.default_rng(33)
    u0 = 0.5 + 0.08 * rng.standard_normal((12, 33))         # in the typical set, ~15 below the peak
    _, loglstar = _centre(om, 33, 1, 24.0)
    dm = device_model(om)
    ops.bound_set(np.eye(33)[None])
    o = ops.slice_batch(dm.model_id(), u0, loglstar, 5e-4, 1, SEED)
    # chains 4 and 6 (found by scanning the oracle) warn at axis 23 and 30 of their 33; chain 0 at axis 0
    refs = {q: OS.slice_chain(u0[q], loglstar, np.eye(33), 5e-4, om, philox.ChainStream(SEED, q), 1) for q in (0, 4, 6)}
    for q, k in ((0, 0), (4, 23), (6, 30)):
        r = refs[q]
        assert r['warn_step'] == k and r['expansion_warning_set']
        assert sum(r['doublings'][:k + 1]) == 0 and all(d > 0 for d in r['doublings'][k + 1:])
    _check(o, refs, refs)


# ---- the direction-length cap ---------------------------------------------------------------------------------------
def test_direction_cap_edge_slice():
    """slice, axes 0.5 I, n = 4: scale 2.0 gives |d| = sqrt(n) / 2 exactly (no cap); the next double caps."""
    om = _g(4)
    rng = np.random.default_rng(4)
    u0 = 0.5 + 0.02 * rng.standard_normal((6, 4))
    loglstar = float(om.loglike(om.prior_transform(np.full(4, 0.5)))) - 3.0
    for scale, capped in ((2.0, False), (np.nextafter(2.0, 3.0), True)):
        for dbl in (False, True):
            o, refs = _run('slice', om, u0, loglstar, 0.5 * np.eye(4), scale, 2, doubling=dbl)
            assert all(r['n_capped'] == (8 if capped else 0) for r in refs), (scale, dbl)
            _check(o, refs)


@pytest.mark.parametrize('n', [4, 50])
def test_direction_cap_large_scale_rslice(n):
    om = _g(n)
    rng = np.random.default_rng(n)
    u0 = 0.5 + 0.02 * rng.standard_normal((6, n))
    loglstar = float(om.loglike(om.prior_transform(np.full(n, 0.5)))) - n
    for dbl in (False, True):
        o, refs = _run('rslice', om, u0, loglstar, 0.1 * np.eye(n), 100.0, 3, doubling=dbl)
        assert all(r['n_capped'] == 3 for r in refs)
        _check(o, refs)


# ---- doubling: proposals the acceptance test refuses ----------------------------------------------------------------
def _shell_starts(n, Q, rng):
    om = OL.shells(n)
    d = rng.standard_normal((Q, n))
    d /= np.linalg.norm(d, axis=1)[:, None]
    u0 = (om.p['c1'] + 2.0 * d + 6.0) / 12.0              # on the first shell (radius 2, prior U(-6, 6))
    return om, u0, math.log(1. / math.sqrt(2. * math.pi * 0.01)) - 2.0


@pytest.mark.parametrize('model,n,sampler,slices,scale', [('egg', 2, 'rslice', 3, 1.0), ('egg', 2, 'slice', 1, 0.5),
                                                          ('egg', 4, 'rslice', 3, 0.5), ('egg', 4, 'slice', 1, 0.5),
                                                          ('shell', 2, 'slice', 1, 0.5)])
def test_doubling_accept_rejections(model, n, sampler, slices, scale):
    rng = np.random.default_rng(1 if model == 'egg' else n)
    if model == 'egg':
        om = OL.eggbox(n)
        pts = rng.random((4000, n))
        logl = om.loglike(om.prior_transform(pts))
        loglstar = float(np.quantile(logl, 0.5))
        u0 = pts[logl > loglstar][:16]
    else:
        om, u0, loglstar = _shell_starts(n, 16, rng)
    o, refs = _run(sampler, om, u0, loglstar, 0.3 * np.eye(n), scale, slices, doubling=True)
    assert sum(r['n_doubling_rejects'] for r in refs) > 0
    _check(o, refs)


# ---- long doublings -------------------------------------------------------------------------------------------------
# rslice, n = 4 Gaussian, axes 0.1 I, one doubled step from the prior centre: log10(scale) -> the oracle's doublings of
# chains 0..3 (found by scanning the oracle; the test re-checks them).  30 doublings is where a 2^28 cap on the
# increment first changes the count, 31 the last that fits an int32, 36 where an int32 total wraps negative.
LONG = {-7.5: [28, 29, 28, 30], -7.25: [26, 29, 27, 27], -8.25: [33, 30, 30, 30], -8.5: [33, 34, 32, 31],
        -9.5: [36, 34, 34, 36], -12.0: [44, 44, 42, 42], -13.0: [47, 54, 47, 46]}


@pytest.mark.parametrize('e', sorted(LONG))
def test_long_doublings_rslice(e):
    om = _g(4)
    u0, loglstar = _centre(om, 4, 4)
    o, refs = _run('rslice', om, u0, loglstar, 0.1 * np.eye(4), 10.0**e, 1, doubling=True)
    assert [r['doublings'][0] for r in refs] == LONG[e]
    assert all(r['n_expand'] == 2**d - 1 for r, d in zip(refs, LONG[e]))
    _check(o, refs)


def test_long_doublings_cover_the_edges():
    assert {28, 29, 30, 31, 32} <= {d for v in LONG.values() for d in v}
    assert max(d for v in LONG.values() for d in v) >= 36


@pytest.mark.parametrize('scale', [1e-9, 1e-12])
def test_long_doublings_slice(scale):
    """slice (4 doubled steps per chain, each along one axis): expansions summed over steps past INT32_MAX."""
    om = _g(4)
    u0, loglstar = _centre(om, 4, 3)
    o, refs = _run('slice', om, u0, loglstar, 0.1 * np.eye(4), scale, 1, doubling=True)
    assert min(min(r['doublings']) for r in refs) >= 28
    assert all(r['n_expand'] > INT32_MAX for r in refs)
    _check(o, refs)
    assert np.all(o['n_expand'] == INT32_MAX)


# ---- the stepping-out guard -----------------------------------------------------------------------------------------
def test_runaway_stepping_out_fails():
    """One n = 1 chain whose slice is 2e7 steps wide: past B2N_MAX_EXPAND (4e6) the fill returns B2N_ERR_SLICE_FAIL
    with the chain's failure bit set (the reference would step on)."""
    from dynesty_b200.ops import _chain_args, _chain_outputs, _chain_ptrs, _ctx
    om = _g(1)
    u0, loglstar = _centre(om, 1, 1)
    dm = device_model(om)
    ops.bound_set(np.eye(1)[None])
    ctx = _ctx(None)
    a, keep, Q, n = _chain_args(dm.model_id(), u0, None, loglstar, 2e-8, SEED, 0, None, None)
    o = _chain_outputs('slice', Q, n)
    st = ctx.lib.b2n_rslice_batch(ctx.h, C.byref(a), 1, 0, *_chain_ptrs(o, 'slice'))
    assert st == _lib.ERR_SLICE_FAIL
    assert o['flags'][0] & FAIL_BIT
    # the same chain in a device round: the round's error
    with pytest.raises(RuntimeError):
        ops.rslice_batch(dm.model_id(), u0, loglstar, 2e-8, 1, SEED)


# ---- device rounds ---------------------------------------------------------------------------------------------------
def _rounds(om, dm, sampler, n, N, K, steps, scale0, rounds, doubling0=False):
    """`rounds` device rounds against nsloop.BatchNS, compared after every round; returns the per-round statuses and the
    oracle's per-round (doubling, last round's info)."""
    from test_gpu_nsloop import _bound
    rng = np.random.default_rng(7 + n)
    u = 0.5 + 0.05 * rng.standard_normal((N, n))
    v = om.prior_transform(u)
    l = np.array([float(om.loglike(x)) for x in v])
    seed, chain0 = 56432, 1000
    b = _bound([u])
    o = nsloop.BatchNS(om, u, v, l, K, sampler, steps, seed, chain0=chain0, scale=scale0, logvol=-2.5, logz=-40.0,
                       loglstar=float(l.min()) - 0.5, ncall=500, bound=b, dlogz=1e-6)
    o.doubling = doubling0
    ops.ns_create(dm.model_id(), N, n, K, ('rwalk', 'rslice', 'slice').index(sampler), steps, seed, chain0=chain0,
                  dlogz=1e-6, dead_capacity=rounds * K + 5)
    sts, ors = [], []
    try:
        ops.ns_set_state(u, v, l, -2.5, -40.0, float(l.min()) - 0.5, 500, scale0)
        if doubling0:
            ops.ns_set_counters(0, 500, True)
        for _ in range(rounds):
            lu = o.live_u
            b = _bound([lu])
            o.bound = b
            ops.bound_set(b['axes'], b['ctrs'], b['ams'], b['logvols'])
            assert o.step(), (o.done, o.need_bound)
            st = ops.ns_run(1, 0)
            assert (st['done'], st['need_bound'], st['error']) == (0, 0, 0)
            assert st['ncall'] == o.ncall and bool(st['doubling']) == o.doubling
            assert st['scale'] == pytest.approx(o.scale, rel=1e-10)
            assert st['logz'] == pytest.approx(o.logz, rel=1e-10)
            du, dv, dl, dlv, dnc = ops.ns_get_dead(0, st['it'], n)
            ou, ov, ol, olv, onc = o.dead_arrays()
            assert np.array_equal(dnc, onc) and np.allclose(dl, ol, rtol=1e-9, atol=0)
            assert np.allclose(du, ou, rtol=1e-8, atol=1e-12)
            sts.append(st)
            ors.append((o.doubling, dict(o.last)))
    finally:
        ops.ns_destroy()
    return sts, ors


@pytest.mark.parametrize('sampler,n,steps', [('rslice', 2, 3), ('slice', 2, 1)])
def test_rounds_switch_to_doubling(sampler, n, steps):
    """Round 1 starts at a scale whose slices take > 1000 expansions: a chain warns, the run's doubling switch flips on
    both sides after round 1, and the later rounds run doubled chains."""
    om, dm = _g(n), DL.gauss_corr(n, 0.4, 5.0)
    sts, ors = _rounds(om, dm, sampler, n, 48, 8, steps, 2e-4, 3)
    assert [d for d, _ in ors] == [True, True, True]
    assert sts[0]['doubling'] == 1
    assert ors[0][1]['n_expand'] > 8 * 1000       # round 1 stepped out
    assert ors[1][1]['n_expand'] > 0


def test_round_tune_after_long_doublings():
    """Doubled chains at scale 1e-10 take 36+ doublings each: the round's expansions exceed what an int32 holds, and the
    tune must double the scale as the oracle's does (a wrapped count would halve it)."""
    om, dm = _g(4), DL.gauss_corr(4, 0.4, 5.0)
    sts, ors = _rounds(om, dm, 'rslice', 4, 32, 4, 1, 1e-10, 2, doubling0=True)
    assert ors[0][1]['n_expand'] >= 4 * (2**36 - 1)
    assert sts[0]['scale'] == pytest.approx(2e-10, rel=1e-12) and sts[1]['scale'] == pytest.approx(4e-10, rel=1e-12)


def test_round_guard_sets_the_run_error():
    """A round whose chain steps out past B2N_MAX_EXPAND ends the run with B2N_ERR_SLICE_FAIL."""
    from test_gpu_nsloop import _bound
    om, dm = _g(1), DL.gauss_corr(1, 0.4, 5.0)
    rng = np.random.default_rng(3)
    N, K = 16, 2
    u = 0.5 + 0.01 * rng.standard_normal((N, 1))
    v = om.prior_transform(u)
    l = np.array([float(om.loglike(x)) for x in v])
    b = _bound([u])
    ops.bound_set(b['axes'], b['ctrs'], b['ams'], b['logvols'])
    ops.ns_create(dm.model_id(), N, 1, K, 1, 1, 5, dlogz=1e-9)
    try:
        ops.ns_set_state(u, v, l, -1.0, -40.0, float(l.min()) - 30.0, 10, 1e-9)
        with pytest.raises(RuntimeError):
            ops.ns_run(1, 0)
        st = ops.ns_status()
        assert st['error'] == _lib.ERR_SLICE_FAIL and st['done'] == 1
    finally:
        ops.ns_destroy()


# ---- host loop, hand-back, checkpoint / resume -----------------------------------------------------------------------
def _sampler(sample='rslice', **kw):
    s = nested.NestedSampler(DL.gauss_corr(4, 0.4, 5.0), nlive=200, bound='multi', sample=sample, seed=21,
                             queue_size=20, slices=3, **kw)
    s.internal_sampler_next.scale = 1e-5     # the first bounded fill steps out ~1e4 times per slice
    return s


def test_host_loop_warning_sets_slice_doubling():
    s = _sampler()
    with pytest.warns(UserWarning, match='doubling'):
        res = s.run_nested(loop='host', dlogz=0.5)
    assert s.internal_sampler.sampler_kwargs['slice_doubling'] is True
    assert np.all(np.diff(res.logl) >= 0)


def test_device_rounds_hand_back_slice_doubling():
    s = _sampler()
    res = s.run_nested(loop='device', batch=10, dlogz=0.5)
    assert s.internal_sampler.sampler_kwargs.get('slice_doubling') is True
    assert np.all(np.diff(res.logl) >= 0) and s.device_rounds > 3


def test_checkpoint_resume_keeps_slice_doubling(tmp_path):
    from test_gpu_nsloop import _abort_at
    ref = _sampler().run_nested(loop='device', batch=10)
    f = str(tmp_path / 'ckpt.pkl')
    s = _sampler()
    with pytest.raises(KeyboardInterrupt):
        s.run_nested(loop='device', batch=10, checkpoint_file=f, checkpoint_every=0., on_checkpoint=_abort_at(3))
    del s
    r = nested.NestedSampler.restore(f)
    assert r._dev_snap['doubling'] == 1 and r._dev_snap['rounds'] > 0
    res = r.run_nested(resume=True)
    assert res.niter == ref.niter and res.ncall == ref.ncall
    assert np.array_equal(res.logl, ref.logl) and np.array_equal(res.samples_u, ref.samples_u)
    assert r.internal_sampler.sampler_kwargs.get('slice_doubling') is True


# ---- a user CUDA model ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('sampler', ['rslice', 'slice'])
def test_user_model_edges(sampler):
    """The NVRTC image of a user likelihood instantiates slice_kernel in its own B2N_US_SLICE slots: the warning and
    switch, and 30+ doublings, through it."""
    from test_gpu_user_model import _models
    om, dm, um = _models('diag', 4)
    u0, loglstar = _centre(om, 4, 8)
    # stepping out past 1000 expansions in some chains, then doubling
    o, refs = _run(sampler, om, u0, loglstar, 0.05 * np.eye(4), 0.02 if sampler == 'rslice' else 0.019, 2, dm=um)
    assert any(r['warn_step'] == 0 and sum(r['doublings'][1:]) > 0 for r in refs)
    _check(o, refs)
    o, refs = _run(sampler, om, u0[:3], loglstar, 0.05 * np.eye(4), 1e-9, 1, doubling=True, dm=um)
    assert max(max(r['doublings']) for r in refs) >= 30
    _check(o, refs)

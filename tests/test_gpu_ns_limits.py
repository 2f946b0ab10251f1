"""GPU tier: the device-resident rounds (csrc/b2n_ns.cu: ns_sort_kernel, ns_step_kernel = ns_commit_body +
ns_propose_body) against oracle.nsstrands.StrandBatchNS where their one-CTA loops change form (oracle/nslimits.py):
sort and merge widths past the thread count, the K-strided propose / commit loops past 1024 and on 256 / 512
threads, exact logl ties, the contains test past one lane pass and on the boundary, many ellipsoids, the growth of
the dead buffer, the stops, and the host's shared-memory refusals.

Standard of comparison, after every round: the status counters (it, ncall, rounds, done, need_bound, error) are
equal, ln X and logZ agree to 1e-13 / rel 1e-10.  At the end: the dead rows' live slot and birth counter
(b2n_ns_get_strands) and the per-slot counters (b2n_ns_get_live_it) are EQUAL -- they spell out the (logl, row)
order of every round's K lowest, ties included -- as are the dead call counts and the logl of every dead row the
caller supplied.  A logl the device computed matches the oracle's to the last bits only (its own summation
order), rel 1e-11 for prior draws and 1e-9 after random walks; with the quantized likelihood it is equal.  Unit-cube
draws are bit-equal; live sets are compared as sets (tests/test_gpu_nsloop.py explains why).

The width, random-walk and thread cases run ceil(N / K) + 1 rounds.  The unit-cube cases start from a live set in
the likelihood's low tail, so that prior draws clear the threshold in a few tries and land above the starting rows:
every row live at the start dies inside the window (asserted), so every position of every merged order is seen in
the dead slots.  One survivor (K = N - 1) is run at N = 2 and 3 only: each such round shrinks the prior volume by
a factor N, so the oracle's prior draws cost O(N) tries per chain from the second round on."""
import math

import numpy as np
import pytest

from oracle import nsstrands, nslimits as NL, likelihoods as OL
from dynesty_b200 import ops, _lib, likelihoods as DL
from test_gpu_nsloop import _bound, _live, _models

pytestmark = pytest.mark.gpu

SEED, CHAIN0 = 4242, 77
HUGE = 1 << 62
UNIT_CUBE = dict(unit_cube_phase=True, first_min_ncall=HUGE, first_min_eff=100.)


def _device():
    """(SM count, opt-in shared memory per block in bytes) of cuda:0."""
    import torch
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, int(getattr(p, 'shared_memory_per_block_optin', 227 * 1024))


def _tail_live(om, n, N, rng, over=40):
    """N prior draws from the lowest 1 / over of the likelihood, in random row order."""
    u = rng.random((over * N, n))
    l = om.loglike(om.prior_transform(u))
    u = u[rng.permutation(np.argsort(l, kind='stable')[:N])]
    v = om.prior_transform(u)
    return u, v, np.array([float(om.loglike(x)) for x in v])


def _status(st, o):
    assert (st['it'], st['ncall'], st['rounds'], st['done'], st['need_bound'], st['error']) == \
        (o.it, o.ncall, o.round, o.done, o.need_bound, o.error)
    assert st['logvol'] == pytest.approx(o.logvol, rel=0, abs=1e-13)
    assert st['logz'] == pytest.approx(o.logz, rel=1e-10)
    assert st['scale'] == pytest.approx(o.scale, rel=1e-10)


def _records(o, n, rtol, exact_u=False, ctx=None):
    """Dead rows, strands, live-slot counters and live set against the oracle's."""
    it = o.it
    du, dv, dl, dlv, dnc = ops.ns_get_dead(0, it, n, ctx=ctx)
    ou, ov, ol, olv, onc = o.dead_arrays()
    dslot, dit = ops.ns_get_strands(0, it, ctx=ctx)
    oslot, oit = o.strand_arrays()
    assert np.array_equal(dslot, oslot) and np.array_equal(dit, oit)
    assert np.array_equal(ops.ns_get_live_it(o.N, ctx=ctx), o.live_it)
    assert np.array_equal(dnc, onc)
    given = oit == 0                                   # rows the caller supplied: copies, equal
    assert np.array_equal(dl[given], ol[given])
    np.testing.assert_allclose(dl, ol, rtol=rtol, atol=0)
    np.testing.assert_allclose(dlv, olv, rtol=0, atol=1e-13)
    if exact_u:
        assert np.array_equal(du, ou)
        np.testing.assert_allclose(dv, ov, rtol=1e-13, atol=1e-15)
    else:
        np.testing.assert_allclose(du, ou, rtol=1e-8, atol=1e-12)
    lu, lv_, ll = ops.ns_get_live(o.N, n, ctx=ctx)
    pd, po = np.argsort(ll, kind='stable'), np.argsort(o.live_logl, kind='stable')
    np.testing.assert_allclose(ll[pd], o.live_logl[po], rtol=rtol, atol=1e-10)
    np.testing.assert_allclose(lu[pd], o.live_u[po], rtol=1e-8, atol=1e-12)


def _every_start_row_died(o):
    slot, it = o.strand_arrays()
    assert len(np.unique(slot[it == 0])) == o.N


def _unitcube_case(N, K, rounds=None, seed=0, **kw):
    """Unit-cube-phase rounds of the 3-D Gaussian from a tail live set, compared round by round."""
    n = 3
    dm, om = _models('gauss', n)
    rng = np.random.default_rng(seed + N + 7 * K)
    u, v, l = _tail_live(om, n, N, rng)
    rounds = rounds or -(-N // K) + 1
    o = nsstrands.StrandBatchNS(om, u, v, l, K, 'rwalk', 1, SEED, chain0=CHAIN0, ncall=N, dlogz=0.0, **UNIT_CUBE, **kw)
    ops.ns_create(dm.model_id(), N, n, K, 0, 1, SEED, chain0=CHAIN0, dlogz=0.0, dead_capacity=rounds * K, **UNIT_CUBE,
                  **kw)
    try:
        ops.ns_set_state(u, v, l, 0.0, -1e300, -1e300, N, 1.0)
        for _ in range(rounds):
            assert o.step()
            _status(ops.ns_run(1, 0), o)
        _records(o, n, 1e-11, exact_u=True)
    finally:
        ops.ns_destroy()
    return o


QUANTIZED_SRC = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    double s = 0.0;
    for (int i = lane; i < n; i += 32) s += v[i] * v[i];
    return floor(p[0] * (-0.5 * b2n_warp_sum(s))) / p[0];
}
'''
_QUANT = {}
FINE_Q = 65536.0


def _quantized(q=4.0):
    """(device model, fresh oracle model) of oracle.nslimits.QuantizedGauss: 3-D, prior U(-2, 2)^3, levels 1 / q."""
    om = NL.QuantizedGauss(3, q)
    if q not in _QUANT:
        _QUANT[q] = DL.DeviceModel.from_cuda(3, QUANTIZED_SRC, params=[om.q], prior_kind=_lib.PRIOR_UNIFORM,
                                             prior_p0=om.lo, prior_p1=om.width, name='quantized_gauss3_%g' % q)
    return _QUANT[q], om


def _ells(points, kell, rng):
    """Ellipsoid 0 bounds every live point (so every start is inside); the others bound random subsets.  The
    log-volumes are weights of the volume-weighted pick only (rwalk reads nothing else from them): shifted by -1000
    -- the range of a bound in a few hundred dimensions -- and spread over > 700 nats, so that the pick must work
    with differences of log-volumes and some ellipsoids never receive a chain."""
    b = _bound([points] + [points[rng.choice(len(points), 12, replace=False)] for _ in range(kell - 1)])
    if kell > 1:
        head = np.array([0.0, -0.4, -1.1, -2.3])[:kell]
        b['logvols'] = -1000.0 + np.concatenate([head, np.linspace(-30.0, -760.0, kell - len(head))])
    return b


def _rwalk_case(N, K, kell, seed=0):
    """Bounded random-walk rounds on the finely quantized Gaussian.  A chain that never moves returns a clone of its
    start whose logl the device recomputes: quantized, it ties EXACTLY with the original's (a continuous logl may
    differ in the last bit and swap the pair in the (logl, row) order of one side only)."""
    n, walks = 3, 2
    dm, om = _quantized(FINE_Q)
    rng = np.random.default_rng(seed + N + 7 * K + kell)
    u, v, l, _ = _live(om, n, N, rng)
    rounds = -(-N // K) + 1
    lstar = float(l.min()) - 0.5
    o = nsstrands.StrandBatchNS(om, u, v, l, K, 'rwalk', walks, SEED, chain0=CHAIN0, scale=0.7, logvol=-2.5,
                                logz=-40.0, loglstar=lstar, ncall=500, dlogz=0.0)
    ops.ns_create(dm.model_id(), N, n, K, 0, walks, SEED, chain0=CHAIN0, dlogz=0.0, dead_capacity=rounds * K)
    counts = []
    try:
        ops.ns_set_state(u, v, l, -2.5, -40.0, lstar, 500, 0.7)
        for _ in range(rounds):
            o.bound = _ells(o.live_u, kell, rng)
            ops.bound_set(o.bound['axes'], o.bound['ctrs'], o.bound['ams'], o.bound['logvols'])
            assert o.step()
            _status(ops.ns_run(1, 0), o)
            counts.append(np.bincount(o.last['ell'], minlength=kell))
        _records(o, n, 0.0)
    finally:
        ops.ns_destroy()
    assert om.min_frac >= 1e-9, om.min_frac
    return o, np.array(counts)


# ---- 1. sort and merge widths ----------------------------------------------------------------------------------
@pytest.mark.parametrize('N,K', NL.WIDTH_CASES)
def test_sort_and_merge_widths(N, K):
    _, optin = _device()
    assert NL.sort_accepts(N, optin) and NL.run_accepts(N, K, 3, 1, optin)
    o = _unitcube_case(N, K)
    _every_start_row_died(o)


@pytest.mark.parametrize('N,K,kell', NL.RWALK_CASES)
def test_rwalk_rounds_past_the_threads(N, K, kell):
    """Start rows, contains, start points and worklist past 1024 chains; the volume-weighted pick and the grouped
    worklist over many ellipsoids (groups without a chain, groups split over several CTAs, more ellipsoids than
    chains)."""
    sms, _ = _device()
    o, counts = _rwalk_case(N, K, kell)
    assert K > NL.THREADS or kell > K
    if kell > 1:
        assert (counts == 0).any(axis=1).all()                             # some ellipsoids get no chain
        assert (counts[:, 1:].sum(axis=1) > 0).all()                       # ... while more than one does
        if K > NL.THREADS:
            assert counts.max() > NL.rwalk_warp_cpc(K, sms)                 # a group over several CTAs


# ---- 2. thread count -------------------------------------------------------------------------------------------
@pytest.mark.parametrize('threads,sampler,N,K', NL.THREAD_CASES)
def test_step_kernel_threads(monkeypatch, threads, sampler, N, K):
    """B2N_NS_THREADS = 256 / 512: the same rounds on fewer threads, against the oracle."""
    assert NL.limits(N, K, threads)['loop_passes'] > 1
    monkeypatch.setenv('B2N_NS_THREADS', str(threads))
    if sampler == 'unitcube':
        _unitcube_case(N, K, seed=threads)
    else:
        _rwalk_case(N, K, 1, seed=threads)


# ---- 3. exact ties ---------------------------------------------------------------------------------------------
# (N, K, stop): unit-cube rounds until the run stops -- with the plateau error (the K-th lowest is the top level:
# nothing above the threshold) or with every live point on the top level (key[0] == lmax)
TIE_RUNS = [(256, 32, 'plateau'), (64, 8, 'flat')]


@pytest.mark.parametrize('N,K,stop', TIE_RUNS)
def test_exact_ties_unit_cube_until_stop(N, K, stop):
    dm, om = _quantized()
    n = 3
    rng = np.random.default_rng(N + K)
    u = rng.random((N, n))
    v = om.prior_transform(u)
    l = np.array([float(om.loglike(x)) for x in v])
    o = nsstrands.StrandBatchNS(om, u, v, l, K, 'rwalk', 1, SEED, chain0=CHAIN0, ncall=N, dlogz=0.0, **UNIT_CUBE)
    ops.ns_create(dm.model_id(), N, n, K, 0, 1, SEED, chain0=CHAIN0, dlogz=0.0, dead_capacity=400 * K, **UNIT_CUBE)
    tied = 0
    try:
        ops.ns_set_state(u, v, l, 0.0, -1e300, -1e300, N, 1.0)
        for _ in range(400):
            sl = np.sort(o.live_logl)
            tied += int(np.count_nonzero(sl[K:] == sl[K - 1]) > 0)
            ran = o.step()
            try:
                st = ops.ns_run(1, 0)
            except RuntimeError as e:
                assert 'status 13' in str(e)
                st = ops.ns_status()
            _status(st, o)
            if not ran:
                break
        assert o.done == 1 and not ran
        assert o.error == (13 if stop == 'plateau' else 0)
        assert tied >= o.round // 2 and o.round >= 3                     # survivors tie with the threshold
        _records(o, n, 0.0, exact_u=True)
    finally:
        ops.ns_destroy()
    assert om.min_frac >= 1e-9, om.min_frac


def test_exact_ties_rwalk_start_rows():
    """Bounded random-walk rounds on the quantized likelihood: start rows strictly above a threshold that
    survivors share, new points tying with survivors, merged by (logl, row)."""
    dm, om = _quantized()
    N, K, n, walks, rounds = 256, 32, 3, 3, 9
    rng = np.random.default_rng(11)
    u = rng.random((N, n))
    v = om.prior_transform(u)
    l = np.array([float(om.loglike(x)) for x in v])
    lstar = float(l.min()) - 1.0
    o = nsstrands.StrandBatchNS(om, u, v, l, K, 'rwalk', walks, SEED, chain0=CHAIN0, scale=0.5, logvol=-1.0,
                                logz=-30.0, loglstar=lstar, ncall=N, dlogz=0.0)
    ops.ns_create(dm.model_id(), N, n, K, 0, walks, SEED, chain0=CHAIN0, dlogz=0.0, dead_capacity=rounds * K)
    tied = 0
    try:
        ops.ns_set_state(u, v, l, -1.0, -30.0, lstar, N, 0.5)
        for _ in range(rounds):
            o.bound = _bound([o.live_u])
            ops.bound_set(o.bound['axes'], o.bound['ctrs'], o.bound['ams'], o.bound['logvols'])
            sl = np.sort(o.live_logl)
            tied += int(sl[K] == sl[K - 1])
            assert o.step()
            _status(ops.ns_run(1, 0), o)
        assert tied >= rounds - 2
        _records(o, n, 0.0)
    finally:
        ops.ns_destroy()
    assert om.min_frac >= 1e-9, om.min_frac


# ---- 4. contains test ------------------------------------------------------------------------------------------
def _boxed(nc, soft, off, strict):
    """N = 16 live points around ctr 0.5 and the ellipsoid am = 16 I (radius 0.25): row 0 sits at 0.5 + off in
    coordinate `soft` only; the other rows are 0.03-offsets in the remaining coordinates, well inside.  The diagonal
    Gaussian barely depends on `soft`, so row 0 has the highest logl; with K = N - 1 it is the one survivor and
    every chain starts from it."""
    N = 16
    ivar = np.ones(nc)
    ivar[soft] = 1e-4
    lnorm = 0.5 * float(np.sum(np.log(ivar / (2 * math.pi))))
    om = OL.Model(nc, OL.PRIOR_UNIFORM, OL.LIKE_GAUSS_DIAG, lo=np.full(nc, -5.0), width=np.full(nc, 10.0),
                  mean=np.zeros(nc), ivar=ivar, lnorm=lnorm)
    dm = DL.DeviceModel(nc, _lib.PRIOR_UNIFORM, _lib.LIKE_GAUSS_DIAG, prior_p0=-5.0, prior_p1=10.0, like_vec0=0.0,
                        like_vec1=ivar, s0=lnorm, name='boxed%d_%d' % (nc, soft))
    rng = np.random.default_rng(nc + soft)
    u = 0.5 + 0.03 * rng.choice([-1.0, 1.0], (N, nc))
    u[:, soft] = 0.5
    u[0] = 0.5
    u[0, soft] = 0.5 + off
    v = om.prior_transform(u)
    l = np.array([float(om.loglike(x)) for x in v])
    assert np.argmax(l) == 0 and np.count_nonzero(l == l.max()) == 1
    b = dict(ctrs=np.full((1, nc), 0.5), ams=16.0 * np.eye(nc)[None], axes=0.25 * np.eye(nc)[None],
             logvols=np.array([nc * math.log(0.25) + 0.5 * nc * math.log(math.pi) - math.lgamma(nc / 2 + 1)]),
             strict=strict)
    return dm, om, u, v, l, b


def _contains_round(nc, soft, off, strict):
    dm, om, u, v, l, b = _boxed(nc, soft, off, strict)
    N, K, walks = len(l), len(l) - 1, 2
    lstar = float(l.min()) - 1.0
    o = nsstrands.StrandBatchNS(om, u, v, l, K, 'rwalk', walks, SEED, chain0=CHAIN0, scale=0.5, logvol=-1.0,
                                logz=-30.0, loglstar=lstar, ncall=N, dlogz=0.0, bound=b)
    ops.bound_set(b['axes'], b['ctrs'], b['ams'], b['logvols'])
    ops.ns_create(dm.model_id(), N, nc, K, 0, walks, SEED, chain0=CHAIN0, dlogz=0.0, strict_contains=strict,
                  dead_capacity=K)
    try:
        ops.ns_set_state(u, v, l, -1.0, -30.0, lstar, N, 0.5)
        ran = o.step()
        _status(ops.ns_run(1, 0), o)
        if ran:
            _records(o, nc, 1e-9)
    finally:
        ops.ns_destroy()
    return o


@pytest.mark.parametrize('nc,soft', [(33, 32), (65, 32), (65, 64)])
def test_contains_past_one_lane_pass(nc, soft):
    """A start outside the bound only through coordinate 32 (lane 0's second pass) or the odd tail nc - 1 of the
    column-pair loop: need_bound = 2 on both sides."""
    o = _contains_round(nc, soft, 0.2525, True)          # d^2 = 16 x 0.2525^2 = 1.0201
    assert o.need_bound == 2 and o.round == 0


@pytest.mark.parametrize('strict', [True, False])
def test_contains_exactly_on_the_boundary(strict):
    """A start at d^2 = 1.0 exactly (0.75 in one coordinate, am = 16 I): outside for the strict test (multi-
    ellipsoid bounds), inside for the non-strict one (single ellipsoid), where the round runs."""
    o = _contains_round(33, 32, 0.25, strict)
    assert (o.need_bound, o.round) == ((2, 0) if strict else (0, 1))


# ---- 6. dead-buffer growth --------------------------------------------------------------------------------------
@pytest.mark.parametrize('slack', [0, 1])
def test_dead_buffer_growth_keeps_strands(slack):
    """Rounds until the dead buffer is full (it + K == capacity runs, it + K == capacity + 1 raises need_bound = 3),
    then b2n_ns_reserve_dead and more rounds: every column, strands included, survives the reallocation.  A fresh
    context, so that the reservation does reallocate."""
    ctx = _lib.Context(0)
    N, K, n = 300, 100, 3
    dm, om = _models('gauss', n)
    u, v, l = _tail_live(om, n, N, np.random.default_rng(slack))
    cap = 2 * K - slack
    o = nsstrands.StrandBatchNS(om, u, v, l, K, 'rwalk', 1, SEED, chain0=CHAIN0, ncall=N, dlogz=0.0, **UNIT_CUBE)
    ops.ns_create(dm.model_id(ctx), N, n, K, 0, 1, SEED, chain0=CHAIN0, dlogz=0.0, dead_capacity=cap, ctx=ctx,
                  **UNIT_CUBE)
    try:
        ops.ns_set_state(u, v, l, 0.0, -1e300, -1e300, N, 1.0, ctx=ctx)
        while o.it + K <= cap:
            assert o.step()
            _status(ops.ns_run(1, 0, ctx=ctx), o)
        assert (o.it == cap) if slack == 0 else (o.it + K == cap + 1)
        st = ops.ns_run(1, 0, ctx=ctx)
        assert (st['need_bound'], st['rounds'], st['it']) == (3, o.round, o.it)
        ops.ns_reserve_dead(8 * K, ctx=ctx)
        for _ in range(3):
            assert o.step()
            _status(ops.ns_run(1, 0, ctx=ctx), o)
        _records(o, n, 1e-11, exact_u=True, ctx=ctx)
        _every_start_row_died(o)
    finally:
        ops.ns_destroy(ctx=ctx)


# ---- 7. stops ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('stop', ['maxiter', 'maxcall', 'logl_max'])
def test_stops_fire_in_the_same_round(stop):
    N, K, n = 200, 30, 3
    dm, om = _models('gauss', n)
    u, v, l = _tail_live(om, n, N, np.random.default_rng(5))
    kw = dict(maxiter=100) if stop == 'maxiter' else (dict(maxcall=N + 110) if stop == 'maxcall' else
                                                       dict(logl_max=float(np.sort(l)[3 * K + 4])))
    o = nsstrands.StrandBatchNS(om, u, v, l, K, 'rwalk', 1, SEED, chain0=CHAIN0, ncall=N, dlogz=0.0, **UNIT_CUBE, **kw)
    ops.ns_create(dm.model_id(), N, n, K, 0, 1, SEED, chain0=CHAIN0, dlogz=0.0, dead_capacity=20 * K, **UNIT_CUBE,
                  **kw)
    try:
        ops.ns_set_state(u, v, l, 0.0, -1e300, -1e300, N, 1.0)
        for _ in range(20):
            ran = o.step()
            _status(ops.ns_run(1, 0), o)
            if not ran:
                break
        assert not ran and o.done == 1 and o.error == 0 and o.round >= 3
        _records(o, n, 1e-11, exact_u=True)
        st = ops.ns_run(3, 0)                                              # stays stopped
        assert (st['rounds'], st['done']) == (o.round, 1)
    finally:
        ops.ns_destroy()
    if stop == 'maxiter':
        assert o.it - K < 100 <= o.it
    elif stop == 'maxcall':
        assert o.ncall >= N + 110
    else:
        assert o.live_logl.min() > kw['logl_max']


# ---- 8. shared-memory refusals -----------------------------------------------------------------------------------
def test_sort_refusal_at_the_limit():
    """The largest nlive the one-CTA sort takes runs; one more is refused at b2n_ns_set_state."""
    _, optin = _device()
    Nmax = NL.sort_limit(optin)
    assert NL.sort_accepts(Nmax, optin) and not NL.sort_accepts(Nmax + 1, optin)
    dm, om = _models('gauss', 3)
    u, v, l = _tail_live(om, 3, Nmax + 1, np.random.default_rng(1), over=2)
    ops.ns_create(dm.model_id(), Nmax + 1, 3, 1, 0, 1, SEED, dlogz=0.0, **UNIT_CUBE)
    try:
        with pytest.raises(NotImplementedError, match='nlive too large'):
            ops.ns_set_state(u, v, l, 0.0, -1e300, -1e300, Nmax + 1, 1.0)
    finally:
        ops.ns_destroy()


def _refusal_ks():
    _, optin = _device()
    N = NL.sort_limit(optin)
    bands = NL.refused_bands(N, 3, 1, optin)
    return N, bands, sorted({k for a, b in bands for k in (a - 1, a, b, b + 1) if 1 <= k < N})


def test_batch_refusals_at_the_sort_limit():
    """At the largest sorted nlive the rounds' shared memory is not monotone in K (Kpad doubles past 2^k while
    nlive - K shrinks): the K on both sides of every edge of every refused band.  Inside a band b2n_ns_run refuses;
    outside, one round matches the oracle."""
    _, optin = _device()
    N, bands, ks = _refusal_ks()
    assert bands and bands[-1][1] < N - 1                                # accepted again above the last band
    dm, om = _models('gauss', 3)
    for K in ks:
        if NL.run_accepts(N, K, 3, 1, optin):
            _unitcube_case(N, K, rounds=1)
            continue
        u, v, l = _tail_live(om, 3, N, np.random.default_rng(K), over=2)
        ops.ns_create(dm.model_id(), N, 3, K, 0, 1, SEED, dlogz=0.0, **UNIT_CUBE)
        try:
            ops.ns_set_state(u, v, l, 0.0, -1e300, -1e300, N, 1.0)
            with pytest.raises(NotImplementedError, match='nlive / batch too large'):
                ops.ns_run(1, 0)
        finally:
            ops.ns_destroy()

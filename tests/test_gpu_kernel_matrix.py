"""GPU: every instantiation of the chain kernels, and the switches of the device-resident rounds, against the float64
oracle (oracle/samplers.py, oracle/nsloop.py) on the same Philox streams.

The chain entry points pick one of many kernels by shape, likelihood, prior, dimension flags, queue length and the
B2N_RWALK_IMPL switch (csrc/b2n_rwalk.cu: rwalk_plan, csrc/b2n_slice.cu: slice_batch_impl, csrc/b2n_unif.cu).  Most
of them share fragment and draw code, so comparing one lock-step variant with another (tests/test_gpu_rwalk.py) does
not notice a change that moves all of them.  Here every case names the instantiation it is meant to reach, the
shared-memory plan that decides where the matrices live is recomputed from the device's SM count and opt-in limit,
and the kernel that really ran is read from a CUDA-activity trace (torch.profiler).

Standard of comparison, for every compared chain q (stream ChainStream(seed, chain0 + q)):
  accept / reject / call / expand / contract counts equal exactly;
  u, v, logl equal to rtol 1e-9 (device libm and FMA contraction differ from numpy in the last bits);
  and, for every chain of the queue, (v, logl) equal to the model evaluated on the returned u.
Queues are several CTAs long with a partial last one, over K = 3 ellipsoids with a random assignment; where the
oracle cannot afford every chain, the first and last chain of each ellipsoid group, the last chain of the queue and a
random sample are compared.
"""
import math
import re

import numpy as np
import pytest

from dynesty_b200 import ops
from helpers import device_model, close
from oracle import samplers as OS, philox, bounding as OB, likelihoods as OL, nsloop

pytestmark = pytest.mark.gpu

PREC, DIAG, EGG, SHELL = OL.LIKE_GAUSS_PREC, OL.LIKE_GAUSS_DIAG, OL.LIKE_EGGBOX, OL.LIKE_SHELLS
RWALK_ENV = ('B2N_RWALK_IMPL',)
SEED = 4242
RTOL = 1e-9


# ---- device facts and the launch plans (mirrors of the host code that chooses a kernel) --------------------------
def _device():
    """(SM count, opt-in shared memory per block in bytes) of cuda:0."""
    import torch
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, int(getattr(p, 'shared_memory_per_block_optin', 227 * 1024))


def _chain_warps(Q, sms, max_warps):
    """b2n_chain_grid (b2n_rwalk.cu): one CTA per SM up to 16 x SMs chains, two beyond; warps = chains per
    CTA capped at 16 and at what fits."""
    ctas = sms if Q <= 16 * sms else 2 * sms
    cpc = max(1, -(-Q // ctas))
    return max(1, min(max_warps, 16, cpc))


def _rwalk_warp_plan(n, nc, like, Q, sms, limit):
    """(axes in shared memory, precision matrix in shared memory) of rwalk_kernel (b2n_rwalk.cu: rwalk_plan)."""
    npad = (n + 1) & ~1
    per_warp = 6 * npad * 8
    flags_b = ((((n + 3) >> 2) << 1) + 4 * npad) * 8
    warps = _chain_warps(Q, sms, min(16, (limit - flags_b) // per_warp))
    fixed = per_warp * warps + flags_b
    ax_b = nc * ((nc + 15) & ~15) * 8
    pr_b = n * ((n + 15) & ~15) * 8 if like == PREC else 0
    ax_s = fixed + ax_b <= limit
    return ax_s, pr_b > 0 and fixed + (ax_b if ax_s else 0) + pr_b <= limit


def _slice_plan(n, like, Q, sms, limit):
    """(axes in shared memory, precision matrix in shared memory) of slice_kernel (b2n_slice.cu: slice_batch_impl)."""
    npad = (n + 1) & ~1
    per_warp, model_b = 6 * npad * 8, 4 * npad * 8
    warps = _chain_warps(Q, sms, min(16, (limit - model_b) // per_warp))
    fixed = per_warp * warps + model_b
    ax_b = n * ((n + 15) & ~15) * 8
    pr_b = ax_b if like == PREC else 0
    ax_s = fixed + ax_b <= limit
    return ax_s, pr_b > 0 and fixed + (ax_b if ax_s else 0) + pr_b <= limit


def _trace(fn):
    import torch
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()            # nothing of an earlier call is still in flight when the trace starts
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, sorted({re.sub(r'\s+', '', e.key) for e in prof.key_averages()})


def _run_traced(fn, expect):
    """fn() under a CUDA-activity trace; asserts that a kernel whose name (blanks removed) contains `expect` ran.
    A trace now and then lacks the record of a kernel that did run: seen on a module's first launch, and as a
    trace that holds the runtime calls (cudaLaunchKernel) but no device-side record at all.  So a call whose trace
    misses the kernel is run once more untraced, which leaves nothing of a first launch to the next trace, and then
    traced again, up to four times; every repeat must give the same outputs bit for bit."""
    out, names = _trace(fn)
    for _ in range(4):
        if any(expect in k for k in names):
            break
        fn()
        again, names = _trace(fn)
        for k in out:
            assert np.array_equal(again[k], out[k]), k
    assert any(expect in k for k in names), (expect, names)
    return out


# ---- models and queues --------------------------------------------------------------------------------------------
def _prec_ppf(n):
    """The C2 precision-matrix Gaussian behind a normal-ppf prior (not an affine prior: the generic chain phase)."""
    g = OL.gauss_corr(n, 0.4, 5.)
    rng = np.random.default_rng(n)
    return OL.Model(n, OL.PRIOR_NORMAL_PPF, PREC, mu=0.2 * rng.standard_normal(n), sigma=1.0 + rng.random(n),
                    mean=g.p['mean'], prec=g.p['prec'], lnorm=g.p['lnorm'])


def _model(kind, n):
    return {'prec': lambda: OL.gauss_corr(n, 0.4, 5.), 'precppf': lambda: _prec_ppf(n),
            'diag': lambda: OL.iid_normal_ppf(n), 'egg': lambda: OL.eggbox(n), 'shell': lambda: OL.shells(n)}[kind]()


def _cloud(kind, n, npts, rng):
    if kind == 'egg':       # the central peak of the eggbox: prod cos(t/2) stays O(1), far from round-off
        return 0.5 + 0.005 * rng.standard_normal((npts, n))
    u = 0.5 + 0.03 * rng.standard_normal((npts, n))
    if kind == 'shell':     # on the first shell (centre -3.5, radius 2, prior U(-6, 6))
        u[:, 0] += (-1.5 / 12.0)
    return u


def _queue(kind, m, nc, Q, rng, K=3):
    """Start points above a threshold, K ellipsoids fitted to the first nc coordinates, a random ellipsoid per chain."""
    n = m.ndim
    pts = _cloud(kind, n, max(3000, 8 * K * n), rng)
    pts[:, nc:] = rng.random((len(pts), n - nc))     # what a proposal draws for the coordinates outside the bound
    logl = m.loglike(m.prior_transform(pts))
    loglstar = float(np.quantile(logl, 0.3))
    good = pts[logl > loglstar]
    axes = np.array([OB.bounding_ellipsoid(good[i::K, :nc]).axes for i in range(K)])
    u0 = good[rng.integers(len(good), size=Q)]
    ell = rng.integers(K, size=Q).astype(np.int32)
    return u0, loglstar, axes, ell


def _pick(ell, rng, extra):
    """First and last chain of each ellipsoid group, the last chain of the queue, `extra` more at random."""
    Q = len(ell)
    idx = {0, Q - 1}
    for k in np.unique(ell):
        w = np.flatnonzero(ell == k)
        idx.update((int(w[0]), int(w[-1])))
    idx.update(int(i) for i in rng.choice(Q, size=min(extra, Q), replace=False))
    return sorted(idx)


def _check_consistent(m, o):
    """(v, logl) of every chain == the model at the returned u."""
    v = m.prior_transform(o['u'])
    close(o['v'], v, rtol=1e-12)
    np.testing.assert_allclose(o['logl'], m.loglike(v), rtol=1e-10, atol=1e-12)


def _wrap(n):
    """periodic and reflective coordinates (B2N_DIM_PERIODIC = 1, B2N_DIM_REFLECTIVE = 2)."""
    return [0, n // 2], [1, n - 1]


# ---- 1. rwalk: one case per instantiation ---------------------------------------------------------------------------
# rwalk_plan (csrc/b2n_rwalk.cu) chooses:
#   rwalk_mmaws_kernel<KT, PL>   GAUSS_PREC, ncdim == n, n <= 62, full slabs (n in 25..32, 49..52, 57..62),
#                                B2N_RWALK_IMPL unset; PL = affine prior and no dimension flags
#   rwalk_mma_kernel<L, KT>      ncdim == n, 16 <= n <= 64, every other likelihood / shape; with B2N_RWALK_IMPL=mma
#                                every ncdim == n, 4 <= n <= 64 (the shapes of rwalk_mmaws_kernel too)
#   rwalk_mmas_kernel<L>         ncdim == n > 64 and its plan fits in shared memory
#   rwalk_kernel<L, AXS, PRS>    everything else, and B2N_RWALK_IMPL=warp; AXS / PRS from the plan.  <L, false, true>
#                                cannot occur: the precision matrix is at least as large as the axes.
# KT = 8 for n <= 32, 13 for n <= 52, 16 above.
MMA8 = dict(B2N_RWALK_IMPL='mma')
WARP = dict(B2N_RWALK_IMPL='warp')
LIKE = dict(prec=PREC, precppf=PREC, diag=DIAG, egg=EGG, shell=SHELL)


def _kt(n):
    return 8 if n <= 32 else (13 if n <= 52 else 16)


def _b(x):
    return 'true' if x else 'false'


RW = []     # (id, kind, n, ncdim, env, Q = qmul x SMs + 3, expected kernel, dimension flags)
# (prec at 25, 32, 49, 52, 57, 62 and the ppf / flags cases further down: B2N_RWALK_IMPL=mma at the shapes where the
# default is the warp-specialised kernel)
for _kind, _ns in (('prec', (16, 24, 25, 32, 33, 45, 49, 52, 53, 56, 57, 62, 63, 64)), ('diag', (20, 40, 60)),
                   ('egg', (24, 36, 56)), ('shell', (20, 44, 64)), ('precppf', (30, 50, 60))):
    for _n in _ns:
        RW.append(('mma8-%s%d' % (_kind, _n), _kind, _n, None, MMA8, 24,
                   'rwalk_mma_kernel<%d,%d>' % (LIKE[_kind], _kt(_n)), False))
# default switches where the warp-specialised kernel does not apply: slabs not full (24, 45), n > 62 (63, 64), not
# the precision-matrix Gaussian (diag40)
for _kind, _n in (('prec', 24), ('prec', 45), ('prec', 63), ('prec', 64), ('diag', 40)):
    RW.append(('mma8-%s%d-default' % (_kind, _n), _kind, _n, None, {}, 24,
               'rwalk_mma_kernel<%d,%d>' % (LIKE[_kind], _kt(_n)), False))
for _n in (25, 32, 49, 52, 57, 62):
    RW.append(('mmaws-plain-prec%d' % _n, 'prec', _n, None, {}, 24, 'rwalk_mmaws_kernel<%d,true>' % _kt(_n), False))
for _n in (30, 50, 60):
    RW.append(('mmaws-generic-ppf%d' % _n, 'precppf', _n, None, {}, 24, 'rwalk_mmaws_kernel<%d,false>' % _kt(_n),
               False))
for _n in (28, 52, 62):
    RW.append(('mmaws-generic-flags%d' % _n, 'prec', _n, None, {}, 24, 'rwalk_mmaws_kernel<%d,false>' % _kt(_n),
               True))
# dimension flags on rwalk_mma_kernel (its chain phase wraps / reflects)
for _n in (28, 40, 52, 62):
    RW.append(('mma8-flags-prec%d' % _n, 'prec', _n, None, MMA8, 24, 'rwalk_mma_kernel<0,%d>' % _kt(_n), True))
for _kind, _n in (('prec', 65), ('prec', 100), ('prec', 128), ('egg', 80), ('shell', 80), ('diag', 96)):
    RW.append(('mmas-%s%d' % (_kind, _n), _kind, _n, None, {}, 24, 'rwalk_mmas_kernel<%d>' % LIKE[_kind], False))
# warp per chain.  With w warps per CTA (Q ~ (w - 1) x SMs) the plan is, on a 227 KB opt-in limit:
#   prec100: axes + precision matrix 2 x 89.6 KB + 4.8 KB per warp -> both shared up to w = 10, matrix global from 11
#   prec200, ncdim 150: axes 192 KB + 9.6 KB per warp -> shared up to w = 3; the 333 KB matrix never fits
#   diag130: axes 150 KB + 6.2 KB per warp -> shared up to w = 12, global from 13
# The test recomputes the plan from the device's own figures and checks it before the launch.
for cid, kind, n, nc, env, qmul, flags in (
        ('warp-prec6-both-smem', 'prec', 6, None, {}, 8, False),
        ('warp-prec6-flags', 'prec', 6, None, {}, 8, True),
        ('warp-prec6-ncdim4', 'prec', 6, 4, {}, 8, False),
        ('warp-prec100-both-smem', 'prec', 100, None, WARP, 8, False),
        ('warp-prec100-prec-global', 'prec', 100, None, WARP, 11, False),
        ('warp-prec200-ncdim150-axes-smem', 'prec', 200, 150, {}, 2, False),
        ('warp-prec200-ncdim150-both-global', 'prec', 200, 150, {}, 4, False),
        ('warp-diag40-ncdim30', 'diag', 40, 30, {}, 8, False),
        ('warp-diag130-axes-smem', 'diag', 130, None, WARP, 8, False),
        ('warp-diag130-axes-global', 'diag', 130, None, WARP, 13, False),
        ('warp-diag130-ncdim100-axes-smem', 'diag', 130, 100, {}, 16, False),
        ('warp-egg12', 'egg', 12, None, {}, 8, False),
        ('warp-shell10', 'shell', 10, None, {}, 8, False)):
    RW.append((cid, kind, n, nc, env, qmul, ('warp', LIKE[kind]), flags))


@pytest.mark.parametrize('cid,kind,n,nc,env,qmul,expect,wrap', RW, ids=[c[0] for c in RW])
def test_rwalk_instantiations(monkeypatch, cid, kind, n, nc, env, qmul, expect, wrap):
    """One queue per case: the trace must name the instantiation `expect` (template signature included), and the
    chains must match the oracle."""
    for k in RWALK_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    sms, limit = _device()
    Q = qmul * sms + 3
    m = _model(kind, n)
    dm = device_model(m)
    nc = nc or n
    if isinstance(expect, tuple):          # warp per chain: where the matrices live follows from the plan
        ax_s, pr_s = _rwalk_warp_plan(n, nc, expect[1], Q, sms, limit)
        want = {'both-smem': (True, expect[1] == PREC), 'prec-global': (True, False), 'axes-smem': (True, False),
                'both-global': (False, False), 'axes-global': (False, False)}
        for tag, plan in want.items():
            if cid.endswith(tag):
                assert (ax_s, pr_s) == plan, (cid, Q, ax_s, pr_s)
        expect = 'rwalk_kernel<%d,%s,%s>' % (expect[1], _b(ax_s), _b(pr_s))
    rng = np.random.default_rng(1000 + n + 7 * qmul + nc)
    u0, loglstar, axes, ell = _queue(kind, m, nc, Q, rng)
    per = ref = nb = flags = None
    if wrap:
        per, ref = _wrap(n)
        flags = ops.dimflags_from(n, per, ref)
        nb = flags == 0
    scale, walks, chain0 = 0.4, 20, 77 + n
    ops.bound_set(axes)
    o = _run_traced(lambda: ops.rwalk_batch(dm.model_id(), u0, loglstar, scale, walks, SEED, chain0=chain0,
                                            ncdim=nc, ell=ell, dimflags=flags), expect)
    assert np.all(o['ncall'] == walks) and np.all(o['n_accept'] + o['n_reject'] == walks)
    assert np.all(o['logl'] > loglstar)
    assert (o['n_accept'] > 0).mean() > 0.1             # the chains move: end points test the proposal arithmetic
    _check_consistent(m, o)
    for q in _pick(ell, rng, 24):
        r = OS.rwalk_chain(u0[q], loglstar, axes[ell[q]], scale, m, philox.ChainStream(SEED, chain0 + q), walks,
                           periodic=per, reflective=ref, nonbounded=nb)
        assert (o['n_accept'][q], o['n_reject'][q], o['ncall'][q]) == (r['n_accept'], r['n_reject'], r['ncall']), q
        close(o['u'][q], r['u'], rtol=RTOL)
        close(o['v'][q], r['v'], rtol=RTOL)
        assert o['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL)


# ---- 2. slice / rslice ----------------------------------------------------------------------------------------------
# slice_kernel<L, RANDOM_DIR, AXS, PRS>, AXS / PRS from the plan of slice_batch_impl (b2n_slice.cu).  On a 227 KB
# opt-in limit:  n = 50: both matrices (2 x 25.6 KB) shared at any warp count;  n = 100: 2 x 89.6 KB + 4.8 KB per
# warp -> the precision matrix leaves shared memory from 11 warps per CTA (Q > 10 x SMs);  n = 200: the 333 KB axes
# never fit, so both are global at any Q.  <L, false, true> cannot occur (the two matrices are the same size).
SL = []     # (id, kind, n, Q = qmul x SMs + 3, slices (rslice, slice), expected (AXS, PRS))
for cid, kind, n, qmul, slices, plan in (('egg25', 'egg', 25, 2, (6, 1), (True, False)),
                                         ('prec50-both-smem', 'prec', 50, 2, (4, 1), (True, True)),
                                         ('prec100-prec-global', 'prec', 100, 11, (3, 1), (True, False)),
                                         ('prec200-both-global', 'prec', 200, 1, (2, 1), (False, False)),
                                         ('diag200-axes-global', 'diag', 200, 1, (2, 1), (False, False))):
    for sampler in ('rslice', 'slice'):
        for dbl in (False, True):
            SL.append(('%s-%s-%s' % (sampler, cid, 'dbl' if dbl else 'std'), sampler, kind, n, qmul,
                       slices[sampler == 'slice'], dbl, plan))


@pytest.mark.parametrize('cid,sampler,kind,n,qmul,slices,doubling,plan', SL, ids=[c[0] for c in SL])
def test_slice_matrix(cid, sampler, kind, n, qmul, slices, doubling, plan):
    sms, limit = _device()
    Q = qmul * sms + 3
    assert _slice_plan(n, LIKE[kind], Q, sms, limit) == plan
    m = _model(kind, n)
    dm = device_model(m)
    rng = np.random.default_rng(2000 + n + qmul)
    if kind == 'egg':       # C3: the whole cube, threshold at the median (the likelihood is nearly flat in 25-D)
        pts = rng.random((4000, n))
        logl = m.loglike(pts)
        loglstar = float(np.quantile(logl, 0.5))
        good = pts[logl > loglstar]
        axes = np.array([OB.bounding_ellipsoid(good[i::3]).axes for i in range(3)])
        u0 = good[rng.integers(len(good), size=Q)]
        ell = rng.integers(3, size=Q).astype(np.int32)
    else:
        u0, loglstar, axes, ell = _queue(kind, m, n, Q, rng)
    scale, chain0 = 1.0, 300 + n
    fn, chain = (ops.rslice_batch, OS.rslice_chain) if sampler == 'rslice' else (ops.slice_batch, OS.slice_chain)
    ops.bound_set(axes)
    o = _run_traced(lambda: fn(dm.model_id(), u0, loglstar, scale, slices, SEED, chain0=chain0, doubling=doubling,
                               ell=ell),
                    'slice_kernel<%d,%s,%s,%s>' % (LIKE[kind], _b(sampler == 'rslice'), _b(plan[0]), _b(plan[1])))
    assert np.all(o['flags'] == 0)
    assert np.all(o['logl'] > loglstar)
    _check_consistent(m, o)
    extra = 2 if n >= 200 else (6 if sampler == 'slice' and n >= 100 else 16)
    for q in _pick(ell, rng, extra):
        r = chain(u0[q], loglstar, axes[ell[q]], scale, m, philox.ChainStream(SEED, chain0 + q), slices,
                  doubling=doubling)
        assert not r['expansion_warning_set']
        assert (o['ncall'][q], o['n_expand'][q], o['n_contract'][q]) == (r['ncall'], r['n_expand'], r['n_contract']), q
        close(o['u'][q], r['u'], rtol=RTOL)
        close(o['v'][q], r['v'], rtol=RTOL)
        assert o['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL)


# ---- 3. uniform sampling from the bound -----------------------------------------------------------------------------
# unif_kernel<L> (b2n_unif_kernel.cuh): the draw and the membership test run warp_matvec2 over 64-row blocks, so
# ncdim > 64 takes a second block; the cube test reads the dimension flags.
UN = [(10, 10, 1, False), (10, 10, 3, False), (10, 10, 3, True), (50, 50, 3, False), (50, 40, 1, False),
      (100, 100, 1, False), (100, 100, 3, False), (100, 80, 3, False), (100, 100, 3, True)]


@pytest.mark.parametrize('n,nc,K,wrap', UN, ids=['n%d-ncdim%d-K%d%s' % (n, nc, K, '-flags' if w else '')
                                                   for n, nc, K, w in UN])
def test_unif_matrix(n, nc, K, wrap):
    m = OL.gauss_corr(n, 0.4, 5.)
    dm = device_model(m)
    rng = np.random.default_rng(3000 + n + nc + K)
    pts = 0.5 + 0.03 * rng.standard_normal((max(2000, 6 * K * nc), n))
    flags = nb = None
    if wrap:                # the bound crosses u = 0 in the first three coordinates; two of them are not bounded
        pts[:, :3] += 0.04 - 0.5
        flags = np.zeros(n, dtype=np.uint8)
        flags[0], flags[1] = 1, 2
        nb = flags == 0
    ells = [OB.bounding_ellipsoid(pts[i::K, :nc]) for i in range(K)]
    me = OB.MultiEll(ells)
    # threshold: the median likelihood of points drawn from the bound (about one in two draws is accepted)
    e0 = ells[0]
    z = rng.standard_normal((1000, nc))
    x = e0.ctr + (z / np.linalg.norm(z, axis=1)[:, None] * rng.random((1000, 1)) ** (1. / nc)) @ e0.axes.T
    x = np.concatenate([x, rng.random((1000, n - nc))], axis=1)
    loglstar = float(np.median(m.loglike(m.prior_transform(x))))
    ops.bound_set(me.axes, me.ctrs, me.ams, me.logvol_ells)
    Q, chain0 = 8 * 32 + 3, 11
    o = _run_traced(lambda: ops.unif_batch(dm.model_id(), Q, n, loglstar, SEED, chain0=chain0, ncdim=nc,
                                           dimflags=flags), 'unif_kernel<%d>' % PREC)
    assert np.all(o['flags'] & 0xC0000000 == 0)
    _check_consistent(m, o)
    for q in range(Q):
        r = OS.unif_chain(loglstar, me, m, philox.ChainStream(SEED, chain0 + q), n, nonbounded=nb)
        assert (o['ncall'][q], o['nprop'][q]) == (r['ncall'], r['nprop']), q
        close(o['u'][q], r['u'], rtol=RTOL)
        close(o['v'][q], r['v'], rtol=RTOL)
        assert o['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL)
    if wrap:
        assert (o['u'][:, :2] < 0).any() and np.all(o['u'][:, 2:nc] > 0)


# ---- 4. model evaluation ---------------------------------------------------------------------------------------------
def _loglike_ld(m, v):
    """The oracle's likelihood evaluated in np.longdouble."""
    v = v.astype(np.longdouble)
    p = {k: (np.asarray(x, dtype=np.longdouble) if isinstance(x, np.ndarray) else np.longdouble(x))
         for k, x in m.p.items()}
    k = m.like_kind
    if k == PREC:
        d = v - p['mean']
        return -0.5 * np.sum((d @ p['prec']) * d, axis=-1) + p['lnorm']
    if k == DIAG:
        d = v - p['mean']
        return -0.5 * np.sum(p['ivar'] * d * d, axis=-1) + p['lnorm']
    if k == EGG:
        t = 2 * p['tmax'] * v - p['tmax']
        return (2 + np.prod(np.cos(t / 2), axis=-1)) ** p['power']
    if k == SHELL:
        w2 = p['w'] ** 2
        const = -0.5 * np.log(2 * np.pi * w2)
        d1 = np.sqrt(np.sum((v - p['c1']) ** 2, axis=-1))
        d2 = np.sqrt(np.sum((v - p['c2']) ** 2, axis=-1))
        a, b = const - (d1 - p['r']) ** 2 / (2 * w2), const - (d2 - p['r']) ** 2 / (2 * w2)
        hi = np.maximum(a, b)
        return hi + np.log1p(np.exp(np.minimum(a, b) - hi))
    raise ValueError(k)


def _prior_ld(m, u):
    p = m.p
    if m.prior_kind == OL.PRIOR_UNIFORM:
        return np.asarray(p['lo'], np.longdouble) + np.asarray(p['width'], np.longdouble) * u.astype(np.longdouble)
    return u.astype(np.longdouble)


@pytest.mark.parametrize('n', [64, 65, 100, 128, 129, 200])
def test_model_eval_gauss_prec_longdouble(n):
    m = OL.gauss_corr(n, 0.4, 5.)
    dm = device_model(m)
    rng = np.random.default_rng(n)
    u = 0.5 + 0.05 * rng.standard_normal((67, n))
    v, logl = ops.model_eval(dm.model_id(), u)
    ref = _loglike_ld(m, _prior_ld(m, u))
    np.testing.assert_allclose(v, _prior_ld(m, u).astype(float), rtol=1e-15, atol=1e-15)
    np.testing.assert_allclose(logl, ref.astype(float), rtol=1e-12)


def test_model_eval_normal_ppf_tails():
    """v = mu + sigma ndtri(u) at the ends of the Philox stream's range: within CUDA's 5-ulp bound for normcdfinv plus
    the rounding of the affine map."""
    from scipy.special import ndtri
    us = np.array([2.0 ** -53, 1e-10, 0.5, 1 - 1e-10, 1 - 2.0 ** -53])
    n = len(us)
    mu, sigma = np.array([0.3, -1.2, 0.3, 2.5, -0.7]), np.array([1.0, 2.0, 0.5, 3.0, 1.5])
    m = OL.Model(n, OL.PRIOR_NORMAL_PPF, DIAG, mu=mu, sigma=sigma, mean=np.zeros(n), ivar=np.ones(n), lnorm=0.0)
    dm = device_model(m)
    v, _ = ops.model_eval(dm.model_id(), us[None])
    x = ndtri(us)
    tol = sigma * 5 * np.spacing(np.abs(x)) + 2 * np.spacing(np.abs(mu + sigma * x))
    assert np.all(np.abs(v[0] - (mu + sigma * x)) <= tol), (v[0], mu + sigma * x, tol)
    assert np.all(np.isfinite(v))


@pytest.mark.parametrize('kind', ['prec', 'diag', 'egg', 'shell', 'region2d'])
@pytest.mark.parametrize('n', [65, 130])
def test_model_eval_every_likelihood_wide(kind, n):
    """Every likelihood kind where its vector loop takes more than two passes of a warp."""
    rng = np.random.default_rng(7 * n)
    if kind == 'region2d':
        m = OL.region2d('diamond', n)
        from dynesty_b200 import likelihoods as DL
        dm = DL.region2d('diamond', n)
        u = rng.random((64, n))
        v, logl = ops.model_eval(dm.model_id(), u)
        np.testing.assert_array_equal(v, u)
        np.testing.assert_allclose(logl, m.loglike(u), rtol=1e-12, atol=1e-15)
        return
    m = _model(kind, n)
    dm = device_model(m)
    if kind == 'egg':       # the eggbox peaks: cos(t/2) = +-1 at u in {0.1, 0.3, ..., 0.9}
        u = rng.choice([0.1, 0.3, 0.5, 0.7, 0.9], size=(64, n)) + 0.003 * rng.standard_normal((64, n))
    else:
        u = _cloud(kind, n, 64, rng)
    v, logl = ops.model_eval(dm.model_id(), u)
    close(v, m.prior_transform(u), rtol=1e-13)
    vr = m.prior_transform(u) if m.prior_kind == OL.PRIOR_NORMAL_PPF else _prior_ld(m, u)
    np.testing.assert_allclose(logl, _loglike_ld(m, np.asarray(vr)).astype(float), rtol=1e-12)


# ---- 5. device rounds at the product shapes ---------------------------------------------------------------------------
def _bound(groups, enlarge=1.25):
    ells = []
    for p in groups:
        e = OB.bounding_ellipsoid(p)
        e.scale_to_logvol(e.logvol + math.log(enlarge))
        ells.append(e)
    return dict(ctrs=np.array([e.ctr for e in ells]), ams=np.array([e.am for e in ells]),
                axes=np.array([e.axes for e in ells]), logvols=np.array([e.logvol for e in ells]), strict=True)


def _split(lu, two):
    return [lu[lu[:, 0] < 0.5], lu[lu[:, 0] >= 0.5]] if two else [lu]


def _c2_live(om, N, n, rng, two):
    Cm = np.full((n, n), 0.4)
    np.fill_diagonal(Cm, 1.0)
    u = 0.5 + 0.03 * rng.standard_normal((N, n)) @ np.linalg.cholesky(Cm).T
    if two:
        u[: N // 2, 0] -= 0.15
        u[N // 2:, 0] += 0.15
    return u


@pytest.mark.parametrize('case', ['c2-rwalk', 'c2-rwalk-two-ellipsoids', 'c3-rslice'])
def test_rounds_product_shape_match_oracle(case):
    """The device-paced chain kernels (C2: the warp-specialised rwalk kernel; C3: rslice) in three rounds against
    oracle.nsloop, with the assertions of tests/test_gpu_nsloop.py::test_rounds_match_oracle."""
    rng = np.random.default_rng(len(case))
    two = case.endswith('two-ellipsoids')
    if case.startswith('c2'):
        n, N, K, steps, rounds, sampler = 50, 2000, 50, 70, 3, 'rwalk'
        om = OL.gauss_corr(n, 0.4, 5.)
        u = _c2_live(om, N, n, rng, two)
        scale0 = 0.3
    else:
        n, N, K, steps, rounds, sampler = 25, 4000, 80, 28, 2, 'rslice'
        om = OL.eggbox(n)
        u = rng.random((N, n))
        scale0 = 1.0
    dm = device_model(om)
    v = om.prior_transform(u)
    l = om.loglike(v)
    seed, chain0 = 56432, 1000
    o = nsloop.BatchNS(om, u, v, l, K, sampler, steps, seed, chain0=chain0, scale=scale0, logvol=-2.5, logz=-40.0,
                       loglstar=float(l.min()) - 0.5, ncall=500, bound=_bound(_split(u, two)), dlogz=1e-6)
    ops.ns_create(dm.model_id(), N, n, K, ('rwalk', 'rslice').index(sampler), steps, seed, chain0=chain0, dlogz=1e-6,
                  dead_capacity=rounds * K + 5)
    try:
        ops.ns_set_state(u, v, l, -2.5, -40.0, float(l.min()) - 0.5, 500, scale0)
        for r in range(rounds):
            b = _bound(_split(o.live_u, two))
            o.bound = b
            ops.bound_set(b['axes'], b['ctrs'], b['ams'], b['logvols'])
            assert o.step(), (o.done, o.need_bound)
            st = ops.ns_run(1, 0)
        assert (st['done'], st['need_bound'], st['error']) == (0, 0, 0)
        assert st['rounds'] == rounds and st['it'] == rounds * K
        assert st['ncall'] == o.ncall
        du, dv, dl, dlv, dnc = ops.ns_get_dead(0, st['it'], n)
        ou, ov, ol, olv, onc = o.dead_arrays()
        assert np.array_equal(dl[:K], ol[:K])
        assert np.allclose(dl, ol, rtol=1e-9, atol=0) and np.allclose(du, ou, rtol=1e-8, atol=1e-12)
        assert np.allclose(dlv, olv, rtol=0, atol=1e-13)
        assert np.array_equal(dnc, onc)
        lu, lv_, ll = ops.ns_get_live(N, n)
        pd, po = np.argsort(ll, kind='stable'), np.argsort(o.live_logl, kind='stable')
        assert np.allclose(ll[pd], o.live_logl[po], rtol=1e-8, atol=1e-10)
        assert np.allclose(lu[pd], o.live_u[po], rtol=1e-8, atol=1e-12)
        assert np.allclose(lv_[pd], o.live_v[po], rtol=1e-8, atol=1e-11)
        assert st['logz'] == pytest.approx(o.logz, rel=1e-10)
        assert st['logvol'] == pytest.approx(o.logvol, abs=1e-13)
        assert st['scale'] == pytest.approx(o.scale, rel=1e-10)
        assert st['loglstar'] == pytest.approx(o.loglstar, rel=1e-9)
        if sampler == 'rwalk':
            assert 0 < o.last['n_accept'] < K * steps
    finally:
        ops.ns_destroy()


# ---- 6. switches of the device rounds ---------------------------------------------------------------------------------
def _switch_run(monkeypatch, n, sampler, env):
    """One device run in a fresh context: 1 round, 40 rounds, a device bound update (which fits the live set on the
    two Gaussian shells with a number of ellipsoids other than the three it started with), 1 round, 40 rounds.
    Returns everything it left."""
    from dynesty_b200 import _lib
    for k in ('B2N_NS_GRAPH', 'B2N_NS_THREADS'):
        monkeypatch.delenv(k, raising=False)
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    ctx = _lib.Context(0)
    om = OL.shells(n)
    dm = device_model(om)
    N, K = (400, 8) if n <= 6 else (1000, 10)
    steps = 10 if sampler == 'rwalk' else 3
    u = 0.5 + 0.03 * np.random.default_rng(n).standard_normal((N, n))
    u[: N // 2, 0] -= 3.5 / 12
    u[N // 2:, 0] += 3.5 / 12
    v, l = om.prior_transform(u), om.loglike(om.prior_transform(u))
    b = _bound([u[: N // 2], u[N // 2: 3 * N // 4], u[3 * N // 4:]], enlarge=3.0 ** n)       # axes x 3
    ops.bound_set(b['axes'], b['ctrs'], b['ams'], b['logvols'], ctx=ctx)
    ops.ns_create(dm.model_id(ctx), N, n, K, ('rwalk', 'rslice').index(sampler), steps, 9, chain0=3, dlogz=1e-9,
                  ctx=ctx)
    try:
        ops.ns_set_state(u, v, l, 0.0, -1e300, -1e300, 0, 0.3, ctx=ctx)
        sts = [ops.ns_run(1, 0, ctx=ctx), ops.ns_run(40, 0, ctx=ctx)]
        nells = ops.ns_update_bound(True, 2.0 ** n, ctx=ctx)       # (axes x 2: the starts stay inside)
        ops.ns_bound_updated(ctx=ctx)
        sts += [ops.ns_run(1, 0, ctx=ctx), ops.ns_run(40, 0, ctx=ctx)]
        dead = ops.ns_get_dead(0, sts[-1]['it'], n, ctx=ctx)
        live = ops.ns_get_live(N, n, ctx=ctx)
    finally:
        ops.ns_destroy(ctx=ctx)
    return sts, nells, dead, live


SW = [(6, 'rwalk'), (50, 'rwalk'), (6, 'rslice')]


@pytest.mark.parametrize('n,sampler', SW, ids=['%s%d' % (s, n) for n, s in SW])
def test_ns_graph_equals_plain_launches(monkeypatch, n, sampler):
    """B2N_NS_GRAPH=1: rounds replayed from a captured CUDA graph (from the second b2n_ns_run of a launch key, 16
    rounds at a time, captured again after the bound changed) give bit-identical runs."""
    a = _switch_run(monkeypatch, n, sampler, {})
    g = _switch_run(monkeypatch, n, sampler, dict(B2N_NS_GRAPH='1'))
    sa, sg = a[0], g[0]
    assert sa[1]['rounds'] == 41 and a[1][0] != 3         # the graph was used before and after the bound changed
    assert sa[3]['rounds'] > 41 + 16
    assert sa == sg and a[1] == g[1]
    for x, y in zip(a[2] + a[3], g[2] + g[3]):
        assert np.array_equal(x, y)


@pytest.mark.parametrize('threads', ['256', '512'])
def test_ns_threads_equal_default(monkeypatch, threads):
    """B2N_NS_THREADS (threads of the one-CTA step kernel, read at b2n_ns_create) changes no result: same dead order
    and counts, logZ to 1e-12."""
    a = _switch_run(monkeypatch, 20, 'rwalk', dict(B2N_NS_THREADS='1024'))
    t = _switch_run(monkeypatch, 20, 'rwalk', dict(B2N_NS_THREADS=threads))
    for sa, st in zip(a[0], t[0]):
        assert {k: x for k, x in sa.items() if k not in ('logz', 'delta_logz')} == \
            {k: x for k, x in st.items() if k not in ('logz', 'delta_logz')}
        assert st['logz'] == pytest.approx(sa['logz'], rel=1e-12)
    assert a[1] == t[1]
    for x, y in zip(a[2] + a[3], t[2] + t[3]):
        assert np.array_equal(x, y)

"""GPU: a chain's result depends only on its own inputs -- start point, ellipsoid, seed and chain id chain0 + q -- never
on the launch it is part of (include/b200nest.h: b2n_set_chain_pack; csrc/b2n_rwalk.cu: rwalk_plan).  Sharded
multi-GPU runs, replicas with packed CTAs and the device-resident rounds rely on it.

Rule of comparison: a reference launch (Q chains from chain0, K = 3 ellipsoids, a random ellipsoid per chain) and a
variant return the same bytes -- u, v, logl, every counter and the flags -- for every chain they share.  No tolerance,
no sample: all chains.  Every variant also shows that it changed the launch: the chains per CTA, warps per CTA, where
the matrices live and the groups per CTA are recomputed from the host formulas (the plan mirrors of
tests/test_gpu_kernel_matrix.py, extended by the chain pack), and the kernel that ran -- its template arguments say
where the matrices live -- is read from a CUDA-activity trace and must match them.  A variant whose geometry equals the reference's fails.

Variants: shards of the queue (a single chain, a cut inside a lock-step group, a cut at a CTA boundary, a cut that
leaves a shard under 16 x SMs chains while the whole queue is over it); contexts with b2n_set_chain_pack(k); the same
chains inside a longer queue, across the thresholds of the warp-per-chain plans and past 8 / 16 chains per CTA of the
lock-step kernels; other chains moved to other ellipsoids, and resident ellipsoids that no chain uses; chain ids
across 2^32 (with the chains at the carry also against the float64 oracle).  Then the device-resident rounds and
whole runs with chain pack 1 against 4 / 8.
"""
import re
import time

import numpy as np
import pytest

from helpers import device_model, close
from oracle import samplers as OS, philox, bounding as OB, likelihoods as OL
from test_gpu_kernel_matrix import (_device, _chain_warps, _rwalk_warp_plan, _slice_plan, _model, _queue,
                                    _kt, LIKE, _bound)
from test_gpu_user_model import _user_restatement


def _have_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:       # noqa: BLE001 -- no torch / no driver: the file is collected and skipped
        return False


pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not _have_cuda(), reason='needs a CUDA device')]

PREC = OL.LIKE_GAUSS_PREC
USER = 5                    # B2N_LIKE_USER
SEED = 90210
RTOL = 1e-9
WALKS = 13                  # not a multiple of the lock-step kernels' ring depth: the last ring is partial
RWALK_ENV = ('B2N_RWALK_IMPL', 'B2N_NS_GRAPH', 'B2N_NS_THREADS')


def _cdiv(a, b):
    return -(-a // b)


# ---- launch plans (host mirrors) --------------------------------------------------------------------------------------
def _plan(fam, n, nc, like, Q, pack, sms, limit):
    """Launch geometry of a chain entry point: dict(cpc chains per CTA, threads, ch chains per lock-step group (warps
    per CTA for the warp-per-chain kernels), ax_s / pr_s where the matrices live).
      mma / ws  rwalk_mma_kernel, rwalk_mmaws_kernel: two CTAs per SM, cpc = max(min(pack, 8), ceil(Q / 2 SMs));
      mmas      rwalk_mmas_kernel: one CTA per SM, cpc = max(min(pack, 16), ceil(Q / SMs));
      warp / slice  rwalk_kernel, slice_kernel (b2n_chain_grid): one CTA per SM up to 16 x SMs chains, two beyond,
                cpc = max(min(pack, 16), ceil(Q / CTAs)), warps = min(cpc, 16, what fits), matrices by the plan;
      unif      unif / unitcube / friends_unif kernels: four chains per 128-thread CTA, no pack."""
    if fam in ('mma', 'ws'):
        return dict(cpc=max(min(pack, 8), _cdiv(Q, 2 * sms)), threads=384 if fam == 'ws' else 256, ch=8,
                    ax_s=None, pr_s=None)
    if fam == 'mmas':
        return dict(cpc=max(min(pack, 16), _cdiv(Q, sms)), threads=512, ch=16, ax_s=None, pr_s=None)
    if fam == 'unif':
        return dict(cpc=4, threads=128, ch=4, ax_s=None, pr_s=None)
    npad = (n + 1) & ~1
    per_warp = 6 * npad * 8
    base = 4 * npad * 8 if fam == 'slice' else ((((n + 3) >> 2) << 1) + 4 * npad) * 8
    max_warps = min(16, (limit - base) // per_warp)
    ctas = sms if Q <= 16 * sms else 2 * sms
    cpc = max(min(pack, 16), _cdiv(Q, ctas))
    warps = max(1, min(max_warps, 16, cpc))
    fixed = per_warp * warps + base
    ax_b = nc * ((nc + 15) & ~15) * 8
    pr_b = n * ((n + 15) & ~15) * 8 if like == PREC else 0
    ax_s = fixed + ax_b <= limit
    pr_s = pr_b > 0 and fixed + (ax_b if ax_s else 0) + pr_b <= limit
    if pack == 1:           # the kernel matrix's mirrors say the same
        assert warps == _chain_warps(Q, sms, max_warps)
        want = _slice_plan(n, like, Q, sms, limit) if fam == 'slice' else _rwalk_warp_plan(n, nc, like, Q, sms, limit)
        assert (ax_s, pr_s) == want
    return dict(cpc=cpc, threads=32 * warps, ch=warps, ax_s=ax_s, pr_s=pr_s)


def _worklist(ell, K, cpc):
    """b2n_build_worklist (csrc/b2n_rwalk.cu): chains grouped by ellipsoid (stable), each group split into
    ceil(count / cpc) CTAs of equal size.  Returns (order, [(first, count, ellipsoid)] per CTA)."""
    order = np.argsort(ell, kind='stable')
    counts = np.bincount(ell, minlength=K)
    cta, start = [], 0
    for k in range(K):
        c = int(counts[k])
        if c:
            parts = _cdiv(c, cpc)
            for i in range(parts):
                lo, hi = start + c * i // parts, start + c * (i + 1) // parts
                cta.append((lo, hi - lo, k))
        start += c
    return order, cta


def _geometry(fam, n, nc, like, Q, pack, ell, K):
    """The plan and where each chain sits: pos[q] = (CTA, group within the CTA, slot within the group, ellipsoid)."""
    sms, limit = _device()
    pl = _plan(fam, n, nc, like, Q, pack, sms, limit)
    pos = np.empty((Q, 4), dtype=np.int64)
    if fam == 'unif':
        q = np.arange(Q)
        pos[:, 0], pos[:, 1], pos[:, 2], pos[:, 3] = q // 4, 0, q % 4, 0
        ncta, groups = _cdiv(Q, 4), 1
    else:
        order, cta = _worklist(ell if ell is not None else np.zeros(Q, np.int32), K, pl['cpc'])
        for j, (lo, cnt, k) in enumerate(cta):
            off = np.arange(cnt)
            pos[order[lo:lo + cnt]] = np.stack([np.full(cnt, j), off // pl['ch'], off % pl['ch'], np.full(cnt, k)], 1)
        ncta, groups = len(cta), max(_cdiv(c, pl['ch']) for _, c, _ in cta)
    return dict(pl, ncta=ncta, groups=groups, pos=pos)


def _shape(g):
    """The launch geometry a variant has to change (everything but the chain positions)."""
    return tuple((k, g[k]) for k in ('cpc', 'threads', 'ch', 'ax_s', 'pr_s', 'ncta', 'groups'))


# ---- traced launches ---------------------------------------------------------------------------------------------------
# A CUDA-activity trace now and then holds the runtime calls of a launch and the device records of what follows it (a
# flags kernel, the copies back) but not the record of the kernel itself: more often late in a long test process, and
# in a short window -- a lone kernel traced without a margin has lost its record in nine traces of ten on one H100
# while another H100 kept every one.  The profiler keeps only the device records that fall inside its capture window,
# so the window is padded with idle time on both sides, more on every retry.
PADS = (0.02, 0.1, 0.3, 1.0, 2.0)


def _trace(fn, pad):
    import torch
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()            # nothing of an earlier call is still in flight when the trace starts
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(pad)
        out = fn()
        torch.cuda.synchronize()
        time.sleep(pad)
    return out, sorted({re.sub(r'\s+', '', e.key) for e in prof.key_averages()})


def _traced(fn, expect):
    """fn() under a CUDA-activity trace; asserts that a kernel whose name (blanks removed) contains `expect` ran.
    As test_gpu_kernel_matrix._run_traced: a trace that misses the kernel is followed by one untraced call (a
    module's first launch can go unrecorded) and traced again, here with a wider window (PADS); every repeat must
    give the same outputs bit for bit."""
    out, names = _trace(fn, PADS[0])
    for pad in PADS[1:]:
        if any(expect in k for k in names):
            break
        fn()
        again, names = _trace(fn, pad)
        for k in out:
            assert np.array_equal(again[k], out[k]), k
    assert any(expect in k for k in names), (expect, names)
    return out


# ---- comparison ---------------------------------------------------------------------------------------------------------
def _raw(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8).reshape(len(a), -1)


def _same(ref, var, rows_ref, rows_var, where):
    """Every output of the chains ref[rows_ref] == var[rows_var], byte for byte; a failure names the first differing
    chain and where it sat in both launches."""
    rows_ref, rows_var = np.asarray(rows_ref), np.asarray(rows_var)
    assert set(ref) == set(var)
    for k in sorted(ref):
        bad = np.flatnonzero((_raw(ref[k][rows_ref]) != _raw(var[k][rows_var])).any(axis=1))
        if bad.size:
            i = int(bad[0])
            raise AssertionError('%s differs at %d of %d chains; first: reference chain %d, %s' % (
                k, bad.size, len(rows_ref), rows_ref[i], where(int(rows_ref[i]), int(rows_var[i]))))


# ---- the chain entry points ---------------------------------------------------------------------------------------------
MMA = dict(B2N_RWALK_IMPL='mma')
WARP = dict(B2N_RWALK_IMPL='warp')


class Case:
    def __init__(self, cid, sampler, kind, n, nc=None, env=None, fam=None, expect=None, wrap=False, doubling=False,
                 slices=None, user=False, qmul=20):
        self.cid, self.sampler, self.kind, self.n, self.nc = cid, sampler, kind, n, nc or n
        self.env, self.fam, self.expect, self.wrap, self.doubling = env or {}, fam, expect, wrap, doubling
        self.slices, self.user, self.qmul = slices, user, qmul

    def __repr__(self):
        return self.cid


def _warp(like, geo):
    return 'rwalk_kernel<%d,%s,%s>' % (like, 'true' if geo['ax_s'] else 'false', 'true' if geo['pr_s'] else 'false')


def _slice_name(like, rdir, geo):
    b = lambda x: 'true' if x else 'false'
    return 'slice_kernel<%d,%s,%s,%s>' % (like, b(rdir), b(geo['ax_s']), b(geo['pr_s']))


CASES = [
    # rwalk_kernel<L, AXS, PRS>: (true, true), (true, false) and (false, false); <L, false, true> cannot occur
    Case('warp-prec6', 'rwalk', 'prec', 6, fam='warp'),
    Case('warp-prec6-flags', 'rwalk', 'prec', 6, fam='warp', wrap=True),
    Case('warp-prec6-ncdim4', 'rwalk', 'prec', 6, nc=4, fam='warp'),
    Case('warp-diag40-ncdim30', 'rwalk', 'diag', 40, nc=30, fam='warp'),
    Case('warp-egg12', 'rwalk', 'egg', 12, fam='warp'),
    Case('warp-shell10', 'rwalk', 'shell', 10, fam='warp'),
    Case('warp-diag130-axes-global', 'rwalk', 'diag', 130, env=WARP, fam='warp', qmul=13),
    # rwalk_mma_kernel<L, KT> at KT 8 / 13 / 16
    Case('mma-prec16', 'rwalk', 'prec', 16, fam='mma'),
    Case('mma-diag40', 'rwalk', 'diag', 40, fam='mma'),
    Case('mma-shell64', 'rwalk', 'shell', 64, fam='mma'),
    Case('mma-egg36-forced', 'rwalk', 'egg', 36, env=MMA, fam='mma'),
    # rwalk_mmaws_kernel<KT, true | false>
    Case('mmaws-plain-prec30', 'rwalk', 'prec', 30, fam='ws'),
    Case('mmaws-plain-prec50', 'rwalk', 'prec', 50, fam='ws'),
    Case('mmaws-plain-prec60', 'rwalk', 'prec', 60, fam='ws'),
    Case('mmaws-generic-ppf50', 'rwalk', 'precppf', 50, fam='ws'),
    Case('mmaws-generic-flags28', 'rwalk', 'prec', 28, fam='ws', wrap=True),
    # rwalk_mmas_kernel<L>
    Case('mmas-prec80', 'rwalk', 'prec', 80, fam='mmas'),
    Case('mmas-shell70', 'rwalk', 'shell', 70, fam='mmas'),
    # slice_kernel<L, RANDOM_DIR, AXS, PRS>
    Case('rslice-prec50', 'rslice', 'prec', 50, fam='slice', slices=3),
    Case('slice-prec50-dbl', 'slice', 'prec', 50, fam='slice', slices=1, doubling=True),
    Case('rslice-egg25-dbl', 'rslice', 'egg', 25, fam='slice', slices=4, doubling=True),
    Case('slice-egg25', 'slice', 'egg', 25, fam='slice', slices=1),
    Case('rslice-prec200-both-global', 'rslice', 'prec', 200, fam='slice', slices=2, qmul=1),
    # one warp per chain, four per CTA
    Case('unif-prec10', 'unif', 'prec', 10, fam='unif', qmul=2),
    Case('unitcube-shell4', 'unitcube', 'shell', 4, fam='unif', qmul=2),
    Case('friends-unif-diag6', 'friends', 'diag', 6, fam='unif', qmul=2),
    # user models (NVRTC images): the warp-per-chain rwalk slot, the rslice slot, the unif slot
    Case('user-rwalk-diag10', 'rwalk', 'diag', 10, fam='warp', user=True),
    Case('user-rslice-shell8', 'rslice', 'shell', 8, fam='slice', slices=3, user=True),
    Case('user-unif-prec10', 'unif', 'prec', 10, fam='unif', user=True, qmul=2),
]
BYID = {c.cid: c for c in CASES}
ELL = [c for c in CASES if c.fam != 'unif']                 # per-chain ellipsoids, chain pack, regrouping
REGISTRY = [c for c in CASES if not c.user]


def _expect(case, like, geo):
    """Name (or names) of the kernel the case must reach at this geometry."""
    n = case.n
    if case.user:           # NVRTC image: demangled or not, the template's name is in the record
        return {'rwalk': 'rwalk_kernel', 'rslice': 'slice_kernel', 'unif': 'unif_kernel'}[case.sampler]
    if case.fam == 'warp':
        return _warp(like, geo)
    if case.fam == 'mma':
        return 'rwalk_mma_kernel<%d,%d>' % (like, _kt(n))
    if case.fam == 'ws':
        return 'rwalk_mmaws_kernel<%d,%s>' % (_kt(n), 'true' if case.kind == 'prec' and not case.wrap else 'false')
    if case.fam == 'mmas':
        return 'rwalk_mmas_kernel<%d>' % like
    if case.fam == 'slice':
        return _slice_name(like, case.sampler == 'rslice', geo)
    return {'unif': 'unif_kernel<%d>', 'unitcube': 'unitcube_kernel<%d>',
            'friends': 'friends_unif_kernel<%d>'}[case.sampler] % like


class Problem:
    """A case's model and a pool of start points / ellipsoid indices (the first Q of them make a queue)."""

    def __init__(self, case, Q):
        self.case = case
        n = case.n
        m = self.m = _model(case.kind, n)
        self.like = USER if case.user else LIKE[case.kind]
        self.dm = _user_restatement(case.kind, m) if case.user else device_model(m)
        rng = np.random.default_rng(sum(map(ord, case.cid)))
        self.K = 3
        self.flags = self.per = self.ref = self.nb = None
        if case.wrap:
            self.per, self.ref = [0, n // 2], [1, n - 1]
            from dynesty_b200 import ops
            self.flags = ops.dimflags_from(n, self.per, self.ref)
            self.nb = self.flags == 0
        if case.sampler in ('rwalk', 'rslice', 'slice'):
            if case.kind == 'egg' and case.sampler != 'rwalk':     # as the kernel matrix: C3 over the whole cube
                pts = rng.random((4000, n))
                logl = m.loglike(pts)
                self.loglstar = float(np.quantile(logl, 0.5))
                good = pts[logl > self.loglstar]
                self.axes = np.array([OB.bounding_ellipsoid(good[i::3]).axes for i in range(3)])
                self.u0 = good[rng.integers(len(good), size=Q)]
                self.ell = rng.integers(3, size=Q).astype(np.int32)
            else:
                self.u0, self.loglstar, self.axes, self.ell = _queue(case.kind, m, case.nc, Q, rng)
            self.bound = dict(axes=self.axes)
        elif case.sampler == 'unif':
            pts = 0.5 + 0.03 * rng.standard_normal((2000, n))
            if case.kind == 'shell':
                pts[:, 0] += -1.5 / 12.0
            self.me = OB.MultiEll([OB.bounding_ellipsoid(pts[i::3]) for i in range(3)])
            self.loglstar = float(np.quantile(m.loglike(m.prior_transform(pts)), 0.3))
            self.bound = dict(axes=self.me.axes, ctrs=self.me.ctrs, ams=self.me.ams, logvols=self.me.logvol_ells)
            self.ell = None
        elif case.sampler == 'unitcube':
            self.loglstar = float(np.quantile(m.loglike(m.prior_transform(rng.random((4000, n)))), 0.9))
            self.bound, self.ell = None, None
        else:
            pts = 0.5 + 0.03 * rng.standard_normal((300, n))
            self.pts = pts
            self.loglstar = float(np.quantile(m.loglike(m.prior_transform(pts)), 0.3))
            self.bound, self.ell = None, None

    def load(self, ctx, axes=None):
        """Make this problem's bound (or `axes`) and model resident in ctx; returns the model id."""
        from dynesty_b200 import ops
        if self.case.sampler == 'friends':
            f = ops.friends_update(self.pts, 'balls', use_clustering=False, ctx=ctx)
            ops.friends_set('balls', self.pts, f['axes'], f['axes_inv'], ctx=ctx)
        elif self.bound is not None:
            b = dict(self.bound)
            if axes is not None:
                b = dict(axes=axes)
            ops.bound_set(b['axes'], b.get('ctrs'), b.get('ams'), b.get('logvols'), ctx=ctx)
        return self.dm.model_id(ctx)

    def run(self, ctx, rows, chain0, ell=None, axes=None, pack=1, trace=False):
        """Launch the chains u0[rows] (or len(rows) draws) with ids chain0 + i in ctx; returns (outputs, geometry).
        trace: the kernel that ran must be the one the plan names (a CUDA-activity trace per launch; kept to the
        launches whose plan the test is about, since a process that records hundreds of traces stops getting the
        device-side records; the NVRTC images of user models are not traced)."""
        from dynesty_b200 import ops
        c = self.case
        Q = len(rows)
        mid = self.load(ctx, axes)
        K = len(axes) if axes is not None else self.K
        if ell is None and self.ell is not None:
            ell = self.ell[rows]
        geo = _geometry(c.fam, c.n, c.nc, self.like, Q, pack, ell, K)
        if c.sampler == 'rwalk':
            fn = lambda: ops.rwalk_batch(mid, self.u0[rows], self.loglstar, 0.4, WALKS, SEED, chain0=chain0, ncdim=c.nc,
                                         ell=ell, dimflags=self.flags, ctx=ctx)
        elif c.sampler in ('rslice', 'slice'):
            f = ops.rslice_batch if c.sampler == 'rslice' else ops.slice_batch
            fn = lambda: f(mid, self.u0[rows], self.loglstar, 1.0, c.slices, SEED, chain0=chain0, doubling=c.doubling,
                           ell=ell, ctx=ctx)
        elif c.sampler == 'unif':
            fn = lambda: ops.unif_batch(mid, Q, c.n, self.loglstar, SEED, chain0=chain0, ctx=ctx)
        elif c.sampler == 'unitcube':
            fn = lambda: ops.unitcube_batch(mid, Q, c.n, self.loglstar, SEED, chain0=chain0, ctx=ctx)
        else:
            fn = lambda: ops.friends_unif_batch(mid, Q, c.n, self.loglstar, SEED, chain0=chain0, ctx=ctx)
        out = _traced(fn, _expect(c, self.like, geo)) if trace and not c.user else fn()
        if 'flags' in out and c.sampler != 'slice' and c.sampler != 'rslice':
            assert np.all(out['flags'] & 0xC0000000 == 0)
        elif 'flags' in out:
            assert np.all(out['flags'] == 0)
        assert np.all(out['logl'] > self.loglstar)
        return out, geo

    def oracle(self, q, chain):
        """The float64 oracle's chain q (start u0[q], ellipsoid ell[q]) on ChainStream(SEED, chain)."""
        c, m, st = self.case, self.m, philox.ChainStream(SEED, chain)
        if c.sampler == 'rwalk':
            return OS.rwalk_chain(self.u0[q], self.loglstar, self.axes[self.ell[q]], 0.4, m, st, WALKS,
                                  periodic=self.per, reflective=self.ref, nonbounded=self.nb)
        if c.sampler in ('rslice', 'slice'):
            f = OS.rslice_chain if c.sampler == 'rslice' else OS.slice_chain
            return f(self.u0[q], self.loglstar, self.axes[self.ell[q]], 1.0, m, st, c.slices, doubling=c.doubling)
        if c.sampler == 'unif':
            return OS.unif_chain(self.loglstar, self.me, m, st, c.n)
        if c.sampler == 'unitcube':
            return OS.unitcube_chain(self.loglstar, m, st, c.n)
        return None


_PROBLEMS = {}
_CTX = {}


def _problem(case, Q):
    key = (case.cid, Q)
    if key not in _PROBLEMS:
        _PROBLEMS.clear()                   # one case at a time: the pools of the large shapes are not small
        _PROBLEMS[key] = Problem(case, Q)
    return _PROBLEMS[key]


def _ctx(pack):
    """A context of its own per chain pack (b2n_set_chain_pack), made once per session."""
    from dynesty_b200 import _lib
    if pack not in _CTX:
        c = _lib.Context(0)
        if pack != 1:
            c.set_chain_pack(pack)
        _CTX[pack] = c
    return _CTX[pack]


def _env(monkeypatch, case):
    for k in RWALK_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in case.env.items():
        monkeypatch.setenv(k, v)


def _where(ga, gb):
    f = lambda g, q: 'CTA %d group %d slot %d ellipsoid %d' % tuple(g['pos'][q])
    return lambda qa, qb: 'reference %s, variant %s' % (f(ga, qa), f(gb, qb))


def _qref(case):
    sms, _ = _device()
    return case.qmul * sms + 3


# ---- A1. shards -------------------------------------------------------------------------------------------------------
def _cuts(case, geo, Q):
    """Shard cuts a (chains [0, a) and [a, Q)): one chain; inside a lock-step group (chains a - 1 and a share CTA
    and group); at a CTA boundary (a opens a CTA, a - 1 closes the one before); and, where the queue is longer than
    16 x SMs, a first shard under it."""
    pos = geo['pos']
    sms, _ = _device()
    cuts = {'one-chain': 1}
    same = [a for a in range(2, Q) if pos[a - 1][0] == pos[a][0] and pos[a - 1][1] == pos[a][1]]
    assert same, 'no two consecutive chains share a group'
    cuts['in-group'] = same[len(same) // 2]
    ends = {}
    for j in np.unique(pos[:, 0]):
        w = np.flatnonzero(pos[:, 0] == j)
        ends[j] = (w[np.lexsort((pos[w, 2], pos[w, 1]))][0], w[np.lexsort((pos[w, 2], pos[w, 1]))][-1])
    bnd = [a for a in range(1, Q) if pos[a][0] != pos[a - 1][0] and ends[pos[a][0]][0] == a
           and ends[pos[a - 1][0]][1] == a - 1]
    assert bnd, 'no CTA boundary between consecutive chains'
    cuts['cta-boundary'] = bnd[len(bnd) // 2]
    if Q > 16 * sms and case.fam in ('warp', 'slice'):
        cuts['under-16-per-sm'] = 16 * sms - 5
    return cuts


@pytest.mark.parametrize('case', CASES, ids=[c.cid for c in CASES])
def test_shards(monkeypatch, case):
    _env(monkeypatch, case)
    Q = _qref(case)
    P = _problem(case, Q)
    ctx = _ctx(1)
    chain0 = 1000 + case.n
    rows = np.arange(Q)
    ref, g = P.run(ctx, rows, chain0, trace=True)
    cuts = _cuts(case, g, Q)
    for tag, a in cuts.items():
        seen = False
        for lo, hi in ((0, a), (a, Q)):
            out, gv = P.run(ctx, rows[lo:hi], chain0 + lo)
            _same(ref, out, rows[lo:hi], np.arange(hi - lo), _where(g, gv))
            seen = seen or _shape(gv) != _shape(g)
        assert seen, (tag, a, _shape(g))     # the shards launch differently from the whole queue
        if tag == 'under-16-per-sm':
            assert Q > 16 * _device()[0] >= a
        if tag == 'in-group':
            assert g['pos'][a - 1][:2].tolist() == g['pos'][a][:2].tolist()


# ---- A2. chain packing ------------------------------------------------------------------------------------------------
def _packs(case):
    return (3, 8, 9) if case.fam in ('mma', 'ws') else (3, 8, 9, 16, 17)


@pytest.mark.parametrize('case', ELL, ids=[c.cid for c in ELL])
def test_chain_pack(monkeypatch, case):
    """Contexts with b2n_set_chain_pack(k): one partial lock-step group, a full one, a second group with one live
    chain, the caps (8 for rwalk_mma / mmaws, 16 for the others)."""
    _env(monkeypatch, case)
    sms, limit = _device()
    Q = (2 if case.fam in ('mma', 'ws') else 1) * sms - 5          # one chain per CTA at pack 1
    P = _problem(case, Q)
    rows = np.arange(Q)
    chain0 = 7 + case.n
    ref, g = P.run(_ctx(1), rows, chain0)
    assert g['cpc'] == 1
    cap = 8 if case.fam in ('mma', 'ws') else 16
    for k in _packs(case):
        out, gv = P.run(_ctx(k), rows, chain0, pack=k, trace=k == 16 and case.cid.startswith('warp-diag130'))
        assert gv['cpc'] == min(k, cap) and _shape(gv) != _shape(g), (k, _shape(gv))
        _same(ref, out, rows, rows, _where(g, gv))


# ---- A3. the same chains inside a longer queue ---------------------------------------------------------------------
# (case, reference Q, longer Qs as (SM multiple, extra), what must change)
SMS_Q = [
    ('warp-prec100', 'rwalk', 'prec', 100, WARP, 'warp', (8, 3), [(11, 3)]),
    ('warp-diag130', 'rwalk', 'diag', 130, WARP, 'warp', (8, 3), [(13, 3)]),
    ('rslice-prec100', 'rslice', 'prec', 100, {}, 'slice', (2, 3), [(11, 3)]),
    ('mma-shell20', 'rwalk', 'shell', 20, {}, 'mma', (2, -5), [(16, 9), (32, 9)]),
    ('mmaws-prec50', 'rwalk', 'prec', 50, {}, 'ws', (2, -5), [(16, 9), (32, 9)]),
    ('mmas-shell80', 'rwalk', 'shell', 80, {}, 'mmas', (1, -5), [(8, 1), (16, 1)]),
]


@pytest.mark.parametrize('cid,sampler,kind,n,env,fam,q0,longer', SMS_Q, ids=[c[0] for c in SMS_Q])
def test_longer_queue(monkeypatch, cid, sampler, kind, n, env, fam, q0, longer):
    """Reference: Q chains; variant: the same chains followed by others.  Warp per chain: the longer queue moves the
    precision matrix (prec100), the axes (diag130) or the slice kernel's precision matrix to global memory.
    Lock-step: chains per CTA past 8 and 16 (a second and a third group per CTA)."""
    case = Case(cid, sampler, kind, n, env=env, fam=fam, slices=2 if sampler == 'rslice' else None)
    _env(monkeypatch, case)
    sms, _ = _device()
    Qs = [m * sms + e for m, e in [q0] + longer]
    P = _problem(case, max(Qs))
    chain0 = 55
    warp = fam in ('warp', 'slice')         # (the lock-step kernels' names do not change with the queue length)
    ref, g = P.run(_ctx(1), np.arange(Qs[0]), chain0, trace=warp)
    cpcs = []
    for Ql in Qs[1:]:
        out, gv = P.run(_ctx(1), np.arange(Ql), chain0, trace=warp)
        if fam in ('warp', 'slice'):
            assert (g['ax_s'], g['pr_s']) != (gv['ax_s'], gv['pr_s']), (Ql, g['ax_s'], g['pr_s'])
        _same(ref, out, np.arange(Qs[0]), np.arange(Qs[0]), _where(g, gv))
        cpcs.append(gv['cpc'])
    if fam in ('mma', 'ws', 'mmas'):      # 1 chain per CTA, then past 8 and past 16
        assert g['cpc'] == 1 and 8 < cpcs[0] <= 16 < cpcs[1], cpcs


# ---- A4. regrouping ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', ELL, ids=[c.cid for c in ELL])
def test_regrouping(monkeypatch, case):
    """Chain q keeps its start point and ellipsoid; (a) the other chains move to other ellipsoids, so q sits in
    another CTA / group / slot; (b) two more ellipsoids are resident, unused, and the used ones move up one index."""
    _env(monkeypatch, case)
    Q = _qref(case)
    P = _problem(case, Q)
    rows = np.arange(Q)
    chain0 = 31
    ctx = _ctx(1)
    ref, g = P.run(ctx, rows, chain0)
    keep = rows[rows % 2 == 0]
    ell2 = P.ell[:Q].copy()
    ell2[1::2] = (ell2[1::2] + 1) % P.K
    out, gv = P.run(ctx, rows, chain0, ell=ell2)
    moved = (g['pos'][keep, :3] != gv['pos'][keep, :3]).any(axis=1)
    assert moved.mean() > 0.5 and (g['pos'][keep, 1:3] != gv['pos'][keep, 1:3]).any(axis=1).mean() > 0.1
    _same(ref, out, keep, keep, _where(g, gv))
    n = P.axes.shape[1]
    extra = np.concatenate([P.axes[:1] * 1.5, P.axes, P.axes[1:2] * 0.7])
    out, gv = P.run(ctx, rows, chain0, ell=P.ell[:Q] + 1, axes=extra)
    assert np.all(gv['pos'][:, 3] == g['pos'][:, 3] + 1) and extra.shape == (5, n, n)
    _same(ref, out, rows, rows, _where(g, gv))


# ---- A5. chain ids across 2^32 ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', REGISTRY, ids=[c.cid for c in REGISTRY])
def test_chain_ids_across_2_32(monkeypatch, case):
    """chain0 = 2^32 - a: chains [0, a) have ids below 2^32, [a, Q) above.  The whole queue against the two shards
    split at the carry, and the chains on either side against the oracle (the kernel matrix's standard)."""
    _env(monkeypatch, case)
    Q = _qref(case)
    P = _problem(case, Q)
    rows = np.arange(Q)
    a = Q // 2 + 1
    chain0 = (1 << 32) - a
    ctx = _ctx(1)
    ref, g = P.run(ctx, rows, chain0)
    for lo, hi in ((0, a), (a, Q)):
        out, gv = P.run(ctx, rows[lo:hi], chain0 + lo)
        assert _shape(gv) != _shape(g) or (g['pos'][lo:hi, :3] != gv['pos'][:, :3]).any()
        _same(ref, out, rows[lo:hi], np.arange(hi - lo), _where(g, gv))
    if case.sampler == 'friends':
        return              # (no oracle of the friends draws at a likelihood threshold; the shards above still apply)
    for q in (a - 2, a - 1, a, a + 1):
        r = P.oracle(q, chain0 + q)
        for k in ('n_accept', 'n_reject', 'ncall', 'n_expand', 'n_contract', 'nprop'):
            if k in ref and k in r:
                assert ref[k][q] == r[k], (q, k)
        close(ref['u'][q], r['u'], rtol=RTOL)
        close(ref['v'][q], r['v'], rtol=RTOL)
        assert ref['logl'][q] == pytest.approx(r['logl'], rel=RTOL, abs=RTOL)


# ---- B. device-resident rounds -------------------------------------------------------------------------------------------
ROUNDS = [(6, 'rwalk', 'shell', 'warp'), (20, 'rwalk', 'shell', 'mma'), (50, 'rwalk', 'prec', 'ws'),
          (80, 'rwalk', 'shell', 'mmas'), (6, 'rslice', 'shell', 'slice')]


def _rounds(monkeypatch, pack, n, sampler, kind, env):
    """One device run in a context with chain pack `pack`: 1 round (traced), 40 rounds, a device bound update,
    1 round, 40 rounds (the pattern of test_gpu_kernel_matrix._switch_run).  Returns what it left."""
    from dynesty_b200 import _lib, ops
    for k in RWALK_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    ctx = _lib.Context(0)
    if pack != 1:
        ctx.set_chain_pack(pack)
    om = OL.shells(n) if kind == 'shell' else OL.gauss_corr(n, 0.4, 5.)
    dm = device_model(om)
    N, K = (400, 8) if n <= 6 else (1000, 10)
    steps = 10 if sampler == 'rwalk' else 3
    rng = np.random.default_rng(n)
    if kind == 'shell':
        u = 0.5 + 0.03 * rng.standard_normal((N, n))
        u[: N // 2, 0] -= 3.5 / 12
        u[N // 2:, 0] += 3.5 / 12
    else:
        Cm = np.full((n, n), 0.4)
        np.fill_diagonal(Cm, 1.0)
        u = 0.5 + 0.03 * rng.standard_normal((N, n)) @ np.linalg.cholesky(Cm).T
        u[: N // 2, 0] -= 0.15
        u[N // 2:, 0] += 0.15
    v, l = om.prior_transform(u), om.loglike(om.prior_transform(u))
    b = _bound([u[: N // 2], u[N // 2: 3 * N // 4], u[3 * N // 4:]], enlarge=3.0 ** n)
    ops.bound_set(b['axes'], b['ctrs'], b['ams'], b['logvols'], ctx=ctx)
    ops.ns_create(dm.model_id(ctx), N, n, K, ('rwalk', 'rslice').index(sampler), steps, 9, chain0=3, dlogz=1e-9,
                  ctx=ctx)
    try:
        ops.ns_set_state(u, v, l, 0.0, -1e300, -1e300, 0, 0.3, ctx=ctx)
        sts = [ops.ns_run(1, 0, ctx=ctx), ops.ns_run(40, 0, ctx=ctx)]
        nells = ops.ns_update_bound(True, 2.0 ** n, ctx=ctx)
        ops.ns_bound_updated(ctx=ctx)
        sts += [ops.ns_run(1, 0, ctx=ctx), ops.ns_run(40, 0, ctx=ctx)]
        dead = ops.ns_get_dead(0, sts[-1]['it'], n, ctx=ctx)
        live = ops.ns_get_live(N, n, ctx=ctx)
    finally:
        ops.ns_destroy(ctx=ctx)
        ctx.close()
    return (sts, nells, dead, live), K


def _rounds_equal(a, b):
    assert a[0] == b[0] and a[1] == b[1]
    for x, y in zip(a[2] + a[3], b[2] + b[3]):
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()


@pytest.mark.parametrize('n,sampler,kind,fam', ROUNDS, ids=['%s%d-%s' % (s, n, f) for n, s, k, f in ROUNDS])
def test_rounds_chain_pack(monkeypatch, n, sampler, kind, fam):
    """b2n_ns_run builds its worklist on the device with the context's chains per CTA: chain pack 1, 4 and 8 give
    the same status dicts, dead and live arrays and bound update bit for bit; and so does B2N_NS_GRAPH=1 with pack 4
    (the graph key mixes the chain pack)."""
    sms, limit = _device()
    like = LIKE[kind] if kind != 'shell' else OL.LIKE_SHELLS
    runs, shapes = {}, {}
    for pack, env in ((1, {}), (4, {}), (8, {}), ('4g', dict(B2N_NS_GRAPH='1'))):
        k = 4 if pack == '4g' else pack
        res, K = _rounds(monkeypatch, k, n, sampler, kind, env)
        pl = _plan(fam, n, n, like, K, k, sms, limit)
        runs[pack], shapes[pack] = res, (pl['cpc'], pl['threads'])
    assert shapes[1] != shapes[4] != shapes[8] and shapes[1][0] == 1
    assert runs[1][0][1]['rounds'] == 41 and runs[1][1][0] != 3       # the bound update changed the ellipsoid count
    for pack in (4, 8, '4g'):
        _rounds_equal(runs[1], runs[pack])


# ---- C. whole runs ------------------------------------------------------------------------------------------------------
def test_nested_run_chain_pack():
    """NestedSampler(..., ctx).run_nested(loop='device') in a context with chain pack 4 == pack 1: every key of
    the results."""
    from dynesty_b200 import _lib, nested
    dm = device_model(OL.shells(4))
    res = {}
    for pack in (1, 4):
        ctx = _lib.Context(0)
        if pack != 1:
            ctx.set_chain_pack(pack)
        s = nested.NestedSampler(dm, nlive=300, bound='multi', sample='rwalk', walks=20, seed=77, ctx=ctx)
        res[pack] = s.run_nested(loop='device', dlogz=0.5, batch=16)
        ctx.close()
    a, b = res[1], res[4]
    assert set(a.keys()) == set(b.keys())
    for k in a.keys():
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), k


def test_replicas_chain_pack():
    """replicas.run_replicas with chain_pack=4 (the logZ ensemble's setting) == chain_pack=1 on 4 seeds."""
    from dynesty_b200 import replicas, likelihoods as DL
    m = DL.gauss_corr(8, 0.4, 5.0)
    kw = dict(nlive=300, bound='multi', sample='rwalk', sampler_kwargs=dict(walks=20), dlogz=0.5, batch=10,
              max_in_flight=4, keep_results=True)
    one, _ = replicas.run_replicas(m, [5, 6, 7, 8], chain_pack=1, **kw)
    four, _ = replicas.run_replicas(m, [5, 6, 7, 8], chain_pack=4, **kw)
    for a, b in zip(one, four):
        assert (a['seed'], a['niter'], a['ncall'], a['logz'], a['logzerr']) == \
            (b['seed'], b['niter'], b['ncall'], b['logz'], b['logzerr'])
        x, y = np.asarray(a['results']['logl']), np.asarray(b['results']['logl'])
        assert x.tobytes() == y.tobytes()

"""GPU: the stepped random walk (csrc/b2n_rwalk_step.cu: rwalk_step_kernel, driven by b2n_rwalk_step for host fills
and by b2n_ns_step / b2n_ns_rwalk_step for the device rounds) at the launch shapes, dimensions, likelihood edge values
and round limits where it changes form.

Two references:
* the fused kernel: a user CUDA model run by rwalk_batch (rwalk_kernel), and the same model wrapped as a TorchModel
  whose loglike is the model's own eval kernel (test_gpu_torch_model.wrap), give EQUAL bytes -- u, v, logl, n_accept,
  n_reject, ncall; at every new n the eval kernel is first shown to give the chain kernel's bits;
* the float64 oracle: oracle.samplers.rwalk_chain on the same Philox streams -- counts and the stream tick exact,
  u / v / logl to rtol 1e-9.

1. launch invariance: a chain's bytes, its tick and in_cube included, depend only on its start, ellipsoid, seed and
   chain id -- across shards, chain packs, longer queues (warps that walk >= 3 chains per launch), regrouped and
   unused ellipsoids, and chain ids across 2^32;
2. shapes: n from 1 to 129 across the lane passes and the 64-row bases of the mat-vec, ncdim < n across 32 / 64
   non-clustered dims, dimension flags, 1 and 2 walks, the warp-count edge of the shared-memory plan, the largest n
   the plan accepts and the first one it refuses;
3. likelihood edge values from torch: NaN, -inf and +inf regions and exact ties with loglstar; loglstar = -inf;
   chains that never accept; priors that return their input, a copy or a non-contiguous tensor;
4. device rounds: ns_run_stepped against b2n_ns_run on the same user model, block by block, at the shapes of
   test_gpu_ns_limits.py that apply, with stops that fire inside a block.

Every launch-shape case recomputes its geometry from a host mirror of b2n_rwalk_step_plan / b2n_chain_grid /
b2n_build_worklist -- warps per CTA, chains per CTA, chains per warp, CTAs -- and asserts that it differs from the
reference run's.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from dynesty_b200 import TorchModel, _lib, ops
from dynesty_b200.likelihoods import DeviceModel
from oracle import philox, samplers as OS
from test_gpu_kernel_matrix import _device
from test_gpu_launch_invariance import _cdiv, _raw, _worklist
from test_gpu_ns_limits import _ells
from test_gpu_nsloop import _bound
from test_gpu_torch_model import DIAG, _dev, wrap

pytestmark = pytest.mark.gpu

SEED = 31337
SCALE = 0.7
WALKS = 13
RTOL = 1e-9
CHAIN_KEYS = ('u', 'v', 'logl', 'n_accept', 'n_reject', 'ncall')
STATE_KEYS = CHAIN_KEYS + ('tick', 'in_cube')


# ---- host mirrors of the launch plan ----------------------------------------------------------------------------------
def _step_plan(n, Q, pack=1):
    """b2n_rwalk_step_plan + b2n_chain_grid: two npad-double vectors per warp, warps limited to what the opt-in shared
    memory holds; one CTA per SM up to 16 x SMs chains, two beyond.  None: the plan refuses n."""
    sms, optin = _device()
    npad = (n + 1) & ~1
    max_warps = min(16, optin // (16 * npad))
    if max_warps < 1:
        return None
    cpc = max(min(pack, 16), _cdiv(Q, sms if Q <= 16 * sms else 2 * sms))
    return dict(cpc=cpc, warps=max(1, min(max_warps, 16, cpc)), max_warps=max_warps)


def _geometry(n, Q, ell, K, pack=1):
    """The plan and where each chain runs: pos[q] = (CTA, warp, chains that warp walks before q, ellipsoid) -- the
    kernel's `for (c = warp; c < count; c += nwarps)`."""
    pl = _step_plan(n, Q, pack)
    w = pl['warps']
    order, cta = _worklist(np.zeros(Q, np.int32) if ell is None else np.asarray(ell), K, pl['cpc'])
    pos = np.empty((Q, 4), dtype=np.int64)
    for j, (lo, cnt, k) in enumerate(cta):
        off = np.arange(cnt)
        pos[order[lo:lo + cnt]] = np.stack([np.full(cnt, j), off % w, off // w, np.full(cnt, k)], 1)
    counts = [c for _, c, _ in cta]
    return dict(pl, K=K, ncta=len(cta), per_cta=max(counts), per_warp=max(_cdiv(c, w) for c in counts), pos=pos)


def _shape(g):
    """What a variant must change: warps per CTA, chains per CTA (planned, largest), chains per warp, CTAs, resident
    ellipsoids."""
    return tuple((k, g[k]) for k in ('warps', 'cpc', 'per_cta', 'per_warp', 'ncta', 'K'))


def _lanes(n, nc):
    """The kernel's lane-level form at (n, nc): npad, lane passes over n, 64-row bases of matvec2o, lane passes of the
    non-clustered uniforms, and whether ball_direction draws its normals in one Philox round (nb <= 31)."""
    return dict(npad=(n + 1) & ~1, passes=_cdiv(n, 32), bases=_cdiv(nc, 64), upasses=_cdiv(n - nc, 32),
                one_round=(nc + 1) // 2 <= 31)


# ---- models -------------------------------------------------------------------------------------------------------------
class NpModel:
    """The oracle's model interface over a numpy loglike of one point (identity prior); records every value."""

    def __init__(self, like):
        self.like, self.seen = like, []

    def prior_transform(self, u):
        return np.array(u, dtype=float)

    def loglike(self, v):
        l = float(self.like(v))
        self.seen.append(l)
        return l


def _diag(n, rng):
    """test_gpu_torch_model's diagonal Gaussian (user CUDA source DIAG, identity prior): (user model, numpy model,
    torch restatement).  The eval kernel's shared memory grows with n; past ~1800 dimensions only the torch
    restatement can run."""
    mean, ivar = 0.5 + 0.05 * rng.standard_normal(n), 1.0 / (0.05 + 0.1 * rng.random(n)) ** 2
    c = -0.5 * n * math.log(2 * math.pi) + 0.5 * np.log(ivar).sum()
    um = DeviceModel.from_cuda(n, DIAG, params=np.concatenate([mean, ivar, [c]]), name='user_diag') \
        if n <= 1800 else None
    om = NpModel(lambda v: -0.5 * np.sum(ivar * (v - mean) ** 2) + c)
    tm_mean, tm_ivar = torch.as_tensor(mean, device=_dev()), torch.as_tensor(ivar, device=_dev())
    tm = TorchModel(n, lambda v: -0.5 * torch.sum(tm_ivar * (v - tm_mean) ** 2, dim=1) + c, lambda u: u,
                    name='torch_diag')
    return um, om, tm


def _axes(K, nc, rng, s=0.03):
    """K random nc x nc ellipsoid axes of scale s (lower-triangular factors of random SPD matrices)."""
    out = []
    for _ in range(K):
        a = rng.standard_normal((nc, nc))
        out.append(s * np.linalg.cholesky(a @ a.T / nc + np.eye(nc)) / math.sqrt(2.0))
    return np.array(out)


def _starts(Q, n, nc, rng):
    """Start points near the centre in the clustered dims, uniform in the others (what a proposal draws there)."""
    u = np.clip(0.5 + 0.03 * rng.standard_normal((Q, n)), 0.02, 0.98)
    u[:, nc:] = rng.random((Q, n - nc))
    return u


# ---- fills ------------------------------------------------------------------------------------------------------------
def _stepped(tm, u0, loglstar, walks, chain0, ell=None, df=None, nc=None, ctx=None):
    """ops.rwalk_stepped, also returning the step state after the last launch: every chain's tick and in_cube."""
    ctx = ops._ctx(ctx)
    dev = tm.device(ctx)
    u0 = torch.as_tensor(u0, dtype=torch.float64, device=dev).contiguous()
    a, keep, Q, n = ops._chain_args(-1, u0, nc, loglstar, SCALE, SEED, chain0, ell, None)
    st, bufs = ops._step_state(Q, n, dev, df, worklist=True)
    o = dict(u=torch.empty((Q, n), dtype=torch.float64, device=dev),
             v=torch.empty((Q, n), dtype=torch.float64, device=dev), logl=torch.empty(Q, dtype=torch.float64, device=dev))
    for k in _lib.CHAIN_OUTPUTS['rwalk'][:3]:
        o[k] = torch.empty(Q, dtype=torch.int32, device=dev)
    args = ops._chain_ptrs(o, 'rwalk')
    with ops._torch_stream(ctx, dev):
        ops._step_through(tm, int(walks), lambda s: ctx.check(
            ctx.lib.b2n_rwalk_step(ctx.h, C.byref(a), int(walks), s, C.byref(st), *args)), st, u0, bufs['u_prop'])
        out = {k: t.cpu().numpy() for k, t in o.items()}
        out['tick'], out['in_cube'] = bufs['tick'].cpu().numpy(), bufs['in_cube'].cpu().numpy()
    return out


def _fused(um, u0, loglstar, walks, chain0, ell=None, df=None, nc=None, ctx=None):
    return ops.rwalk_batch(um.model_id(ctx), u0, loglstar, SCALE, walks, SEED, chain0=chain0, ncdim=nc, ell=ell,
                           dimflags=df, ctx=ctx)


def _equal(ref, var, rows_ref, rows_var, keys, where=None):
    """ref[k][rows_ref] == var[k][rows_var] byte for byte for every k; a failure names the first differing chain."""
    rows_ref, rows_var = np.asarray(rows_ref), np.asarray(rows_var)
    for k in keys:
        bad = np.flatnonzero((_raw(ref[k][rows_ref]) != _raw(var[k][rows_var])).any(axis=1))
        if bad.size:
            i = int(bad[0])
            raise AssertionError('%s differs at %d of %d chains; first: reference chain %d%s' % (
                k, bad.size, len(rows_ref), rows_ref[i], '' if where is None else ', ' + where(rows_ref[i], rows_var[i])))


def _where(ga, gb):
    f = lambda g, q: 'CTA %d warp %d pass %d ellipsoid %d' % tuple(g['pos'][q])
    return lambda qa, qb: 'reference %s, variant %s' % (f(ga, qa), f(gb, qb))


def _eval_matches_chain(um, f):
    """The eval kernel gives the chain kernel's bits for the same v (else the fused comparison could not be exact)."""
    _, le = um.evaluate(f['v'])
    assert le.tobytes() == f['logl'].tobytes()


def _logl_close(a, b):
    if np.isfinite(b):
        assert abs(a - b) <= RTOL * max(1.0, abs(b)), (a, b)
    else:
        assert (np.isnan(a) and np.isnan(b)) or a == b, (a, b)


def _oracle(out, q, u0, loglstar, axes, chain, om, walks, per=None, ref=None, df=None):
    """Chain q of a stepped fill against the float64 oracle on ChainStream(SEED, chain)."""
    r = OS.rwalk_chain(u0[q], loglstar, axes, SCALE, om, philox.ChainStream(SEED, chain), walks,
                       periodic=per, reflective=ref, nonbounded=None if df is None else (df == 0))
    assert (out['n_accept'][q], out['n_reject'][q], out['ncall'][q]) == (r['n_accept'], r['n_reject'], r['ncall']), q
    if 'tick' in out:
        assert int(out['tick'][q]) == r['ticks'], q
    for k in ('u', 'v'):
        np.testing.assert_allclose(out[k][q], r[k], rtol=RTOL, atol=RTOL * max(1.0, np.abs(r[k]).max()))
    _logl_close(out['logl'][q], r['logl'])
    return r


# ---- 1. launch invariance ---------------------------------------------------------------------------------------------
class Problem:
    """The reference problem of section 1: 12 dimensions, 9 clustered, one periodic and one reflective dim, K = 3
    ellipsoids, a pool of starts and ellipsoid indices (the first Q make a queue)."""
    n, nc, K = 12, 9, 3

    def __init__(self, Q):
        rng = np.random.default_rng(12)
        self.Q = Q
        self.um, self.om, _ = _diag(self.n, rng)
        self.tm = wrap(self.um)
        self.per, self.ref = [0], [1]
        self.df = ops.dimflags_from(self.n, self.per, self.ref)
        self.axes = _axes(self.K, self.nc, rng)
        self.u0 = _starts(Q, self.n, self.nc, rng)
        self.ell = rng.integers(self.K, size=Q).astype(np.int32)
        _, l = self.um.evaluate(_starts(4000, self.n, self.nc, rng))
        self.loglstar = float(np.quantile(l, 0.3))

    def run(self, ctx, rows, chain0, ell=None, axes=None, pack=1):
        axes = self.axes if axes is None else axes
        ell = self.ell[rows] if ell is None else ell
        ops.bound_set(axes, ctx=ctx)
        out = _stepped(self.tm, self.u0[rows], self.loglstar, WALKS, chain0, ell=ell, df=self.df, nc=self.nc, ctx=ctx)
        return out, _geometry(self.n, len(rows), ell, len(axes), pack)

    def oracle(self, out, q, chain):
        """Chain q of `out`, started from u0[q] on ellipsoid ell[q] with id `chain`, against the oracle."""
        _oracle(out, q, self.u0, self.loglstar, self.axes[self.ell[q]], chain, self.om, WALKS, self.per, self.ref,
                self.df)


_P = {}
_CTX = {}


def _problem():
    """The pool of the longest queue of section 1 (100 x SMs + 7 chains), made once."""
    if 'p' not in _P:
        _P['p'] = Problem(100 * _device()[0] + 7)
    return _P['p']


def _ctx(pack):
    """A context of its own per chain pack (b2n_set_chain_pack), made once per session."""
    if pack not in _CTX:
        c = _lib.Context(0)
        if pack != 1:
            c.set_chain_pack(pack)
        _CTX[pack] = c
    return _CTX[pack]


def _qref():
    return 20 * _device()[0] + 3


def _reference():
    """The reference run (Q = 20 x SMs + 3 chains, pack 1), checked against the fused kernel and, on a sample of
    chains, against the oracle."""
    P = _problem()
    if 'ref' not in _P:
        Q = _qref()
        rows = np.arange(Q)
        ref, g = P.run(_ctx(1), rows, 1000)
        f = _fused(P.um, P.u0[:Q], P.loglstar, WALKS, 1000, ell=P.ell[:Q], df=P.df, nc=P.nc, ctx=_ctx(1))
        _eval_matches_chain(P.um, f)
        _equal(f, ref, rows, rows, CHAIN_KEYS, _where(g, g))
        for q in (0, 1, Q // 2, Q - 1):
            P.oracle(ref, q, 1000 + q)
        _P['ref'], _P['ref_g'] = ref, g
    return P, _P['ref'], _P['ref_g']


def _ref_geometry():
    """The reference run's geometry, from the mirror alone."""
    P = _problem()
    return _geometry(P.n, _qref(), P.ell[:_qref()], P.K)


def _cuts(g, Q):
    """Shard cuts a (chains [0, a) and [a, Q)): one chain; inside a CTA (a - 1 and a share it); at a CTA boundary (a
    opens a CTA, a - 1 closes the one before); a first shard under 16 x SMs while the whole queue is over it."""
    pos, sms = g['pos'], _device()[0]
    cuts = {'one-chain': 1}
    same = [a for a in range(2, Q) if pos[a - 1][0] == pos[a][0]]
    cuts['in-cta'] = same[len(same) // 2]
    first = {j: int(np.flatnonzero(pos[:, 0] == j).min()) for j in np.unique(pos[:, 0])}
    last = {j: int(np.flatnonzero(pos[:, 0] == j).max()) for j in np.unique(pos[:, 0])}
    bnd = [a for a in range(1, Q) if pos[a][0] != pos[a - 1][0] and first[pos[a][0]] == a
           and last[pos[a - 1][0]] == a - 1]
    cuts['cta-boundary'] = bnd[len(bnd) // 2]
    cuts['under-16-per-sm'] = 16 * sms - 5
    return cuts


@pytest.mark.parametrize('cut', ['one-chain', 'in-cta', 'cta-boundary', 'under-16-per-sm'])
def test_shards(cut):
    P, ref, g = _reference()
    Q, sms = len(ref['u']), _device()[0]
    a = _cuts(g, Q)[cut]
    rows = np.arange(Q)
    assert Q > 16 * sms and g['cpc'] == _cdiv(Q, 2 * sms)      # the whole queue: two CTAs per SM
    if cut == 'in-cta':
        assert g['pos'][a - 1][0] == g['pos'][a][0]
    if cut == 'cta-boundary':
        assert g['pos'][a - 1][0] != g['pos'][a][0]
    if cut == 'under-16-per-sm':
        assert a <= 16 * sms < Q
    seen = False
    for lo, hi in ((0, a), (a, Q)):
        out, gv = P.run(_ctx(1), rows[lo:hi], 1000 + lo)
        _equal(ref, out, rows[lo:hi], np.arange(hi - lo), STATE_KEYS, _where(g, gv))
        seen = seen or _shape(gv) != _shape(g)
    assert seen, (cut, a, _shape(g))
    if cut == 'under-16-per-sm':                              # the short shard: one CTA per SM, 16 chains each
        assert _geometry(P.n, a, P.ell[:a], P.K)['cpc'] == _cdiv(a, sms) == 16


@pytest.mark.parametrize('pack', [3, 8, 9, 16, 17])
def test_chain_pack(pack):
    """Q = SMs - 5 chains: one per CTA at pack 1; b2n_set_chain_pack(k) puts min(k, 16) in a CTA, one warp each."""
    P, _, _ = _reference()
    Q = _device()[0] - 5
    rows = np.arange(Q)
    ref, g = P.run(_ctx(1), rows, 7)
    assert g['cpc'] == 1 and g['warps'] == 1
    out, gv = P.run(_ctx(pack), rows, 7, pack=pack)
    assert gv['cpc'] == gv['warps'] == min(pack, 16) and _shape(gv) != _shape(g)
    _equal(ref, out, rows, rows, STATE_KEYS, _where(g, gv))


def test_longer_queue_three_chains_per_warp():
    """The reference chains at the head of a queue of 100 x SMs + 7 chains: 51 chains per CTA, so that every
    warp walks three or four chains per launch -- and reuses its shared-memory slots and the chain's worklist entry
    at every later step."""
    P, ref, g = _reference()
    Ql = P.Q
    out, gv = P.run(_ctx(1), np.arange(Ql), 1000)
    assert g['per_warp'] == 1 and gv['warps'] == 16 and gv['per_warp'] >= 3 and _shape(gv) != _shape(g)
    Q = len(ref['u'])
    assert (gv['pos'][:Q, 2] >= 2).any()                    # reference chains walked third (or later) by their warp
    _equal(ref, out, np.arange(Q), np.arange(Q), STATE_KEYS, _where(g, gv))


def test_regrouping():
    """(a) the odd chains move to other ellipsoids, so the even ones sit in other CTAs and warps; (b) 40 ellipsoids
    resident, the three used ones at 5, 17 and 33."""
    P, ref, g = _reference()
    Q = len(ref['u'])
    rows = np.arange(Q)
    keep = rows[rows % 2 == 0]
    ell2 = P.ell[:Q].copy()
    ell2[1::2] = (ell2[1::2] + 1) % P.K
    out, gv = P.run(_ctx(1), rows, 1000, ell=ell2)
    assert (g['pos'][keep, :3] != gv['pos'][keep, :3]).any(axis=1).mean() > 0.5
    _equal(ref, out, keep, keep, STATE_KEYS, _where(g, gv))
    used = np.array([5, 17, 33])
    extra = _axes(40, P.nc, np.random.default_rng(40), s=0.05)
    extra[used] = P.axes
    out, gv = P.run(_ctx(1), rows, 1000, ell=used[P.ell[:Q]].astype(np.int32), axes=extra)
    assert np.array_equal(gv['pos'][:, 3], used[g['pos'][:, 3]]) and _shape(gv) != _shape(g)
    _equal(ref, out, rows, rows, STATE_KEYS, _where(g, gv))


def test_chain_ids_across_2_32():
    """chain0 = 2^32 - a: the whole queue against the two shards split at the carry, and the four chains around it
    against the oracle (counter words 2 and 3 of the Philox counter)."""
    P, _, _ = _reference()
    Q = _qref()
    rows = np.arange(Q)
    a = Q // 2 + 1
    chain0 = (1 << 32) - a
    ref, g = P.run(_ctx(1), rows, chain0)
    for lo, hi in ((0, a), (a, Q)):
        out, gv = P.run(_ctx(1), rows[lo:hi], chain0 + lo)
        assert _shape(gv) != _shape(g)
        _equal(ref, out, rows[lo:hi], np.arange(hi - lo), STATE_KEYS, _where(g, gv))
    for q in (a - 2, a - 1, a, a + 1):
        P.oracle(ref, q, chain0 + q)


def test_harness_catches_a_broken_fill():
    """The byte comparison fails on a fill whose chain ids are off by one, and on a likelihood one ulp off at one
    chain -- there, at that chain's logl only."""
    P, ref, g = _reference()
    Q = 2 * _device()[0] + 1
    rows = np.arange(Q)
    ops.bound_set(P.axes, ctx=_ctx(1))
    good = _stepped(P.tm, P.u0[:Q], P.loglstar, WALKS, 1000, ell=P.ell[:Q], df=P.df, nc=P.nc, ctx=_ctx(1))
    _equal(ref, good, rows, rows, STATE_KEYS)
    off = _stepped(P.tm, P.u0[:Q], P.loglstar, WALKS, 1001, ell=P.ell[:Q], df=P.df, nc=P.nc, ctx=_ctx(1))
    with pytest.raises(AssertionError):
        _equal(ref, off, rows, rows, CHAIN_KEYS)
    q = Q // 3
    base = P.tm.loglike

    def nudged(v):
        l = base(v).clone()
        l[q] = torch.nextafter(l[q], torch.tensor(math.inf, dtype=torch.float64, device=l.device))
        return l
    bad = _stepped(TorchModel(P.n, nudged, lambda u: u), P.u0[:Q], P.loglstar, WALKS, 1000, ell=P.ell[:Q], df=P.df,
                   nc=P.nc, ctx=_ctx(1))
    with pytest.raises(AssertionError, match='logl differs at 1 of %d chains; first: reference chain %d' % (Q, q)):
        _equal(ref, bad, rows, rows, CHAIN_KEYS)
    others = rows[rows != q]
    _equal(ref, bad, others, others, STATE_KEYS)


# ---- 2. shapes ----------------------------------------------------------------------------------------------------------
# (id, n, ncdim, flags, walks)
SHAPES = [('n%d' % n, n, n, None, WALKS) for n in (1, 2, 31, 33, 63, 64, 65, 128, 129)] + [
    ('n34-nc3', 34, 3, None, WALKS),          # n - nc = 31
    ('n40-nc8', 40, 8, None, WALKS),          # 32
    ('n96-nc63', 96, 63, None, WALKS),        # 33
    ('n100-nc36', 100, 36, None, WALKS),      # 64
    ('n130-nc65', 130, 65, None, WALKS),      # 65, two 64-row bases
    ('n12-per', 12, 12, 'per', WALKS),
    ('n40-nc30-ref', 40, 30, 'ref', WALKS),
    ('n65-both', 65, 65, 'both', WALKS),
    ('n10-walks1', 10, 10, None, 1),
    ('n33-nc20-walks2', 33, 20, None, 2),
]


def _flags(n, kind):
    per = [0, n - 1] if kind in ('per', 'both') else None
    ref = [min(1, n - 1)] if kind in ('ref', 'both') else None
    if per is not None and ref is not None:
        ref = [1, n // 2]
    return per, ref, ops.dimflags_from(n, per, ref)


def _shape_case(n, nc, kind, walks, Q, K=2, seed=0, check=8):
    """A fill at (n, nc): fused == stepped byte for byte, and `check` chains (the first, the last, a sample) against
    the oracle.  Returns (stepped outputs, geometry)."""
    rng = np.random.default_rng(seed + 1000 * n + nc)
    um, om, _ = _diag(n, rng)
    tm = wrap(um)
    per, ref, df = _flags(n, kind)
    axes = _axes(K, nc, rng)
    u0 = _starts(Q, n, nc, rng)
    ell = rng.integers(K, size=Q).astype(np.int32)
    _, l = um.evaluate(_starts(2000, n, nc, rng))
    loglstar = float(np.quantile(l, 0.3))
    ctx = _ctx(1)
    ops.bound_set(axes, ctx=ctx)
    f = _fused(um, u0, loglstar, walks, 50 + n, ell=ell, df=df, nc=nc, ctx=ctx)
    _eval_matches_chain(um, f)
    s = _stepped(tm, u0, loglstar, walks, 50 + n, ell=ell, df=df, nc=nc, ctx=ctx)
    g = _geometry(n, Q, ell, K)
    _equal(f, s, np.arange(Q), np.arange(Q), CHAIN_KEYS, _where(g, g))
    assert 0 < s['n_accept'].sum() < walks * Q                   # both branches of the accept half ran
    assert _shape(g) != _shape(_ref_geometry())
    for q in sorted({0, Q - 1} | set(rng.choice(Q, size=check, replace=False).tolist())):
        _oracle(s, q, u0, loglstar, axes[ell[q]], 50 + n + q, om, walks, per, ref, df)
    return s, g


@pytest.mark.parametrize('cid,n,nc,kind,walks', SHAPES, ids=[c[0] for c in SHAPES])
def test_shapes(cid, n, nc, kind, walks):
    """Q = 40 x SMs + 1 chains: 21 per CTA, so every CTA has warps that walk a second chain."""
    sms = _device()[0]
    Q = 40 * sms + 1
    s, g = _shape_case(n, nc, kind, walks, Q)
    assert g['warps'] == 16 and g['per_warp'] == 2 and (g['pos'][:, 2] == 1).any()
    lanes, ref = _lanes(n, nc), _lanes(Problem.n, Problem.nc)
    assert lanes != ref
    if n in (1, 2):
        assert lanes['npad'] == 2 and lanes['passes'] == 1
    if nc in (65, 128, 129):
        assert lanes['bases'] >= 2 and not lanes['one_round']
    if n - nc in (33, 64, 65):
        assert lanes['upasses'] >= 2


def _warp_edge():
    """(largest n that gets 16 warps, the next n): 16 warps x 2 x npad doubles fit in the opt-in shared memory."""
    _, optin = _device()
    npad = (optin // (16 * 16)) & ~1
    return npad, npad + 1


@pytest.mark.parametrize('side', ['last-16-warps', 'first-15-warps'])
def test_warp_limit_edge(side):
    """ncdim = 2 and a tiny bound: the shared memory of the stepped kernel depends on n only.  Q = 16 x SMs: one CTA
    per SM with 16 chains, walked by 16 warps on one side of the edge and by 15 on the other, one warp taking two."""
    sms = _device()[0]
    n16, n15 = _warp_edge()
    n = n16 if side == 'last-16-warps' else n15
    Q = 16 * sms
    pl = _step_plan(n, Q)
    assert pl['max_warps'] == (16 if n == n16 else 15)
    s, g = _shape_case(n, 2, None, 5, Q, check=3)
    if n == n16:
        assert g['warps'] == 16 and g['per_warp'] == 1
    else:
        assert g['warps'] == 15 and g['per_warp'] == 2 and g['per_cta'] == 16
        assert (g['pos'][:, 2] == 1).any()                      # chains their warp walks second


def _n_limit():
    """The largest n the plan accepts: one warp's two npad-double vectors fill the opt-in shared memory."""
    _, optin = _device()
    return (optin // 16) & ~1


def test_largest_n_against_the_oracle():
    """The largest n of the plan (one warp per CTA), with the torch restatement (the eval kernel has no room for a
    point at that n), against the float64 oracle on a few chains."""
    n = _n_limit()
    assert _step_plan(n, 6)['max_warps'] == 1 and _step_plan(n + 1, 6) is None
    rng = np.random.default_rng(n)
    _, om, tm = _diag(n, rng)
    Q, nc, walks = 6, 2, 5
    axes = _axes(2, nc, rng)
    u0 = _starts(Q, n, nc, rng)
    ell = (np.arange(Q) % 2).astype(np.int32)
    loglstar = float(np.quantile([om.like(x) for x in _starts(40, n, nc, rng)], 0.5))
    ctx = _ctx(1)
    ops.bound_set(axes, ctx=ctx)
    g = _geometry(n, Q, ell, 2)
    assert (g['warps'], g['per_warp'], g['ncta']) == (1, 1, Q) and _shape(g) != _shape(_ref_geometry())
    s = _stepped(tm, u0, loglstar, walks, 3, ell=ell, nc=nc, ctx=ctx)
    for q in range(Q):
        _oracle(s, q, u0, loglstar, axes[ell[q]], 3 + q, om, walks)
    assert 0 < s['n_accept'].sum() < walks * Q


def test_past_the_largest_n_refuses():
    """One n past the limit: the host fill and the device rounds refuse with 'ndim too large' before any launch."""
    n = _n_limit() + 1
    assert _step_plan(n, 4) is None
    tm = TorchModel(n, lambda v: torch.zeros(v.shape[0], dtype=torch.float64, device=v.device), lambda u: u)
    ctx = _lib.Context(0)
    try:
        ops.bound_set(0.01 * np.eye(2)[None], np.full((1, 2), 0.5), 1e4 * np.eye(2)[None],
                      np.array([math.log(math.pi * 1e-4)]), ctx=ctx)
        n0 = ctx.launch_count()
        with pytest.raises(NotImplementedError, match='ndim too large for the stepped rwalk kernel'):
            _stepped(tm, np.full((4, n), 0.5), -1e300, 3, 0, nc=2, ctx=ctx)
        assert ctx.launch_count() == n0
        N = 8
        u = np.full((N, n), 0.5)
        ops.ns_create(-1, N, n, 2, 0, 3, SEED, ncdim=2, ctx=ctx)
        try:
            ops.ns_set_state(u, u, np.zeros(N), 0.0, -1e300, -1e300, N, 1.0, ctx=ctx)
            n0 = ctx.launch_count()
            with pytest.raises(NotImplementedError, match='ndim too large for the stepped rwalk kernel'):
                ops.ns_run_stepped(tm, 2, ctx=ctx)
            assert ctx.launch_count() == n0
        finally:
            ops.ns_destroy(ctx=ctx)
    finally:
        ctx.close()


# ---- 3. likelihood edge values ----------------------------------------------------------------------------------------
# -inf for v0 < p0, NaN for v0 > p1, +inf within sqrt(p2) of the centre, else -|v - 0.5|^2 quantised to steps 1 / p3
EDGE = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    double s = 0.0;
    for (int i = lane; i < n; i += 32) {
        const double d = v[i] - 0.5;
        s = fma(d, d, s);
    }
    s = b2n_warp_sum(s);
    if (v[0] < p[0]) return __longlong_as_double(0xfff0000000000000ULL);
    if (v[0] > p[1]) return __longlong_as_double(0x7ff8000000000000ULL);
    if (s < p[2]) return __longlong_as_double(0x7ff0000000000000ULL);
    return floor(-p[3] * s) / p[3];
}
'''
EDGE_P = (0.44, 0.56, 0.03 ** 2, 200.0)


def _edge_np(v):
    s = float(np.sum((v - 0.5) ** 2))
    if v[0] < EDGE_P[0]:
        return -np.inf
    if v[0] > EDGE_P[1]:
        return np.nan
    if s < EDGE_P[2]:
        return np.inf
    return math.floor(-EDGE_P[3] * s) / EDGE_P[3]


_EDGE = {}


def _edge_problem():
    """n = 5: 256 chains, a tenth starting in the +inf ball, the rest between the -inf and NaN slabs."""
    if not _EDGE:
        n, Q = 5, 256
        rng = np.random.default_rng(5)
        um = DeviceModel.from_cuda(n, EDGE, params=list(EDGE_P), name='user_edges')
        u0 = np.clip(0.5 + 0.04 * rng.standard_normal((Q, n)), 0.0, 1.0)
        u0[:, 0] = 0.5 + 0.05 * (2 * rng.random(Q) - 1)
        u0[::10] = 0.5 + 0.004 * rng.standard_normal((len(u0[::10]), n))
        _, l = um.evaluate(u0)
        assert np.isposinf(l[::10]).all() and np.isfinite(l).sum() > Q // 2
        fin = l[np.isfinite(l)]
        _EDGE.update(um=um, u0=u0, n=n, Q=Q, axes=np.array([0.04 * np.eye(n), 0.025 * np.eye(n)]),
                     ell=(np.arange(Q) % 2).astype(np.int32), level=float(np.sort(fin)[len(fin) // 2]))
    return _EDGE


@pytest.mark.parametrize('lstar', ['level', '-inf', 'above-every-level'])
def test_edge_values(lstar):
    """stepped == fused byte for byte; every chain against the oracle (counts exact); the oracle saw NaN, -inf and
    +inf proposals and, at a quantised level, exact ties (which must reject: the test is strict >); chains that never
    accepted return their start's (u, v, logl)."""
    E = _edge_problem()
    um, u0, Q, n = E['um'], E['u0'], E['Q'], E['n']
    loglstar = {'level': E['level'], '-inf': -math.inf, 'above-every-level': 1e300}[lstar]
    ctx = _ctx(1)
    ops.bound_set(E['axes'], ctx=ctx)
    f = _fused(um, u0, loglstar, WALKS, 400, ell=E['ell'], ctx=ctx)
    _eval_matches_chain(um, f)
    s = _stepped(wrap(um), u0, loglstar, WALKS, 400, ell=E['ell'], ctx=ctx)
    _equal(f, s, np.arange(Q), np.arange(Q), CHAIN_KEYS)
    om = NpModel(_edge_np)
    for q in range(Q):
        _oracle(s, q, u0, loglstar, E['axes'][E['ell'][q]], 400 + q, om, WALKS)
    seen = np.array(om.seen)
    assert np.isnan(seen).any() and np.isneginf(seen).any() and np.isposinf(seen).any()
    if lstar == 'level':
        assert (seen == loglstar).sum() >= 10
    still = np.flatnonzero(s['n_accept'] == 0)
    if lstar != '-inf':                                           # (at -inf every finite proposal is accepted)
        assert still.size > (Q // 2 if lstar == 'above-every-level' else 0)
    _, l0 = um.evaluate(u0[still])
    assert s['u'][still].tobytes() == u0[still].tobytes() and s['v'][still].tobytes() == u0[still].tobytes()
    assert s['logl'][still].tobytes() == l0.tobytes()
    if lstar == '-inf':                                           # everything finite or +inf is accepted
        assert np.isfinite(s['logl']).sum() + np.isposinf(s['logl']).sum() == Q
    if lstar == 'above-every-level':                              # only the +inf ball accepts
        assert np.isposinf(s['logl'][s['n_accept'] > 0]).all()


def test_prior_returning_its_input_a_copy_or_a_strided_view():
    """v_prop may BE u_prop (an identity prior that returns its input): the same bytes as a prior that returns
    u.clone() and as one that returns a non-contiguous tensor of the same values."""
    E = _edge_problem()
    um, u0, Q = E['um'], E['u0'], E['Q']
    base = wrap(um)
    strided = lambda u: u.t().contiguous().t()
    probe = torch.rand((7, E['n']), dtype=torch.float64, device=_dev())
    assert strided(probe).data_ptr() != probe.data_ptr() and not strided(probe).is_contiguous()
    ctx = _ctx(1)
    ops.bound_set(E['axes'], ctx=ctx)
    outs = {}
    for name, prior in (('input', lambda u: u), ('clone', lambda u: u.clone()), ('strided', strided)):
        tm = TorchModel(E['n'], base.loglike, prior, name='edges_' + name)
        outs[name] = _stepped(tm, u0, E['level'], WALKS, 400, ell=E['ell'], ctx=ctx)
    assert 0 < outs['input']['n_accept'].sum()
    for name in ('clone', 'strided'):
        _equal(outs['input'], outs[name], np.arange(Q), np.arange(Q), STATE_KEYS)


# ---- 4. device rounds ---------------------------------------------------------------------------------------------------
def _snapshot(ctx, N, n, it):
    du, dv, dl, dlv, dnc = ops.ns_get_dead(0, it, n, ctx=ctx)
    slot, dit = ops.ns_get_strands(0, it, ctx=ctx)
    lu, lv, ll = ops.ns_get_live(N, n, ctx=ctx)
    return [du, dv, dl, dlv, dnc, slot, dit, ops.ns_get_live_it(N, ctx=ctx), lu, lv, ll]


def _same_snapshot(a, b):
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), i


def _block(fn, ctx):
    """A block of rounds; a run that stops with an error status gives the status it left."""
    try:
        return fn()
    except RuntimeError:
        return ops.ns_status(ctx=ctx)


def _fixed_bound(u, kell, rng):
    """A bound that holds every point the rounds will start from: ellipsoid 0 bounds the live set, enlarged 3x in
    every direction; kell > 1 adds test_gpu_ns_limits' ellipsoids on random subsets, with log-volume weights spread
    so that some of them receive no chain.  Fixed for the whole run, so that the rounds do not depend on the blocks
    they are issued in."""
    big = _bound([u], enlarge=3.0 ** u.shape[1])
    if kell == 1:
        return big
    b = _ells(u, kell, rng)
    for k in ('ctrs', 'ams', 'axes'):
        b[k][0] = big[k][0]
    return b


# (id, model, n, ncdim, flags, N, K, walks, kell, pack, threads, stop, blocks of rounds; None: around the stop)
ROUNDS = [
    ('k1100', 'diag', 3, 3, None, 1400, 1100, 2, 1, 1, None, None, [1, 1, 1]),
    ('threads256', 'diag', 4, 4, None, 700, 300, 3, 1, 1, '256', None, [1, 2, 2]),
    ('threads512', 'diag', 4, 4, None, 1500, 600, 2, 1, 1, '512', None, [1, 2]),
    ('multi-ell', 'diag', 3, 3, None, 400, 90, 3, 6, 1, None, None, [1, 2, 2]),
    ('ties', 'quant', 3, 3, None, 256, 32, 3, 1, 1, None, None, [1, 2, 3, 3]),
    ('ncdim-flags', 'diag', 8, 5, 'both', 300, 40, 4, 1, 1, None, None, [1, 3, 3]),
    ('pack4', 'diag', 6, 6, None, 300, 100, 3, 3, 4, None, None, [1, 3]),
    ('pack8', 'diag', 6, 6, None, 300, 100, 3, 3, 8, None, None, [1, 3]),
    ('maxiter', 'diag', 3, 3, None, 200, 30, 2, 1, 1, None, 'maxiter', None),
    ('maxcall', 'diag', 3, 3, None, 200, 30, 2, 1, 1, None, 'maxcall', None),
    ('dlogz', 'diag', 3, 3, None, 200, 30, 2, 1, 1, None, 'dlogz', None),
    ('long-block', 'diag', 3, 3, None, 200, 30, 2, 1, 1, None, 'dlogz', [400]),
]


@pytest.mark.parametrize('cid,model,n,nc,flags,N,K,walks,kell,pack,threads,stop,blocks', ROUNDS,
                         ids=[r[0] for r in ROUNDS])
def test_device_rounds(monkeypatch, cid, model, n, nc, flags, N, K, walks, kell, pack, threads, stop, blocks):
    """b2n_ns_run(user model), one round at a time in a context with chain pack 1, against ns_run_stepped(the
    wrapped model) in blocks of rounds in a context with chain pack `pack`: after every block the whole status dict
    equals the fused run's after the same round; at the end the dead rows, strands, live-slot counters and live set
    are equal byte for byte.  A stop fires in the second round of a block (blocks=None: the blocks are cut around the
    round the fused run stopped in), or inside one block of 400 rounds; the launches the stop skips -- the rest of
    the block and one more block -- change nothing."""
    monkeypatch.delenv('B2N_NS_THREADS', raising=False)
    if threads:
        monkeypatch.setenv('B2N_NS_THREADS', threads)
    rng = np.random.default_rng(N + K + n)
    if model == 'quant':
        # the edge model with its -inf / NaN / +inf regions off: -|v - 0.5|^2 in steps of 1 / 64
        um = DeviceModel.from_cuda(n, EDGE, params=[-1.0, 2.0, 0.0, 64.0], name='quantized_identity')
        u = rng.random((N, n))
    else:
        um, _, _ = _diag(n, rng)
        u = np.clip(0.5 + 0.05 * rng.standard_normal((N, n)), 0.01, 0.99)
    tm = wrap(um)
    _, l = um.evaluate(u)
    df = _flags(n, flags)[2] if flags else None
    limit = {'maxiter': dict(maxiter=100), 'maxcall': dict(maxcall=N + 5 * K * walks + 7), 'dlogz': dict(dlogz=0.5),
             None: dict(dlogz=0.0)}[stop]
    b = _fixed_bound(u[:, :nc], kell, rng)
    if pack != 1:
        assert _step_plan(n, K, pack)['cpc'] != _step_plan(n, K)['cpc']
    lstar = float(l.min()) - 0.5
    cf, cs = _lib.Context(0), _lib.Context(0)
    if pack != 1:
        cs.set_chain_pack(pack)
    try:
        for c, mid in ((cf, um.model_id(cf)), (cs, -1)):
            ops.bound_set(b['axes'], b['ctrs'], b['ams'], b['logvols'], ctx=c)
            ops.ns_create(mid, N, n, K, 0, walks, SEED, chain0=9, ncdim=nc, dimflags=df, ctx=c, **limit)
            ops.ns_set_state(u, u, l, -2.5, -40.0, lstar, N, SCALE, ctx=c)
        # the fused run, one round at a time: fused[r] is its status after round r
        fused = [None]
        cap = 400 if stop else sum(blocks)
        while len(fused) <= cap:
            st = _block(lambda: ops.ns_run(1, 0, ctx=cf), cf)
            fused.append(st)
            assert not st['need_bound'] and not st['error'], st
            if st['done']:
                break
        last = len(fused) - 1
        if stop:
            assert fused[last]['done'] and last >= 3, last
        if blocks is None:
            blocks = [last - 2, 6]
        end = 0
        for R in blocks:
            s = _block(lambda: ops.ns_run_stepped(tm, R, ctx=cs), cs)
            end = min(end + R, last)
            assert s == fused[end], (R, end, s, fused[end])
        if stop:
            start = sum(blocks[:-1])
            assert end == last and start < last < start + blocks[-1]   # inside the last block, before its end
            snap = _snapshot(cs, N, n, s['it'])
            assert ops.ns_run_stepped(tm, 5, ctx=cs) == s             # a whole block of skipped launches
            _same_snapshot(snap, _snapshot(cs, N, n, s['it']))
        if stop == 'maxiter':
            assert s['it'] - K < 100 <= s['it']
        elif stop == 'maxcall':
            assert s['ncall'] >= N + 5 * K * walks + 7
        elif stop == 'dlogz':
            assert s['delta_logz'] < 0.5
        _same_snapshot(_snapshot(cf, N, n, s['it']), _snapshot(cs, N, n, s['it']))
        if model == 'quant':                                         # new points tie with survivors and each other
            dl = ops.ns_get_dead(0, s['it'], n, ctx=cf, positions=False)[2]
            assert len(np.unique(dl)) < len(dl) // 4
    finally:
        for c in (cf, cs):
            ops.ns_destroy(ctx=c)
            c.close()

"""GPU: TorchModel -- likelihoods written as batched PyTorch functions, run between the launches of the stepped
random walk (csrc/b2n_rwalk_step.cu).

* oracle parity: torch restatements of the diagonal Gaussian (normal-ppf prior), the precision-matrix Gaussian and
  the shell at n = 10 and 200, with ncdim < n and with periodic / reflective dims, against oracle.samplers.rwalk_chain
  on the same Philox streams: counts exact, u / v / logl to rtol 1e-9;
* bit identity with the fused kernel: a user CUDA model (identity prior) wrapped as a TorchModel, whose loglike is the
  model's own eval kernel, gives array_equal fills to rwalk_batch (B2N_RWALK_IMPL=warp), and array_equal whole runs
  (host loop, device rounds, dynamic sampler);
* evidence of likelihoods the registry lacks, written only in torch;
* no host round trip inside a fill or a block of rounds (torch.profiler).
"""
import math

import numpy as np
import pytest
import torch

from dynesty_b200 import TorchModel, _lib, dynamic, nested, ops
from dynesty_b200.likelihoods import DeviceModel
from oracle import bounding as OB, likelihoods as OL, philox, samplers as OS

pytestmark = pytest.mark.gpu

SEED = 56432
RTOL = 1e-9

DIAG = r'''
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
    double s = 0.0;
    for (int i = lane; i < n; i += 32) {
        const double d = v[i] - p[i];
        s = fma(p[n + i] * d, d, s);
    }
    s = b2n_warp_sum(s);
    return fma(-0.5, s, p[2 * n]);
}
'''


def close(a, b, rtol=RTOL):
    np.testing.assert_allclose(a, b, rtol=rtol, atol=rtol * max(np.abs(np.asarray(b)).max(), 1e-300))


def _dev():
    return torch.device('cuda', _lib.default_context().device)


# ---- torch restatements of the oracle models ---------------------------------------------------------------------
def torch_restatement(om):
    """A TorchModel computing what the oracle model computes."""
    p, n, dev = om.p, om.ndim, _dev()
    t = lambda a: torch.as_tensor(np.broadcast_to(np.asarray(a, dtype=float), (n,)).copy(), device=dev)
    if om.prior_kind == OL.PRIOR_UNIFORM:
        lo, wd = t(p['lo']), t(p['width'])
        prior = lambda u: lo + wd * u
    elif om.prior_kind == OL.PRIOR_NORMAL_PPF:
        mu, sg = t(p['mu']), t(p['sigma'])
        prior = lambda u: mu + sg * torch.special.ndtri(u)
    else:
        prior = lambda u: u
    if om.like_kind == OL.LIKE_GAUSS_DIAG:
        mean, ivar = t(p['mean']), t(p['ivar'])
        like = lambda v: -0.5 * torch.sum(ivar * (v - mean) ** 2, dim=1) + p['lnorm']
    elif om.like_kind == OL.LIKE_GAUSS_PREC:
        mean, prec = t(p['mean']), torch.as_tensor(np.asarray(p['prec'], dtype=float), device=dev)
        like = lambda v: -0.5 * torch.sum((v - mean) @ prec * (v - mean), dim=1) + p['lnorm']
    else:
        c1, c2 = t(p['c1']), t(p['c2'])
        r, w = p['r'], p['w']
        cst = math.log(1.0 / math.sqrt(2.0 * math.pi * w * w))

        def like(v):
            a = torch.sqrt(torch.sum((v - c1) ** 2, dim=1))
            b = torch.sqrt(torch.sum((v - c2) ** 2, dim=1))
            return torch.logaddexp(cst - (a - r) ** 2 / (2 * w * w), cst - (b - r) ** 2 / (2 * w * w))
    return TorchModel(n, like, prior, name='torch_%d' % om.like_kind)


_OM = {'diag': lambda n: OL.iid_normal_ppf(n), 'shell': lambda n: OL.shells(n),
       'prec': lambda n: OL.gauss_corr(n, 0.4, 5.)}


def _queue(kind, om, Q, nc, rng, K=2):
    n = om.ndim
    pts = 0.5 + 0.03 * rng.standard_normal((max(2000, 8 * K * n), n))
    if kind == 'shell':
        pts[:, 0] += (-1.5 / 12.0)
    logl = om.loglike(om.prior_transform(pts))
    loglstar = float(np.quantile(logl, 0.3))
    good = pts[logl > loglstar]
    ells = [OB.bounding_ellipsoid(good[i::K, :nc]) for i in range(K)]
    u0 = np.ascontiguousarray(good[rng.integers(len(good), size=Q)])
    return u0, loglstar, np.array([e.axes for e in ells]), rng.integers(K, size=Q).astype(np.int32)


@pytest.mark.parametrize('kind', ['diag', 'shell', 'prec'])
@pytest.mark.parametrize('n,ncdim,flags', [(10, 10, None), (10, 7, None), (10, 10, 'per'), (200, 200, None),
                                           (200, 150, 'ref')])
def test_stepped_fill_matches_oracle(kind, n, ncdim, flags):
    om = _OM[kind](n)
    tm = torch_restatement(om)
    rng = np.random.default_rng(7 * n + ncdim)
    Q = 301 if n == 10 else 40
    u0, loglstar, axes, ell = _queue(kind, om, Q, ncdim, rng)
    ops.bound_set(axes)
    per = [0, 3] if flags == 'per' else None
    ref = [1, 4] if flags == 'ref' else None
    df = ops.dimflags_from(n, per, ref)
    walks, scale, chain0 = 25, 0.6, 90 + n
    o = ops.rwalk_stepped(tm, u0, loglstar, scale, walks, SEED, chain0=chain0, ell=ell, dimflags=df, ncdim=ncdim)
    assert np.all(o['ncall'] == walks)
    for q in sorted({0, Q - 1} | set(rng.choice(Q, size=min(12, Q), replace=False).tolist())):
        r = OS.rwalk_chain(u0[q], loglstar, axes[ell[q]], scale, om, philox.ChainStream(SEED, chain0 + q), walks,
                           periodic=per, reflective=ref,
                           nonbounded=None if df is None else (df != 0))
        assert o['n_accept'][q] == r['n_accept'] and o['n_reject'][q] == r['n_reject'], q
        close(o['u'][q], r['u'])
        close(o['v'][q], r['v'])
        close(o['logl'][q], r['logl'])


# ---- the user CUDA model and its TorchModel wrapper ----------------------------------------------------------------
def _user_diag(n, rng):
    mean, ivar = 0.5 + 0.05 * rng.standard_normal(n), 1.0 / (0.05 + 0.1 * rng.random(n)) ** 2
    prm = np.concatenate([mean, ivar, [-0.5 * n * math.log(2 * math.pi) + 0.5 * np.log(ivar).sum()]])
    return DeviceModel.from_cuda(n, DIAG, params=prm, name='user_diag')


def wrap(um):
    """The user model as a TorchModel: identity prior, loglike = the model's eval kernel (b2n_model_eval) on the
    torch tensor, enqueued on torch's current stream."""
    ctx = _lib.default_context()
    dev = _dev()

    def loglike(v):
        out = torch.empty(v.shape[0], dtype=torch.float64, device=dev)
        v = v.contiguous()
        if ctx.mode == _lib.PTR_DEVICE:           # inside a stepped fill / block of rounds: already on torch's stream
            ctx.check(ctx.lib.b2n_model_eval(ctx.h, um.ids(ctx)[1], v.data_ptr(), v.shape[0], None, out.data_ptr()))
        else:
            with ops._torch_stream(ctx, dev):
                ctx.check(ctx.lib.b2n_model_eval(ctx.h, um.ids(ctx)[1], v.data_ptr(), v.shape[0], None,
                                                 out.data_ptr()))
        return out

    return TorchModel(um.ndim, loglike, lambda u: u, name='wrapped_' + um.name)


@pytest.mark.parametrize('n,ncdim,flags', [(10, 10, None), (10, 6, 'per'), (200, 200, None), (200, 160, 'ref')])
def test_stepped_fill_bit_identical_to_fused(monkeypatch, n, ncdim, flags):
    rng = np.random.default_rng(n + ncdim)
    um = _user_diag(n, rng)
    tm = wrap(um)
    Q = 301 if n == 10 else 40
    pts = 0.5 + 0.03 * rng.standard_normal((4000, n))
    _, l = um.evaluate(pts)
    loglstar = float(np.quantile(l, 0.3))
    good = pts[l > loglstar]
    axes = np.array([OB.bounding_ellipsoid(good[i::2, :ncdim]).axes for i in range(2)])
    u0 = np.ascontiguousarray(good[rng.integers(len(good), size=Q)])
    ell = rng.integers(2, size=Q).astype(np.int32)
    df = ops.dimflags_from(n, [0, 2] if flags == 'per' else None, [1, 3] if flags == 'ref' else None)
    ops.bound_set(axes)
    monkeypatch.setenv('B2N_RWALK_IMPL', 'warp')
    f = ops.rwalk_batch(um.model_id(), u0, loglstar, 0.7, 25, SEED, chain0=11, ncdim=ncdim, ell=ell, dimflags=df)
    monkeypatch.delenv('B2N_RWALK_IMPL')
    # the eval kernel gives the chain kernel's bits for the same v (else the comparison below could not be exact)
    _, le = um.evaluate(f['v'])
    assert np.array_equal(le, f['logl'])
    s = ops.rwalk_stepped(tm, u0, loglstar, 0.7, 25, SEED, chain0=11, ell=ell, dimflags=df, ncdim=ncdim)
    for k in ('u', 'v', 'logl', 'n_accept', 'n_reject', 'ncall'):
        assert np.array_equal(s[k], f[k]), k


def _results_equal(a, b):
    assert a['niter'] == b['niter'] and a['ncall'] == b['ncall']
    assert np.array_equal(a['logl'], b['logl']) and np.array_equal(a['logvol'], b['logvol'])
    assert a['logz'][-1] == b['logz'][-1]


@pytest.fixture(scope='module')
def pair():
    um = _user_diag(8, np.random.default_rng(3))
    return um, wrap(um)


def test_host_loop_run_bit_identical(pair):
    um, tm = pair
    kw = dict(nlive=200, bound='multi', sample='rwalk', seed=5, live_init='host')
    a = nested.NestedSampler(um, **kw).run_nested(dlogz=0.5, loop='host')
    b = nested.NestedSampler(tm, **kw).run_nested(dlogz=0.5, loop='host')
    _results_equal(a, b)


@pytest.mark.parametrize('maxcall', [None, 23000])     # 23000: the run stops partway through a block of rounds
def test_device_rounds_run_bit_identical(pair, maxcall):
    um, tm = pair
    kw = dict(nlive=200, bound='multi', sample='rwalk', seed=9, live_init='host')
    a = nested.NestedSampler(um, **kw).run_nested(dlogz=0.1, loop='device', device_init=False, maxcall=maxcall)
    b = nested.NestedSampler(tm, **kw).run_nested(dlogz=0.1, loop='device', maxcall=maxcall)
    _results_equal(a, b)


def test_dynamic_run_bit_identical(pair):
    um, tm = pair
    kw = dict(nlive=150, bound='multi', sample='rwalk', seed=4, live_init='host')
    a = dynamic.DynamicNestedSampler(um, device_init=False, **kw).run_nested(maxbatch=2, nlive_batch=100)
    b = dynamic.DynamicNestedSampler(tm, **kw).run_nested(maxbatch=2, nlive_batch=100)
    _results_equal(a, b)


# ---- evidence of likelihoods the registry lacks ------------------------------------------------------------------
def _mixture(n=10, h=10.0):
    """test_gpu_user_model.py's mixture: 0.3 N(m1, 1) + 0.7 N(m2, 0.6^2), m1 / m2 = -2.5 / +2.5 in the first two
    coordinates, prior U(-h, h)^n."""
    dev = _dev()
    m1, m2 = torch.zeros(n, dtype=torch.float64, device=dev), torch.zeros(n, dtype=torch.float64, device=dev)
    m1[:2], m2[:2] = -2.5, 2.5
    s1, s2, w1, w2 = 1.0, 0.6, math.log(0.3), math.log(0.7)
    c = 0.5 * n * math.log(2 * math.pi)

    def like(v):
        l1 = w1 - 0.5 * torch.sum((v - m1) ** 2, 1) / s1 ** 2 - n * math.log(s1) - c
        l2 = w2 - 0.5 * torch.sum((v - m2) ** 2, 1) / s2 ** 2 - n * math.log(s2) - c
        return torch.logaddexp(l1, l2)
    return TorchModel(n, like, lambda u: 2 * h * u - h, name='mixture'), -n * math.log(2 * h)


def _solve_gauss(n=20):
    dev = _dev()
    rng = np.random.default_rng(1)
    a = rng.standard_normal((n, n))
    cov = 0.002 * (a @ a.T / n + np.eye(n))
    covt = torch.as_tensor(cov, device=dev)
    lnorm = -0.5 * n * math.log(2 * math.pi) - 0.5 * np.linalg.slogdet(cov)[1]

    def like(v):
        d = v - 0.5
        return -0.5 * torch.sum(d * torch.linalg.solve(covt, d.T).T, 1) + lnorm
    return TorchModel(n, like, lambda u: u, name='solve_gauss'), 0.0     # the mass lies well inside the unit cube


@pytest.mark.parametrize('which', ['mixture', 'solve'])
def test_evidence_of_torch_only_likelihoods(which):
    tm, lnz = _mixture() if which == 'mixture' else _solve_gauss()
    for seed in (1, 2):
        r = nested.NestedSampler(tm, nlive=400, bound='multi', seed=seed).run_nested(dlogz=0.05, loop='device')
        assert abs(r['logz'][-1] - lnz) < 4 * r['logzerr'][-1], (seed, r['logz'][-1], lnz, r['logzerr'][-1])


# ---- no host round trip inside a fill or a block of rounds --------------------------------------------------------
def _d2h(prof):
    return [e for e in prof.events() if e.device_type.name == 'CUDA' and 'memcpy' in e.name.lower()
            and 'dtoh' in e.name.lower()]


def _stepped_records(prof):
    return [e for e in prof.events() if e.device_type.name == 'CUDA' and e.name.startswith('rwalk_step_kernel')]


# A CUDA-activity trace now and then lacks the device record of a kernel that did run, more often late in a long test
# process and near the edges of the capture window (test_gpu_launch_invariance.py, PADS).  So the window is padded with
# idle time on both sides, and a trace that misses a record is taken again with a wider pad; the launches themselves
# are counted by the library (b2n_launch_count), which sees every one.
PADS = (0.05, 0.3, 1.0, 2.0)


def _traced(fn, pad):
    import time
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()            # nothing of an earlier call is still in flight when the trace starts
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        time.sleep(pad)
        out = fn()
        torch.cuda.synchronize()
        time.sleep(pad)
    return out, prof


def test_no_round_trip_inside_a_fill_or_a_block():
    ctx = _lib.default_context()
    om = OL.gauss_corr(10, 0.4, 5.)
    tm = torch_restatement(om)
    rng = np.random.default_rng(2)
    u0, loglstar, axes, ell = _queue('prec', om, 200, 10, rng)
    ops.bound_set(axes)
    u0t = torch.as_tensor(u0, device=_dev())
    walks = 12
    fill = lambda: ops.rwalk_stepped(tm, u0t, loglstar, 0.6, walks, SEED, ell=ell)
    ref = fill()                                                         # warm-up (first-call checks)
    # one fill = walks + 1 stepped launches, and no copy to the host before the last of them has run
    for pad in PADS:
        n0 = ctx.launch_count()
        out, prof = _traced(fill, pad)
        assert ctx.launch_count() - n0 == walks + 1
        for k in ref:
            assert np.array_equal(out[k], ref[k]), k
        k = _stepped_records(prof)
        if len(k) == walks + 1:
            break
    assert len(k) == walks + 1, (len(k), walks + 1)
    last = max(e.time_range.end for e in k)
    d2h = _d2h(prof)
    assert d2h and all(e.time_range.start >= last for e in d2h)         # only the read of the outputs
    # a block of rounds: no copy to the host between two status reads
    s = nested.NestedSampler(tm, nlive=200, seed=3)
    s.update_bound_if_needed(nested.LOWL, force=True)                    # the first bound, on the host
    ops.ns_create(-1, 200, 10, 5, 0, walks, 3, ncdim=10)
    try:
        ops.ns_set_state(s.live_u, s.live_v, s.live_logl, -3.0, -1e300, -1e300, 0, 1.0)
        s._ensure_resident()
        ops.ns_run_stepped(tm, 2)
        rounds = 4
        n0 = ctx.launch_count()
        st, prof = _traced(lambda: ops.ns_run_stepped(tm, rounds), PADS[1])
        assert not (st['done'] or st['need_bound'] or st['error'])
        # per round one round-kernel launch and walks + 1 stepped launches, then the closing commit
        assert ctx.launch_count() - n0 == rounds * (1 + walks + 1) + 1
        assert len(_d2h(prof)) <= 1                                      # the one status read at the end of the block
    finally:
        ops.ns_destroy()

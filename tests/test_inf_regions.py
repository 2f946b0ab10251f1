"""CPU tier: runs whose log-likelihood is -inf on part of the prior, on the oracle-backed stand-in for the C ABI
(tests/fake_backend.py).

The initial live points are uniform over the region where logl is finite, of prior volume f < 1.  A run that starts
at ln X = 0 integrates over a volume 1/f too large: its evidence is high by -ln f.  Both inits estimate f by
rejection sampling, f = nlive / D with D the prior draws spent (``NestedSampler.initial_logvol``), and every volume
-- host loop, device rounds, the final live points, the dynamic sampler's merged record -- starts at ln f.  Checked
here: the exact bookkeeping of both inits, that a likelihood finite everywhere leaves every run as it was, the
refusal of non-finite supplied live points, and the evidence of the diamond (the reference's
tests/test_sampling.py region) against its quadrature."""
import math

import numpy as np
import pytest
from scipy import integrate

from dynesty_b200 import dynamic as D, likelihoods as DL, nested
from oracle import likelihoods as OL, philox, samplers as OS

SEED = 56432
NLIVE = 200


def _diamond_truth():
    """ln Z and f of the diamond by quadrature: logl = D2 - 1/4 where D2 = squared distance to the nearest corner of
    the unit square is > 1/4, -inf inside the four quarter discs.  One quarter of the square (x, y < 1/2, nearest
    corner the origin) times four."""
    def inner(x):
        y0 = math.sqrt(max(0.25 - x * x, 0.0))
        return integrate.quad(lambda y: math.exp(x * x + y * y - 0.25), y0, 0.5, epsabs=1e-14, epsrel=1e-13)[0]
    z = 4 * integrate.quad(inner, 0.0, 0.5, epsabs=1e-14, epsrel=1e-13, limit=200)[0]
    return math.log(z), 1.0 - math.pi / 4


DIAMOND_LOGZ, DIAMOND_F = _diamond_truth()


def test_diamond_truth():
    assert abs(DIAMOND_LOGZ - (-1.4682353)) < 1e-6


def _device_draws(model, nlive, seed):
    """Prior draws the device init spends: the oracle's unit-cube chains at threshold -inf, chain ids 2^61 + i."""
    return sum(OS.unitcube_chain(-np.inf, model, philox.ChainStream(seed, (1 << 61) + i), model.ndim)['ncall']
               for i in range(nlive))


def _host_draws(model, nlive, seed):
    """Prior draws the host init spends: batches of nlive from default_rng(seed), finite points taken in order,
    counted up to the last point taken."""
    rng = np.random.default_rng(seed)
    have, d = 0, 0
    while True:
        logl = model.loglike(model.prior_transform(rng.random((nlive, model.ndim))))
        ok = np.nonzero(np.isfinite(logl))[0][:nlive - have]
        have += len(ok)
        if have == nlive:
            return d + int(ok[-1]) + 1
        d += nlive


@pytest.mark.parametrize('live_init', ['device', 'host'])
def test_initial_volume_bookkeeping(fake_ops, live_init):
    """logvol_init = ln(nlive / D) with D the draws spent; ncall starts at D; the first dead point sits one ln X step
    below logvol_init, and the final live points of a run with no dead point start from logvol_init."""
    N = 50
    om = OL.region2d('diamond')
    d = (_device_draws if live_init == 'device' else _host_draws)(om, N, SEED)
    assert d > N
    s = nested.NestedSampler(DL.region2d('diamond'), nlive=N, bound='single', sample='unif', seed=SEED,
                             live_init=live_init)
    assert s.logvol_init == math.log(N / d) and s.ncall == d
    assert np.all(np.isfinite(s.live_logl)) and s.live_u.shape == (N, 2)
    np.testing.assert_array_equal(s.live_logl, om.loglike(s.live_v))
    # the final live points alone (a run with no dead point, as a dynamic batch can end)
    e = np.empty((0, 2))
    r0 = s._finalize(e, e, np.empty(0), np.empty(0), np.empty(0, dtype=np.int64), None, True)
    np.testing.assert_array_equal(r0.logvol, s.logvol_init + np.log(1. - (np.arange(N) + 1.) / (N + 1.)))
    assert np.isfinite(r0.logzerr[-1]) and np.isfinite(r0.information[-1])
    res = s.run_nested(dlogz=None, maxiter=30)
    assert res.logvol[0] == s.logvol_init - math.log((N + 1.) / N)
    assert res.ncall >= d + res.niter


def test_finite_likelihood_keeps_every_run_as_it_was(fake_ops):
    """With logl finite everywhere both inits spend exactly nlive draws: logvol_init is exactly 0.0, and the host init
    takes one (nlive, ndim) block from rstate, as it always did, so the rest of the run draws the same numbers."""
    m = DL.gauss_test3d()
    for live_init in ('device', 'host'):
        s = nested.NestedSampler(m, nlive=60, bound='single', sample='unif', seed=7, live_init=live_init)
        assert s.logvol_init == 0.0 and s.ncall == 60
    rng = np.random.default_rng(7)
    np.testing.assert_array_equal(s.live_u, rng.random((60, 3)))
    assert s.rstate.random() == rng.random()
    r = s.run_nested(dlogz=None, maxiter=20)
    dlv = math.log(61. / 60.)
    np.testing.assert_array_equal(r.logvol[:r.niter], -dlv * np.arange(1, r.niter + 1))


@pytest.mark.parametrize('bad', [np.nan, np.inf, -np.inf])
def test_supplied_live_points_need_finite_logl(fake_ops, bad):
    m = DL.gauss_test3d()
    rng = np.random.default_rng(3)
    u = rng.random((40, 3))
    v, logl = m.evaluate(u)
    logl = logl.copy()
    logl[17] = bad
    with pytest.raises(ValueError, match='live point 17'):
        nested.NestedSampler(m, nlive=40, bound='single', sample='unif', live_points=(u, v, logl))
    logl[17] = 0.0
    s = nested.NestedSampler(m, nlive=40, bound='single', sample='unif', live_points=(u, v, logl))
    assert s.logvol_init == 0.0 and s.ncall == 40


class _Stub:
    """A model whose host evaluation returns a fixed logl for every point (host init only)."""
    ndim = 2
    nblob = 0

    def __init__(self, value):
        self.value = value

    def evaluate(self, u, ctx=None):
        return np.array(u), np.full(len(u), self.value)


def test_host_init_errors(fake_ops):
    """NaN or +inf logl during the host init is an error (sampler.py:176-178); so is no finite point in 1000
    batches."""
    for value in (np.nan, np.inf):
        with pytest.raises(ValueError, match='invalid'):
            nested.NestedSampler(_Stub(value), nlive=10, bound='none', sample='unif', live_init='host')
    with pytest.raises(RuntimeError, match='1000 batches'):
        nested.NestedSampler(_Stub(-np.inf), nlive=10, bound='none', sample='unif', live_init='host')


def _tolerance(res, f, nlive):
    """4 sigma: the run's logzerr and the scatter of ln f-hat from the init draws, (1 - f) / nlive."""
    return 4 * math.sqrt(res.logzerr[-1] ** 2 + (1. - f) / nlive)


@pytest.mark.parametrize('live_init', ['device', 'host'])
@pytest.mark.parametrize('loop', ['host', 'device'])
def test_diamond_evidence(fake_ops, live_init, loop):
    """Host loop, and the device rounds of the stand-in backend after a host-loop prior phase: ln Z of the diamond
    within 4 sigma of the quadrature, sigma including the scatter of ln f-hat; finite logzerr and information."""
    s = nested.NestedSampler(DL.region2d('diamond'), nlive=NLIVE, bound='single', sample='unif', seed=SEED,
                             live_init=live_init)
    res = s.run_nested(dlogz=0.01, loop=loop, device_init=False)
    assert abs(res.logz[-1] - DIAMOND_LOGZ) < _tolerance(res, DIAMOND_F, NLIVE), (res.logz[-1], DIAMOND_LOGZ)
    assert np.isfinite(res.logzerr[-1]) and np.isfinite(res.information[-1])
    assert abs(s.logvol_init - math.log(DIAMOND_F)) < 4 * math.sqrt((1 - DIAMOND_F) / NLIVE)


def test_diamond_dynamic_record_starts_at_initial_volume(fake_ops):
    """The dynamic sampler's merged record is integrated from the baseline's logvol_init, and a batch joins it there."""
    d = D.DynamicNestedSampler(DL.region2d('diamond'), nlive=100, bound='single', sample='unif', seed=SEED)
    r0 = d.sample_initial(dlogz=0.05, round_size=10)
    assert d.logvol_init == d.base_sampler.logvol_init < -1.0
    assert r0.logvol[0] == d.logvol_init - math.log(101. / 100.)
    lv, _, lz, _, _ = D.integrate_record(d.saved, d.logvol_init)
    np.testing.assert_array_equal(lv, r0.logvol)
    res = d.add_batch(nlive=60, logl_bounds=(0.05, 0.2), round_size=6)
    assert d.batch == 1 and res.niter > r0.niter and np.all(np.diff(res.logvol) < 0)
    assert res.logvol[0] == d.logvol_init - math.log(101. / 100.)
    assert np.isfinite(res.logzerr[-1]) and np.isfinite(res.information[-1])
    assert abs(res.logz[-1] - DIAMOND_LOGZ) < _tolerance(res, DIAMOND_F, 100), (res.logz[-1], DIAMOND_LOGZ)


def test_resume_keeps_initial_volume(fake_ops, tmp_path):
    """logvol_init travels in the pickle: a run restored from a checkpoint of its device phase ends as the
    uninterrupted one."""
    m = DL.region2d('diamond')
    mk = lambda: nested.NestedSampler(m, nlive=100, bound='single', sample='unif', seed=11)
    ref = mk().run_nested(dlogz=0.05, loop='device', batch=10)
    f = str(tmp_path / 'ckpt.pkl')
    s = mk()
    n = []

    def stop(k):
        n.append(k)
        if k == 2:
            raise KeyboardInterrupt

    with pytest.raises(KeyboardInterrupt):
        s.run_nested(dlogz=0.05, loop='device', batch=10, checkpoint_file=f, checkpoint_every=0., on_checkpoint=stop)
    r = nested.NestedSampler.restore(f)
    assert r.logvol_init == s.logvol_init < -1.0
    res = r.run_nested(resume=True)
    assert res.niter == ref.niter and res.logz[-1] == ref.logz[-1]
    np.testing.assert_array_equal(res.logvol, ref.logvol)
    assert res.logvol[0] == r.logvol_init - math.log(101. / 100.)

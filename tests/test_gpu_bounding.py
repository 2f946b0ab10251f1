"""GPU: bounding-ellipsoid construction / decomposition vs fixtures produced by the
UNMODIFIED reference (tests/golden, oracle/make_golden.py) and vs the oracle.

float64 tolerances (stated): the reference uses LAPACK eigh, the CUDA path a cyclic
Jacobi solver -> eigenvector signs / order in degenerate subspaces are not comparable;
sign-invariant quantities are compared: ctr, cov, logvol 1e-9; am 1e-7 (am carries the
condition number); axes through axes @ axes.T = cov and sorted axis lengths."""
import numpy as np
import pytest

from dynesty_b200 import _lib, ops
from helpers import close, SEED
from oracle import bounding as OB, philox

pytestmark = pytest.mark.gpu


def check_ell(o, g, p, am_rtol=1e-7):
    close(o['ctr'], g[p + 'ctr'])
    close(o['cov'], g[p + 'cov'])
    close(o['am'], g[p + 'am'], rtol=am_rtol)
    close(o['axes'] @ o['axes'].T, g[p + 'cov'])
    close(np.sort(o['axlens']), np.sort(g[p + 'axlens']))
    assert abs(o['logvol'] - float(g[p + 'logvol'])) < 1e-8
    # internal consistency of the CUDA eigen-decomposition
    close(o['cov'] @ o['am'], np.eye(len(o['ctr'])), rtol=1e-6)
    assert np.all(np.diff(o['axlens']) >= 0)           # ascending like LAPACK
    close(np.linalg.norm(o['axes'], axis=0), o['axlens'])


@pytest.mark.parametrize('name', ['g20', 'g3', 'g50', 'few', 'illcond'])
def test_bounding_ellipsoid_golden(golden, name):
    g = golden['bounding']
    pts = g['be_%s_points' % name]
    o = ops.bounding_ellipsoid(pts)
    check_ell(o, g, 'be_%s_' % name, am_rtol=1e-6 if name == 'illcond' else 1e-7)
    d2 = ops.membership(pts, o['ctr'], o['am'], want_d2=True)[2]
    assert d2.max() < 1                                  # bounding.py:1438-1453
    assert o['warn'] == 0


def test_bounding_rank_deficient(golden):
    """tests/test_ellipsoid.py:258-264 (test_bounding_crazy): must not raise and must
    still bound every point; ndim 1, 10, 100."""
    g = golden['bounding']
    pts = g['be_rank1_points']
    o = ops.bounding_ellipsoid(pts)
    assert ops.membership(pts, o['ctr'], o['am'], want_d2=True)[2].max() < 1
    assert np.all(np.linalg.eigvalsh(o['cov']) > 0)
    # the rescale factor of a rank-deficient fit is set by round-off in the null space
    # (1/l_min ~ 1e11 times noise^2): only pinned loosely
    close(np.sort(o['axlens'])[-1], np.sort(g['be_rank1_axlens'])[-1], rtol=1e-4)
    rng = np.random.default_rng(1)
    for ndim in (1, 10, 100, 150):       # 150: sliced eigensolver + host-driven repair ladder
        x = rng.random(200)
        p = 0.5 + (x[:, None] - 0.5) * np.ones((1, ndim)) * 0.2
        o = ops.bounding_ellipsoid(p)
        assert ops.membership(p, o['ctr'], o['am'], want_d2=True)[2].max() < 1


def test_bounding_errors():
    with pytest.raises(ValueError):                       # bounding.py:1405-1407
        ops.bounding_ellipsoid(np.full((1, 3), 0.5))
    with pytest.raises(ValueError):
        ops.multi_decompose(np.full((1, 3), 0.5))


@pytest.mark.parametrize('N,n', [(2000, 50), (8000, 200), (500, 3), (64, 2)])
def test_bounding_vs_oracle_sizes(N, n):
    """BASELINE sizes (C2 2000x50, C4 8000x200): compared with the oracle directly."""
    rng = np.random.default_rng(N + n)
    A = rng.standard_normal((n, n)) / np.sqrt(n)
    pts = 0.5 + 0.05 * rng.standard_normal((N, n)) @ (np.eye(n) + 0.5 * A)
    o = ops.bounding_ellipsoid(pts)
    e = OB.bounding_ellipsoid(pts)
    close(o['ctr'], e.ctr, rtol=1e-12)
    close(o['cov'], e.cov, rtol=1e-9)
    close(o['am'], e.am, rtol=1e-7)
    close(np.sort(o['axlens']), np.sort(e.axlens), rtol=1e-9)
    assert abs(o['logvol'] - e.logvol) < 1e-8
    close(o['axes'] @ o['axes'].T, e.cov, rtol=1e-9)


@pytest.mark.parametrize('name', ['iso', 'cap', 'shrink'])
def test_scale_to_logvol_golden(golden, name):
    g = golden['bounding']
    # the CUDA routine needs axes/axlens in matching (ascending) order: rebuild from cov
    o = ops.bounding_ellipsoid(g['be_g20_points'])
    covs, ams, axes = o['cov'][None].copy(), o['am'][None].copy(), o['axes'][None].copy()
    axlens, logvols = o['axlens'][None].copy(), np.array([o['logvol']])
    target = logvols + float(g['stl_%s_dlv' % name])
    ops.scale_to_logvol(covs, ams, axes, axlens, logvols, target)
    p = 'stl_%s_' % name
    close(covs[0], g[p + 'cov'])
    close(ams[0], g[p + 'am'], rtol=1e-7)
    close(np.sort(axlens[0]), np.sort(g[p + 'axlens']))
    close(axes[0] @ axes[0].T, g[p + 'cov'])
    assert abs(logvols[0] - float(g[p + 'logvol'])) < 1e-9


@pytest.mark.parametrize('name', ['c8', 'c2', 'blob', 'ring'])
def test_multi_decompose_golden(golden, name):
    g = golden['multi']
    p = 'me_%s_' % name
    pts = g[p + 'points']
    o = ops.multi_decompose(pts)
    assert o['nells'] == len(g[p + 'logvols'])
    # leaf ORDER depends on eigenvector signs (see tests/test_oracle_golden.py): compare as sets
    o1, o2 = np.argsort(o['ctrs'][:, 0]), np.argsort(g[p + 'ctrs'][:, 0])
    close(o['ctrs'][o1], g[p + 'ctrs'][o2])
    close(o['covs'][o1], g[p + 'covs'][o2])
    close(o['ams'][o1], g[p + 'ams'][o2], rtol=1e-7)
    close(o['logvols'][o1], g[p + 'logvols'][o2], rtol=1e-10)
    # labels: every point is inside the ellipsoid it is assigned to
    lab = o['labels']
    assert lab.min() >= 0 and lab.max() < o['nells']
    mask = ops.membership(pts, o['ctrs'], o['ams'])[0]
    assert mask[np.arange(len(pts)), lab].all()
    # enlarge like Sampler.update_bound (sampler.py:506-508): scalar target -> per-ellipsoid shift
    from scipy.special import logsumexp
    covs, ams, axes = o['covs'].copy(), o['ams'].copy(), o['axes'].copy()
    axlens, logvols = o['axlens'].copy(), o['logvols'].copy()
    ops.scale_to_logvol(covs, ams, axes, axlens, logvols, logvols + np.log(1.25))
    close(logvols[o1], g[p + 'enl_logvols'][o2], rtol=1e-10)
    close(ams[o1], g[p + 'enl_ams'][o2], rtol=1e-7)
    assert abs(logsumexp(logvols) - (float(g[p + 'logvol']) + np.log(1.25))) < 1e-9


def test_number_clusters():
    """tests/test_ellipsoid.py:267-286: 6^4 grid clusters recovered within 10 %."""
    rng = np.random.default_rng(SEED)
    ndim, npt, nper = 4, 30, 6
    g1 = np.linspace(0, 1, nper + 2)[1:-1]
    grid = np.array(np.meshgrid(*[g1] * ndim)).reshape(ndim, -1).T
    pts = (grid[:, None, :] + 1e-4 * rng.standard_normal((len(grid), npt, ndim))).reshape(-1, ndim)
    o = ops.multi_decompose(pts, max_ells=4000)
    assert abs(o['nells'] / len(grid) - 1) < 0.1


@pytest.mark.parametrize('multi', [0, 1])
def test_bootstrap_expand_golden(golden, multi):
    g = golden['multi']
    got = ops.bootstrap_expand(g['me_c2_points'], multi, 4, SEED, 1000)
    np.testing.assert_allclose(got, g['boot_%d_expand' % multi], rtol=1e-8)


@pytest.mark.parametrize('case', ['gauss2000x50', 'clusters4000x25', 'two20000x8', 'illcond600x12', 'grid'])
def test_candidate_path_equals_eigen_path(case, monkeypatch):
    """The candidates of the multi-ellipsoid tree go through the Cholesky / matrix-squaring kernel
    (chol_node_kernel), only the accepted leaves through the eigen path; B2N_BOUND_FAST=0 forces the eigen
    path for every node.  Same tree, same leaves: nells equal, centres / covariances / log-volumes to
    round-off (the leaf fits see the points in a different order), every point inside its ellipsoid.
    'two20000x8' has two leaves; 'illcond600x12' and 'grid' (exactly degenerate spectra) have nodes the
    candidate path cannot certify: it must fall back."""
    if case == 'grid':
        g1 = np.linspace(0.2, 0.8, 5)
        pts = np.array(np.meshgrid(g1, g1, g1)).reshape(3, -1).T
        pts = np.concatenate([pts, pts + 1e-3, pts - 1e-3, pts + 2e-3])
    else:
        pts = _clouds(case)
    monkeypatch.setenv('B2N_BOUND_FAST', '0')
    slow = ops.multi_decompose(pts)
    monkeypatch.setenv('B2N_BOUND_FAST', '1')
    fast = ops.multi_decompose(pts)
    assert fast['nells'] == slow['nells']
    a, b = np.lexsort(fast['ctrs'].T[::-1]), np.lexsort(slow['ctrs'].T[::-1])
    close(fast['ctrs'][a], slow['ctrs'][b], rtol=1e-12)
    close(fast['covs'][a], slow['covs'][b], rtol=1e-9)
    close(fast['logvols'][a], slow['logvols'][b], rtol=1e-11)
    close(fast['ams'][a], slow['ams'][b], rtol=1e-7)
    mask = ops.membership(pts, fast['ctrs'], fast['ams'])[0]
    assert mask[np.arange(len(pts)), fast['labels']].all()
    if case == 'clusters4000x25':
        assert fast['nells'] == 8


def _clouds(case):
    rng = np.random.default_rng(SEED)
    if case == 'gauss2000x50':
        Cm = np.full((50, 50), 0.4)
        np.fill_diagonal(Cm, 1.0)
        return 0.5 + 0.02 * rng.standard_normal((2000, 50)) @ np.linalg.cholesky(Cm).T
    if case == 'clusters4000x25':
        ctrs = 0.2 + 0.6 * rng.random((8, 25))
        return np.concatenate([c + 0.01 * rng.standard_normal((500, 25)) for c in ctrs])
    if case == 'two20000x8':            # 2500 rows per k-means CTA: more than its shared-memory stage holds
        return np.concatenate([0.3 + 0.02 * rng.standard_normal((12000, 8)), 0.7 + 0.02 * rng.standard_normal((8000, 8))])
    if case == 'illcond600x12':         # the root's covariance needs the repair ladder: its speculative fit is not adopted
        p = 0.5 + 0.05 * rng.standard_normal((600, 12))
        p[:, 11] = p[:, 0] + 1e-9 * rng.standard_normal(600)
        return p
    raise KeyError(case)


@pytest.mark.parametrize('case', ['gauss2000x50', 'clusters4000x25', 'two20000x8', 'illcond600x12'])
def test_speculative_root_fit_equals_refit(case, monkeypatch):
    """b2n_spec_root_*: the root's eigen fit runs on a side stream while the candidate tree is expanded and is
    adopted when the root is the accepted leaf (gauss2000x50; the others have several leaves or a root whose
    covariance needs the repair ladder, and are re-fitted after the tree).  The adopted fit runs the kernels of
    bounding_ellipsoid on the same rows in the same order: equal to the bit.  Every case is reproducible call to
    call."""
    pts = _clouds(case)
    monkeypatch.setenv('B2N_BOUND_FAST', '1')           # attempt the candidate path whatever this context saw before
    b = ops.multi_decompose(pts)
    b2 = ops.multi_decompose(pts)
    assert b['nells'] == b2['nells']
    for k in ('labels', 'ctrs', 'covs', 'ams', 'axes', 'logvols'):
        assert np.array_equal(b[k], b2[k]), k
    if case == 'gauss2000x50':
        a = ops.bounding_ellipsoid(pts)
        assert b['nells'] == 1
        for k, kb in (('ctr', 'ctrs'), ('cov', 'covs'), ('am', 'ams'), ('axes', 'axes'), ('axlens', 'axlens')):
            assert np.array_equal(b[kb][0], a[k]), k
        assert b['logvols'][0] == a['logvol']
    for k in range(b['nells']):
        close(b['axes'][k] @ b['axes'][k].T, b['covs'][k], rtol=1e-9)
    mask = ops.membership(pts, b['ctrs'], b['ams'])[0]
    assert mask[np.arange(len(pts)), b['labels']].all()


def _indefinite(n):
    """A symmetric matrix with two negative eigenvalues: improve_covar runs its repair ladder."""
    rng = np.random.default_rng(n)
    A = rng.standard_normal((n, n))
    lam, V = np.linalg.eigh(A @ A.T / n)
    lam[:2] = -lam[:2]
    M = (V * lam) @ V.T
    return 0.5 * (M + M.T)


def _line150():
    """Collinear points in 150 dimensions: the sliced eigensolver's repair ladder and the second pass."""
    x = np.random.default_rng(1).random(200)
    return 0.5 + (x[:, None] - 0.5) * np.ones((1, 150)) * 0.2


# One call of each bound-update entry point, on a fresh context (no state carried over, such as the eigen path taken
# for a while after a candidate could not be certified).  n = 50 / 40 keep the eigen solve in one CTA's shared
# memory; n = 150 takes the sliced solver.
LAUNCH_CALLS = {
    'bounding_ellipsoid-n50': lambda ctx: ops.bounding_ellipsoid(_clouds('gauss2000x50'), ctx=ctx),
    'bounding_ellipsoid-n150': lambda ctx: ops.bounding_ellipsoid(_line150(), ctx=ctx),
    'improve_covar-n40': lambda ctx: ops.improve_covar(_indefinite(40), ctx=ctx),
    'improve_covar-n150': lambda ctx: ops.improve_covar(_indefinite(150), ctx=ctx),
    'moments-n50': lambda ctx: ops.moments(_clouds('gauss2000x50'), ctx=ctx),
    'moments-n150': lambda ctx: ops.moments(_line150(), ctx=ctx),
    'multi_decompose-gauss2000x50': lambda ctx: ops.multi_decompose(_clouds('gauss2000x50'), ctx=ctx),
    'multi_decompose-clusters4000x25': lambda ctx: ops.multi_decompose(_clouds('clusters4000x25'), ctx=ctx),
    'multi_decompose-two20000x8': lambda ctx: ops.multi_decompose(_clouds('two20000x8'), ctx=ctx),
    'multi_decompose-illcond600x12': lambda ctx: ops.multi_decompose(_clouds('illcond600x12'), ctx=ctx),
    'bootstrap_expand-single': lambda ctx: ops.bootstrap_expand(_clouds('clusters4000x25'), 0, 2, SEED, 1000, ctx=ctx),
    'bootstrap_expand-multi': lambda ctx: ops.bootstrap_expand(_clouds('clusters4000x25'), 1, 2, SEED, 1000, ctx=ctx),
    'friends_update': lambda ctx: ops.friends_update(_clouds('gauss2000x50'), 'balls', ctx=ctx),
}
LAUNCHES = {'bounding_ellipsoid-n50': 7, 'bounding_ellipsoid-n150': 24, 'improve_covar-n40': 1,
            'improve_covar-n150': 9, 'moments-n50': 4, 'moments-n150': 4, 'multi_decompose-gauss2000x50': 55,
            'multi_decompose-clusters4000x25': 99, 'multi_decompose-two20000x8': 137,
            'multi_decompose-illcond600x12': 137, 'bootstrap_expand-single': 18, 'bootstrap_expand-multi': 141,
            'friends_update': 12}


@pytest.mark.parametrize('call', sorted(LAUNCH_CALLS))
def test_bound_update_launches(call, monkeypatch):
    """Kernel launches per call of the bound-update entry points (B2N_BOUND_FAST unset: the default path)."""
    monkeypatch.delenv('B2N_BOUND_FAST', raising=False)
    ctx = _lib.Context(0)
    try:
        before = ctx.launch_count()
        LAUNCH_CALLS[call](ctx)
        assert ctx.launch_count() - before == LAUNCHES[call]
    finally:
        ctx.close()


# ---- improve_covar_mat on its own (b2n_improve_covar): the reference's test matrices (tests/test_ellipsoid.py:242-255)
@pytest.mark.parametrize('name', ['zero', 'rank1', 'neg', 'good'])
def test_improve_covar_mat_fixtures(golden, name):
    """The repair ladder fed a RAW matrix: `zero` / `neg` take the failed == 2 identity blend
    (bounding.py:1366-1371), `rank1` the eigenvalue clamp (:1362-1365), `good` passes untouched.  The clamp /
    blend outputs are deterministic functions of the eigen-decomposition, compared with the reference's own
    outputs (fixtures) at 1e-6 -- the bar of tests/test_oracle_golden.py for the oracle."""
    g = golden['bounding']
    good, cov, am, axes, warn = ops.improve_covar(g['icm_%s_in' % name])
    assert good == bool(g['icm_%s_good' % name])
    assert warn == 0
    close(cov, g['icm_%s_cov' % name], rtol=1e-6)
    assert np.all(np.linalg.eigvalsh(cov) > 0)
    close(cov @ am, np.eye(cov.shape[0]), rtol=1e-3)
    close(axes @ axes.T, cov, rtol=1e-6)


def test_improve_covar_identity_fallback():
    """A matrix no blend can repair (NaN: eigh(check_finite=False) returns NaN, every trial fails) ends in the
    identity fallback with the reference's warning (bounding.py:1373-1378); the oracle agrees."""
    import warnings
    bad = np.full((5, 5), np.nan)
    good, cov, am, axes, warn = ops.improve_covar(bad)
    assert not good and warn & 1
    for a in (cov, am, axes):
        assert np.array_equal(a, np.eye(5))
    try:                    # (LAPACK may refuse NaN input instead of returning NaN: the reference catches that, :1358)
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            og, oc, oa, ox, _ = OB.improve_covar_mat(bad)
        assert not og and np.array_equal(oc, np.eye(5))
    except np.linalg.LinAlgError:
        pass


@pytest.mark.parametrize('n', [3, 40, 130])
def test_improve_covar_vs_oracle_random(n):
    """Singular, indefinite and ill-conditioned random matrices (n = 130: the sliced eigensolver's ladder)."""
    rng = np.random.default_rng(n)
    A = rng.standard_normal((n, n))
    S = A @ A.T / n
    lam, V = np.linalg.eigh(S)
    for kind in ('illcond', 'indefinite', 'singular'):
        l2 = lam.copy()
        if kind == 'illcond':
            l2[0] = l2[-1] * 1e-15
        elif kind == 'indefinite':
            l2[:2] = -l2[:2]
        else:
            l2[:max(1, n // 4)] = 0.0
        M = (V * l2) @ V.T
        M = 0.5 * (M + M.T)
        good, cov, am, axes, warn = ops.improve_covar(M)
        og, oc, oa, ox, _ = OB.improve_covar_mat(M)
        assert good == og and warn == 0
        close(cov, oc, rtol=1e-6)
        w = np.linalg.eigvalsh(cov)
        assert w.min() > 0 and w.max() / w.min() < 1.05e11      # clamped at 10 max / 1e12 (:1362-1365)
        close(cov @ am, np.eye(n), rtol=1e-3)


def test_bounding_identical_and_collinear_points():
    """Clouds that drive the ladder through `failed == 2` from the POINT side: identical points (zero covariance)
    and collinear points (rank 1) -- bounding_ellipsoid must still return a bound containing every point."""
    rng = np.random.default_rng(7)
    same = np.tile(rng.random(6), (40, 1))
    line = np.outer(np.linspace(0.2, 0.8, 60), np.ones(6)) + 0.1
    for name, pts in (('same', same), ('line', line)):
        o = ops.bounding_ellipsoid(pts)
        d2 = ops.membership(pts, o['ctr'], o['am'], want_d2=True)[2]
        assert d2.max() < 1 + 1e-9
        assert np.all(np.linalg.eigvalsh(o['cov']) > 0)
        # (no comparison of the VOLUME with the oracle: the covariance of coincident / collinear points is pure
        #  round-off of the mean -- 1e-34 -- so which rung of the ladder repairs it depends on the summation order)
        assert np.isfinite(o['logvol'])

"""GPU: the multi-ellipsoid decomposition (csrc/b2n_multi.cu, b2n_bounding.cu, b2n_eig_sliced.cu) against the
float64 oracle node by node (oracle/bounding.py candidate_tree), at the shapes where its kernels change form.

Each case's form is derived from the device limits by mirroring the host's formulas (km_stage_max / stage_cap
in decompose(), the Cholesky candidates' shared-memory bound `csm`, the eigen kernel's and the sliced solver's),
the way test_gpu_kernel_matrix.py mirrors rwalk_plan, and the test asserts that the case reaches the form it
names.  Every cloud is well-posed by the oracle's margins (tests/test_oracle_multi.py) before anything is
compared, so the tree must match exactly:
  - every node's member set (a node's rows are a SET: partitions only permute inside segments), its children,
    the split sizes of refused splits and the accepted leaves;
  - every node's log-volume to 1e-9 relative -- the Cholesky candidates' included, which otherwise only feed
    the host's accept / reject decisions;
  - the leaves of ops.multi_decompose: centres 1e-12, covariances 1e-9, am 1e-7, axes @ axes.T = cov, and its
    labels equal to the tree's member sets."""
import os

import numpy as np
import pytest

from dynesty_b200 import ops
from helpers import close
from oracle import bounding as OB, multicases as MC, philox
from oracle.make_golden import SEED

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'multi_edges.npz')
KM_CLUSTER = 8


def _optin():
    import torch
    return int(torch.cuda.get_device_properties(0).shared_memory_per_block_optin)


# ---- the host's formulas (b2n_multi.cu decompose / multi_run, b2n_bounding.cu b2n_fit_nodes, b2n_eig_sliced.cu)
def km_stage_max(n, optin):
    nw = 16
    while (6 * n + nw * 2 * n) * 8 + nw * 2 * 4 > optin and nw > 1:
        nw >>= 1
    base = (6 * n + nw * 2 * n) * 8 + (nw * 2 + 2) * 4
    room = min(optin, 120 * 1024)
    return (room - base) // ((n | 1) * 8 + 1) if room > base else 0


def chol_fits(n, optin):
    return (2 * n * (n | 1) + 3 * n + 32 + 2 * (n + 2)) * 8 <= optin


def eig_single_cta(n, optin):
    half = ((n + 1) & ~1) // 2
    return (2 * half + 2 * n + 32) * 8 + 2 * n * (n | 1) * 8 <= optin


def eig_sliced_fits(n, optin):
    half = ((n + 1) & ~1) // 2
    npk = n * (n + 1) // 2
    return (((npk + 1) & ~1) + n * ((n + 7) // 8) + 3 * half + 32) * 8 + 2 * half * 4 <= optin


def km_forms(tree, n, optin):
    """{depth: set of (node, CTA form)}: a k-means CTA runs the thread-per-row loop if all its rows fit the
    level's stage (stage_cap = min(km_stage_max, ceil(max count / 8) + 1)), else the warp-per-row loop."""
    smax = km_stage_max(n, optin)
    out = {}
    for d in sorted({nd['depth'] for nd in tree['nodes']}):
        split = [i for i, nd in enumerate(tree['nodes']) if nd['depth'] == d and nd['split'] is not None]
        if not split:
            continue
        maxc = max(len(tree['nodes'][i]['members']) for i in split)
        cap = min(smax, (maxc + KM_CLUSTER - 1) // KM_CLUSTER + 1)
        forms = set()
        for i in split:
            c = len(tree['nodes'][i]['members'])
            for r in range(KM_CLUSTER):
                rows = c * (r + 1) // KM_CLUSTER - c * r // KM_CLUSTER
                forms.add((i, 'empty' if rows == 0 else 'thread' if rows <= cap else 'warp'))
        out[d] = forms
    return out


# ---- comparison with the oracle
def check_tree(pts, g, t, lv_atol=0.0):
    """g: ops.multi_tree, t: OB.candidate_tree.  Structure exact, log-volumes 1e-9 relative (+ lv_atol)."""
    N = len(pts)
    perm = g['perm']
    assert np.array_equal(np.sort(perm), np.arange(N))
    key = OB.tree_by_members(t)
    T = len(g['start'])
    assert T == len(t['nodes'])
    ids = [key[tuple(np.sort(perm[s:s + c]))] for s, c in zip(g['start'], g['count'])]
    assert sorted(ids) == list(range(T))
    leaves = set(t['leaves'])
    for i, j in enumerate(ids):
        nd = t['nodes'][j]
        ch = g['children'][i]
        if nd['children'] is None:
            assert np.all(ch == -1), (i, j)
        else:
            assert sorted(ids[c] for c in ch) == sorted(nd['children']), (i, j)
        if nd['split'] is None:
            assert np.all(g['split'][i] == -1), (i, j)
        else:
            assert sorted(g['split'][i]) == sorted(nd['split']), (i, j)
        assert bool(g['leaf'][i]) == (j in leaves), (i, j)
        assert abs(g['logvol'][i] - nd['logvol']) <= lv_atol + 1e-9 * max(1.0, abs(nd['logvol'])), \
            (i, j, g['logvol'][i], nd['logvol'])
    return ids


def check_leaves(pts, t, am_rtol=1e-7, lv_atol=0.0, cov_rtol=1e-9):
    """ops.multi_decompose: the oracle's accepted leaves, labels = their member sets."""
    o = ops.multi_decompose(pts)
    assert o['nells'] == len(t['leaves'])
    key = {tuple(t['nodes'][i]['members']): i for i in t['leaves']}
    for k in range(o['nells']):
        e = t['nodes'][key[tuple(np.flatnonzero(o['labels'] == k))]]['ell']
        close(o['ctrs'][k], e.ctr, rtol=1e-12)
        close(o['covs'][k], e.cov, rtol=cov_rtol)
        close(o['ams'][k], e.am, rtol=am_rtol)
        close(o['axes'][k] @ o['axes'][k].T, e.cov, rtol=cov_rtol)
        assert abs(o['logvols'][k] - e.logvol) <= lv_atol + 1e-9 * max(1.0, abs(e.logvol))
    return o


_TREES = {}


def oracle_tree(name):
    if name not in _TREES:
        t = OB.candidate_tree(MC.cloud(name))
        assert t['km_margin'] > 1e-9 and t['eig_gap'] > 1e-6 and OB.decision_margin(t) > 1e-6, name
        _TREES[name] = t
    return _TREES[name]


# name: (B2N_BOUND_FAST, path the tree must come from, the form the case is there for)
CASES = {
    'two20000x8': ('1', 'cholesky', 'km-warp-root'),
    'three2100x50': ('1', 'cholesky', 'km-mixed-node'),
    'gauss2000x50': ('1', 'cholesky', 'spec-root'),
    'few7x1': ('1', 'cholesky', 'km-empty-cta'),
    'few18x2': ('1', 'cholesky', 'km-tiny'),
    'two3600x33': ('1', 'cholesky', 'km-odd-n'),
    'two640x64': ('1', 'cholesky', 'chol-4x2'),
    'two640x65': ('1', 'cholesky', 'chol-8x4'),
    'two600x119': ('1', 'cholesky', 'chol-8x4'),
    'two600x120': ('1', 'eigen', 'sliced'),
    'two700x150': ('1', 'eigen', 'sliced'),
    'mix300x2late': ('1', 'cholesky', 'late'),
    'mix300x2test2': ('1', 'cholesky', 'test2'),
    'illcond600x12': ('1', 'eigen', 'uncertified'),
    # the eigen path for every candidate, forced
    'three2100x50/eigen': ('0', 'eigen', 'km-mixed-node'),
    'mix300x2test2/eigen': ('0', 'eigen', 'test2'),
}


def check_form(name, form, t, pts, optin):
    N, n = pts.shape
    forms = km_forms(t, n, optin)
    if form == 'km-warp-root':
        assert {f for _, f in forms[0]} == {'warp'}
        assert {f for _, f in forms[1]} == {'thread'}
    elif form == 'km-mixed-node':
        assert {f for _, f in forms[0]} == {'thread', 'warp'}          # one node, CTAs in both forms
    elif form == 'spec-root':
        assert t['leaves'] == [0] and N >= 4 * n and eig_single_cta(n, optin)
    elif form == 'km-empty-cta':
        assert any('empty' in {f for _, f in fs} for fs in forms.values())
    elif form == 'km-tiny':              # n = 2: a splittable node has 4 n = 8 rows or more, a few per CTA
        assert all(len(nd['members']) < 3 * KM_CLUSTER for nd in t['nodes'])
    elif form == 'km-odd-n':
        assert n % 2 == 1 and n > 32
        assert {f for _, f in forms[0]} == {'warp'} and 'thread' in {f for _, f in forms[1]}
    elif form == 'chol-4x2':
        assert chol_fits(n, optin) and n <= 64
    elif form == 'chol-8x4':
        assert chol_fits(n, optin) and n > 64
    elif form == 'sliced':
        assert not chol_fits(n, optin) and not eig_single_cta(n, optin) and eig_sliced_fits(n, optin)
        assert len(t['leaves']) >= 2 and len({t['nodes'][i]['depth'] for i in t['leaves']}) == 1
    elif form == 'late':
        assert t['late']
    elif form == 'test2':
        assert 2 in {nd['accept'] for nd in t['nodes']}
        assert any(nd['split'] is not None and nd['children'] is None for nd in t['nodes'])
    elif form == 'uncertified':
        pass
    else:
        raise KeyError(form)


@pytest.mark.parametrize('case', list(CASES))
def test_multi_tree_vs_oracle(case, monkeypatch):
    name = case.split('/')[0]
    fast, path, form = CASES[case]
    pts = MC.cloud(name)
    t = oracle_tree(name)
    check_form(name, form, t, pts, _optin())
    monkeypatch.setenv('B2N_BOUND_FAST', fast)
    g = ops.multi_tree(pts)
    assert g['path'] == path
    # illcond: every node's covariance goes through the repair ladder, whose clamped eigenvalue 10 lam_max / 1e12
    # both eigensolvers recompute to an absolute eps lam_max, i.e. to ~2e-5 relative: ln det and am inherit that,
    # and the covariance through the rescale factor (its fmax weighs the clamped direction by 1 / lam_min)
    ill = name.startswith('illcond')
    check_tree(pts, g, t, lv_atol=2e-5 if ill else 0.0)
    o = check_leaves(pts, t, am_rtol=1e-4 if ill else 1e-7, lv_atol=2e-5 if ill else 0.0, cov_rtol=1e-7 if ill else 1e-9)
    if form == 'spec-root':         # the root's speculative eigen fit is the result: the oracle's bounding_ellipsoid
        e = OB.bounding_ellipsoid(pts)
        close(o['ctrs'][0], e.ctr, rtol=1e-12)
        close(o['covs'][0], e.cov, rtol=1e-9)
        close(o['ams'][0], e.am, rtol=1e-7)


def test_retry_sets_the_skip_count(monkeypatch):
    """A candidate that cannot be certified sends the update to the eigen path and the next 16 calls of the
    context skip the Cholesky candidates (unless B2N_BOUND_FAST=1 forces the attempt); the tree is the oracle's
    either way."""
    from dynesty_b200 import _lib
    ctx = _lib.Context(0)
    monkeypatch.delenv('B2N_BOUND_FAST', raising=False)
    ill, good = MC.cloud('illcond600x12'), MC.cloud('two640x64')
    assert ops.multi_tree(ill, ctx=ctx)['path'] == 'eigen'
    for _ in range(16):
        g = ops.multi_tree(good, ctx=ctx)
        assert g['path'] == 'eigen'
    check_tree(good, g, oracle_tree('two640x64'))
    g = ops.multi_tree(good, ctx=ctx)
    assert g['path'] == 'cholesky'
    check_tree(good, g, oracle_tree('two640x64'))


@pytest.mark.parametrize('name', ['two640x65', 'mix300x2late', 'mix300x2test2'])
def test_multi_decompose_vs_reference_fixture(name):
    """The unmodified reference's leaves (tests/golden/multi_edges.npz, oracle/make_golden_multi.py)."""
    g = np.load(GOLDEN)
    p = name + '_'
    pts = g[p + 'points']
    o = ops.multi_decompose(pts)
    K = len(g[p + 'logvols'])
    assert o['nells'] == K
    want = {tuple(g[p + 'members_%d' % k]): k for k in range(K)}
    for j in range(K):
        k = want[tuple(np.flatnonzero(o['labels'] == j))]
        close(o['ctrs'][j], g[p + 'ctrs'][k], rtol=1e-12)
        close(o['covs'][j], g[p + 'covs'][k], rtol=1e-9)
        close(o['ams'][j], g[p + 'ams'][k], rtol=1e-7)
        assert abs(o['logvols'][j] - g[p + 'logvols'][k]) <= 1e-9 * max(1.0, abs(g[p + 'logvols'][k]))


def _expected_expands(pts, multi, nboot, chain0):
    out = []
    for r in range(nboot):
        s = philox.ChainStream(SEED, chain0 + r)
        sel = OB.bootstrap_split(len(pts), s.integers(len(pts), len(pts)))
        if multi:
            t = OB.candidate_tree(pts[sel])
            assert t['km_margin'] > 1e-9 and t['eig_gap'] > 1e-6 and OB.decision_margin(t) > 1e-6
        out.append((OB.bootstrap_expand(pts, sel, bool(multi)), sel))
    return out


@pytest.mark.parametrize('name', MC.BOOT_CLOUDS)
@pytest.mark.parametrize('multi', [0, 1])
def test_bootstrap_expand_vs_oracle(name, multi):
    """nboot = 8 replicas from chain0 = 77, each against OB.bootstrap_expand on the same Philox selection."""
    pts = MC.boot_cloud(name)
    N, n = pts.shape
    want = _expected_expands(pts, multi, 8, 77)
    got = ops.bootstrap_expand(pts, multi, 8, SEED, 77)
    for r, (w, sel) in enumerate(want):
        assert abs(got[r] - w) <= 1e-9 * w, (r, got[r], w)
    nin = [int(sel.sum()) for _, sel in want]
    if name == 'odd401x5':
        assert N % 2 == 1
    elif name == 'split999x8' and multi:
        assert all(len(OB.candidate_tree(pts[sel])['leaves']) >= 2 for _, sel in want)
    elif name == 'small45x10':
        assert max(nin) < 4 * n


@pytest.mark.parametrize('name', ['two640x65', 'odd401x5', 'split999x8'])
@pytest.mark.parametrize('multi', [0, 1])
def test_bootstrap_expand_vs_reference_fixture(name, multi):
    g = np.load(GOLDEN)
    want = g['boot_%s_%d' % (name, multi)]
    got = ops.bootstrap_expand(g[name + '_points'], multi, len(want), SEED, 2000)
    np.testing.assert_allclose(got, want, rtol=1e-9)

"""CPU tier: the oracle's multi-ellipsoid decomposition (oracle/bounding.py candidate_tree) against the unmodified
reference (tests/golden/multi_edges.npz, oracle/make_golden_multi.py) and scipy, and the well-posedness of every
cloud tests/test_gpu_multi.py compares the CUDA decomposition with (oracle/multicases.py): no point within a
relative 1e-9 of the k-means bisector, no split node whose two largest eigenvalues lie within a relative 1e-6 (the
major axis seeds the k-means), no volume test within 1e-6 of its threshold."""
import os

import numpy as np
import pytest
import scipy.cluster.vq as vq

from helpers import close
from oracle import bounding as OB, multicases as MC, philox
from oracle.make_golden import SEED
from oracle.make_golden_multi import BOOT, BOOT_CHAIN0, CLOUDS as FIXTURE_CLOUDS

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'multi_edges.npz')


@pytest.fixture(scope='module')
def edges():
    return np.load(GOLDEN)


@pytest.mark.parametrize('name', FIXTURE_CLOUDS)
def test_candidate_tree_vs_reference(edges, name):
    """The leaves of the oracle's candidate tree are the reference's: member sets exact, centres 1e-12,
    covariances 1e-9, log-volumes 1e-10.  Matched by member set: the sign LAPACK gives the major axis decides
    which end point seeds cluster 0, and with it the order of the leaves."""
    p = name + '_'
    pts = edges[p + 'points']
    assert np.array_equal(pts, MC.cloud(name))
    t = OB.candidate_tree(pts)
    K = len(edges[p + 'logvols'])
    assert len(t['leaves']) == K
    want = {tuple(edges[p + 'members_%d' % k]): k for k in range(K)}
    for i in t['leaves']:
        nd = t['nodes'][i]
        k = want[tuple(nd['members'])]
        close(nd['ell'].ctr, edges[p + 'ctrs'][k], rtol=1e-12)
        close(nd['ell'].cov, edges[p + 'covs'][k], rtol=1e-9)
        assert abs(nd['logvol'] - edges[p + 'logvols'][k]) <= 1e-10 * max(1.0, abs(edges[p + 'logvols'][k]))
    # and the recursion it restates gives the same leaves
    ells, members = OB.bounding_ellipsoids(pts)
    assert [list(m) for m in members] == [list(t['nodes'][i]['members']) for i in t['leaves']]


@pytest.mark.parametrize('name', BOOT)
@pytest.mark.parametrize('multi', [0, 1])
def test_bootstrap_expand_vs_reference(edges, name, multi):
    pts = edges[name + '_points']
    for r, want in enumerate(edges['boot_%s_%d' % (name, multi)]):
        s = philox.ChainStream(SEED, BOOT_CHAIN0 + r)
        sel = OB.bootstrap_split(len(pts), s.integers(len(pts), len(pts)))
        assert abs(OB.bootstrap_expand(pts, sel, bool(multi)) - want) <= 1e-9 * want


@pytest.mark.parametrize('name', ['two20000x8', 'three2100x50', 'two3600x33', 'two640x65', 'mix300x2late', 'few7x1'])
def test_kmeans2_matrix_vs_scipy(name):
    """kmeans2_matrix (and the traced copy candidate_tree uses) against scipy.cluster.vq.kmeans2(minit='matrix',
    iter=10) at the root of the cloud, from the reference's start centres."""
    pts = MC.cloud(name)
    scale = pts.std(axis=0)[None, :]
    p1, p2 = OB.bounding_ellipsoid(pts).major_axis_endpoints()
    start = np.vstack((p1, p2)) / scale
    code, lab = OB.kmeans2_matrix(pts / scale, start, 10)
    want_code, want_lab = vq.kmeans2(pts / scale, start.copy(), iter=10, minit='matrix')
    assert np.array_equal(lab, want_lab)
    close(code, want_code, rtol=1e-12)
    lab2, margin, _ = OB.kmeans2_trace(pts / scale, start, 10)
    assert np.array_equal(lab2, lab) and margin > 0


def _tree(name, cache={}):
    if name not in cache:
        cache[name] = OB.candidate_tree(MC.cloud(name))
    return cache[name]


@pytest.mark.parametrize('name', MC.CLOUDS)
def test_case_cloud_is_well_posed(name):
    t = _tree(name)
    assert t['km_margin'] > 1e-9
    assert t['eig_gap'] > 1e-6
    assert OB.decision_margin(t) > 1e-6
    ells, members = OB.bounding_ellipsoids(MC.cloud(name))
    assert [list(m) for m in members] == [list(t['nodes'][i]['members']) for i in t['leaves']]


def test_case_clouds_reach_every_decision():
    """Between them the clouds hit every outcome of a split: refused by the 2n minimum, rejected by both volume
    tests, accepted by the first, accepted by the second only; and labels that change in the 10th iteration."""
    t = _tree('mix300x2test2')
    assert {0, 1, 2} <= {nd['accept'] for nd in t['nodes']}
    for name in ('mix300x2late', 'mix300x2test2'):
        n = MC.cloud(name).shape[1]
        assert any(nd['split'] is not None and min(nd['split']) < 2 * n for nd in _tree(name)['nodes'])
    assert _tree('mix300x2late')['late']
    # resolve() with n (n + 1) / 2 parameters instead of n (n + 3) / 2 accepts another set of leaves here
    assert OB.candidate_tree(MC.cloud('mix300x2test2'), nparam=3)['leaves'] != t['leaves']


@pytest.mark.parametrize('name', MC.BOOT_CLOUDS)
def test_bootstrap_cloud_is_well_posed(name):
    pts = MC.boot_cloud(name)
    for r in range(8):
        s = philox.ChainStream(SEED, 77 + r)
        sel = OB.bootstrap_split(len(pts), s.integers(len(pts), len(pts)))
        t = OB.candidate_tree(pts[sel])
        assert t['km_margin'] > 1e-9 and t['eig_gap'] > 1e-6 and OB.decision_margin(t) > 1e-6

"""CPU tier: oracle/friends.py (RadFriends / SupFriends restated) against tests/golden/friends.npz and
friends_edges.npz, which the UNMODIFIED reference generated (oracle/make_golden.py gen_friends,
oracle/make_golden_friends.py; its draws replayed on the Philox stream); the clustering against scipy's single
linkage; the row-chunked pairwise distances against the whole-block arithmetic they replace."""
import math
import os

import numpy as np
import pytest

from oracle import friends as F, philox
from conftest import GOLDEN

SEED = 56432


def load_cases():
    """friends.npz and friends_edges.npz as one mapping; the n40 cloud's points and queries (stored once) appear
    under the per-kind keys of the other clouds."""
    g = dict(np.load(os.path.join(GOLDEN, 'friends.npz')))
    g.update(np.load(os.path.join(GOLDEN, 'friends_edges.npz')))
    for kind in ('balls', 'cubes'):
        for k in ('points', 'query', 'enlarge'):
            g['fr_n40_%s_%s' % (kind, k)] = g['fr_n40_' + k]
    return g


@pytest.fixture(scope='module')
def g():
    return load_cases()


def close(a, b, rtol=1e-9):
    np.testing.assert_allclose(a, b, rtol=rtol, atol=rtol * max(np.abs(b).max(), 1e-300))


@pytest.mark.parametrize('cname', ['blob', 'two', 'n40'])
@pytest.mark.parametrize('kind', ['balls', 'cubes'])
def test_friends_update_and_queries(g, cname, kind):
    p = 'fr_%s_%s_' % (cname, kind)
    pts = g[p + 'points']
    n = pts.shape[1]
    enlarge = float(g.get(p + 'enlarge', math.log(1.25)))
    b = F.Friends(n, kind)
    for rep in (1, 2):
        sub = pts if rep == 1 else pts[::-1][:len(pts) - 10]
        assert F.threshold_gap(sub, b.am) > 1e-9                  # the partition does not hinge on a last bit
        b.update(sub)                                             # leave-one-out radius
        q = p + 'u%d_' % rep
        close(b.cov, g[q + 'cov'])
        close(b.am, g[q + 'am'], rtol=1e-7)
        close(b.axes, g[q + 'axes'], rtol=1e-8)
        close(b.axes_inv, g[q + 'axes_inv'], rtol=1e-7)
        assert abs(b.logvol - float(g[q + 'logvol'])) < 1e-8
        b.scale_to_logvol(b.logvol + enlarge)                     # the Sampler's enlarge step (sampler.py:506-508)
    xs = g[p + 'query']
    assert F.query_gap(xs, b.ctrs, b.axes_inv, kind) > 1e-9
    assert np.array_equal(np.array([b.overlap(x) for x in xs]), g[p + 'overlap'])
    assert np.array_equal(np.array([b.contains(x) for x in xs]), g[p + 'contains'])
    pt = np.dot(b.ctrs, b.axes_inv)
    close(F.loo_radius(pt, kind), g[p + 'loo'], rtol=1e-7)
    boot = [F.bootstrap_radius(pt, kind, philox.ChainStream(SEED, 400 + r).integers(len(pt), len(pt))) for r in range(3)]
    close(np.array(boot), g[p + 'boot'], rtol=1e-7)
    draws, qs = [], []
    for c in range(30):
        draws.append(b.sample(philox.ChainStream(SEED, 500 + c)))
        x, qq = b.sample(philox.ChainStream(SEED, 600 + c), return_q=True)
        draws.append(x)
        qs.append(qq)
    close(np.array(draws), g[p + 'draws'], rtol=1e-8)
    assert np.array_equal(np.array(qs), g[p + 'draw_q'])
    assert all(b.contains(x) for x in draws)
    b.scale_to_logvol(b.logvol + 0.3)
    close(b.am, g[p + 'scaled_am'], rtol=1e-7)
    close(b.axes, g[p + 'scaled_axes'], rtol=1e-8)


def test_clusters_are_connected_components():
    rng = np.random.default_rng(3)
    pts = np.concatenate([0.2 + 0.01 * rng.standard_normal((40, 2)), 0.8 + 0.01 * rng.standard_normal((35, 2))])
    am = np.linalg.inv(np.cov(pts[:40], rowvar=False)) / 9.0       # distance 1 = 3 sigma of one blob
    lab = F.components_within(pts, am)
    assert lab.max() == 1 and len(set(lab[:40])) == 1 and len(set(lab[40:])) == 1 and lab[0] != lab[-1]
    try:
        from scipy import cluster, spatial
    except ImportError:
        return
    ref = cluster.hierarchy.fcluster(cluster.hierarchy.single(spatial.distance.pdist(pts, 'mahalanobis', VI=am)), 1.0,
                                     criterion='distance')
    assert len(set(zip(lab, ref))) == 2                            # same partition, labels aside


@pytest.mark.parametrize('kind', ['balls', 'cubes'])
def test_path_cloud_update(g, kind):
    """Three shuffled curves (friends_edges.npz path_*): the labels need more than 8 sweeps of the kernel's rule,
    i.e. cross two of the host's 4-sweep batches; the update clustering under path_am0 matches the reference."""
    pts, am0 = g['path_points'], g['path_am0']
    adj = F.mahalanobis_pairs(pts, am0) <= 1.0
    lab, sweeps = F.label_sweeps(adj)
    assert sweeps > 8
    assert F.threshold_gap(pts, am0) > 1e-9
    assert len(set(lab)) == 3 and F.components_within(pts, am0).max() == 2
    assert len(set(zip(lab, F.components_within(pts, am0)))) == 3          # the same partition
    b = F.Friends(2, kind)
    b.am = am0
    b.update(pts)
    q = 'path_%s_' % kind
    close(b.cov, g[q + 'cov'])
    close(b.am, g[q + 'am'], rtol=1e-7)
    close(b.axes, g[q + 'axes'], rtol=1e-8)
    close(b.axes_inv, g[q + 'axes_inv'], rtol=1e-7)
    assert abs(b.logvol - float(g[q + 'logvol'])) < 1e-8


def _scipy_clusters(pts, am):
    from scipy import cluster, spatial
    return cluster.hierarchy.fcluster(cluster.hierarchy.single(spatial.distance.pdist(pts, 'mahalanobis', VI=am)), 1.0,
                                      criterion='distance')


@pytest.mark.parametrize('cloud', ['path', 'singletons'])
def test_components_match_single_linkage(g, cloud):
    """components_within == fcluster(single(pdist)) cut at 1, on the path cloud and on 12 curves, 8 of them single
    points (clusters of one)."""
    pytest.importorskip('scipy')
    if cloud == 'path':
        pts, am = g['path_points'], g['path_am0']
    else:
        pts, am = F.chain_cloud(np.random.default_rng(8), (7, 1, 5, 1, 1, 9, 1, 1, 3, 1, 1, 1), 3)
    assert F.threshold_gap(pts, am) > 1e-9
    lab, ref = F.components_within(pts, am), _scipy_clusters(pts, am)
    k = lab.max() + 1
    assert k == ref.max() == (3 if cloud == 'path' else 12)
    assert len(set(zip(lab, ref))) == k                                       # same partition, labels aside
    assert np.array_equal(np.unique(F.label_sweeps(F.mahalanobis_pairs(pts, am) <= 1.0)[0], return_inverse=True)[1], lab)


def test_row_chunks_are_bit_identical(g):
    """The row-chunked pairwise distances equal, bit for bit, the whole (N, N, n) block arithmetic they replace, for
    chunks of one row, of a few rows and of the whole block."""
    def whole_mahal(pts, am):
        d = pts[:, None, :] - pts[None, :, :]
        return np.sqrt(np.clip(np.einsum('ijk,kl,ijl->ij', d, am, d), 0.0, None))

    def whole_dist(a, b, kind):
        d = a[:, None, :] - b[None, :, :]
        return np.sqrt((d * d).sum(-1)) if kind == 'balls' else np.abs(d).max(-1)

    for cname in ('blob', 'two'):
        for kind in ('balls', 'cubes'):
            p = 'fr_%s_%s_' % (cname, kind)
            pts = g[p + 'points']
            am, axes_inv = g[p + 'u1_am'], g[p + 'u1_axes_inv']
            pt = np.dot(pts, axes_inv)
            N, n = pts.shape
            idxs = philox.ChainStream(SEED, 400).integers(N, N)
            sel = F.bootstrap_split(N, idxs)
            for budget in (1, 7 * N * n, None):
                assert F._row_chunks(N, N, n, budget)[0].stop == (N if budget is None else max(1, (budget // (N * n))))
                assert np.array_equal(F.mahalanobis_pairs(pts, am, budget), whole_mahal(pts, am))
                assert np.array_equal(F.components_within(pts, am, budget=budget),
                                      F.components_within(pts, am, budget=N * N * n))
                assert np.array_equal(F.loo_radius(pt, kind, budget), np.sort(whole_dist(pt, pt, kind), axis=1)[:, 1])
                assert F.bootstrap_radius(pt, kind, idxs, budget) == whole_dist(pt[~sel], pt[sel], kind).min(1).max()

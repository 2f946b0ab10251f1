"""Point clouds for the checks of the multi-ellipsoid decomposition (csrc/b2n_multi.cu) against the oracle.

TEST INFRASTRUCTURE.  Each cloud sits where a kernel of the bound update changes form; tests/test_gpu_multi.py
derives which form from the device limits, and tests/test_oracle_multi.py checks that every cloud is well-posed
(k-means margins, eigengaps and volume-test margins, oracle.bounding.candidate_tree).  Seeded: the same arrays on
every machine.
"""
import numpy as np

SEED = 56432


def _two(rng, sizes, n, lo=0.3, hi=0.7, spread=0.02):
    return np.concatenate([lo + spread * rng.standard_normal((sizes[0], n)),
                           hi + spread * rng.standard_normal((sizes[1], n))])


def _crossed(rng, sizes, n):
    """Two clusters, each wide in one half of the dimensions and thin in the other: splitting them shrinks the
    volume by far more than the reference's threshold, even where n (n + 3) / 2 parameters make it large."""
    wide = np.where(np.arange(n) < n // 2, 0.03, 0.003)
    return np.concatenate([0.35 + wide * rng.standard_normal((sizes[0], n)),
                           0.65 + wide[::-1] * rng.standard_normal((sizes[1], n))])


def _mix(seed, n, k, npts, spread):
    """k Gaussian clusters of Dirichlet sizes and uneven axis scales, shuffled."""
    rng = np.random.default_rng(seed)
    ctrs = 0.2 + 0.6 * rng.random((k, n))
    w = rng.dirichlet(np.ones(k) * 2)
    sizes = np.maximum(1, (w * npts).astype(int))
    parts = [c + spread * rng.standard_normal((s, n)) * rng.uniform(0.3, 1.5, n) for c, s in zip(ctrs, sizes)]
    return rng.permutation(np.concatenate(parts))


def cloud(name):
    rng = np.random.default_rng(SEED + sum(map(ord, name)))
    if name == 'two20000x8':          # the root's k-means CTAs hold 2500 rows: more than their stage, deeper nodes fit
        return _two(rng, (12000, 8000), 8)
    if name == 'three2100x50':        # 262 or 263 rows per CTA: the root's CTAs straddle the stage at n = 50
        ctrs = 0.2 + 0.6 * rng.random((3, 50))
        return rng.permutation(np.concatenate([c + 0.02 * rng.standard_normal((s, 50))
                                               for c, s in zip(ctrs, (1100, 600, 400))]))
    if name == 'gauss2000x50':        # the C2 shape: unimodal, the root is the accepted leaf
        cm = np.full((50, 50), 0.4)
        np.fill_diagonal(cm, 1.0)
        return 0.5 + 0.02 * rng.standard_normal((2000, 50)) @ np.linalg.cholesky(cm).T
    if name == 'few7x1':              # 7 rows over the 8 CTAs of a k-means node
        return np.concatenate([0.2 + 0.01 * rng.standard_normal((3, 1)), 0.8 + 0.01 * rng.standard_normal((4, 1))])
    if name == 'few18x2':             # every node has fewer rows than CTAs
        return np.concatenate([c + 0.01 * rng.standard_normal((s, 2))
                               for c, s in zip(([0.2, 0.2], [0.8, 0.3], [0.5, 0.8]), (7, 6, 5))])
    if name == 'two3600x33':          # odd n: unequal column halves; two lane passes of the warp loop at the root
        return _two(rng, (2000, 1600), 33)
    if name in ('two640x64', 'two640x65'):     # the two register tilings of the Cholesky candidates
        return _crossed(rng, (320, 320), int(name[-2:]))
    if name == 'two600x119':          # the largest n of the Cholesky candidates
        return _crossed(rng, (300, 300), 119)
    if name == 'two600x120':          # eigen-path candidates, sliced solver
        return _crossed(rng, (300, 300), 120)
    if name == 'two700x150':
        return _crossed(rng, (350, 350), 150)
    if name == 'mix300x2late':        # labels still change in the 10th Lloyd iteration; refused and rejected splits
        return _mix(0, 2, 3, 300, 0.06)
    if name == 'mix300x2test2':       # a split accepted by the second volume test only; refused and rejected splits
        return _mix(0, 2, 3, 300, 0.1)
    if name == 'illcond600x12':       # the root's covariance needs the repair ladder: no certified candidate
        p = 0.5 + 0.05 * rng.standard_normal((600, 12))
        p[:, 11] = p[:, 0] + 1e-9 * rng.standard_normal(600)
        return p
    raise KeyError(name)


CLOUDS = ('two20000x8', 'three2100x50', 'gauss2000x50', 'few7x1', 'few18x2', 'two3600x33', 'two640x64',
          'two640x65', 'two600x119', 'two600x120', 'two700x150', 'mix300x2late', 'mix300x2test2', 'illcond600x12')


def boot_cloud(name):
    """Clouds of the bootstrap-expansion checks: odd N, an in-bag set that splits (n = 8), one too small to
    split, n = 65."""
    rng = np.random.default_rng(SEED + 7 + sum(map(ord, name)))
    if name == 'odd401x5':
        return 0.5 + 0.05 * rng.standard_normal((401, 5))
    if name == 'split999x8':
        return _two(rng, (600, 399), 8)
    if name == 'small45x10':          # ~29 rows in the bag: fewer than the 4 n = 40 a split needs
        return 0.5 + 0.05 * rng.standard_normal((45, 10))
    if name == 'two641x65':
        return _crossed(rng, (321, 320), 65)
    raise KeyError(name)


BOOT_CLOUDS = ('odd401x5', 'split999x8', 'small45x10', 'two641x65')

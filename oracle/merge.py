"""Merging runs (the reference's merge_runs), restated in numpy.

TEST INFRASTRUCTURE (see oracle/__init__.py).  What is restated (reference py/dynesty/utils.py):
  merge_runs         :1817-1900   base runs as a pairwise tree, then the add-on runs one at a time
  _merge_two         :2045-2225   the walk: order (ties to the base side) and live counts (low-edge rule)
  ln X of _merge_two :2159-2187   ln((n+1)/n) per point, the plateau rule inside a group of equal logl
  compute_integrals  :1411-1467   dynesty_b200.nested._integrate (same quadrature)
Same contract as ``dynesty_b200.ops.merge_runs`` (include/b200nest.h, b2n_merge_runs).
"""
import numpy as np


def _rule(lb, nb, ln, nn, eb, en):
    """_merge_two's count of the merged point (:2131-2145) from the base / new runs' current logl and counts."""
    return np.where((lb > en) & (ln > eb), nb + nn, np.where(lb <= en, nb, nn))


def merge_two(la, na, lb, nb, ea, eb):
    """One _merge_two walk of two ascending records, vectorised: A's point i goes to i + #{b < a}, B's point j to
    j + #{a <= b}; each takes the other run's logl / count at the other run's pointer (+inf / 0 once exhausted).
    Returns (pos_a, pos_b, n): the merged positions and the merged counts."""
    j = np.searchsorted(lb, la, side='left')
    i = np.searchsorted(la, lb, side='right')
    bl = np.where(j < len(lb), lb[np.minimum(j, len(lb) - 1)], np.inf)
    bn = np.where(j < len(lb), nb[np.minimum(j, len(lb) - 1)], 0)
    al = np.where(i < len(la), la[np.minimum(i, len(la) - 1)], np.inf)
    an = np.where(i < len(la), na[np.minimum(i, len(la) - 1)], 0)
    pos_a, pos_b = np.arange(len(la)) + j, np.arange(len(lb)) + i
    n = np.empty(len(la) + len(lb), dtype=np.int64)
    n[pos_a] = _rule(la, na, bl, bn, ea, eb)
    n[pos_b] = _rule(al, an, lb, nb, ea, eb)
    return pos_a, pos_b, n


def _merge_nodes(x, y):
    """Merge two nodes dict(logl, n, src, edge), x the base side."""
    pa, pb, n = merge_two(x['logl'], x['n'], y['logl'], y['n'], x['edge'], y['edge'])
    out = dict(n=n, edge=min(x['edge'], y['edge']))
    for k in ('logl', 'src'):
        v = np.empty(len(n), dtype=x[k].dtype)
        v[pa], v[pb] = x[k], y[k]
        out[k] = v
    return out


def merge_order_counts(logl, samples_n, run_ptr, nbase, lowedge=None):
    """The merged order and counts of merge_runs (:1859-1896): (perm, n)."""
    logl, n = np.asarray(logl, dtype=float), np.asarray(samples_n, dtype=np.int64)
    R = len(run_ptr) - 1
    le = np.full(R, -np.inf) if lowedge is None else np.asarray(lowedge, dtype=float)
    nodes = [dict(logl=logl[a:b], n=n[a:b], src=np.arange(a, b, dtype=np.int64), edge=float(le[r]))
             for r, (a, b) in enumerate(zip(run_ptr[:-1], run_ptr[1:]))]
    base = nodes[:nbase]
    while len(base) > 1:
        base = [_merge_nodes(base[k], base[k + 1]) if k + 1 < len(base) else base[k] for k in range(0, len(base), 2)]
    acc = base[0]
    for x in nodes[nbase:]:
        acc = _merge_nodes(acc, x)
    return acc['src'], acc['n']


def flat_order_counts(logl, samples_n, run_ptr):
    """The flat rule equal to the base tree when every low edge is -inf (DESIGN.md section 15.2): a stable sort of the
    concatenation by logl, and at every merged point the sum over runs of each run's count at its first point not yet
    merged (0 once exhausted).  Returns (perm, n)."""
    logl, n = np.asarray(logl, dtype=float), np.asarray(samples_n, dtype=np.int64)
    N = len(logl)
    perm = np.argsort(logl, kind='stable')
    pos = np.empty(N, dtype=np.int64)
    pos[perm] = np.arange(N)
    # run r contributes n_r[k] on merged positions pos_r[k-1] + 1 .. pos_r[k], and 0 after its last point
    diff = np.zeros(N + 1, dtype=np.int64)
    for a, b in zip(run_ptr[:-1], run_ptr[1:]):
        p, c = pos[a:b], n[a:b]
        np.add.at(diff, np.r_[0, p[:-1] + 1], c - np.r_[0, c[:-1]])
        diff[p[-1] + 1] -= c[-1]
    return perm, np.cumsum(diff)[:N]


def log_t(logl, n):
    """ln t per merged point (:2159-2187): -ln((n+1)/n), and inside a group of m >= 2 equal logl whose first point has
    count n, ln((n-k)/(n-k+1)) for its k-th point (X falls by X_0 / (n+1) at each of them)."""
    logl, n = np.asarray(logl, dtype=float), np.asarray(n, dtype=np.int64)
    start = np.searchsorted(logl, logl, side='left')
    k = np.arange(len(logl)) - start
    with np.errstate(divide='ignore', invalid='ignore'):
        return -np.log1p(1.0 / (n[start] - k).astype(float))


def merge_runs(logl, samples_n, run_ptr, nbase, lowedge=None, arrays=True):
    """Same contract as ``dynesty_b200.ops.merge_runs``."""
    from dynesty_b200.nested import _integrate
    perm, n = merge_order_counts(logl, samples_n, np.asarray(run_ptr, dtype=np.int64), int(nbase), lowedge)
    lm = np.asarray(logl, dtype=float)[perm]
    logvol = np.cumsum(log_t(lm, n))
    logwt, logz, logzvar, h = _integrate(lm, logvol)
    o = dict(perm=perm, samples_n=n, logz_end=float(logz[-1]), logzerr_end=float(np.sqrt(abs(logzvar[-1]))),
             h_end=float(h[-1]))
    if arrays:
        o.update(logvol=logvol, logwt=logwt, logz=logz, logzvar=logzvar, h=h)
    return o

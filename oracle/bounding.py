"""numpy restatement of dynesty's ellipsoid bounding (single + multi).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Citations are to
py/dynesty/bounding.py unless noted.
"""
import math
import numpy as np
from scipy.special import gammaln, logsumexp

ONE_MINUS_A_BIT = 1.0 - 1e-3          # bounding.py:1418-1424
MAX_COND = 1e12                       # bounding.py:1311
EIG_MULT = 10.0                       # bounding.py:1326


def logvol_prefactor(n):
    """ln volume of the unit n-ball (bounding.py:1271-1285, p=2)."""
    return n * math.log(2.) + n * gammaln(1.5) - gammaln(n / 2. + 1)


class Ell:
    """State of one ellipsoid (bounding.py:201-240)."""

    def __init__(self, ctr, cov, am=None, axes=None):
        self.ctr = np.asarray(ctr, dtype=float)
        self.cov = np.asarray(cov, dtype=float)
        self.ndim = self.ctr.shape[0]
        lam, vec = np.linalg.eigh(self.cov)                      # :212
        if not np.all((lam > 0.) & np.isfinite(lam)):             # :213,218
            raise ValueError("singular ellipsoid")
        self.axlens = np.sqrt(lam)                                # :214
        self.logvol = logvol_prefactor(self.ndim) + 0.5 * np.log(lam).sum()  # :217
        self.axes = vec * self.axlens if axes is None else axes   # :227-230
        self.am = (vec / lam) @ vec.T if am is None else am       # :232-236

    @classmethod
    def unit_default(cls, ndim):
        """Ellipsoid(ndim) with no centre: ctr = 0 (sic), cov = I n/4 (:203-205)."""
        return cls(np.zeros(ndim), np.identity(ndim) * ndim / 4)

    def major_axis_endpoints(self):                               # :278-284
        i = int(np.argmax(self.axlens))
        v = self.axes[:, i]
        return self.ctr - v, self.ctr + v

    def mahal2(self, x):
        """Squared normalised distance of each row of x (:286-300)."""
        d = np.atleast_2d(x) - self.ctr
        return np.einsum('ij,jk,ik->i', d, self.am, d)

    def scale_to_logvol(self, logvol):                            # :242-276
        n = self.ndim
        logf = logvol - self.logvol
        max_log_axlen = math.log(math.sqrt(n) / 2)
        log_axlen = np.log(self.axlens)
        if log_axlen.max() < max_log_axlen - logf / n:
            f = math.exp(logf / n)
            self.cov = self.cov * f**2
            self.am = self.am * (1. / f**2)
            self.axlens = self.axlens * f
            self.axes = self.axes * f
        else:
            logfax = np.zeros(n)
            cur, left = logf, n
            lam, vec = np.linalg.eigh(self.cov)
            for i in np.argsort(lam)[::-1]:
                delta = max(min(max_log_axlen - log_axlen[i], cur / left), 0)
                logfax[i] = delta
                cur -= delta
                left -= 1
            fax = np.exp(logfax)
            lam1 = lam * fax**2
            self.cov = (vec * lam1) @ vec.T
            self.am = (vec * (1. / lam1)) @ vec.T
            self.axlens = self.axlens * fax
            self.axes = self.axes * fax
        self.logvol = logvol


def improve_covar_mat(covar0, ntries=100):
    """Condition-number repair ladder (bounding.py:1311-1384).
    Returns (good, covar, am, axes, status) ; status 0 ok / 1 fell back to identity."""
    n = covar0.shape[0]
    covar = np.array(covar0, dtype=float)
    coeffmin = 1e-10
    failed = 0
    for trial in range(ntries):
        failed = 0
        lam, vec = np.linalg.eigh(covar)
        mx, mn = lam.max(), lam.min()
        if np.isfinite(lam).all():
            if mx <= 0:
                failed = 2
            elif mn < mx / MAX_COND:
                failed = 1
            else:
                axes = vec * lam**.5
                break
        else:
            failed = 2
        if failed == 1:
            lam_fix = np.maximum(lam, EIG_MULT * mx / MAX_COND)
            covar = (vec * lam_fix) @ vec.T
        else:
            coeff = coeffmin * (1. / coeffmin)**(trial * 1. / (ntries - 1))
            covar = (1. - coeff) * covar + coeff * np.eye(n)
    if failed > 0:
        covar = np.eye(n)
        return False, covar, covar.copy(), covar.copy(), 1
    am = (vec * (1. / lam)) @ vec.T
    return trial == 0, covar, am, axes, 0


def bounding_ellipsoid(points):
    """bounding.py:1387-1461."""
    points = np.asarray(points, dtype=float)
    npts, n = points.shape
    if npts == 1:
        raise ValueError("single point")
    ctr = points.mean(axis=0)
    covar = np.atleast_2d(np.cov(points, rowvar=False))          # ddof=1
    delta = points - ctr
    for i in range(2):
        good, covar, am, axes, _ = improve_covar_mat(covar)
        fmax = np.einsum('ij,jk,ik->i', delta, am, delta).max()
        if i == 0 and fmax > ONE_MINUS_A_BIT:
            mult = fmax / ONE_MINUS_A_BIT
            covar = covar * mult
            am = am / mult
            axes = axes * math.sqrt(mult)
        if i == 1 and fmax >= 1:
            raise RuntimeError("Failed to initialize the ellipsoid")
        if good:
            break
    return Ell(ctr, covar, am=am, axes=axes)


def kmeans2_matrix(data, centres, niter=10):
    """scipy.cluster.vq.kmeans2(data, k=centres, iter=niter, minit='matrix')
    restated (scipy 1.18.1 cluster/vq.py kmeans2 loop): nearest-centre labels
    (ties -> lowest index), centroid = member mean, an empty cluster keeps its
    previous centre; the returned labels are those of the LAST assignment, i.e.
    computed before the final centroid update."""
    code = np.array(centres, dtype=float)
    k = code.shape[0]
    label = None
    for _ in range(niter):
        d2 = ((data[:, None, :] - code[None, :, :])**2).sum(axis=2)
        label = np.argmin(d2, axis=1)
        new = code.copy()
        for j in range(k):
            m = label == j
            if m.any():
                new[j] = data[m].mean(axis=0)
        code = new
    return code, label


def bounding_ellipsoids(points, ell=None, scale=None, idx=None):
    """bounding.py:1464-1563 / 1566-1590.  Returns (ells, members) where
    members[k] is the sorted index array (into the top-level `points`) of the
    points that ellipsoid k was fitted to."""
    points = np.asarray(points, dtype=float)
    npts, n = points.shape
    if idx is None:
        idx = np.arange(npts)
    if ell is None:
        ell = bounding_ellipsoid(points)
    min_size = 2 * n
    if npts < 2 * min_size:                                       # :1493
        return [ell], [idx]
    p1, p2 = ell.major_axis_endpoints()                           # :1500
    start = np.vstack((p1, p2))
    if scale is None:
        scale = points.std(axis=0)[None, :]                       # :1503-1504 (ddof=0)
    _, labels = kmeans2_matrix(points / scale, start / scale, 10)  # :1510-1515
    sel = [labels == 0, labels == 1]
    if min(sel[0].sum(), sel[1].sum()) < min_size:                # :1521
        return [ell], [idx]
    kids = [bounding_ellipsoid(points[s]) for s in sel]           # :1525
    nparam = (n * (n + 3)) // 2
    log_vol_dec = nparam * math.log(npts) / npts                  # :1541-1542
    out_e, out_m = [], []
    for s, kid in zip(sel, kids):                                 # :1548-1549
        e, m = bounding_ellipsoids(points[s], kid, scale, idx[s])
        out_e += e
        out_m += m
    if np.logaddexp(kids[0].logvol, kids[1].logvol) - ell.logvol < -log_vol_dec:
        return out_e, out_m                                       # :1552-1554
    if (logsumexp([e.logvol for e in out_e]) - ell.logvol <
            -log_vol_dec * (len(out_e) - 1)):                     # :1558-1560
        return out_e, out_m
    return [ell], [idx]


class MultiEll:
    """Stacked arrays of a MultiEllipsoid (bounding.py:440-476)."""

    def __init__(self, ells):
        self.ells = list(ells)
        self.refresh()

    def refresh(self):
        self.nells = len(self.ells)
        self.ctrs = np.array([e.ctr for e in self.ells])
        self.covs = np.array([e.cov for e in self.ells])
        self.ams = np.array([e.am for e in self.ells])
        self.axes = np.array([e.axes for e in self.ells])
        self.logvol_ells = np.array([e.logvol for e in self.ells])
        self.logvol = logsumexp(self.logvol_ells)

    def mahal2(self, x):
        """(M, K) squared normalised distances (bounding.py:506-507)."""
        d = np.atleast_2d(x)[:, None, :] - self.ctrs[None, :, :]
        return np.einsum('mai,aij,maj->ma', d, self.ams, d)

    def within_mask(self, x):                                     # :502-510 strict <
        return self.mahal2(x) < 1

    def scale_to_logvol(self, logvol):                            # :478-495
        if np.ndim(logvol) > 0:
            new = np.asarray(logvol, dtype=float)
        else:
            new = self.logvol_ells + (logvol - self.logvol)
        for e, lv in zip(self.ells, new):
            e.scale_to_logvol(lv)
        self.refresh()


def multi_update(points):
    """MultiEllipsoid.update without bootstrap (bounding.py:665-686)."""
    points = np.asarray(points, dtype=float)
    if points.shape[0] == 1:
        raise RuntimeError("single point")
    first = bounding_ellipsoid(points)
    ells, members = bounding_ellipsoids(points, first)
    me = MultiEll(ells)
    if not me.within_mask(points).any(axis=1).all():              # :683-685
        raise RuntimeError('Rejecting invalid MultiEllipsoid region')
    return me, members


def bootstrap_split(npoints, idxs):
    """In/out masks given the resampled indices (bounding.py:1603-1616)."""
    sel = np.zeros(npoints, dtype=bool)
    sel[np.unique(idxs)] = True
    n_in = sel.sum()
    if n_in < 2:
        sel[:2] = True
    if n_in > npoints - 1:
        sel[0] = False
    return sel


def bootstrap_expand(points, sel_in, multi):
    """bounding.py:1619-1648 given the in-bag mask."""
    pin, pout = points[sel_in], points[~sel_in]
    ell = bounding_ellipsoid(pin)
    if not multi:
        d = np.sqrt(ell.mahal2(pout))
    else:
        ells, _ = bounding_ellipsoids(pin, ell)
        d = np.min(np.array([np.sqrt(e.mahal2(pout)) for e in ells]), axis=0)
    return max(1., float(np.max(d)))


# ---- the whole candidate tree of bounding_ellipsoids, with what makes a comparison with it well-posed
def kmeans2_trace(data, centres, niter=10):
    """kmeans2_matrix with its conditioning: (labels, margin, late) where margin is the smallest relative
    distance gap |d0 - d1| / (d0 + d1) of any point in any of the niter assignments (two centres) and late
    says whether the last assignment changed any label of the one before."""
    code = np.array(centres, dtype=float)
    margin, prev, late = np.inf, None, False
    for _ in range(niter):
        d2 = ((data[:, None, :] - code[None, :, :])**2).sum(axis=2)
        label = np.argmin(d2, axis=1)
        s = d2[:, 0] + d2[:, 1]
        gap = np.abs(d2[:, 0] - d2[:, 1])
        margin = min(margin, float(np.min(np.where(s > 0, gap / np.where(s > 0, s, 1.0), 0.0))))
        late = prev is not None and bool(np.any(label != prev))
        prev = label
        for j in range(2):
            m = label == j
            if m.any():
                code[j] = data[m].mean(axis=0)
    return prev, margin, late


def candidate_tree(points, nparam=None):
    """bounding_ellipsoids restated to return the WHOLE candidate tree (the reference fits both children of every
    split before it applies its volume tests, :1525-1560, so the tree does not depend on the tests).

    Returns dict(nodes, leaves, km_margin, eig_gap, late).  nodes[i]: members (sorted indices into `points`),
    ell (its bounding_ellipsoid), logvol, depth, children (two node ids or None), split (the k-means cluster sizes,
    None if no split was attempted), accept (None: no children; 0 rejected, 1 accepted by the first volume test
    :1552, 2 by the second :1558) and dist (how far the evaluated tests lie from their thresholds, in ln volume).
    leaves: the accepted leaves in the reference's order.  km_margin: smallest relative k-means margin over every
    split node, point and Lloyd iteration; eig_gap: smallest relative gap between the two largest eigenvalues of a
    split node's covariance (it fixes the major axis and so the start centres); late: some split node's labels
    still changed in the last Lloyd iteration.  nparam overrides n (n + 3) / 2 (:1541)."""
    points = np.asarray(points, dtype=float)
    npts, n = points.shape
    min_size = 2 * n
    scale = points.std(axis=0)[None, :]
    if nparam is None:
        nparam = (n * (n + 3)) // 2
    nodes = []
    cond = dict(km_margin=np.inf, eig_gap=np.inf, late=False)

    def expand(idx, ell, depth):
        i = len(nodes)
        nodes.append(dict(members=idx, ell=ell, logvol=ell.logvol, depth=depth, children=None, split=None,
                          accept=None, dist=()))
        if len(idx) < 2 * min_size:                               # :1493
            return i
        lam = np.sort(ell.axlens)**2
        if n > 1:
            cond['eig_gap'] = min(cond['eig_gap'], (lam[-1] - lam[-2]) / lam[-1])
        p1, p2 = ell.major_axis_endpoints()
        labels, margin, late = kmeans2_trace(points[idx] / scale, np.vstack((p1, p2)) / scale)
        cond['km_margin'] = min(cond['km_margin'], margin)
        cond['late'] = cond['late'] or late
        sel = [labels == 0, labels == 1]
        nodes[i]['split'] = (int(sel[0].sum()), int(sel[1].sum()))
        if min(nodes[i]['split']) < min_size:                      # :1521
            return i
        nodes[i]['children'] = [expand(idx[s], bounding_ellipsoid(points[idx[s]]), depth + 1) for s in sel]
        return i

    def resolve(i):
        nd = nodes[i]
        if nd['children'] is None:
            return [i]
        c0, c1 = nd['children']
        sub = resolve(c0) + resolve(c1)
        cnt = len(nd['members'])
        dec = nparam * math.log(cnt) / cnt                       # :1541-1542
        t1 = np.logaddexp(nodes[c0]['logvol'], nodes[c1]['logvol']) - nd['logvol'] + dec
        t2 = logsumexp([nodes[s]['logvol'] for s in sub]) - nd['logvol'] + dec * (len(sub) - 1)
        if t1 < 0:
            nd['accept'], nd['dist'] = 1, (abs(t1),)
            return sub
        nd['dist'] = (abs(t1), abs(t2))
        nd['accept'] = 2 if t2 < 0 else 0
        return sub if t2 < 0 else [i]

    expand(np.arange(npts), bounding_ellipsoid(points), 0)
    leaves = resolve(0)
    return dict(nodes=nodes, leaves=leaves, **cond)


def decision_margin(tree):
    """Smallest distance of an evaluated volume test from its threshold (inf if nothing was split)."""
    return min([d for nd in tree['nodes'] for d in nd['dist']], default=np.inf)


def tree_by_members(tree):
    """{tuple(sorted members): node id}: children are matched by their member SETS, because the sign of the
    major-axis eigenvector (LAPACK's or the CUDA solver's) decides which end point seeds cluster 0."""
    return {tuple(nd['members']): i for i, nd in enumerate(tree['nodes'])}

"""Generate tests/golden/multi_edges.npz by running the UNMODIFIED reference's MultiEllipsoid.

TEST INFRASTRUCTURE.  Run where the reference copy oracle/_ref exists (oracle/install_ref.py):

    python -m oracle.make_golden_multi

The conventions are those of oracle/make_golden.py gen_multi (same seed, same output directory, the bootstrap
draws replayed on the Philox stream through ``oracle.philox.ScriptedGenerator``).  The clouds are three of
oracle/multicases.py, where tests/golden/multi.npz (n <= 10, N <= 1600) does not reach:
  two640x65      n = 65: the wider register tiling of the Cholesky candidates, two accepted leaves;
  mix300x2late   labels that still change in the 10th Lloyd iteration, refused and rejected splits;
  mix300x2test2  a split accepted by the second volume test only.
Keys per cloud <name>_: points, and per leaf k (the reference's order) ctrs, covs, ams, logvols and the member
set members_<k> (row indices of the points the leaf was fitted to).  The reference does not return member sets:
they are read off by wrapping its bounding_ellipsoid while MultiEllipsoid.update runs, so every number is still
the reference's own.  boot_<name>_<multi>: _ellipsoid_bootstrap_expand for chains 2000 + rep, rep < 3, on the
clouds two640x65 and oracle.multicases.boot_cloud odd401x5 / split999x8 (whose points are stored too).
tests/test_oracle_multi.py checks the oracle against this file and tests/test_gpu_multi.py the kernels.
"""
import os

import numpy as np

from . import multicases, philox, refshim
from .make_golden import OUT, SEED

CLOUDS = ('two640x65', 'mix300x2late', 'mix300x2test2')
BOOT = ('two640x65', 'odd401x5', 'split999x8')
BOOT_CHAIN0 = 2000


def leaves_with_members(B, pts):
    """MultiEllipsoid.update on pts; (me, members) with members[k] the rows leaf k was fitted to."""
    fitted = {}
    orig = B.bounding_ellipsoid

    def recording(points):
        ell = orig(points)
        fitted[id(ell)] = np.array(points, copy=True)
        return ell

    rows = {p.tobytes(): i for i, p in enumerate(pts)}
    assert len(rows) == len(pts)
    B.bounding_ellipsoid = recording
    try:
        me = B.MultiEllipsoid(pts.shape[1])
        me.update(pts)
    finally:
        B.bounding_ellipsoid = orig
    members = [np.sort([rows[p.tobytes()] for p in fitted[id(e)]]) for e in me.ells]
    return me, members


def gen_multi_edges(B):
    out = {}
    for name in CLOUDS:
        pts = multicases.cloud(name)
        me, members = leaves_with_members(B, pts)
        p = name + '_'
        out[p + 'points'] = pts
        out[p + 'ctrs'], out[p + 'covs'], out[p + 'ams'] = me.ctrs, me.covs, me.ams
        out[p + 'logvols'] = np.array([e.logvol for e in me.ells])
        for k, m in enumerate(members):
            out[p + 'members_%d' % k] = m.astype(np.int32)
    for name in BOOT:
        pts = multicases.cloud(name) if name in CLOUDS else multicases.boot_cloud(name)
        if name not in CLOUDS:
            out[name + '_points'] = pts
        for multi in (0, 1):
            out['boot_%s_%d' % (name, multi)] = np.array([
                B._ellipsoid_bootstrap_expand((bool(multi), pts, philox.ScriptedGenerator(SEED, BOOT_CHAIN0 + r)))
                for r in range(3)])
    np.savez_compressed(os.path.join(OUT, 'multi_edges.npz'), **out)
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    refshim.import_reference()
    from dynesty import bounding as B
    gen_multi_edges(B)
    f = os.path.join(OUT, 'multi_edges.npz')
    print('wrote', f, os.path.getsize(f))


if __name__ == '__main__':
    main()

"""Generate tests/golden/friends_edges.npz by running the UNMODIFIED reference's RadFriends / SupFriends.

TEST INFRASTRUCTURE.  Run where the reference copy oracle/_ref exists (oracle/install_ref.py):

    python -m oracle.make_golden_friends

The fixture conventions are those of oracle/make_golden.py gen_friends (same seed, same output directory, draws
replayed on the Philox stream through ``oracle.philox.ScriptedGenerator``).  The clouds sit where the CUDA kernels of
csrc/b2n_friends.cu change form and friends.npz does not reach:
  n40   40 dimensions (the lane loops of the transform, overlap and draw kernels take two passes), two clusters of
        130 points: the keys of gen_friends under the prefix fr_n40_<kind>_, the points and queries once (fr_n40_points,
        fr_n40_query).  Each update is followed by an enlargement of fr_n40_enlarge in log-volume (every axis x 4)
        instead of gen_friends' log 1.25: the Chebyshev radius of 260 points in 40-D is so short that, enlarged
        less, the cubes' second update would cluster every point on its own (a zero covariance);
  path  three shuffled curves of 150, 110 and 40 points in 2-D (oracle.friends.chain_cloud): label propagation
        needs more than 8 sweeps to join each curve (oracle.friends.label_sweeps), so the labels cross several of
        the host's 4-sweep batches.  One update per kind clustering under the metric path_am0.
tests/test_oracle_friends.py checks the oracle against this file and tests/test_gpu_friends.py the kernels.
"""
import os

import numpy as np

from . import friends, philox, refshim
from .make_golden import OUT, SEED


def gen_friends_edges(B):
    rng = np.random.default_rng(SEED + 11)
    out = {}
    n = 40
    pts = np.concatenate([0.25 + 0.02 * rng.standard_normal((130, n)), 0.75 + 0.02 * rng.standard_normal((130, n))])
    out['fr_n40_points'] = pts
    xs = np.concatenate([pts[:20] + 0.01 * rng.standard_normal((20, n)), 0.25 + 0.5 * rng.random((20, n))])
    out['fr_n40_query'] = xs
    out['fr_n40_enlarge'] = enlarge = np.float64(n * np.log(4.0))
    for kind, cls in (('balls', B.RadFriends), ('cubes', B.SupFriends)):
        p = 'fr_n40_%s_' % kind
        b = cls(n)
        for rep in (1, 2):
            sub = pts if rep == 1 else pts[::-1][:len(pts) - 10]
            b.update(sub, rstate=np.random.default_rng(1), bootstrap=0)
            b.ctrs = sub
            q = p + 'u%d_' % rep
            out[q + 'cov'], out[q + 'am'], out[q + 'axes'] = b.cov.copy(), b.am.copy(), np.real(b.axes).copy()
            out[q + 'axes_inv'], out[q + 'logvol'] = np.real(b.axes_inv).copy(), np.float64(b.logvol)
            b.scale_to_logvol(b.logvol + enlarge)               # as gen_friends: keeps the pairs off distance 1
        out[p + 'overlap'] = np.array([b.overlap(x) for x in xs])
        out[p + 'contains'] = np.array([b.contains(x) for x in xs])
        pt = np.dot(b.ctrs, np.real(b.axes_inv))
        out[p + 'loo'] = B._friends_leaveoneout_radius(pt, kind)
        out[p + 'boot'] = np.array([B._friends_bootstrap_radius((pt, kind, philox.ScriptedGenerator(SEED, 400 + r)))
                                    for r in range(3)])
        xs1, qs = [], []
        for c in range(30):
            xs1.append(b.sample(rstate=philox.ScriptedGenerator(SEED, 500 + c)))
            x, qq = b.sample(rstate=philox.ScriptedGenerator(SEED, 600 + c), return_q=True)
            xs1.append(x)
            qs.append(qq)
        out[p + 'draws'] = np.array(xs1)
        out[p + 'draw_q'] = np.array(qs)
        b.scale_to_logvol(b.logvol + 0.3)
        out[p + 'scaled_am'], out[p + 'scaled_axes'] = b.am.copy(), np.real(b.axes).copy()
    pts, am0 = friends.chain_cloud(rng, (150, 110, 40), 2)
    out['path_points'], out['path_am0'] = pts, am0
    for kind, cls in (('balls', B.RadFriends), ('cubes', B.SupFriends)):
        q = 'path_%s_' % kind
        b = cls(2)
        b.am = am0.copy()
        b.update(pts, rstate=np.random.default_rng(1), bootstrap=0)
        out[q + 'cov'], out[q + 'am'], out[q + 'axes'] = b.cov.copy(), b.am.copy(), np.real(b.axes).copy()
        out[q + 'axes_inv'], out[q + 'logvol'] = np.real(b.axes_inv).copy(), np.float64(b.logvol)
    np.savez_compressed(os.path.join(OUT, 'friends_edges.npz'), **out)
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    refshim.import_reference()
    from dynesty import bounding as B
    gen_friends_edges(B)
    f = os.path.join(OUT, 'friends_edges.npz')
    print('wrote', f, os.path.getsize(f))


if __name__ == '__main__':
    main()

"""Equal-weight posterior draws (the reference's resample_equal / Results.samples_equal, utils.py:895-903,
1120-1187), restated in numpy on the B2N stream.

TEST INFRASTRUCTURE (see oracle/__init__.py).  The semantics are those of include/b200nest.h (b2n_resample_equal,
b2n_jitter_equal, b2n_resample_equal_runs) and DESIGN.md section 15.5:
  tick 0   u = one uniform;   c = np.cumsum(w), wsum = c[-1], C = c / wsum;   pos_i = (u + i) / M;
  draw_i   = the smallest j with pos_i < C_j (N - 1 if none: a position that rounded to 1.0);
  tick 1   perm = the stable argsort of one uniform vector event of M elements (ChainStream.permutation);
  idx      = draw[perm];   counts = np.bincount(draw, minlength=N).
Realisation r of a jitter / resample call draws on the stream (seed, EQUAL_CHAIN0 + chain0 + r) with the weights of
oracle.posterior (jitter_weights / resample_weights).
"""
import numpy as np

from . import jitter, philox, posterior, resample

EQUAL_CHAIN0 = 1 << 62


class ScriptedEqualGenerator(philox.ScriptedGenerator):
    """ScriptedGenerator that also scripts ``permutation(x)`` (utils.py:1187 ``rstate.permutation(samples[idx])``) as
    x[ChainStream.permutation(len(x))]: with it the unmodified reference's resample_equal consumes the numbers of one
    B2N stream, ``random()`` at tick 0 and the permutation at tick 1."""

    def permutation(self, x):
        if np.ndim(x) == 0:
            return self._s.permutation(int(x))
        x = np.asarray(x)
        return x[self._s.permutation(len(x))]


def draw(w, M, seed, chain):
    """dict(idx (M), counts (N), wsum) of one weight vector w (N) on the stream (seed, chain), and the positions pos
    (M), the normalised cumsum c (N) and the permutation perm (M) behind them."""
    w = np.asarray(w, dtype=np.float64)
    N = len(w)
    s = philox.ChainStream(seed, chain)
    u = s.uniform()
    c = np.cumsum(w)
    wsum = float(c[-1])
    c /= c[-1]
    pos = (u + np.arange(M)) / M
    d = np.minimum(np.searchsorted(c, pos, side='right'), N - 1)
    perm = s.permutation(M)
    return dict(idx=d[perm], counts=np.bincount(d, minlength=N), wsum=wsum, pos=pos, c=c, perm=perm)


def _stack(rs):
    return dict(idx=np.array([r['idx'] for r in rs]), counts=np.array([r['counts'] for r in rs]),
                wsum=np.array([r['wsum'] for r in rs]))


def resample_equal(w, M, seed, chain0=0):
    """Same contract as ``dynesty_b200.ops.resample_equal`` (counts always)."""
    w = np.atleast_2d(np.asarray(w, dtype=np.float64))
    return _stack([draw(wr, M, seed, chain0 + r) for r, wr in enumerate(w)])


def jitter_equal(logl, samples_n, R, M, seed, chain0=0, approx=False, logwt_ref=None, logz_ref=None):
    """Same contract as ``dynesty_b200.ops.jitter_equal`` (counts always, no gather)."""
    o = jitter.jitter_runs(logl, samples_n, R, seed, chain0, approx, logwt_ref, logz_ref)
    o.update(_stack([draw(posterior.jitter_weights(logl, samples_n, seed, chain0 + r, approx), M, seed,
                          EQUAL_CHAIN0 + chain0 + r) for r in range(R)]))
    return o


def resample_equal_runs(logl, strand, base, piece_ptr, piece_strand, end, R, M, seed, chain0=0, logwt_ref=None,
                        logz_ref=None):
    """Same contract as ``dynesty_b200.ops.resample_equal_runs`` (counts always, no gather)."""
    o = resample.resample_runs(logl, strand, base, piece_ptr, piece_strand, end, R, seed, chain0, logwt_ref, logz_ref)
    rs = []
    for r in range(R):
        W, _, present = posterior.resample_weights(logl, strand, base, piece_ptr, piece_strand, end, seed, chain0 + r)
        rs.append(draw(np.where(present, W, 0.0), M, seed, EQUAL_CHAIN0 + chain0 + r))
    o.update(_stack(rs))
    return o

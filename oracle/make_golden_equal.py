"""Generate tests/golden/equal_ref.npz by running the UNMODIFIED reference's resample_equal through
oracle.equal.ScriptedEqualGenerator.

TEST INFRASTRUCTURE.  Run where the reference copy oracle/_ref exists (oracle/install_ref.py):

    python -m oracle.make_golden_equal

Cases (samples = np.arange(N), so the reference returns the drawn indices; stream (SEED, EQ_CHAIN + case number)):
  doc       N = 4, the reference docstring's weights [0.6, 0.2, 0.15, 0.05]
  r1000     N = 1000 random weights, normalised
  r70000    N = 70 000 random weights, normalised
  zeros     N = 500, every third weight 0 and the last ten 0
  one       N = 300, one non-zero weight
  sum_hi    N = 2000 summing to 1 + 1e-6 (the renormalisation warning)
  sum_lo    N = 2000 summing to 1 - 1e-6 (the renormalisation warning)
Per case: <name>_w (the weights), <name>_chain, <name>_idx (the reference's output), <name>_warned.
"""
import os
import warnings

import numpy as np

from . import equal, refshim
from .make_golden import OUT, SEED

EQ_CHAIN = 12000
NAMES = ('doc', 'r1000', 'r70000', 'zeros', 'one', 'sum_hi', 'sum_lo')


def cases():
    rng = np.random.default_rng(SEED + 15)
    out = {'doc': np.array([0.6, 0.2, 0.15, 0.05])}
    for n in (1000, 70000):
        w = rng.exponential(size=n) * rng.random(n) ** 3
        out['r%d' % n] = w / w.sum()
    w = rng.random(500)
    w[::3] = 0.0
    w[-10:] = 0.0
    out['zeros'] = w / w.sum()
    w = np.zeros(300)
    w[137] = 1.0
    out['one'] = w
    for name, f in (('sum_hi', 1.0 + 1e-6), ('sum_lo', 1.0 - 1e-6)):
        w = rng.random(2000)
        out[name] = w / w.sum() * f
    return out


def gen_equal(U):
    out = dict(eq_seed=np.int64(SEED), eq_names=np.array(NAMES))
    for k, (name, w) in enumerate(sorted(cases().items(), key=lambda t: NAMES.index(t[0]))):
        chain = EQ_CHAIN + k
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter('always')
            idx = U.resample_equal(np.arange(len(w)), w, rstate=equal.ScriptedEqualGenerator(SEED, chain))
        out[name + '_w'] = w
        out[name + '_chain'] = np.int64(chain)
        out[name + '_idx'] = np.asarray(idx, dtype=np.int32)
        out[name + '_warned'] = np.bool_(any('renormalized' in str(c.message) for c in caught))
    np.savez_compressed(os.path.join(OUT, 'equal_ref.npz'), **out)
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    refshim.import_reference()
    from dynesty import utils as U
    gen_equal(U)
    print('wrote', os.path.join(OUT, 'equal_ref.npz'), os.path.getsize(os.path.join(OUT, 'equal_ref.npz')))


if __name__ == '__main__':
    main()

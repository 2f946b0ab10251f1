"""Record tests/golden/mmaws_outputs.npz: the outputs of rwalk_mmaws_kernel (the warp-specialised C2 chain kernel) on
seeded queues, for tests/test_gpu_mmaws_golden.py to compare byte for byte.

    python scripts/make_golden_mmaws.py [--out tests/golden/mmaws_outputs.npz]        (one H100)

Cases: the precision-matrix Gaussian at every n in NS (all three k-tile counts, first and last n of each), once with
an affine prior and no dimension flags (the PLAIN instantiation) and once behind a normal-ppf prior with periodic and
reflective coordinates (the generic one).  Two queues over K = 3 ellipsoids, Q = 3 x SMs + 5 (2 chains per CTA) and
Q = 16 x SMs + 5 (8 or 9 chains per CTA: a full group of 8 and a partial one), 24 walks: three ring buffers, the last
one partial.  Every input is drawn from numpy's PCG64 stream of the case; the threshold is stored with the outputs.
Saved per case: logl and the accept / reject / call counters in full, SHA-256 digests of the u and v arrays (Q x n
each), and u, v of a few chains."""
import argparse
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from oracle import likelihoods as OL  # noqa: E402

NS = (25, 32, 49, 50, 52, 57, 62)
QMULS = (3, 16)
KINDS = ('plain', 'generic')
SEED, WALKS, SCALE, K = 4343, 24, 0.4, 3
OUT = os.path.join(ROOT, 'tests', 'golden', 'mmaws_outputs.npz')


def case_inputs(kind, n, Q):
    """(oracle model, u0 (Q, n), axes (K, n, n), ell (Q,), dimension flags or None) of a case."""
    rng = np.random.default_rng(9000 + 2 * n + KINDS.index(kind))
    g = OL.gauss_corr(n, 0.4, 5.)
    flags = None
    if kind == 'plain':
        m = g
    else:
        from dynesty_b200 import ops
        m = OL.Model(n, OL.PRIOR_NORMAL_PPF, OL.LIKE_GAUSS_PREC, mu=0.2 * rng.standard_normal(n),
                     sigma=1.0 + rng.random(n), mean=g.p['mean'], prec=g.p['prec'], lnorm=g.p['lnorm'])
        flags = ops.dimflags_from(n, [0, n // 2], [1, n - 1])
    u0 = 0.5 + 0.03 * rng.standard_normal((Q, n))
    axes = 0.03 * (np.eye(n) + 0.2 * rng.standard_normal((K, n, n)))
    ell = rng.integers(K, size=Q).astype(np.int32)
    return m, u0, axes, ell, flags


def run_case(kind, n, Q, loglstar=None):
    """The chains of a case through ops.rwalk_batch; loglstar None = the 0.3 quantile of logl at the start points."""
    from dynesty_b200 import ops
    from helpers import device_model
    m, u0, axes, ell, flags = case_inputs(kind, n, Q)
    if loglstar is None:
        loglstar = float(np.quantile(m.loglike(m.prior_transform(u0)), 0.3))
    ops.bound_set(axes)
    o = ops.rwalk_batch(device_model(m).model_id(), u0, loglstar, SCALE, WALKS, SEED, chain0=100 * n, ell=ell,
                        dimflags=flags)
    return loglstar, o


def digest(x):
    return hashlib.sha256(np.ascontiguousarray(x, dtype=np.float64).tobytes()).hexdigest()


def sample_rows(Q):
    """Chains saved in full: the first and last of the queue and a few between."""
    return np.unique(np.r_[0, 1, 7, 8, Q // 2, Q - 9, Q - 1])


def queue_lengths():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return [qm * sms + 5 for qm in QMULS]


def record(rec, qm, Q, kind, n):
    loglstar, o = run_case(kind, n, Q)
    key = 'q%d_%s%d_' % (qm, kind, n)
    rec[key + 'loglstar'] = np.float64(loglstar)
    rec[key + 'logl'] = o['logl']
    for c in ('n_accept', 'n_reject', 'ncall'):
        rec[key + c] = o[c]
    for c in ('u', 'v'):
        rec[key + c + '_sha256'] = np.array(digest(o[c]))
        rec[key + c + '_rows'] = o[c][sample_rows(Q)]
    print('%-8s n=%2d  Q=%d  mean accept %.3f' % (kind, n, Q, o['n_accept'].mean() / WALKS))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=OUT)
    a = ap.parse_args()
    rec = {}
    for qm, Q in zip(QMULS, queue_lengths()):
        rec['q%d_Q' % qm] = np.int64(Q)
        for kind in KINDS:
            for n in NS:
                record(rec, qm, Q, kind, n)
    np.savez_compressed(a.out, **rec)
    print('wrote', a.out)


if __name__ == '__main__':
    main()

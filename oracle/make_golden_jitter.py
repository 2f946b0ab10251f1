"""Generate tests/golden/jitter.npz by running the UNMODIFIED reference's jitter_run / kld_error.

TEST INFRASTRUCTURE.  Run where the reference copy oracle/_ref exists (oracle/install_ref.py):

    python -m oracle.make_golden_jitter

The fixture conventions are those of oracle/make_golden.py (same seed, same output directory, same oracle-backed
stand-in for the runs whose records are used).  The draws are scripted with ``oracle.jitter.ScriptedJitterGenerator``
so that the reference consumes the B2N streams b2n_jitter_runs consumes; tests/test_jitter.py checks the numpy
restatement (oracle/jitter.py) and tests/test_gpu_jitter.py the kernel against this file.
"""
import os

import numpy as np

from . import jitter, refshim
from .make_golden import OUT, SEED

# realisations recorded by gen_jitter: chain ids JITTER_CHAIN0 + r
JITTER_CHAIN0, JITTER_R = 7000, (0, 1, 2, 5)


def gen_jitter(U):
    """The reference's jitter_run / kld_error (utils.py:1273-1408, 1932-1997), driven by ScriptedJitterGenerator(SEED,
    JITTER_CHAIN0 + r), on two records: the device-round run of integrals.npz (samples_n a sawtooth of rounds, then the
    add_live tail) and a merged dynamic run with irregular samples_n (the run of tests/test_dynamic.py on the oracle
    backend).  approx off and on; _find_decrease's output too."""
    import sys
    from _pytest.monkeypatch import MonkeyPatch
    sys.path.insert(0, os.path.join(os.path.dirname(OUT)))
    import fake_backend
    mp = MonkeyPatch()
    try:
        fake_backend.install(mp)
        from dynesty_b200 import dynamic as D, likelihoods as DL
        d = D.DynamicNestedSampler(DL.gauss_test3d(), nlive=80, bound='multi', sample='rwalk', walks=10, seed=4)
        d.sample_initial(dlogz=0.5, round_size=8)
        dyn = d.run_nested(nlive_batch=60, maxbatch=2, n_effective=1e9, round_size=6)
    finally:
        mp.undo()
    g = np.load(os.path.join(OUT, 'integrals.npz'))
    records = {'golden': (g['wt_logl'], g['wt_samples_n'], g['wt_logwt'], g['wt_logz']),
               'dyn': (np.asarray(dyn.logl), np.asarray(dyn.samples_n), np.asarray(dyn.logwt), np.asarray(dyn.logz))}
    out = dict(jit_seed=np.int64(SEED), jit_chain0=np.int64(JITTER_CHAIN0), jit_r=np.array(JITTER_R, dtype=np.int64))
    for name, (logl, sn, logwt, logz) in records.items():
        p = 'jit_%s_' % name
        N = len(logl)
        sn = np.asarray(sn, dtype=np.int64)
        out.update({p + 'logl': logl, p + 'samples_n': sn, p + 'logwt': logwt, p + 'logz': logz})
        flag, nstart, bounds = U._find_decrease(sn)
        out[p + 'flag'] = flag
        out[p + 'nstart'] = np.asarray(nstart, dtype=np.int64)
        out[p + 'bounds'] = np.array(bounds, dtype=np.int64).reshape(-1, 2)
        res = U.Results(dict(samples_u=np.zeros((N, 1)), samples=np.zeros((N, 1)), samples_id=np.zeros(N, dtype=int),
                             logl=logl, samples_n=sn, logvol=np.zeros(N), logwt=logwt, logz=logz, logzerr=np.zeros(N),
                             information=np.zeros(N)))
        for approx in (False, True):
            q = p + 'a%d_' % approx
            cols = {k: [] for k in ('logvol', 'logwt', 'logz', 'logzerr', 'h', 'kld', 'ticks')}
            for r in JITTER_R:
                rs = jitter.ScriptedJitterGenerator(SEED, JITTER_CHAIN0 + r)
                kld, new = U.kld_error(res, 'jitter', rstate=rs, return_new=True, approx=approx)
                for k in ('logvol', 'logwt', 'logz', 'logzerr'):
                    cols[k].append(np.asarray(new[k]))
                cols['h'].append(U.compute_integrals(logl=logl, logvol=new['logvol'])[3])
                cols['kld'].append(kld)
                cols['ticks'].append(rs.tick)
            out.update({q + k: np.array(v) for k, v in cols.items()})
    np.savez_compressed(os.path.join(OUT, 'jitter.npz'), **out)
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    refshim.import_reference()
    from dynesty import utils as U
    gen_jitter(U)
    print('wrote', os.path.join(OUT, 'jitter.npz'), os.path.getsize(os.path.join(OUT, 'jitter.npz')))


if __name__ == '__main__':
    main()

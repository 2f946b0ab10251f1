"""Generate tests/golden/jitter.npz and jitter_edges.npz by running the UNMODIFIED reference's jitter_run / kld_error.

TEST INFRASTRUCTURE.  Run where the reference copy oracle/_ref exists (oracle/install_ref.py):

    python -m oracle.make_golden_jitter [jitter] [jitter_edges]

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


def gen_jitter_edges(U):
    """The reference's jitter_run / kld_error (approx off), driven by ScriptedJitterGenerator(SEED, JITTER_CHAIN0 + r)
    for r = 0, 1, on two records of tests/test_jitter.py at b2n_jitter_runs' piece boundaries: [2, 1] repeated
    JT_TILE + 1 times (one segment more than a scan tile) and one stretch JT_CHUNK + 1, .., 1 (a scan of one chunk
    plus two exponentials).  Writes tests/golden/jitter_edges.npz: per record its logl, samples_n, logwt, logz, and
    per realisation (the new_ keys) full logvol / logwt / logz / kld and the final logzerr and h."""
    import sys
    sys.path.insert(0, os.path.dirname(OUT))
    from test_jitter import EDGES
    names = ('pairs_Tp1', 'stretch_Cp1')
    R = 2
    out = dict(seed=np.int64(SEED), chain0=np.int64(JITTER_CHAIN0), r=np.arange(R), names=np.array(names))
    for name in names:
        rec = jitter.expected_record(EDGES[name][0])
        p = 'edge_%s_' % name
        out.update({p + k: rec[k] for k in ('logl', 'samples_n', 'logwt', 'logz')})
        N = len(rec['logl'])
        res = U.Results(dict(samples_u=np.zeros((N, 1)), samples=np.zeros((N, 1)), samples_id=np.zeros(N, dtype=int),
                             logl=rec['logl'], samples_n=rec['samples_n'], logvol=rec['logvol'], logwt=rec['logwt'],
                             logz=rec['logz'], logzerr=np.zeros(N), information=np.zeros(N)))
        cols = {k: [] for k in ('logvol', 'logwt', 'logz', 'kld', 'logzerr', 'h')}
        for r in range(R):
            rs = jitter.ScriptedJitterGenerator(SEED, JITTER_CHAIN0 + r)
            kld, new = U.kld_error(res, 'jitter', rstate=rs, return_new=True, approx=False)
            for k in ('logvol', 'logwt', 'logz'):
                cols[k].append(np.asarray(new[k]))
            cols['kld'].append(kld)
            cols['logzerr'].append(new['logzerr'][-1])
            cols['h'].append(U.compute_integrals(logl=rec['logl'], logvol=new['logvol'])[3][-1])
        out.update({p + 'new_' + k: np.array(v) for k, v in cols.items()})
    np.savez_compressed(os.path.join(OUT, 'jitter_edges.npz'), **out)
    return out


def main(argv=()):
    """All fixtures, or only those named on the command line (jitter, jitter_edges)."""
    os.makedirs(OUT, exist_ok=True)
    refshim.import_reference()
    from dynesty import utils as U
    for name, gen in (('jitter', gen_jitter), ('jitter_edges', gen_jitter_edges)):
        if not argv or name in argv:
            gen(U)
            f = os.path.join(OUT, name + '.npz')
            print('wrote', f, os.path.getsize(f))


if __name__ == '__main__':
    import sys
    main(sys.argv[1:])

"""Generate tests/golden/resample.npz by running the UNMODIFIED reference's resample_run / kld_error(error='resample').

TEST INFRASTRUCTURE.  Run where the reference copy oracle/_ref exists (oracle/install_ref.py):

    python -m oracle.make_golden_resample

Records with one point removed per iteration (where the reference's live-count rule holds), made on the oracle
backend (tests/fake_backend.py plus ``oracle.nsstrands``): a host-loop run, device-round runs with batch = 1
with and without the final live points, and a merged dynamic record.  The draws are scripted with
``oracle.resample.ScriptedResampleGenerator`` so that the reference consumes the B2N streams b2n_resample_runs consumes;
tests/test_resample.py checks the numpy restatement (oracle/resample.py) and tests/test_gpu_resample.py the kernel
against this file.
"""
import os

import numpy as np

from . import nsstrands, refshim, resample
from .make_golden import OUT, SEED

# realisations recorded: chain ids RESAMPLE_CHAIN0 + r
RESAMPLE_CHAIN0, RESAMPLE_R = 9000, (0, 1, 3)


def records():
    """name -> our Results of the four K = 1 records (oracle backend)."""
    import sys
    from _pytest.monkeypatch import MonkeyPatch
    sys.path.insert(0, os.path.join(os.path.dirname(OUT)))
    import fake_backend
    mp = MonkeyPatch()
    try:
        fake_backend.install(mp)
        from dynesty_b200 import dynamic as D, likelihoods as DL, nested as N
        nsstrands.install(mp, fake_backend._state)
        out = {}
        s = N.NestedSampler(DL.gauss_test3d(), nlive=40, bound='multi', sample='rwalk', walks=25, seed=SEED)
        out['host'] = s.run_nested(dlogz=0.5, loop='host', strands=True)
        for name, add_live in (('dev', True), ('devnolive', False)):
            s = N.NestedSampler(DL.gauss_test3d(), nlive=40, bound='multi', sample='rwalk', walks=25, seed=SEED + 1)
            out[name] = s.run_nested(dlogz=0.5, loop='device', batch=1, add_live=add_live, strands=True)
        d = D.DynamicNestedSampler(DL.gauss_test3d(), nlive=40, bound='multi', sample='rwalk', walks=25, seed=SEED + 2)
        out['dyn'] = d.run_nested(dlogz_init=0.5, nlive_batch=30, maxbatch=2, n_effective=1e9, round_size=1,
                                  strands=True)
    finally:
        mp.undo()
    return out


def ref_results(U, res):
    """The reference's Results of one of our records."""
    N = len(res['logl'])
    d = dict(samples_u=np.zeros((N, 1)), samples=np.zeros((N, 1)), samples_id=np.asarray(res['samples_id']),
             samples_it=np.asarray(res['samples_it']), logl=np.asarray(res['logl']), logvol=np.asarray(res['logvol']),
             logwt=np.asarray(res['logwt']), logz=np.asarray(res['logz']), logzerr=np.asarray(res['logzerr']),
             information=np.asarray(res['information']), ncall=np.asarray(res['ncall_per_it']), blob=np.zeros(N))
    if 'samples_batch' in res:
        d.update(samples_n=np.asarray(res['samples_n']), samples_batch=np.asarray(res['samples_batch']),
                 batch_logl_bounds=np.array(res['batch_bounds'], dtype=float))
    else:
        d.update(nlive=int(len(set(np.asarray(res['samples_id']).tolist()))), niter=int(res['niter']))
    return U.Results(d)


def gen_resample(U):
    out = dict(rs_seed=np.int64(SEED), rs_chain0=np.int64(RESAMPLE_CHAIN0), rs_r=np.array(RESAMPLE_R, dtype=np.int64))
    for name, res in records().items():
        p = 'rs_%s_' % name
        for k in ('logl', 'samples_id', 'samples_it', 'samples_n', 'logwt', 'logz', 'logvol', 'ncall_per_it',
                  'samples_batch'):
            if k in res:
                out[p + k] = np.asarray(res[k])
        out[p + 'niter'] = np.int64(res['niter'])
        if 'batch_bounds' in res:
            out[p + 'batch_bounds'] = np.array(res['batch_bounds'], dtype=float)
        rr = ref_results(U, res)
        for r in RESAMPLE_R:
            q = p + 'r%d_' % r
            g = resample.ScriptedResampleGenerator(SEED, RESAMPLE_CHAIN0 + r)
            new, idx = U.resample_run(rr, rstate=g, return_idx=True)
            out[q + 'ticks'] = np.int64(g.tick)
            g = resample.ScriptedResampleGenerator(SEED, RESAMPLE_CHAIN0 + r)
            kld = U.kld_error(rr, error='resample', rstate=g)
            out[q + 'idx'] = np.asarray(idx)
            out[q + 'kld'] = np.asarray(kld)
            for k in ('samples_n', 'logvol', 'logwt', 'logz'):
                out[q + k] = np.asarray(new[k])
            out[q + 'h'] = np.asarray(new['information'])
            out[q + 'logzerr'] = np.asarray(new['logzerr'])
    np.savez_compressed(os.path.join(OUT, 'resample.npz'), **out)
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    refshim.import_reference()
    from dynesty import utils as U
    gen_resample(U)
    print('wrote', os.path.join(OUT, 'resample.npz'), os.path.getsize(os.path.join(OUT, 'resample.npz')))


if __name__ == '__main__':
    main()

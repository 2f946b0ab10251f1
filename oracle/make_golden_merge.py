"""Generate tests/golden/merge.npz by running the UNMODIFIED reference's merge_runs.

TEST INFRASTRUCTURE.  Run where the reference copy oracle/_ref exists (oracle/install_ref.py):

    python -m oracle.make_golden_merge

Runs made on the oracle backend (tests/fake_backend.py plus ``oracle.nsstrands``) and two synthetic records, merged
by the reference.  Every input sample's index in the concatenation that b2n_merge_runs takes (the runs in
``dynesty_b200.utils.merge_order``) is passed as the reference's ``blob``, which _merge_two carries through, so the
merged ``blob`` is the kernel's ``perm``.  Cases:
  static3 / static5  three / five device-round runs (batch 4, final live points): the odd run passes up two levels
  hostnolive         a host-loop run and a run without its final live points (the reference's nrun == niter branch)
  dynstatic          a dynamic record and a static run
  unravel_host       unravel_run of a host-loop run (one removal per iteration, 40 strands) merged back
  unravel_dyn        unravel_run of a dynamic record: base strands, then the add-on strands one at a time
  ties               two synthetic records with quantised logl: ties inside and across runs, plateaus spanning both
  single             one run
tests/test_merge.py checks the numpy restatement (oracle/merge.py) and dynesty_b200.utils.merge_runs, and
tests/test_gpu_merge.py the kernel, against this file.
"""
import os
import sys

import numpy as np

from . import nsstrands, refshim
from .make_golden import OUT, SEED

IN_KEYS = ('logl', 'logvol', 'samples_n', 'samples_id', 'samples_it', 'samples_batch', 'ncall_per_it', 'niter', 'nlive')


def runs():
    """name -> our Results of the runs the cases are made of (oracle backend)."""
    from _pytest.monkeypatch import MonkeyPatch
    sys.path.insert(0, os.path.dirname(OUT))
    import fake_backend
    mp = MonkeyPatch()
    try:
        fake_backend.install(mp)
        from dynesty_b200 import dynamic as D, likelihoods as DL, nested as N
        nsstrands.install(mp, fake_backend._state)
        out = {}
        for k in range(5):
            s = N.NestedSampler(DL.gauss_test3d(), nlive=40, bound='multi', sample='rwalk', walks=25, seed=SEED + 10 + k)
            out['dev%d' % k] = s.run_nested(dlogz=0.5, loop='device', batch=4, add_live=True, strands=True)
        for name, add_live, seed in (('host', True, SEED), ('hostnolive', False, SEED + 20)):
            s = N.NestedSampler(DL.gauss_test3d(), nlive=40, bound='multi', sample='rwalk', walks=25, seed=seed)
            out[name] = s.run_nested(dlogz=0.5, loop='host', add_live=add_live, strands=True)
        d = D.DynamicNestedSampler(DL.gauss_test3d(), nlive=40, bound='multi', sample='rwalk', walks=25, seed=SEED + 2)
        out['dyn'] = d.run_nested(dlogz_init=0.5, nlive_batch=30, maxbatch=2, n_effective=1e9, round_size=1,
                                  strands=True)
    finally:
        mp.undo()
    return out


def synthetic(nlive, ndead, seed):
    """A static record (ndead points at nlive, then the final nlive) with logl quantised to integers."""
    from dynesty_b200.nested import Results, _integrate
    rng = np.random.default_rng(seed)
    N = ndead + nlive
    logl = np.floor(np.sort(rng.uniform(-20.0, 0.0, N)))
    n = np.r_[np.full(ndead, nlive), np.arange(nlive, 0, -1)].astype(np.int64)
    logvol = np.cumsum(np.log(n / (n + 1.)))
    logwt, logz, logzvar, h = _integrate(logl, logvol)
    return Results(logl=logl, samples_n=n, niter=ndead, logvol=logvol, logwt=logwt, logz=logz,
                   logzerr=np.sqrt(logzvar), information=h, ncall_per_it=np.ones(N, dtype=np.int64),
                   samples_id=np.zeros(N, dtype=np.int64), samples_it=np.zeros(N, dtype=np.int64))


def cases():
    from dynesty_b200 import utils as DU
    r = runs()
    return dict(static3=[r['dev0'], r['dev1'], r['dev2']],
                static5=[r['dev%d' % k] for k in range(5)],
                hostnolive=[r['host'], r['hostnolive']],
                dynstatic=[r['dyn'], r['dev3']],
                unravel_host=DU.unravel_run(r['host']),
                unravel_dyn=DU.unravel_run(r['dyn']),
                ties=[synthetic(10, 60, SEED + 30), synthetic(8, 50, SEED + 31)],
                single=[r['host']])


def ref_results(U, res, blob):
    """The reference's Results of one of our runs: static (nlive, niter) when its counts are a static run's, else
    with samples_n (and its batches when it has them)."""
    from dynesty_b200 import utils as DU
    N = len(res['logl'])
    n = DU.samples_n_of(res)
    d = dict(samples_u=np.zeros((N, 1)), samples=np.zeros((N, 1)), logl=np.asarray(res['logl'], dtype=float),
             samples_id=np.asarray(res['samples_id']), samples_it=np.asarray(res['samples_it']),
             ncall=np.asarray(res['ncall_per_it']), blob=blob)
    d.update({k: np.asarray(res[k]) for k in ('logvol', 'logwt', 'logz', 'logzerr', 'information')})
    if 'samples_batch' in res:
        d.update(samples_batch=np.asarray(res['samples_batch']),
                 batch_logl_bounds=np.array([tuple(b) for b in res['batch_bounds']], dtype=float))
    niter = int(res['niter'])
    nlive = int(res['nlive']) if 'nlive' in res else int(n.max())
    static = np.minimum(np.arange(N, 0, -1), nlive) if N == niter + nlive else np.full(N, nlive)
    if N in (niter, niter + nlive) and np.array_equal(n, static) and 'samples_batch' not in res:
        d.update(nlive=nlive, niter=niter)
    else:
        d['samples_n'] = n
        if 'samples_batch' not in res:
            d.update(samples_batch=np.zeros(N, dtype=int), batch_logl_bounds=np.array([(-np.inf, np.inf)]))
    return U.Results(d)


def gen_merge(U):
    from dynesty_b200 import utils as DU
    out = dict()
    for name, res_list in cases().items():
        p = 'c_%s_' % name
        order, nbase = DU.merge_order(res_list)
        runs_ = [res_list[i] for i in order]
        sizes = np.array([len(r['logl']) for r in runs_], dtype=np.int64)
        run_ptr = np.r_[0, np.cumsum(sizes)]
        lowedge = []
        for r in runs_:
            b, bounds = DU._batches(r)
            lowedge.append(float(np.min(bounds[b])))
        out.update({p + 'logl': np.concatenate([np.asarray(r['logl'], dtype=float) for r in runs_]),
                    p + 'samples_n': np.concatenate([DU.samples_n_of(r) for r in runs_]),
                    p + 'run_ptr': run_ptr, p + 'nbase': np.int64(nbase), p + 'lowedge': np.array(lowedge),
                    p + 'nin': np.int64(len(res_list))})
        for i, r in enumerate(res_list):
            q = p + 'in%d_' % i
            for k in IN_KEYS:
                if k in r:
                    out[q + k] = np.asarray(r[k])
            if 'batch_bounds' in r:
                out[q + 'batch_bounds'] = np.array([tuple(b) for b in r['batch_bounds']], dtype=float)
        rr = [None] * len(res_list)
        for pos, i in enumerate(order):
            rr[i] = ref_results(U, res_list[i], np.arange(run_ptr[pos], run_ptr[pos + 1]))
        m = U.merge_runs(rr, print_progress=False)
        out[p + 'ref_perm'] = np.asarray(m['blob'], dtype=np.int64)
        out[p + 'ref_samples_n'] = np.asarray(U._get_nsamps_samples_n(m)[1], dtype=np.int64)
        for k in ('logl', 'logvol', 'logwt', 'logz', 'logzerr', 'information'):
            out[p + 'ref_' + k] = np.asarray(m[k], dtype=float)
        out[p + 'ref_niter'] = np.int64(m['niter'])
        out[p + 'ref_nlive'] = np.int64(m['nlive'] if 'nlive' in m.keys() else -1)
    np.savez_compressed(os.path.join(OUT, 'merge.npz'), **out)
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    refshim.import_reference()
    from dynesty import utils as U
    gen_merge(U)
    print('wrote', os.path.join(OUT, 'merge.npz'), os.path.getsize(os.path.join(OUT, 'merge.npz')))


if __name__ == '__main__':
    main()

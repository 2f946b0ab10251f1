"""Strand records of the batched-replacement rounds (b2n_ns_get_strands / b2n_ns_set_live_it / b2n_ns_get_live_it),
restated on the CPU.

TEST INFRASTRUCTURE (see oracle/__init__.py): the checker of the strand columns of csrc/b2n_ns.cu.  ``StrandBatchNS``
is ``oracle.nsloop.BatchNS`` plus what the commit kernel records for every removal: the j-th removal of a round
records the live slot it occupied and the slot's birth counter (the dead rows recorded before its occupant entered
the live set), then the slot's new occupant gets it + K, the dead rows after the round -- its birth threshold is the
round threshold, the logl of dead row it + K - 1.  Phase-0 (unit-cube) and uniform-sampler rounds commit through the
same ``_commit`` and record the same.
"""
import numpy as np

from . import nsloop


class StrandBatchNS(nsloop.BatchNS):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.live_it = np.zeros(self.N, dtype=np.int64)       # b2n_ns_set_state sets every counter to 0
        self.dead_slot, self.dead_it = [], []

    def _commit(self, order, sl, thr, out):
        slots = np.asarray(order[:self.K])
        self.dead_slot.extend(int(s) for s in slots)
        self.dead_it.extend(int(x) for x in self.live_it[slots])
        self.live_it[slots] = self.it + self.K
        super()._commit(order, sl, thr, out)

    def strand_arrays(self):
        """(slot int32, it int64) of every dead row: b2n_ns_get_strands."""
        return np.array(self.dead_slot, dtype=np.int32), np.array(self.dead_it, dtype=np.int64)


def install(monkeypatch, state):
    """On top of the oracle backend of the device rounds (tests/fake_backend.py, whose rounds are ``nsloop.BatchNS``
    objects kept in ``state['ns']``): make those rounds ``StrandBatchNS`` and answer ops.ns_get_strands /
    ns_set_live_it / ns_get_live_it from them."""
    from dynesty_b200 import ops
    monkeypatch.setattr(nsloop, 'BatchNS', StrandBatchNS)

    def ns_get_strands(first, count, ctx=None):
        slot, it = state['ns'].strand_arrays()
        return slot[first:first + count], it[first:first + count]

    def ns_set_live_it(live_it, ctx=None):
        state['ns'].live_it = np.array(live_it, dtype=np.int64)

    def ns_get_live_it(nlive, ctx=None):
        return state['ns'].live_it.copy()

    for f in (ns_get_strands, ns_set_live_it, ns_get_live_it):
        monkeypatch.setattr(ops, f.__name__, f)

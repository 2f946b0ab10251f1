"""GPU: rwalk_mmaws_kernel reproduces, bit for bit, the outputs recorded in tests/golden/mmaws_outputs.npz
(scripts/make_golden_mmaws.py) on seeded queues at every k-tile count, with the PLAIN and the generic chain phase;
and one FP64 m16n8k4 MMA gives the bits of two m8n8k4 (scripts/dmma_shapes.py's probe), which is what lets the
kernel's direction product run on the larger shape without changing a result."""
import os

import numpy as np
import pytest

from scripts import dmma_shapes, make_golden_mmaws as G

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'mmaws_outputs.npz')
CASES = [(qm, kind, n) for qm in G.QMULS for kind in G.KINDS for n in G.NS]


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def test_dmma_16x8x4_is_two_8x8x4():
    pr = dmma_shapes.probe()
    assert pr['k4_maxerr_normal'] < 1e-12 and pr['k8_maxerr_normal'] < 1e-12, pr     # fragment layouts
    assert all(v == 0 for v in pr['k4_vs_2x884_differ'].values()), pr


@pytest.mark.parametrize('qm,kind,n', CASES, ids=['q%d-%s%d' % c for c in CASES])
def test_mmaws_matches_golden(monkeypatch, qm, kind, n):
    monkeypatch.delenv('B2N_RWALK_IMPL', raising=False)
    g = np.load(GOLDEN)
    Q = G.queue_lengths()[G.QMULS.index(qm)]
    if Q != int(g['q%d_Q' % qm]):
        pytest.skip('recorded for a queue of %d chains (the SM count of the recording GPU), not %d'
                    % (int(g['q%d_Q' % qm]), Q))
    key = 'q%d_%s%d_' % (qm, kind, n)
    _, o = G.run_case(kind, n, Q, loglstar=float(g[key + 'loglstar']))
    for c in ('n_accept', 'n_reject', 'ncall'):
        assert np.array_equal(o[c], g[key + c]), c
    rows = G.sample_rows(Q)
    for c in ('u', 'v'):
        assert _same_bits(o[c][rows], g[key + c + '_rows']), c
        assert G.digest(o[c]) == str(g[key + c + '_sha256']), c
    assert _same_bits(o['logl'], g[key + 'logl'])

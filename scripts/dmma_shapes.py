"""The FP64 MMA shapes of sm_90 side by side: throughput, dependent-issue latency and bit identity.

    python scripts/dmma_shapes.py [--iters 20000] [--tiles 512] [--out FILE]

Throughput: b2n_fp64_peak, 16 independent accumulator chains per thread on every SM, for the m8n8k4 shape the chain
kernels use and for m16n8k4, m16n8k8, m16n8k16 (TFLOP/s; best of 4 launches).  Latency: b2n_fp64_latency, one warp
issuing one dependency chain (SM clocks per instruction).  Bit identity: b2n_dmma_probe on seeded tiles with
cancellation, mixed magnitudes (1e+-300), subnormals and signed zeros: one m16n8k4 must give the bits of two m8n8k4
(rows 0..7 and 8..15); how often one m16n8k8 differs from two chained k4 steps is counted for information.  The
card's name, power limit and SM clock are read in the same call.  Prints one JSON line and the go / no-go verdict of
moving a k4 contraction from m8n8k4 to m16n8k4 (bit-identical, and at least 1.6 x the flop rate)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dynesty_b200 import ops  # noqa: E402

SHAPES = ('fma', 'mma', 'mma16x8x4', 'mma16x8x8', 'mma16x8x16')
CLASSES = ('normal', 'cancel', 'mixed', 'subnormal', 'zeros')


def probe_tiles(per_class=128, seed=90):
    """(a (T, 16, 8), b (T, 8, 8), c (T, 16, 8), class label per tile), `per_class` tiles of each of CLASSES."""
    rng = np.random.default_rng(seed)
    A, B, Cc, lab = [], [], [], []

    def signed(shape, lo, hi):
        return rng.choice([-1.0, 1.0], size=shape) * 10.0 ** rng.uniform(lo, hi, size=shape)

    for cls in CLASSES:
        T = per_class
        if cls == 'normal':
            a, b, c = rng.standard_normal((T, 16, 8)), rng.standard_normal((T, 8, 8)), rng.standard_normal((T, 16, 8))
        elif cls == 'cancel':
            # products that cancel in pairs (a[:, 1] = -a[:, 0], b[1] = b[0], the same in k 4..7) on top of
            # accumulators that cancel the whole exact sum: every bit left is the rounding of the hardware
            a, b = rng.standard_normal((T, 16, 8)), rng.standard_normal((T, 8, 8))
            a[:, :, 1] = -a[:, :, 0] * (1.0 + 2.0 ** -40 * rng.standard_normal((T, 16)))
            b[:, 1] = b[:, 0]
            a[:, :, 5] = -a[:, :, 4]
            b[:, 5] = b[:, 4]
            c = -np.einsum('tik,tkj->tij', a[:, :, :4], b[:, :4]) * (1.0 + 2.0 ** -50 * rng.standard_normal((T, 16, 8)))
        elif cls == 'mixed':
            a, b, c = signed((T, 16, 8), -150, 150), signed((T, 8, 8), -150, 150), signed((T, 16, 8), -300, 300)
        elif cls == 'subnormal':
            a, b = signed((T, 16, 8), -170, -150), signed((T, 8, 8), -170, -150)
            c = rng.choice([-1.0, 1.0], size=(T, 16, 8)) * 5e-324 * rng.integers(0, 1 << 40, size=(T, 16, 8))
        else:
            a, b, c = rng.standard_normal((T, 16, 8)), rng.standard_normal((T, 8, 8)), rng.standard_normal((T, 16, 8))
            for x in (a, b, c):
                z = rng.random(x.shape) < 0.5
                x[z] = np.copysign(0.0, rng.choice([-1.0, 1.0], size=int(z.sum())))
        A.append(a); B.append(b); Cc.append(c); lab += [cls] * T
    return np.concatenate(A), np.concatenate(B), np.concatenate(Cc), np.array(lab)


def bits_differ(x, y):
    """Elements whose bit patterns differ."""
    return np.ascontiguousarray(x).view(np.uint64) != np.ascontiguousarray(y).view(np.uint64)


def probe(per_class=128, seed=90):
    a, b, c, lab = probe_tiles(per_class, seed)
    r = ops.dmma_probe(a, b, c)
    d4, d8 = bits_differ(r['k4'], r['k4x2rows']), bits_differ(r['k8'], r['k4x2steps'])
    # fragment layouts: the 'normal' tiles against float64 numpy (a layout error is O(1), round-off ~1e-15)
    nm = lab == 'normal'
    ref4 = np.einsum('tik,tkj->tij', a[nm][:, :, :4], b[nm][:, :4]) + c[nm]
    ref8 = np.einsum('tik,tkj->tij', a[nm], b[nm]) + c[nm]
    return dict(tiles=int(len(lab)),
                k4_vs_2x884_differ={k: int(d4[lab == k].sum()) for k in CLASSES},
                k8_vs_2k4_differ={k: int(d8[lab == k].sum()) for k in CLASSES},
                elements_per_class=int(per_class * 128),
                k4_maxerr_normal=float(np.abs(r['k4'][nm] - ref4).max()),
                k8_maxerr_normal=float(np.abs(r['k8'][nm] - ref8).max()))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                            '--format=csv,noheader', '-i', '0'], capture_output=True, text=True, timeout=30).stdout
        return [s.strip() for s in q.strip().split(',')[:4]]
    except Exception as e:                                   # the numbers still stand; say why the card is unknown
        return ['unknown (%r)' % (e,)] + ['unknown'] * 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20000)
    ap.add_argument('--tiles', type=int, default=128, help='probe tiles per input class')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    peak = {k: ops.fp64_peak(k, a.iters)[0] for k in SHAPES}
    lat = {k: ops.fp64_latency(k) for k in SHAPES}
    name, plim, sm, smmax = card()
    pr = probe(a.tiles)
    ratio = peak['mma16x8x4'] / peak['mma']
    ident = all(v == 0 for v in pr['k4_vs_2x884_differ'].values())
    out = dict(card=name, power_limit=plim, sm_clock_after=sm, sm_clock_max=smmax,
               tflops=peak, latency_cycles=lat, ratio_16x8x4_over_8x8x4=ratio, probe=pr,
               go=bool(ident and ratio >= 1.6))
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')
    print('16x8x4 bit-identical to 2 x 8x8x4: %s; flop rate %.2f x 8x8x4 (bar 1.6): %s'
          % (ident, ratio, 'GO' if out['go'] else 'NO-GO'))


if __name__ == '__main__':
    main()

"""Where the one-CTA kernels of the device rounds (csrc/b2n_ns.cu) change form, restated on the CPU.

TEST INFRASTRUCTURE (see oracle/__init__.py): the case table of tests/test_gpu_ns_limits.py and the host formulas
it is derived from, so that tests/test_oracle_nsloop.py can check without a GPU that the table reaches every limit.

The step kernel (ns_propose_body + ns_commit_body) runs on ONE CTA of ``threads`` threads (1024, or 512 / 256 under
B2N_NS_THREADS); the start-up sort always runs on 1024.  The loops that change form:
  sort      bitonic over Npad = next power of two >= N (>= 2); Npad / 2 pairs per stage, ceil(Npad / 2 / 1024)
            pairs per thread; rows >= N are +inf padding
  merge     bitonic over the K new keys padded to Kpad (>= 2); Kpad / 2 pairs per stage over ``threads``
  commit    dead records / evidence / binary searches: ``for (j = tid; j < K; j += threads)``
  propose   start rows / ellipsoid picks / start points / worklist: the same stride over K
Shared memory (bytes) is what b2n_ns.cu asks for: the sort is refused when ns_sort_smem exceeds the opt-in limit
(b2n_ns_set_state: "nlive too large"), the rounds when max(ns_propose_smem, ns_commit_smem) + 2048 does
(b2n_ns_run: "nlive / batch too large").  The commit's figure is not monotone in K: Kpad doubles at K = 2^k + 1
while the survivors' part N - K keeps shrinking, so at N = Npad the refused K form bands between accepted
ranges (at N = 16384 on a 227 KB limit: 4097..5381 and 8193..13573).
"""
import math

import numpy as np

THREADS = 1024                  # B2N_NS_THREADS of b2n_ns.cu: the sort, and the step kernel by default
STEP_HEADROOM = 2048            # b2n_ns_run keeps this much room for the step kernel's static shared memory
H100_SMEM_OPTIN = 227 * 1024    # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100


def pad2(x):
    """Npad / Kpad: the next power of two >= x, at least 2."""
    p = 2
    while p < x:
        p <<= 1
    return p


def passes(width, threads):
    """Iterations of ``for (t = tid; t < width; t += threads)`` for thread 0."""
    return -(-width // threads)


def sort_smem(N):
    return pad2(N) * 12 + 64


def commit_smem(N, K):
    NA = N - K
    return (NA + (NA & 1)) * 8 + pad2(K) * 8 + NA * 4 + pad2(K) * 4 + 64


def propose_smem(K, nc, kell):
    return (THREADS // 32) * nc * 8 + ((kell + 1) & ~1) * 8 + K * 8 + (kell + 2) * 4 + 64


def sort_accepts(N, optin):
    return sort_smem(N) <= optin


def run_accepts(N, K, nc, kell, optin):
    return max(propose_smem(K, nc, kell), commit_smem(N, K)) + STEP_HEADROOM <= optin


def sort_limit(optin):
    """Largest nlive the start-up sort accepts."""
    N = 2
    while sort_accepts(2 * N, optin):
        N *= 2
    return N


def refused_bands(N, nc, kell, optin):
    """The batches 1 <= K < N the rounds refuse at nlive N, as a list of inclusive (first, last) ranges."""
    bands, start = [], None
    for K in range(1, N):
        if not run_accepts(N, K, nc, kell, optin):
            start = K if start is None else start
        elif start is not None:
            bands.append((start, K - 1))
            start = None
    if start is not None:
        bands.append((start, N - 1))
    return bands


def limits(N, K, threads=THREADS):
    """What a round of (N, K) on a step kernel of ``threads`` threads reaches."""
    return dict(sort_passes=passes(pad2(N) // 2, THREADS), sort_padding=pad2(N) - N,
                merge_half=pad2(K) // 2, merge_passes=passes(pad2(K) // 2, threads),
                loop_passes=passes(K, threads), one_survivor=K == N - 1)


# ---- the case table of tests/test_gpu_ns_limits.py ------------------------------------------------------------
# unit-cube-phase rounds (prior draws: cheap on both sides), (N, K)
WIDTH_CASES = [
    (2, 1),             # smallest shape: Npad = Kpad = 2, one survivor
    (3, 2),             # N = 2^k + 1: one padding row in the sort; one survivor
    (1025, 512),        # Npad 2048 with 1023 padding rows
    (2048, 1023),       # Npad = N, one sort pass per thread; Kpad / 2 = 512 < threads
    (3000, 1024),       # K = threads
    (2049, 1025),       # two sort passes; Kpad / 2 = threads; K one past the threads
    (4097, 2048),       # four sort passes; K = 2 x threads
    (4097, 2049),       # two merge passes
    (6000, 4097),       # Kpad 8192 over 4097 keys: four merge passes, half of them on padding
    (16384, 8192),      # the largest sort (eight passes); K = 8192 is the last batch before a refused band
]
# bounded random-walk rounds, n = 3, walks = 2: (N, K, number of ellipsoids)
RWALK_CASES = [
    (4096, 2049, 1),    # start rows / contains / start points / worklist loops past 1024, one ellipsoid
    (2048, 1025, 7),    # ... with the serial grouped worklist over seven ellipsoids
    (200, 16, 40),      # more ellipsoids than chains
]
# the step kernel on fewer threads: (threads, sampler, N, K)
THREAD_CASES = [(t, s, N, K) for t in (256, 512) for s, N, K in (('unitcube', 4097, 2049), ('rwalk', 1000, 600))]


def rwalk_warp_cpc(K, sms):
    """Chains per CTA of the warp-per-chain rwalk kernel (b2n_chain_grid, b2n_rwalk.cu), min_cpc 1."""
    ctas = sms if K <= 16 * sms else 2 * sms
    return max(1, -(-K // ctas))


# ---- a likelihood with exact ties ----------------------------------------------------------------------------
class QuantizedGauss:
    """L(v) = floor(q L_g(v)) / q with L_g(v) = -0.5 |v|^2 and the prior U(lo, lo + width)^n.

    Every value is a multiple of 1 / q, so new points tie exactly with survivors and with the round threshold.
    The device evaluates L_g in its own summation order; the floor agrees with this one as long as q L_g is not
    within rounding of an integer, so every evaluation records the distance of q L_g from the nearest integer
    (``min_frac``): a test that relies on the equality checks it."""

    def __init__(self, n, q=4.0, lo=-2.0, width=4.0):
        self.ndim, self.q, self.lo, self.width = int(n), float(q), float(lo), float(width)
        self.min_frac = math.inf

    def prior_transform(self, u):
        return self.lo + self.width * np.asarray(u, dtype=float)

    def loglike(self, v):
        v = np.asarray(v, dtype=float)
        t = self.q * (-0.5 * np.sum(v * v, axis=-1))
        self.min_frac = min(self.min_frac, float(np.min(np.abs(t - np.rint(t)))))
        return np.floor(t) / self.q

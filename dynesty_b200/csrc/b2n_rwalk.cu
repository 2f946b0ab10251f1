// b2n_rwalk.cu -- batched random-walk proposal chains: a warp-per-chain kernel (this comment), and three
// lock-step FP64-tensor-core kernels further down (rwalk_mma_kernel and its warp-specialised form
// rwalk_mmaws_kernel for 16 <= n <= 64, rwalk_mmas_kernel for n > 64).  rwalk_plan picks one per call.
//
// Replaces RWalkSampler.sample -> generic_random_walk -> propose_ball_point
// (reference internal_samplers.py:505-561, 866-986, 989-1035) for a whole queue
// of chains in ONE launch.  Per chain and per step:
//   1. fresh U(0,1) on the non-clustered dims (:1011-1013)       [vector uniform event]
//   2. dr = randsphere(ncdim) (bounding.py:1288-1297)            [normal event + uniform event]
//   3. u' = u + scale * axes @ dr on the clustered dims (:1020-1021)
//   4. periodic wrap / reflect (:1024-1029), unitcheck (:1032); an out-of-cube
//      proposal counts as a call and a reject WITHOUT a likelihood call (:951-954)
//   5. v = prior_transform(u'), logl = loglikelihood(v), accept iff logl > loglstar
// exactly `walks` steps; with zero accepts v/logl are recomputed at the start (:970-975).
//
// Mapping of rwalk_kernel (ncdim < n, n < 16, or B2N_RWALK_IMPL=warp).  The grid is persistent-sized: ~one CTA per SM, each CTA owns an equal share of
// the queue (<= 16 chains in flight, one warp per chain) and only chains of ONE ellipsoid,
// whose axes^T and the precision matrix of a GAUSS_PREC model are staged ONCE into shared
// memory (column stride padded to 128 B so every column read is bank-conflict free) and
// then streamed `walks` times by every warp: HBM sees each matrix once per CTA.  Lane i
// owns rows i, i+32 of each mat-vec, the proposal vector is a warp-private shared vector
// read as 16-byte broadcasts; all shared-memory traffic is explicit b2n_sm[] indexing (no
// generic-pointer fix-ups), the wrap/reflect/cube test and the prior transform are fused
// into the mat-vec epilogue, and the two draw events of a step share one Philox + one log.
// The kernel is shared-memory-pipe bound, not HBM bound: the matrices are read from shared
// memory for every proposal, so DRAM traffic is a tiny fraction of the algorithmic bytes.
#include "b2n_rwalk_kernel.cuh"
#include <algorithm>


// =====================================================================================
// rwalk_mma_kernel -- the same chains, 8 at a time per CTA in LOCK-STEP, with both mat-vecs
// done as FP64 tensor-core MMAs (mma.sync m8n8k4 f64 = DMMA) whose A operands -- 8-row slabs
// of axes and of the precision matrix -- live in REGISTERS for the whole kernel.
//
// Why: the warp-per-chain kernel above streams 40 KB of matrix per proposal out of shared
// memory and is bound by the shared-memory pipe.  All chains of
// a CTA use the same matrices and take the same number of steps, so the per-step work of a
// CTA is Y[n x 8] = A[n x n] X[n x 8]: a small dense contraction.  Distributing A over the
// lanes as DMMA fragments (1 double per lane per 8x4 tile; 13 k-tiles for n = 50 -> 26
// registers per matrix per warp) removes the matrix traffic from shared memory entirely and
// replaces ~500 LDS/DFMA per proposal by ~4 DMMA.  Only the 8 direction vectors go through
// shared memory.  Warp w is (i) the owner of chain w (RNG, wrap/reflect/cube test, prior,
// accept/reject: phases 1,3,5) and (ii) the owner of work item (slab w % S, chain-tile w / S)
// of the two contractions (phases 2,4); the directions (phase 1) come from a ring generated 8 steps ahead
// by all warps (see DEPTH below); 3 CTA barriers per step.
// Used when ncdim == ndim, 16 <= n <= 64 (fragments fit in registers); otherwise the
// warp-per-chain kernel runs.  Results agree with it to round-off (different summation order).
// =====================================================================================
__device__ __forceinline__ void dmma884(double& d0, double& d1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(d0), "+d"(d1)
                 : "d"(a), "d"(b));
}
// Two m8n8k4 stacked: a0 / d[0..1] are rows g of the first 8-row half, a1 / d[2..3] rows g of the second, b shared.
// One DMMA.16x8x4 gives the bits of the two DMMA.8x8x4 (tests/test_gpu_mmaws_golden.py, scripts/dmma_shapes.py).
__device__ __forceinline__ void dmma1684(double (&d)[4], double a0, double a1, double b) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                 : "d"(a0), "d"(a1), "d"(b));
}

// Shared-memory plan of rwalk_mma_kernel, in doubles: the kernel takes its offsets from it, the host its size.
// KT = k-tiles of 4 columns (n <= 4*KT); CH = chains in lock-step per CTA (8 -> 256 threads, two
// CTAs per SM overlap each other's barriers instead of one 16-chain CTA per SM waiting at each).
// DEPTH = direction ring: the draws of a step do not depend on the chain state (the Philox counter
// is a function of (chain, tick = 2 * step) only), so the directions of the next DEPTH steps of all
// live chains of the CTA are generated up front and dealt over ALL warps of the CTA.  A full CTA
// (8 chains) gains a barrier per step; a CTA with few chains -- the small rounds of b2n_ns_run run
// one chain per CTA -- generates its directions on 8 warps in parallel instead of serially on one,
// which is the longest dependency chain of a step (Philox -> log -> sqrt -> sincospi).
template <int KT>
struct MmaLayout {
    static constexpr int CH = 8, DEPTH = 8;
    static constexpr int RS = 8 * ((4 * KT + 7) / 8);                    // rows padded to whole 8-row slabs
    static constexpr int XS = RS + ((RS % 16 == 4) ? 0 : ((20 - RS % 16) % 16));   // chain stride == 4 (mod 16):
                                                                         // the B-fragment loads are conflict free
    static constexpr int YS = RS + 2;
    static constexpr int XB = CH * XS;                                   // one direction buffer (all chains of the CTA)
    int n, npad;
    __host__ __device__ explicit MmaLayout(int n_) : n(n_), npad((n_ + 1) & ~1) {}
    __host__ __device__ int o_fl() const { return 4 * npad; }           // dimension flags, after stage_model's vectors
    // ring: direction z of step s, later delta = v - mean
    __host__ __device__ int o_x() const { return o_fl() + (((n + 3) >> 2) << 1); }
    __host__ __device__ int o_y() const { return o_x() + DEPTH * XB; }  // axes @ z (chain-major)
    __host__ __device__ int o_q() const { return o_y() + CH * YS; }     // per-slab partial quadratic forms
    __host__ __device__ int o_f() const { return o_q() + 8 * CH; }      // step factors scale * U^(1/n) / |z|
    __host__ __device__ int o_st() const { return o_f() + DEPTH * CH; } // per-chain state: ucur, uprop, vcur, vprop
    __host__ __device__ int total() const { return o_st() + CH * 4 * npad; }
};

// The draws use the branch-free math of b2n_fastmath.cuh, two ring items at a time per warp, where lane 31 is idle
// (n <= 62); at n = 63, 64 one item at a time with ball_direction.
template <int LIKE, int KT>
__global__ void __launch_bounds__(256, 2) rwalk_mma_kernel(const RwalkParams p) {
    using L = MmaLayout<KT>;
    constexpr int CH = L::CH, DEPTH = L::DEPTH, XS = L::XS, YS = L::YS, XB = L::XB;
    const int n = p.n;
    const int npad = (n + 1) & ~1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    B2N_DYN_PROLOGUE(p)
    const int3 cd = p.cta[blockIdx.x];
    const int S = (n + 7) >> 3;                     // 8-row slabs
    // ---- shared-memory plan
    const L lay(n);
    const ModelSm ms = stage_model(p.m, 0, n, npad);
    const int op0 = ms.op0, op1 = ms.op1, omu = ms.olv0;
    uint32_t* fl = reinterpret_cast<uint32_t*>(&b2n_sm[lay.o_fl()]);
    for (int i = threadIdx.x; i < n; i += blockDim.x) fl[i] = p.dimflags ? p.dimflags[i] : 0u;
    const int oX = lay.o_x(), oY = lay.o_y(), oQ = lay.o_q(), oF = lay.o_f(), ost = lay.o_st();
    for (int e = threadIdx.x; e < DEPTH * XB; e += blockDim.x) b2n_sm[oX + e] = 0.0;
    // ---- matrix fragments -> registers.  item (s, t): slab s of rows, chain tile t
    const int s_it = warp % S, t_it = warp / S;
    const bool has_item = warp < (CH / 8) * S && t_it < CH / 8;
    double fragA[KT], fragP[KT];
    {
        const double* Ag = p.axesT + (size_t)cd.z * n * n;      // axesT[j*n + i] = axes[i][j]
        const double* Pg = p.m.lmat;
        const int row = 8 * s_it + (lane >> 2);
#pragma unroll
        for (int kt = 0; kt < KT; kt++) {
            const int col = 4 * kt + (lane & 3);
            const bool in = has_item && row < n && col < n;
            fragA[kt] = in ? Ag[(size_t)col * n + row] : 0.0;
            fragP[kt] = (LIKE == B2N_LIKE_GAUSS_PREC && in) ? Pg[(size_t)row * n + col] : 0.0;
        }
    }
    __syncthreads();
    const double inv_n = 1.0 / (double)n;
    const int pk = p.m.prior_kind;

    for (int g0 = 0; g0 < cd.y; g0 += CH) {                     // groups of CH chains
        const int c = warp;                                     // chain slot owned by this warp
        const int nlc = (cd.y - g0) < CH ? (cd.y - g0) : CH;    // live chains of the group
        const bool live = c < nlc;
        const int q = live ? p.order[cd.x + g0 + c] : 0;
        int oucur = ost + c * 4 * npad, ouprop = oucur + npad, ovcur = ouprop + npad, ovprop = ovcur + npad;
        const int oy = oY + c * YS;
        if (live)
            for (int i = lane; i < n; i += 32) b2n_sm[oucur + i] = p.u0[(size_t)(p.start ? p.start[q] : q) * n + i];
        int nacc = 0, nrej = 0;
        double lcur = 0.0;
        for (int step0 = 0; step0 < p.walks; step0 += DEPTH) {
            // ---- phase 1 (all warps): directions in the unit ball of the next DEPTH steps of every
            //      live chain -> X[s][chain], factors -> F[s][chain].  Item w = (step s, chain c2).
            const int nd = (p.walks - step0) < DEPTH ? (p.walks - step0) : DEPTH;
            if (n <= 62) {
                for (int w = warp; w < nd * nlc; w += 2 * CH) {         // items w and w + CH together
                    const int w2 = w + CH;
                    const bool two = w2 < nd * nlc;
                    const int sa = w / nlc, ca = w - sa * nlc;
                    const int sb = two ? w2 / nlc : sa, cb = two ? w2 - sb * nlc : ca;
                    ChainRng ga, gb;
                    ga.init(p.seed, chain0_ + (uint64_t)p.order[cd.x + g0 + ca]);
                    gb.init(p.seed, chain0_ + (uint64_t)p.order[cd.x + g0 + cb]);
                    ga.tick = 2u * (uint32_t)(step0 + sa);
                    gb.tick = 2u * (uint32_t)(step0 + sb);
                    double fa, fb;
                    ball_direction_pair_fast(ga, gb, oX + sa * XB + ca * XS, oX + sb * XB + cb * XS, two, n, lane, inv_n,
                                             fa, fb);
                    if (lane == 0) {
                        b2n_sm[oF + sa * CH + ca] = scale_ * fa;
                        if (two) b2n_sm[oF + sb * CH + cb] = scale_ * fb;
                    }
                }
            } else
            for (int w = warp; w < nd * nlc; w += CH) {
                const int s = w / nlc, c2 = w - s * nlc;
                ChainRng g;
                g.init(p.seed, chain0_ + (uint64_t)p.order[cd.x + g0 + c2]);
                g.tick = 2u * (uint32_t)(step0 + s);             // two draw events per step (:1011-1016)
                const double f = scale_ * ball_direction(g, oX + s * XB + c2 * XS, n, lane, inv_n);
                if (lane == 0) b2n_sm[oF + s * CH + c2] = f;
            }
            __syncthreads();
            for (int s = 0; s < nd; s++) {
            const int oXs = oX + s * XB, ox = oXs + c * XS;
            const double fac = live ? b2n_sm[oF + s * CH + c] : 0.0;
            // ---- phase 2 (item warp): Y[rows of slab][chains of tile] = A_slab @ X
            if (has_item) {
                // NACC independent accumulator pairs: the k-tiles form NACC short DMMA dependency chains instead
                // of one long one (a CTA with one chain -- b2n_ns_run's small rounds -- is bound by that latency)
                double d0 = 0.0, d1 = 0.0, e0 = 0.0, e1 = 0.0;
                const int xb = oXs + (8 * t_it + (lane >> 2)) * XS + (lane & 3);
#pragma unroll
                for (int kt = 0; kt + 1 < KT; kt += 2) {
                    dmma884(d0, d1, fragA[kt], b2n_sm[xb + 4 * kt]);
                    dmma884(e0, e1, fragA[kt + 1], b2n_sm[xb + 4 * kt + 4]);
                }
                if (KT & 1) dmma884(d0, d1, fragA[KT - 1], b2n_sm[xb + 4 * (KT - 1)]);
                d0 += e0;
                d1 += e1;
                const int row = 8 * s_it + (lane >> 2), c0 = 8 * t_it + 2 * (lane & 3);
                b2n_sm[oY + c0 * YS + row] = d0;
                b2n_sm[oY + (c0 + 1) * YS + row] = d1;
            }
            __syncthreads();
            // ---- phase 3 (chain warp): u' = u + fac*y, wrap / reflect / cube test, prior, delta -> X[s][c]
            bool ok = true;
            if (live) {
                for (int i = lane; i < n; i += 32) {
                    double t = fma(fac, b2n_sm[oy + i], b2n_sm[oucur + i]);
                    const uint32_t f = fl[i];
                    if (f & B2N_DIM_PERIODIC) t = mod1(t);
                    if (f & B2N_DIM_REFLECTIVE) t = reflect1(t);
                    ok = ok && in_cube(t, f);
                    const double vi = prior_sm(pk, op0, op1, i, t);
                    b2n_sm[ouprop + i] = t;
                    b2n_sm[ovprop + i] = vi;
                    b2n_sm[ox + i] = vi - b2n_sm[omu + i];
                }
                ok = __all_sync(B2N_FULL, ok);
            }
            double l = 0.0;
            if (LIKE == B2N_LIKE_GAUSS_PREC) {
                __syncthreads();
                // ---- phase 4 (item warp): partial delta^T P delta over the rows of the slab
                if (has_item) {
                    double d0 = 0.0, d1 = 0.0, e0 = 0.0, e1 = 0.0;
                    const int xb = oXs + (8 * t_it + (lane >> 2)) * XS + (lane & 3);
#pragma unroll
                    for (int kt = 0; kt + 1 < KT; kt += 2) {
                        dmma884(d0, d1, fragP[kt], b2n_sm[xb + 4 * kt]);
                        dmma884(e0, e1, fragP[kt + 1], b2n_sm[xb + 4 * kt + 4]);
                    }
                    if (KT & 1) dmma884(d0, d1, fragP[KT - 1], b2n_sm[xb + 4 * (KT - 1)]);
                    d0 += e0;
                    d1 += e1;
                    const int row = 8 * s_it + (lane >> 2), c0 = 8 * t_it + 2 * (lane & 3);
                    double q0 = d0 * b2n_sm[oXs + c0 * XS + row], q1 = d1 * b2n_sm[oXs + (c0 + 1) * XS + row];
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) {
                        q0 += __shfl_xor_sync(B2N_FULL, q0, o);
                        q1 += __shfl_xor_sync(B2N_FULL, q1, o);
                    }
                    if (lane < 4) {
                        b2n_sm[oQ + s_it * CH + c0] = q0;
                        b2n_sm[oQ + s_it * CH + c0 + 1] = q1;
                    }
                }
                __syncthreads();
                // ---- phase 5 (chain warp): logl
                double qf = 0.0;
                for (int s2 = 0; s2 < S; s2++) qf += b2n_sm[oQ + s2 * CH + c];
                l = fma(-0.5, qf, p.m.s0);
            } else {
                if (live && ok) {
                    __syncwarp();
                    l = loglike_sm<LIKE, false>(p.m, ms, nullptr, 0, n, n, ovprop, oy, lane);
                }
                __syncthreads();      // Y (scratch of the likelihood) is rewritten by the next step's phase 2
            }
            if (live) {
                if (!ok) {
                    nrej++;
                } else if (l > loglstar_) {
                    int t = oucur; oucur = ouprop; ouprop = t;
                    t = ovcur; ovcur = ovprop; ovprop = t;
                    lcur = l;
                    nacc++;
                } else {
                    nrej++;
                }
            }
            }   // s
            // the ring is regenerated only after every warp has finished reading it (phase 4 of the
            // last step sits before a barrier; phase 3 of non-GAUSS_PREC likelihoods does too)
        }
        if (live) {
            if (nacc == 0) {   // recompute (v, logl) of the start point (:970-975), warp-local
                for (int i = lane; i < n; i += 32) b2n_sm[ovcur + i] = prior_sm(pk, op0, op1, i, b2n_sm[oucur + i]);
                __syncwarp();
                lcur = loglike_sm<LIKE, false>(p.m, ms, p.m.lmat, 0, n, n, ovcur, oy, lane);
            }
            __syncwarp();
            for (int i = lane; i < n; i += 32) {
                peer_put(p.peer, &p.u[(size_t)q * n + i], b2n_sm[oucur + i]);
                peer_put(p.peer, &p.v[(size_t)q * n + i], b2n_sm[ovcur + i]);
            }
            if (lane == 0) {
                peer_put(p.peer, &p.logl[q], lcur);
                peer_put(p.peer, &p.nacc[q], nacc);
                peer_put(p.peer, &p.nrej[q], nrej);
                peer_put(p.peer, &p.ncall[q], (int)p.walks);
            }
        }
        __syncthreads();
        // X rows of chains that are not live in the next group must read as zero
        for (int e = threadIdx.x; e < DEPTH * XB; e += blockDim.x) b2n_sm[oX + e] = 0.0;
        __syncthreads();
    }
    peer_finish(p.peer);
}

// =====================================================================================
// rwalk_mmaws_kernel -- the lock-step kernel, WARP-SPECIALISED (GAUSS_PREC models): 8 step warps + 4 draw warps.
//
// Why: the draws are a large share of the instructions of rwalk_mma_kernel and the only part of it that is
// bound by instruction issue; the step phases are chains of dependent shared-memory loads, DMMAs, shuffles and
// barriers that leave the schedulers idle most of the time.  The draws of a step do not depend on the chain state, so
// they do not have to sit in the same instruction stream at all:
//   * warps 8..11 (one per scheduler) do nothing but draw: they fill a DOUBLE-BUFFERED ring of directions (8 steps x 8
//     chains per buffer) one buffer ahead of the step warps and issue into the cycles the step warps leave empty.
//     A draw warp deals the Philox blocks of its items -- nb = (n + 1) / 2 Box-Muller pair blocks and one radius block
//     each -- over its lanes as ONE flat space, one block per lane and two side by side, so no lane draws a block
//     nobody uses (a warp per item leaves 32 - nb - 1 lanes idle: 6 at n = 50, 15 at n = 32); each block leaves its
//     share of |z|^2 (or log U) in the warp's scratch, and one LANE per item then sums |z|^2 in the association of
//     the former 32-lane butterfly (ss_butterfly: bit-identical) and forms the step factor scale * U^(1/n) / |z|;
//   * warps 0..7 run the step phases of rwalk_mma_kernel on register-resident DMMA fragments, with every shared-memory
//     offset a compile-time constant and TWO barriers per step instead of three (phase 4 of step s and phase 2 of
//     step s + 1 run back to back, then phase 5 of step s and phase 3 of step s + 1);
//   * the direction product axes @ z (phase 2) runs on DMMA.16x8x4, two slabs per instruction, dealt over all 8 step
//     warps as (slab pair, k-tile parity) items: at KT = 13 a warp issues at most 7 DMMAs per step instead of 13, 52
//     per CTA-step instead of 91.  Each parity is summed in the order of the former per-slab accumulator pair and
//     phase 3 adds the two halves, so the chains keep their bits;
//   * the two roles meet at named barriers only (FULL / EMPTY per ring buffer: bar.arrive on one side, bar.sync on
//     the other), the step warps synchronise among themselves on a 256-thread named barrier;
//   * setmaxnreg moves registers from the draw warps (64) to the step warps (88; the fragments alone are 52 registers):
//     256 x 88 + 128 x 64 = the 384 x 80 the CTA is launched with.  Not kept: 96 / 48 -- two side-by-side blocks
//     need about 64 registers, the draw loop spills at 48 and the launch took 5 % longer (H100 SXM, 700 W); the
//     step warps still spill two fragment doubles at 96.  (Budgets are multiples of 8, so 92 / 56 does not exist.)
// Draw events, ticks and arithmetic are those of rwalk_mma_kernel (the step factor is the same expression); delta^T P
// delta is summed as 2 delta^T U delta (below), so results agree with rwalk_mma_kernel to round-off.
// =====================================================================================
template <int KT>
struct MmaWsLayout {
    static constexpr int CH = 8, DEPTH = 8, NSW = 8, NDW = 4;
    static constexpr int RS = 8 * ((4 * KT + 7) / 8);                    // rows padded to whole slabs (>= n)
    static constexpr int XS = RS + ((RS % 16 == 4) ? 0 : ((20 - RS % 16) % 16));
    static constexpr int YS = RS + 2;
    static constexpr int XB = CH * XS;
    static constexpr int RING = DEPTH * XB;
    static constexpr int SMAX = RS / 8;                                  // slabs at the largest n of this KT
    static constexpr int NTMAX = SMAX * KT - SMAX * (SMAX - 1);          // tiles on or above the diagonal: sum (KT - 2 s)
    static constexpr int TPW = (NTMAX + NSW - 1) / NSW;                  // of them per step warp
    static constexpr int O_P0 = 0, O_P1 = RS, O_MU = 2 * RS;            // prior vectors, likelihood mean
    static constexpr int O_FL = 3 * RS;                                  // dimension flags (RS uint32)
    static constexpr int O_X = O_FL + RS / 2;                            // two rings: direction z, later delta = v - mean
    static constexpr int O_Y = O_X + 2 * RING;                           // axes @ z (chain-major), two buffers (slot parity)
    static constexpr int O_Q = O_Y + 2 * CH * YS;                        // partial quadratic forms per step warp
    static constexpr int O_F = O_Q + 8 * CH;                             // step factors, two rings
    // draw warps' scratch: per warp, one row per item of a buffer (DEPTH * CH / NDW of them) with the |z|^2 share of
    // each pair block and log U of the radius block; row stride (nb + 1) | 1 <= SRMAX (odd: the one-lane-per-item
    // reads of a column are bank-conflict free)
    static constexpr int NBMAX = ((4 * KT < 62 ? 4 * KT : 62) + 1) / 2;  // pair blocks at the largest n of this KT
    static constexpr int SRMAX = (NBMAX + 1) | 1;
    static constexpr int SCW = DEPTH * CH / NDW * SRMAX;
    static constexpr int O_SC = O_F + 2 * DEPTH * CH;
    static constexpr int O_ST = O_SC + NDW * SCW;                        // chain state: ucur, uprop, vcur, vprop
    static constexpr int TOTAL = O_ST + CH * 4 * RS;                     // doubles
};
// Static schedule of the symmetric quadratic form (largest n of a KT: S = SMAX slabs): the tiles (slab s, k-tile k)
// with k >= 2 s, in (s, k) order, TPW consecutive ones per step warp.  Everything below is resolved at compile time
// (W = warp index through a switch), so a warp's phase 4 is straight-line code: its DMMAs with immediate offsets and
// one multiply by delta[rows of the slab] at the end of each run of tiles of one slab.
template <int KT>
struct SymSched {
    using L = MmaWsLayout<KT>;
    static constexpr int NT = L::NTMAX, TPW = L::TPW;
    static constexpr __host__ __device__ int slab(int t) { int s = 0; while (t >= KT - 2 * s) { t -= KT - 2 * s; s++; } return s; }
    static constexpr __host__ __device__ int ktile(int t) { int s = 0; while (t >= KT - 2 * s) { t -= KT - 2 * s; s++; } return 2 * s + t; }
    // position of tile t inside the run of tiles of its slab that belongs to warp t / TPW
    static constexpr __host__ __device__ int runpos(int t) {
        const int first = (t / TPW) * TPW;
        return slab(first) == slab(t) ? t - first : ktile(t) - 2 * slab(t);
    }
    static constexpr __host__ __device__ bool runend(int t) { return (t + 1) % TPW == 0 || t + 1 == NT || slab(t + 1) != slab(t); }
};
template <int KT, int W, int J>
__device__ __forceinline__ void sym_load(double (&fragU)[MmaWsLayout<KT>::TPW], const double* __restrict__ Pg, int n, int lane) {
    using Sch = SymSched<KT>;
    if constexpr (J < Sch::TPW) {
        constexpr int t = W * Sch::TPW + J;
        double u = 0.0;
        if constexpr (t < Sch::NT) {
            constexpr int ts = Sch::slab(t), tk = Sch::ktile(t);
            const int row = 8 * ts + (lane >> 2), col = 4 * tk + (lane & 3);
            if (row < n && col < n && col >= row) u = (col == row ? 0.5 : 1.0) * Pg[(size_t)row * n + col];
        }
        fragU[J] = u;
        sym_load<KT, W, J + 1>(fragU, Pg, n, lane);
    }
}
template <int KT, int W, int J>
__device__ __forceinline__ void sym_tiles(const double (&fragU)[MmaWsLayout<KT>::TPW], int xt, int xr, double& d0, double& d1,
                                          double& e0, double& e1, double& q0, double& q1) {
    using Sch = SymSched<KT>;
    constexpr int XS = MmaWsLayout<KT>::XS;
    constexpr int t = W * Sch::TPW + J;
    if constexpr (J < Sch::TPW && t < Sch::NT) {
        constexpr int s = Sch::slab(t), k = Sch::ktile(t), pos = Sch::runpos(t);
        if constexpr (pos & 1) dmma884(e0, e1, fragU[J], b2n_sm[xt + 4 * k]);
        else dmma884(d0, d1, fragU[J], b2n_sm[xt + 4 * k]);
        if constexpr (Sch::runend(t)) {       // multiply the slab's rows by delta[rows], start the next run from zero
            if constexpr (pos >= 1) {
                q0 = fma(d0 + e0, b2n_sm[xr + 8 * s], q0);
                q1 = fma(d1 + e1, b2n_sm[xr + XS + 8 * s], q1);
                e0 = 0.0; e1 = 0.0;
            } else {
                q0 = fma(d0, b2n_sm[xr + 8 * s], q0);
                q1 = fma(d1, b2n_sm[xr + XS + 8 * s], q1);
            }
            d0 = 0.0; d1 = 0.0;
        }
        sym_tiles<KT, W, J + 1>(fragU, xt, xr, d0, d1, e0, e1, q0, q1);
    }
}
#define B2N_WARP_SWITCH(W_, CALL)                                                                      \
    switch (W_) {                                                                                      \
        case 0: CALL(0); break; case 1: CALL(1); break; case 2: CALL(2); break; case 3: CALL(3); break; \
        case 4: CALL(4); break; case 5: CALL(5); break; case 6: CALL(6); break; default: CALL(7); break; \
    }

__device__ __forceinline__ void nbar_sync(int id, int count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void nbar_arrive(int id, int count) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// PLAIN: no periodic / reflective dimension and a prior that is affine per component (uniform, identity): phase 3 is
// then straight-line code for the (at most) two components of a lane.
// Ring: RB = 2 buffers of DB = 8 steps; the step warps start every buffer with a two-interval prologue.  Not kept: ONE
// pipeline over all ring slots, the next buffer awaited where it is first touched (two steps early) -- the draw warps are
// busy most of the time, and taking two steps of slack away from them makes both roles wait for each other.
template <int KT, bool PLAIN>
__global__ void __launch_bounds__(384, 2) rwalk_mmaws_kernel(const RwalkParams p) {
    using L = MmaWsLayout<KT>;
    constexpr int CH = L::CH, XS = L::XS, YS = L::YS, XB = L::XB, RS = L::RS;
    constexpr int DB = L::DEPTH, RB = 2;
    constexpr int BAR_STEP = 1, BAR_FULL = 2, BAR_EMPTY = 2 + RB;  // named barriers (0 = __syncthreads)
    const int n = p.n;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    B2N_DYN_PROLOGUE(p)
    const int3 cd = p.cta[blockIdx.x];
    uint32_t* fl = reinterpret_cast<uint32_t*>(&b2n_sm[L::O_FL]);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        b2n_sm[L::O_P0 + i] = p.m.pp0 ? p.m.pp0[i] : 0.0;
        b2n_sm[L::O_P1 + i] = p.m.pp1 ? p.m.pp1[i] : 1.0;
        b2n_sm[L::O_MU + i] = p.m.lv0 ? p.m.lv0[i] : 0.0;
        fl[i] = p.dimflags ? p.dimflags[i] : 0u;
    }
    for (int e = threadIdx.x; e < 2 * L::RING; e += blockDim.x) b2n_sm[L::O_X + e] = 0.0;
    __syncthreads();
    const int NB = (p.walks + DB - 1) / DB;                       // ring buffers filled per group of chains

    if (warp >= L::NSW) {
        // =============================== draw warps ===============================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 64;");
        const int dw = warp - L::NSW;
        const double inv_n = 1.0 / (double)n;
        const int nb1 = ((n + 1) >> 1) + 1;                       // Philox blocks per item: pair blocks + the radius block
        const int SR = nb1 | 1, osc = L::O_SC + dw * L::SCW;
        for (int g0 = 0; g0 < cd.y; g0 += CH) {
            const int nlc = (cd.y - g0) < CH ? (cd.y - g0) : CH;
            for (int blk = 0; blk < NB; blk++) {
                const int b = blk & (RB - 1), step0 = blk * DB;
                const int nd = (p.walks - step0) < DB ? (p.walks - step0) : DB;
                const int nit = nd * nlc;
                const int oXb = L::O_X + b * DB * XB;
                if (blk >= RB) nbar_sync(BAR_EMPTY + b, 384);     // the step warps have finished with this buffer
                // this warp's items: w = dw + NDW * k, k < cnt.  Their blocks form one flat space, task t = k * nb1 + j,
                // dealt one block per lane, two tasks (t, t + 32) side by side while both halves are busy
                const int cnt = (nit - dw + L::NDW - 1) / L::NDW, T = cnt * nb1;
                auto task = [&](int t, ChainRng& g, int& j, int& off, int& o) {
                    const int k = t / nb1, w = dw + L::NDW * k;
                    j = t - k * nb1;
                    int s, c2;
                    if (nlc == CH) { s = w >> 3; c2 = w & 7; }
                    else { s = w / nlc; c2 = w - s * nlc; }
                    g.init(p.seed, chain0_ + (uint64_t)p.order[cd.x + g0 + c2]);
                    g.tick = 2u * (uint32_t)(step0 + s);
                    off = oXb + s * XB + c2 * XS;
                    o = osc + k * SR + j;
                };
                int t0 = 0;
                for (; t0 + 32 < T; t0 += 64) {
                    const int tb = t0 + 32 + lane;
                    const bool two = tb < T;
                    ChainRng ga, gb;
                    int ja, offa, oa, jb, offb, ob;
                    task(t0 + lane, ga, ja, offa, oa);
                    task(two ? tb : t0 + lane, gb, jb, offb, ob);
                    ball_block_fast(ga, ja, n, offa, oa, true);
                    ball_block_fast(gb, jb, n, offb, ob, two);
                }
                if (t0 < T) {
                    const bool one = t0 + lane < T;
                    ChainRng g;
                    int j, off, o;
                    task(one ? t0 + lane : t0, g, j, off, o);
                    ball_block_fast(g, j, n, off, o, one);
                }
                __syncwarp();
                if (lane < cnt) {         // step factors, one lane per item (cnt <= DB * CH / NDW = 16)
                    const int w = dw + L::NDW * lane;
                    int s, c2;
                    if (nlc == CH) { s = w >> 3; c2 = w & 7; }
                    else { s = w / nlc; c2 = w - s * nlc; }
                    const int o = osc + lane * SR;
                    const double ss = ss_butterfly<1>(o, nb1 - 1, 0);
                    b2n_sm[L::O_F + b * DB * CH + s * CH + c2] = scale_ * b2n_div(exp(b2n_sm[o + nb1 - 1] * inv_n), b2n_sqrt(ss));
                }
                __syncwarp();             // the next buffer's blocks rewrite the scratch
                __threadfence_block();
                nbar_arrive(BAR_FULL + b, 384);
            }
            // group boundary: both roles meet, the rings are cleared (rows of chains that are not live in the next group)
            __syncthreads();
            for (int e = threadIdx.x; e < 2 * L::RING; e += blockDim.x) b2n_sm[L::O_X + e] = 0.0;
            __syncthreads();
        }
    } else {
        // =============================== step warps ===============================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 88;");
        // axes @ z: item (slab pair pp, k-tile parity kpar) -- the rows of slabs 2 pp, 2 pp + 1 as the two halves of
        // m16n8k4 tiles, over the k-tiles of one parity.  The even items sum the even k-tiles in order, the odd items
        // the odd ones, and phase 3 adds the two: the association of the former per-slab accumulator pair (d, e).
        constexpr int NP = (L::SMAX + 1) / 2;                      // slab pairs (KT = 13: slab 7 of pair 3 is padding)
        constexpr int NKH = (KT + 1) / 2;                          // k-tiles of the even parity; the odd one has KT / 2
        const bool has_item = warp < 2 * NP;
        const int pp = warp % NP, kpar = warp / NP;               // the two parities of a pair on different schedulers
        double fragA[2 * NKH];                                    // k-tile 2 j + kpar: [2 j] slab 2 pp, [2 j + 1] slab 2 pp + 1
        {
            const double* Ag = p.axesT + (size_t)cd.z * n * n;
            const int row = 16 * pp + (lane >> 2);
#pragma unroll
            for (int j = 0; j < NKH; j++) {
                const int col = 4 * (2 * j + kpar) + (lane & 3);
                fragA[2 * j] = (has_item && row < n && col < n) ? Ag[(size_t)col * n + row] : 0.0;
                fragA[2 * j + 1] = (has_item && row + 8 < n && col < n) ? Ag[(size_t)col * n + row + 8] : 0.0;
            }
        }
        // The precision matrix is symmetric: delta^T P delta = 2 delta^T U delta with U = its upper triangle and HALF
        // its diagonal, so only the (slab, k-tile) tiles on or above the diagonal are contracted -- 49 of the 91 at
        // n = 50 -- dealt over all 8 warps by the static schedule SymSched (this kernel runs for S == SMAX only).
        double fragU[L::TPW];
#define B2N_SYM_LOAD(W_) sym_load<KT, W_, 0>(fragU, p.m.lmat, n, lane)
        B2N_WARP_SWITCH(warp, B2N_SYM_LOAD)
#undef B2N_SYM_LOAD
        const int xb_it = (lane >> 2) * XS + (lane & 3);                          // B fragment of k-tile 0
        const int yr_it = 16 * pp + (lane >> 2);                                  // row of d[0], d[1] (chains 2 t, 2 t + 1)
        const int xr_it = 2 * (lane & 3) * XS + (lane >> 2);                      // delta[row 0 of a slab] of chain c0
        const int pk = p.m.prior_kind;
        const int c = warp;                                       // chain slot owned by this warp

        for (int g0 = 0; g0 < cd.y; g0 += CH) {
            const int nlc = (cd.y - g0) < CH ? (cd.y - g0) : CH;
            const bool live = c < nlc;
            const int q = live ? p.order[cd.x + g0 + c] : 0;
            // chain state in shared memory: [u_a | u_b | v_a | v_b]; `par` says which half holds the current point
            const int ost = L::O_ST + c * 4 * RS;
            int par = 0;
#define oucur (ost + par * RS)
#define ouprop (ost + (par ^ 1) * RS)
#define ovcur (ost + 2 * RS + par * RS)
#define ovprop (ost + 2 * RS + (par ^ 1) * RS)
            if (live)
                for (int i = lane; i < n; i += 32) b2n_sm[oucur + i] = p.u0[(size_t)(p.start ? p.start[q] : q) * n + i];
            int nacc = 0, nrej = 0;
            double lcur = 0.0;
            bool ok = true;

            // phase 2 of a ring slot: this warp's half of axes @ z (d) -- the DMMAs are issued in the interval before
            // the one that stores them (phase2_store), so the tensor pipe works on the next-but-one step while the warp
            // walks through the latency chains of phases 5 and 3, and the z rows the DMMAs read are dead by the store
            auto phase2_issue = [&](int oXs, double (&d)[4]) {
                d[0] = 0.0; d[1] = 0.0; d[2] = 0.0; d[3] = 0.0;
                const int xb = oXs + xb_it + 4 * kpar;
#pragma unroll
                for (int j = 0; j < NKH; j++)
                    if (KT % 2 == 0 || j + 1 < NKH || kpar == 0) dmma1684(d, fragA[2 * j], fragA[2 * j + 1], b2n_sm[xb + 8 * j]);
            };
            // the even half goes to Y[buf], the odd half to oo (chain stride so): the z rows of its own ring slot (read by
            // nobody once the slot's DMMAs are issued; phase 3 reads each element before it writes delta over it) or,
            // for slot 0, Y[1].  Rows of the padding slab are not stored: they would run past a chain's row of Y.
            auto phase2_store = [&](int buf, int oo, int so, const double (&d)[4]) {
                const int cs = kpar ? so : YS;
                const int o = (kpar ? oo : L::O_Y + buf * CH * YS) + 2 * (lane & 3) * cs + yr_it;
                b2n_sm[o] = d[0];
                b2n_sm[o + cs] = d[1];
                if (2 * pp + 1 < L::SMAX) {
                    b2n_sm[o + 8] = d[2];
                    b2n_sm[o + cs + 8] = d[3];
                }
            };
            // u' = u + fac*y with y = the even half at oy + the odd half at oz, wrap / reflect / cube test, prior,
            // delta -> X[s][c]
            auto phase3 = [&](int oXs, double fac, int oy, int oz) {
                if (PLAIN) {
                    const int i0 = lane, i1 = lane + 32;
                    const bool v0 = i0 < n, v1 = i1 < n;
                    double t0 = 0.5, t1 = 0.5;
                    if (v0) t0 = fma(fac, b2n_sm[oy + i0] + b2n_sm[oz + i0], b2n_sm[oucur + i0]);
                    if (v1) t1 = fma(fac, b2n_sm[oy + i1] + b2n_sm[oz + i1], b2n_sm[oucur + i1]);
                    const bool good = (t0 > 0.0 && t0 < 1.0) && (t1 > 0.0 && t1 < 1.0);
                    if (v0) {
                        const double vi = fma(b2n_sm[L::O_P1 + i0], t0, b2n_sm[L::O_P0 + i0]);
                        b2n_sm[ouprop + i0] = t0;
                        b2n_sm[ovprop + i0] = vi;
                        b2n_sm[oXs + c * XS + i0] = vi - b2n_sm[L::O_MU + i0];
                    }
                    if (v1) {
                        const double vi = fma(b2n_sm[L::O_P1 + i1], t1, b2n_sm[L::O_P0 + i1]);
                        b2n_sm[ouprop + i1] = t1;
                        b2n_sm[ovprop + i1] = vi;
                        b2n_sm[oXs + c * XS + i1] = vi - b2n_sm[L::O_MU + i1];
                    }
                    ok = __all_sync(B2N_FULL, good);
                    return;
                }
                bool good = true;
                for (int i = lane; i < n; i += 32) {
                    double t = fma(fac, b2n_sm[oy + i] + b2n_sm[oz + i], b2n_sm[oucur + i]);
                    const uint32_t f = fl[i];
                    if (f & B2N_DIM_PERIODIC) t = mod1(t);
                    if (f & B2N_DIM_REFLECTIVE) t = reflect1(t);
                    good = good && in_cube(t, f);
                    const double vi = prior_sm(pk, L::O_P0, L::O_P1, i, t);
                    b2n_sm[ouprop + i] = t;
                    b2n_sm[ovprop + i] = vi;
                    b2n_sm[oXs + c * XS + i] = vi - b2n_sm[L::O_MU + i];
                }
                ok = __all_sync(B2N_FULL, good);
            };
            auto phase4 = [&](int oXs) {          // this warp's tiles of delta^T U delta
                double q0 = 0.0, q1 = 0.0, d0 = 0.0, d1 = 0.0, e0 = 0.0, e1 = 0.0;
                const int xt = oXs + xb_it, xr = oXs + xr_it;
#define B2N_SYM_TILES(W_) sym_tiles<KT, W_, 0>(fragU, xt, xr, d0, d1, e0, e1, q0, q1)
                B2N_WARP_SWITCH(warp, B2N_SYM_TILES)
#undef B2N_SYM_TILES
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) {
                    q0 += __shfl_xor_sync(B2N_FULL, q0, o);
                    q1 += __shfl_xor_sync(B2N_FULL, q1, o);
                }
                if (lane < 4) {
                    b2n_sm[L::O_Q + warp * CH + 2 * lane] = q0;
                    b2n_sm[L::O_Q + warp * CH + 2 * lane + 1] = q1;
                }
            };
            auto phase5 = [&]() {                 // logl = s0 - delta^T U delta, accept / reject
                double qf = 0.0;
#pragma unroll
                for (int w2 = 0; w2 < L::NSW; w2++) qf += b2n_sm[L::O_Q + w2 * CH + c];
                const double l = p.m.s0 - qf;
                if (ok && l > loglstar_) {
                    par ^= 1;
                    lcur = l;
                    nacc++;
                } else {
                    nrej++;
                }
            };

            // Two barrier intervals per step,
            //   I(g) = [store phase 2 of slot g + 1] phase 4 of slot g
            //   C(g) = [issue phase 2 of slot g + 2] phase 5 of slot g, phase 3 of slot g + 1
            // per ring buffer (nd <= 8 slots), with a prologue that stores slot 0 and issues slot 1
            for (int blk = 0; blk < NB; blk++) {
                const int b = blk & 1, step0 = blk * DB;
                const int nd = (p.walks - step0) < DB ? (p.walks - step0) : DB;
                const int oXb = L::O_X + b * DB * XB, oFb = L::O_F + b * DB * CH;
                double d[4];                                      // phase 2 of the next slot, issued and not yet stored
                nbar_sync(BAR_FULL + b, 384);                     // the draw warps have filled this buffer
                if (has_item) {
                    phase2_issue(oXb, d);
                    phase2_store(0, L::O_Y + CH * YS, YS, d);
                    if (nd > 1) phase2_issue(oXb + XB, d);
                }
                nbar_sync(BAR_STEP, 256);
                if (live) phase3(oXb, b2n_sm[oFb + c], L::O_Y + c * YS, L::O_Y + (CH + c) * YS);
                nbar_sync(BAR_STEP, 256);
                for (int s2 = 0; s2 < nd; s2++) {
                    const int oXn = oXb + (s2 + 1) * XB;          // slot s2 + 1
                    if (has_item && s2 + 1 < nd) phase2_store((s2 + 1) & 1, oXn, XS, d);
                    phase4(oXb + s2 * XB);
                    nbar_sync(BAR_STEP, 256);
                    // every read of this ring buffer is done: hand it back to the draw warps (if they will ask for it)
                    if (s2 == nd - 1 && blk + 2 < NB) nbar_arrive(BAR_EMPTY + b, 384);
                    if (has_item && s2 + 2 < nd) phase2_issue(oXb + (s2 + 2) * XB, d);
                    if (live) phase5();
                    if (s2 + 1 < nd) {
                        if (live) phase3(oXn, b2n_sm[oFb + (s2 + 1) * CH + c], L::O_Y + (((s2 + 1) & 1) * CH + c) * YS, oXn + c * XS);
                        nbar_sync(BAR_STEP, 256);
                    }
                }
            }
            if (live) {
                if (nacc == 0) {   // recompute (v, logl) of the start point (:970-975), warp-local
                    const int oy = L::O_Y + c * YS;
                    __syncwarp();
                    for (int i = lane; i < n; i += 32) {
                        const double vi = prior_sm(pk, L::O_P0, L::O_P1, i, b2n_sm[oucur + i]);
                        b2n_sm[ovcur + i] = vi;
                        b2n_sm[oy + i] = vi - b2n_sm[L::O_MU + i];
                    }
                    __syncwarp();
                    lcur = fma(-0.5, quadform_full<false>(p.m.lmat, 0, n, n, oy, lane), p.m.s0);
                }
                __syncwarp();
                for (int i = lane; i < n; i += 32) {
                    peer_put(p.peer, &p.u[(size_t)q * n + i], b2n_sm[oucur + i]);
                    peer_put(p.peer, &p.v[(size_t)q * n + i], b2n_sm[ovcur + i]);
                }
                if (lane == 0) {
                    peer_put(p.peer, &p.logl[q], lcur);
                    peer_put(p.peer, &p.nacc[q], nacc);
                    peer_put(p.peer, &p.nrej[q], nrej);
                    peer_put(p.peer, &p.ncall[q], (int)p.walks);
                }
            }
            __syncthreads();
            for (int e = threadIdx.x; e < 2 * L::RING; e += blockDim.x) b2n_sm[L::O_X + e] = 0.0;
            __syncthreads();
#undef oucur
#undef ouprop
#undef ovcur
#undef ovprop
        }
    }
    peer_finish(p.peer);
}

// =====================================================================================
// rwalk_mmas_kernel -- lock-step DMMA kernel for LARGE n (64 < n: the matrix fragments do not
// fit in registers, and at n = 200 the 320 KB axes matrix does not even fit in shared memory).
// Same phases as rwalk_mma_kernel with 16 chains per CTA, but the A-operand fragments are
// STREAMED from global memory (L2-resident) every step: each 8x4 fragment is loaded once per
// CTA-step and feeds two DMMAs (the two 8-chain tiles), so the L2 traffic per proposal is
// n^2*8/16 bytes instead of the n^2*8 of the warp-per-chain kernel (20 KB vs 320 KB at n=200).
// Warp w owns slabs w, w+16, ...  BASELINE config C4 (200-D, single ellipsoid, rwalk).
// =====================================================================================
// Shared-memory plan of rwalk_mmas_kernel, in doubles: the kernel takes its offsets from it, the host its size.
struct MmasLayout {
    static constexpr int CH = 16;
    int n, npad;
    int RS, XS, YS; // rows padded to whole 8-row slabs; chain strides of X (== 4 mod 16: conflict-free B fragments), Y
    __host__ __device__ explicit MmasLayout(int n_)
        : n(n_), npad((n_ + 1) & ~1), RS(8 * ((n_ + 7) / 8)), XS(RS + ((RS % 16 == 4) ? 0 : ((20 - RS % 16) % 16))),
          YS(RS + 2) {}
    __host__ __device__ int o_fl() const { return 4 * npad; }           // dimension flags, after stage_model's vectors
    // direction z, later delta = v - mean (chain-major)
    __host__ __device__ int o_x() const { return o_fl() + (((n + 3) >> 2) << 1); }
    __host__ __device__ int o_y() const { return o_x() + CH * XS; }     // axes @ z (chain-major)
    __host__ __device__ int o_q() const { return o_y() + CH * YS; }     // per-slab partial quadratic forms
    __host__ __device__ int o_st() const { return o_q() + (RS / 8) * CH; }  // per-chain state: ucur, uprop, vcur, vprop
    // helper scratch: step factors, U^(1/n), current state buffers, cube flags (CH x CH ints)
    __host__ __device__ int o_h() const { return o_st() + CH * 4 * npad; }
    __host__ __device__ int total() const { return o_h() + 3 * CH + CH * CH / 2; }
};

template <int LIKE>
__global__ void __launch_bounds__(512, 1) rwalk_mmas_kernel(const RwalkParams p) {
    constexpr int CH = MmasLayout::CH;
    const int n = p.n;
    const int npad = (n + 1) & ~1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    B2N_DYN_PROLOGUE(p)
    const int3 cd = p.cta[blockIdx.x];
    const int S = (n + 7) >> 3, KT = (n + 3) >> 2;
    const MmasLayout lay(n);
    const int XS = lay.XS, YS = lay.YS;
    const ModelSm ms = stage_model(p.m, 0, n, npad);
    const int op0 = ms.op0, op1 = ms.op1, omu = ms.olv0;
    uint32_t* fl = reinterpret_cast<uint32_t*>(&b2n_sm[lay.o_fl()]);
    for (int i = threadIdx.x; i < n; i += blockDim.x) fl[i] = p.dimflags ? p.dimflags[i] : 0u;
    const int oX = lay.o_x(), oY = lay.o_y(), oQ = lay.o_q(), ost = lay.o_st();
    for (int e = threadIdx.x; e < CH * XS; e += blockDim.x) b2n_sm[oX + e] = 0.0;
    const double* __restrict__ Ag = p.axesT + (size_t)cd.z * n * n;     // axesT[col*n + row] = axes[row][col]
    const double* __restrict__ Pg = p.m.lmat;                             // symmetric
    __syncthreads();
    const double inv_n = 1.0 / (double)n;
    const int pk = p.m.prior_kind;
    const int lr = lane >> 2, lc = lane & 3;

    // ---- helper scratch: step factor, U^(1/n), which state buffer is current, per-helper cube flags
    const int oH = lay.o_h();
    double* facbuf = &b2n_sm[oH];
    double* pwbuf = &b2n_sm[oH + CH];
    int* selbuf = reinterpret_cast<int*>(&b2n_sm[oH + 2 * CH]);
    int* okbuf = reinterpret_cast<int*>(&b2n_sm[oH + 3 * CH]);            // CH x CH

    for (int g0 = 0; g0 < cd.y; g0 += CH) {
        // L chains are live in this pass.  A pass with few chains (the rounds of b2n_ns_run put 1-2 chains on a CTA)
        // used to leave 14 of the 16 warps idle outside the contraction while the chain's own warp generated its
        // 200 normals (4 Philox / log / sincos rounds), U^(1/n) and 200 ndtri's one after the other: H = 16 / L
        // warps now serve a chain -- the owner (h = 0: chain state, accept test, counters) and H - 1 helpers that
        // take their share of the ELEMENTWISE work (normal blocks, the radius power, wrap / cube test / prior / delta
        // of their elements).  Every element is computed by the same instructions as before and every sum is still
        // formed by the owner in the old order (|z|^2 from the stored z), so a chain's result does not depend on
        // how many warps worked on it -- nor, therefore, on the batch it is part of.
        const int L = min(CH, cd.y - g0);
        const int H = CH / L;
        const int c = warp % L, h = warp / L;
        const bool owner = h == 0, helper = h < H;
        const int q = p.order[cd.x + g0 + c];
        const int sbase = ost + c * 4 * npad;
        int oucur = sbase, ouprop = sbase + npad, ovcur = ouprop + npad, ovprop = ovcur + npad;
        const int ox = oX + c * XS, oy = oY + c * YS;
        const bool two = L > 8;                   // chains 8..15 exist: second column tile of the contractions
        ChainRng g;
        g.init(p.seed, chain0_ + (uint64_t)q);
        if (owner) {
            for (int i = lane; i < n; i += 32) b2n_sm[oucur + i] = p.u0[(size_t)(p.start ? p.start[q] : q) * n + i];
            if (lane == 0) selbuf[c] = 0;
        }
        int nacc = 0, nrej = 0;
        double lcur = 0.0;
        const int nb = (n + 1) >> 1;
        __syncthreads();
        for (int step = 0; step < p.walks; step++) {
            // ---- draw events of the step: normal vector (tick 2 step), radius uniform (tick 2 step + 1)
            if (helper) {
                g.tick = 2u * (uint32_t)step;
                for (int b = 32 * h + lane; b < nb; b += 32 * H) {
                    double z0, z1;
                    rng_normal_pair(g, b, z0, z1);
                    if (2 * b + 1 < n) *reinterpret_cast<double2*>(&b2n_sm[ox + 2 * b]) = make_double2(z0, z1);
                    else b2n_sm[ox + 2 * b] = z0;
                }
                if (h == H - 1) {
                    g.tick = 2u * (uint32_t)step + 1u;
                    const double U = rng_uniform(g);
                    const double pw = pow(U, inv_n);
                    if (lane == 0) pwbuf[c] = pw;
                }
            }
            __syncthreads();
            if (owner) {                              // |z|^2 in normals_sm's order, then the step factor
                double ss = 0.0;
                for (int b = lane; b < nb; b += 32) {
                    const double z0 = b2n_sm[ox + 2 * b];
                    ss = fma(z0, z0, ss);
                    if (2 * b + 1 < n) { const double z1 = b2n_sm[ox + 2 * b + 1]; ss = fma(z1, z1, ss); }
                }
                ss = warp_sum(ss);
                if (lane == 0) facbuf[c] = scale_ * (pwbuf[c] / sqrt(ss));
            }
            // ---- Y = A X, fragments of A streamed from L2 (slabs dealt from the LAST warp down: the owners -- warps
            //      0 .. L-1, which have just formed the step factors -- get the fewest)
            for (int s = CH - 1 - warp; s < S; s += CH) {
                const int row = 8 * s + lr;
                const bool rv = row < n;
                const double* ap = Ag + (rv ? row : 0) + (size_t)lc * n;
                const int xb0 = oX + lr * XS + lc, xb1 = xb0 + 8 * XS;
                double d00 = 0, d01 = 0, d10 = 0, d11 = 0;
                if (two) {
#pragma unroll 8
                    for (int kt = 0; kt < KT; kt++) {
                        const bool in = rv && (4 * kt + lc) < n;
                        const double a = in ? __ldg(ap + (size_t)(4 * kt) * n) : 0.0;
                        dmma884(d00, d01, a, b2n_sm[xb0 + 4 * kt]);
                        dmma884(d10, d11, a, b2n_sm[xb1 + 4 * kt]);
                    }
                } else {
                    // (one column tile: the loop is a load and a DMMA -- 25 loads in flight per warp instead of 8,
                    //  the phase is bound by the L2 round trips of its fragment loads)
#pragma unroll 25
                    for (int kt = 0; kt < KT; kt++) {
                        const bool in = rv && (4 * kt + lc) < n;
                        const double a = in ? __ldg(ap + (size_t)(4 * kt) * n) : 0.0;
                        dmma884(d00, d01, a, b2n_sm[xb0 + 4 * kt]);
                    }
                }
                const int c0 = 2 * lc;
                b2n_sm[oY + c0 * YS + row] = d00;
                b2n_sm[oY + (c0 + 1) * YS + row] = d01;
                if (two) {
                    b2n_sm[oY + (8 + c0) * YS + row] = d10;
                    b2n_sm[oY + (9 + c0) * YS + row] = d11;
                }
            }
            __syncthreads();
            // ---- proposal u' = u + fac y, wrap / reflect / cube test, prior, delta: elements dealt over the H warps
            if (helper) {
                const double fac = facbuf[c];
                const int sel = selbuf[c];
                const int ucur_ = sel ? sbase + npad : sbase, uprop_ = sel ? sbase : sbase + npad;
                const int vprop_ = sel ? sbase + 2 * npad : sbase + 3 * npad;
                bool okp = true;
                for (int i = 32 * h + lane; i < n; i += 32 * H) {
                    double t = fma(fac, b2n_sm[oy + i], b2n_sm[ucur_ + i]);
                    const uint32_t f = fl[i];
                    if (f & B2N_DIM_PERIODIC) t = mod1(t);
                    if (f & B2N_DIM_REFLECTIVE) t = reflect1(t);
                    okp = okp && in_cube(t, f);
                    const double vi = prior_sm(pk, op0, op1, i, t);
                    b2n_sm[uprop_ + i] = t;
                    b2n_sm[vprop_ + i] = vi;
                    b2n_sm[ox + i] = vi - b2n_sm[omu + i];
                }
                okp = __all_sync(B2N_FULL, okp);
                if (lane == 0) okbuf[c * CH + h] = okp ? 1 : 0;
            }
            __syncthreads();
            bool ok = true;
            if (owner)
                for (int k = 0; k < H; k++) ok = ok && (okbuf[c * CH + k] != 0);
            double l = 0.0;
            if (LIKE == B2N_LIKE_GAUSS_PREC) {
                for (int s = warp; s < S; s += CH) {
                    const int row = 8 * s + lr;
                    const bool rv = row < n;
                    const double* pp = Pg + (rv ? row : 0) + (size_t)lc * n;
                    const int xb0 = oX + lr * XS + lc, xb1 = xb0 + 8 * XS;
                    double d00 = 0, d01 = 0, d10 = 0, d11 = 0;
#pragma unroll 8
                    for (int kt = 0; kt < KT; kt++) {
                        const bool in = rv && (4 * kt + lc) < n;
                        const double a = in ? __ldg(pp + (size_t)(4 * kt) * n) : 0.0;
                        dmma884(d00, d01, a, b2n_sm[xb0 + 4 * kt]);
                        if (two) dmma884(d10, d11, a, b2n_sm[xb1 + 4 * kt]);
                    }
                    const int c0 = 2 * lc;
                    double q00 = d00 * b2n_sm[oX + c0 * XS + row], q01 = d01 * b2n_sm[oX + (c0 + 1) * XS + row];
                    double q10 = d10 * b2n_sm[oX + (8 + c0) * XS + row], q11 = d11 * b2n_sm[oX + (9 + c0) * XS + row];
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) {
                        q00 += __shfl_xor_sync(B2N_FULL, q00, o);
                        q01 += __shfl_xor_sync(B2N_FULL, q01, o);
                        q10 += __shfl_xor_sync(B2N_FULL, q10, o);
                        q11 += __shfl_xor_sync(B2N_FULL, q11, o);
                    }
                    if (lane < 4) {
                        b2n_sm[oQ + s * CH + c0] = q00;
                        b2n_sm[oQ + s * CH + c0 + 1] = q01;
                        b2n_sm[oQ + s * CH + 8 + c0] = q10;
                        b2n_sm[oQ + s * CH + 9 + c0] = q11;
                    }
                }
                __syncthreads();
                double qf = 0.0;
                for (int s = 0; s < S; s++) qf += b2n_sm[oQ + s * CH + c];
                l = fma(-0.5, qf, p.m.s0);
            } else if (owner && ok) {
                l = loglike_sm<LIKE, false>(p.m, ms, nullptr, 0, n, n, ovprop, oy, lane);
            }
            if (owner) {
                if (!ok) {
                    nrej++;
                } else if (l > loglstar_) {
                    int t = oucur; oucur = ouprop; ouprop = t;
                    t = ovcur; ovcur = ovprop; ovprop = t;
                    lcur = l;
                    nacc++;
                    if (lane == 0) selbuf[c] ^= 1;
                } else {
                    nrej++;
                }
            }
        }
        if (owner) {
            if (nacc == 0) {
                for (int i = lane; i < n; i += 32) b2n_sm[ovcur + i] = prior_sm(pk, op0, op1, i, b2n_sm[oucur + i]);
                __syncwarp();
                lcur = loglike_sm<LIKE, false>(p.m, ms, p.m.lmat, 0, n, n, ovcur, oy, lane);
            }
            __syncwarp();
            for (int i = lane; i < n; i += 32) {
                peer_put(p.peer, &p.u[(size_t)q * n + i], b2n_sm[oucur + i]);
                peer_put(p.peer, &p.v[(size_t)q * n + i], b2n_sm[ovcur + i]);
            }
            if (lane == 0) {
                peer_put(p.peer, &p.logl[q], lcur);
                peer_put(p.peer, &p.nacc[q], nacc);
                peer_put(p.peer, &p.nrej[q], nrej);
                peer_put(p.peer, &p.ncall[q], (int)p.walks);
            }
        }
        __syncthreads();
        for (int e = threadIdx.x; e < CH * XS; e += blockDim.x) b2n_sm[oX + e] = 0.0;
        __syncthreads();
    }
    peer_finish(p.peer);
}

// Host-side grouping of chains by ellipsoid -> per-CTA work descriptors.
// (shared with the slice kernels)
int b2n_build_worklist(b2n_ctx* ctx, int64_t Q, const int32_t* ell, int K, int chains_per_cta,
                       std::vector<int>& order, std::vector<int3>& cta) {
    order.resize(Q);
    cta.clear();
    std::vector<int64_t> count(K + 1, 0);
    if (ell) {
        for (int64_t q = 0; q < Q; q++) {
            if (ell[q] < 0 || ell[q] >= K) return b2n_fail(ctx, B2N_ERR_ARG, "chain ellipsoid index out of range");
            count[ell[q] + 1]++;
        }
    } else {
        count[1] = Q;
    }
    for (int k = 0; k < K; k++) count[k + 1] += count[k];
    std::vector<int64_t> pos(count.begin(), count.end() - 1);
    for (int64_t q = 0; q < Q; q++) order[pos[ell ? ell[q] : 0]++] = (int)q;
    for (int k = 0; k < K; k++) {
        // split the group into equal CTAs (no short tail CTA)
        const int64_t c = count[k + 1] - count[k];
        if (c == 0) continue;
        const int64_t parts = (c + chains_per_cta - 1) / chains_per_cta;
        for (int64_t i = 0; i < parts; i++) {
            const int64_t lo = count[k] + c * i / parts, hi = count[k] + c * (i + 1) / parts;
            cta.push_back(make_int3((int)lo, (int)(hi - lo), k));
        }
    }
    return B2N_OK;
}

int b2n_worklist_dev(b2n_ctx* ctx, int64_t Q, const int32_t* ell, int K, int chains_per_cta, const void** dorder,
                     const void** dcta, unsigned* ncta) {
    const bool trivial = (ell == nullptr || K == 1);
    if (trivial && ell)
        for (int64_t q = 0; q < Q; q++)
            if (ell[q] != 0) return b2n_fail(ctx, B2N_ERR_ARG, "chain ellipsoid index out of range");
    if (trivial && ctx->wl_Q == Q && ctx->wl_cpc == chains_per_cta && ctx->wl_order.p && ctx->wl_cta.p) {
        *dorder = ctx->wl_order.p; *dcta = ctx->wl_cta.p; *ncta = (unsigned)ctx->wl_ncta;
        return B2N_OK;
    }
    std::vector<int> order;
    std::vector<int3> cta;
    B2N_TRY(b2n_build_worklist(ctx, Q, trivial ? nullptr : ell, K, chains_per_cta, order, cta));
    *ncta = (unsigned)cta.size();
    if (trivial) {
        // (the buffers may still be read by an enqueued kernel of a device-pointer caller)
        B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        B2N_CUDA(ctx, ctx->wl_order.ensure(order.size() * sizeof(int)));
        B2N_CUDA(ctx, ctx->wl_cta.ensure(cta.size() * sizeof(int3)));
        B2N_CUDA(ctx, cudaMemcpy(ctx->wl_order.p, order.data(), order.size() * sizeof(int), cudaMemcpyHostToDevice));
        B2N_CUDA(ctx, cudaMemcpy(ctx->wl_cta.p, cta.data(), cta.size() * sizeof(int3), cudaMemcpyHostToDevice));
        ctx->wl_Q = Q; ctx->wl_cpc = chains_per_cta; ctx->wl_ncta = (int)cta.size();
        *dorder = ctx->wl_order.p; *dcta = ctx->wl_cta.p;
        return B2N_OK;
    }
    B2N_TRY(b2n_in_host(ctx, ctx->work0, order.data(), order.size() * sizeof(int), dorder));
    B2N_TRY(b2n_in_host(ctx, ctx->work1, cta.data(), cta.size() * sizeof(int3), dcta));
    return B2N_OK;
}

// Persistent-sized grid: one CTA per SM when every chain can have its own warp
// (Q <= 16 x SMs), two per SM beyond that; warps loop over their CTA's chains.
void b2n_chain_grid(const b2n_ctx* ctx, int64_t Q, int max_warps, int& chains_per_cta, int& warps) {
    const int64_t sms = ctx->sm_count;
    const int64_t ctas = (Q <= 16 * sms) ? sms : 2 * sms;
    chains_per_cta = (int)std::max<int64_t>(std::min(ctx->min_cpc, 16), (Q + ctas - 1) / ctas);
    warps = std::max(1, std::min(max_warps, std::min(16, chains_per_cta)));
}

// The kernel of a b2n_rwalk_batch call and its launch geometry.
enum RwalkKind { RWALK_WARP, RWALK_MMA, RWALK_WS, RWALK_MMAS };
struct RwalkPlan {
    RwalkKind kind;
    int KT;                 // MMA, WS: k-tiles of 4 columns (n <= 4 KT)
    bool plain;             // WS: affine prior and no dimension flag -- the straight-line chain phase
    int warps;              // WARP: chains in flight per CTA, one warp each
    int chains_per_cta;
    size_t smem;            // dynamic shared memory, bytes
    int ldA, ldP;           // WARP: padded column strides of axesT / the precision matrix in shared memory
    bool ax_s, pr_s;        // WARP: axesT / the precision matrix staged in shared memory
};

// The kernel depends on the problem (model, shape, dimension flags) only, never on the queue length: a chain's result
// must not depend on which batch it is part of -- sharded multi-GPU runs rely on that.  The queue length sets the
// chains per CTA (and, for WARP, the warps per CTA and where the matrices live).
//   WS   rwalk_mmaws_kernel: the precision-matrix Gaussian, ncdim == n, n in 25..32, 49..52, 57..62 -- its static
//        schedule of the symmetric quadratic form is laid out for the largest slab count of a KT, and its draws need
//        an idle lane 31 for the radius (n <= 62);
//   MMA  rwalk_mma_kernel: every other registry likelihood with ncdim == n, 16 <= n <= 64;
//   MMAS rwalk_mmas_kernel: ncdim == n > 64 when its plan fits in shared memory;
//   WARP rwalk_kernel: everything else, and a user likelihood at every n (the lock-step kernels have no user
//        instantiation).
// B2N_RWALK_IMPL=warp forces WARP; B2N_RWALK_IMPL=mma forces MMA, for registry likelihoods with ncdim == n, 4 <= n <= 64.
static int rwalk_plan(b2n_ctx* ctx, const B2nModel& m, int n, int nc, int64_t Q, const uint8_t* dimflags,
                      RwalkPlan& pl) {
    // warp per chain: per-warp state always; matrices (128-byte padded columns) when they fit
    const int npad = (n + 1) & ~1;
    const size_t per_warp = (size_t)6 * npad * sizeof(double);
    const size_t flags_b = (size_t)((((n + 3) >> 2) << 1) + 4 * npad) * sizeof(double);
    const size_t limit = (size_t)ctx->max_smem_optin;
    const int max_warps = (int)std::min<size_t>(16, (limit - flags_b) / per_warp);
    if (max_warps < 1) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "ndim too large for the rwalk kernel");
    const char* impl = getenv("B2N_RWALK_IMPL");
    const bool force_warp = impl && !strcmp(impl, "warp"), force_mma = impl && !strcmp(impl, "mma");
    const bool user = m.like_kind == B2N_LIKE_USER;
    if (force_mma) {
        if (user) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "B2N_RWALK_IMPL=mma: the lock-step kernels have no user-likelihood instantiation");
        if (!(nc == n && n >= 4 && n <= 64)) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "B2N_RWALK_IMPL=mma needs ncdim == ndim <= 64");
    }
    pl = RwalkPlan{};
    pl.KT = n <= 32 ? 8 : (n <= 52 ? 13 : 16);
    pl.ldA = (nc + 15) & ~15;
    pl.ldP = (n + 15) & ~15;
    const bool lockstep = !force_warp && !user && nc == n;
    if (force_mma || (lockstep && n >= 16 && n <= 64)) {
        // matrices as register fragments, 8-chain CTAs, two resident per SM
        const int KT = pl.KT;
        const bool full_slabs = ((n + 7) >> 3) == (4 * KT + 7) / 8;
        const bool ws = !force_mma && m.like_kind == B2N_LIKE_GAUSS_PREC && n <= 62 && full_slabs;
        pl.kind = ws ? RWALK_WS : RWALK_MMA;
        const int ctas = 2 * ctx->sm_count;
        pl.chains_per_cta = (int)std::max<int64_t>(std::min(ctx->min_cpc, 8), (Q + ctas - 1) / ctas);
        pl.warps = 8;
        const int total = ws ? (KT == 8 ? MmaWsLayout<8>::TOTAL : (KT == 13 ? MmaWsLayout<13>::TOTAL : MmaWsLayout<16>::TOTAL))
                             : (KT == 8 ? MmaLayout<8>(n).total() : (KT == 13 ? MmaLayout<13>(n).total() : MmaLayout<16>(n).total()));
        pl.smem = (size_t)total * sizeof(double);
        pl.plain = m.prior_kind != B2N_PRIOR_NORMAL_PPF;
        if (dimflags)
            for (int i = 0; i < n; i++) pl.plain = pl.plain && dimflags[i] == 0u;
        return B2N_OK;
    }
    if (lockstep && n > 64 && (size_t)MmasLayout(n).total() * sizeof(double) <= limit) {
        // large n: matrix fragments streamed from L2 (16 chains share each load), one CTA per SM
        pl.kind = RWALK_MMAS;
        const int ctas = ctx->sm_count;
        pl.chains_per_cta = (int)std::max<int64_t>(std::min(ctx->min_cpc, 16), (Q + ctas - 1) / ctas);
        pl.warps = 16;
        pl.smem = (size_t)MmasLayout(n).total() * sizeof(double);
        return B2N_OK;
    }
    pl.kind = RWALK_WARP;
    b2n_chain_grid(ctx, Q, max_warps, pl.chains_per_cta, pl.warps);
    const size_t fixed = per_warp * pl.warps + flags_b;
    const size_t ax_b = (size_t)nc * pl.ldA * sizeof(double);
    const size_t pr_b = (m.like_kind == B2N_LIKE_GAUSS_PREC) ? (size_t)n * pl.ldP * sizeof(double) : 0;
    pl.ax_s = fixed + ax_b <= limit;
    pl.pr_s = pr_b > 0 && fixed + (pl.ax_s ? ax_b : 0) + pr_b <= limit;
    pl.smem = fixed + (pl.ax_s ? ax_b : 0) + (pl.pr_s ? pr_b : 0);
    return B2N_OK;
}

extern "C" int b2n_rwalk_batch(b2n_ctx* ctx, const b2n_chain_args* a, int32_t walks, double* u,
                               double* v, double* logl, int32_t* n_accept, int32_t* n_reject,
                               int32_t* ncall) {
    if (!ctx) return B2N_ERR_ARG;
    // start points by index (b2n_set_start_rows): consumed by THIS call, however it ends
    const int32_t* sidx = ctx->start_idx;
    const int64_t srows = ctx->start_nrows;
    ctx->start_idx = nullptr; ctx->start_nrows = 0;
    B2nModel m;
    B2N_TRY(b2n_chain_begin(ctx, a, false, &m));
    const bool gather = ctx->peer.total > 0;      // outputs may be NULL in gather mode (b2n_peer_result)
    if (!gather && (!u || !v || !logl || !n_accept || !n_reject || !ncall)) return B2N_ERR_ARG;
    const int n = a->ndim, nc = a->ncdim;
    const int64_t Q = a->nchain;
    if (n != m.ndim || nc < 1 || nc > n || walks < 1 || Q < 0 || !a->u0) return B2N_ERR_ARG;
    if (ctx->bK < 1 || ctx->bn != nc) return b2n_fail(ctx, B2N_ERR_ARG, "resident bound missing or of wrong dimension (b2n_bound_set)");
    if (Q == 0) return b2n_chain_none(ctx);
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    ZcScope zc(ctx);          // pinned caller buffers are read / written in place (host-pointer mode)

    RwalkPlan plan;
    B2N_TRY(rwalk_plan(ctx, m, n, nc, Q, a->dimflags, plan));
    const bool dyn = ctx->dyn.active;        // device-paced launch (b2n_ns.cu): worklist + scalars in HBM
    if (dyn) {
        B2N_TRY(b2n_chain_dyn(ctx, plan.chains_per_cta));
        if (ctx->dyn.plan_only) return B2N_OK;
    }
    RwalkParams p;
    p.dyn = dyn ? ctx->dyn.dev : nullptr;
    p.m = m; p.n = n; p.nc = nc; p.walks = walks; p.ldA = plan.ldA; p.ldP = plan.ldP;
    p.loglstar = a->loglstar; p.scale = a->scale; p.seed = a->seed; p.chain0 = a->chain0;
    p.axesT = ctx->b_axesT.as<double>();
    const void *du0, *dorder, *dcta, *dfl = nullptr, *dstart = nullptr;
    // start points by index: u0 is then the whole live set
    if (sidx) {
        if (dyn) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "start rows by index: not in a device-paced launch");
        if (ctx->ptr_mode == B2N_PTR_DEVICE) dstart = sidx;
        else {
            for (int64_t i = 0; i < Q; i++)
                if (sidx[i] < 0 || sidx[i] >= srows) return b2n_fail(ctx, B2N_ERR_ARG, "start row index out of range");
            B2N_TRY(b2n_in_host(ctx, ctx->in1, sidx, (size_t)Q * sizeof(int32_t), &dstart));
        }
    }
    B2N_TRY(b2n_in(ctx, ctx->in0, a->u0, (size_t)(sidx ? srows : Q) * n * sizeof(double), &du0));
    unsigned ncta = 0;
    if (dyn) {
        dorder = ctx->dyn.order; dcta = ctx->dyn.cta;
    } else {
        B2N_TRY(b2n_worklist_dev(ctx, Q, a->ell, ctx->bK, plan.chains_per_cta, &dorder, &dcta, &ncta));
    }
    std::vector<uint32_t> fl;
    if (a->dimflags) {
        fl.assign(a->dimflags, a->dimflags + n);
        B2N_TRY(b2n_in_host(ctx, ctx->in3, fl.data(), fl.size() * sizeof(uint32_t), &dfl));
    }
    void* const out[B2N_NSLOT] = {u, v, logl, n_accept, n_reject, ncall, nullptr};
    void* dev[B2N_NSLOT];
    B2N_TRY(b2n_chain_bind(ctx, n, Q, out, dev, &p.peer));
    p.u0 = (const double*)du0; p.start = (const int*)dstart; p.order = (const int*)dorder; p.cta = (const int3*)dcta;
    p.dimflags = (const uint32_t*)dfl;
    p.u = (double*)dev[0]; p.v = (double*)dev[1]; p.logl = (double*)dev[2];
    p.nacc = (int*)dev[3]; p.nrej = (int*)dev[4]; p.ncall = (int*)dev[5];

    const unsigned grid = dyn ? (unsigned)ctx->dyn.max_cta : ncta;
    const int KT = plan.KT;
    // LAUNCH(threads, kernel): raise the kernel's shared-memory limit to the plan's, then launch it
#define LAUNCH(THREADS, ...)                                                              \
    do {                                                                                  \
        B2N_TRY(b2n_func_smem(ctx, (const void*)(__VA_ARGS__), plan.smem));               \
        __VA_ARGS__<<<grid, THREADS, plan.smem, ctx->stream>>>(p);                        \
    } while (0)
#define CALL_WARP(L)                                                                      \
    if (plan.ax_s && plan.pr_s) LAUNCH(plan.warps * 32, rwalk_kernel<L, true, true>);     \
    else if (plan.ax_s) LAUNCH(plan.warps * 32, rwalk_kernel<L, true, false>);            \
    else if (plan.pr_s) LAUNCH(plan.warps * 32, rwalk_kernel<L, false, true>);            \
    else LAUNCH(plan.warps * 32, rwalk_kernel<L, false, false>);
#define CALL_MMA(L)                                                                       \
    if (KT == 8) LAUNCH(256, rwalk_mma_kernel<L, 8>);                                     \
    else if (KT == 13) LAUNCH(256, rwalk_mma_kernel<L, 13>);                              \
    else LAUNCH(256, rwalk_mma_kernel<L, 16>);
#define CALL_MMAS(L) LAUNCH(512, rwalk_mmas_kernel<L>);
#define CALL_WS(K)                                                                        \
    if (plan.plain) LAUNCH(384, rwalk_mmaws_kernel<K, true>);                             \
    else LAUNCH(384, rwalk_mmaws_kernel<K, false>);
    B2N_TIME_BEGIN(ctx);
    switch (plan.kind) {
    case RWALK_WS:
        if (KT == 8) { CALL_WS(8) }
        else if (KT == 13) { CALL_WS(13) }
        else { CALL_WS(16) }
        break;
    case RWALK_MMA:
        B2N_DISPATCH_LIKE(m.like_kind, CALL_MMA)
        break;
    case RWALK_MMAS:
        B2N_DISPATCH_LIKE(m.like_kind, CALL_MMAS)
        break;
    case RWALK_WARP:
        if (m.like_kind == B2N_LIKE_USER) {
            void* args[] = {(void*)&p};
            B2N_TRY(b2n_user_launch(ctx, a->model_id, B2N_US_RWALK + (plan.ax_s ? 1 : 0), dim3(grid),
                                    dim3(plan.warps * 32), plan.smem, args));
        } else {
            B2N_DISPATCH_LIKE(m.like_kind, CALL_WARP)
        }
        break;
    }
    B2N_TIME_END(ctx);
#undef CALL_WS
#undef CALL_MMAS
#undef CALL_MMA
#undef CALL_WARP
#undef LAUNCH
    B2N_LAUNCH_CHECK(ctx);
    return b2n_chain_end(ctx, n, Q, out, dev, nullptr, 0);
}

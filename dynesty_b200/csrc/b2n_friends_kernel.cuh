// b2n_friends_kernel.cuh -- UniformBoundSampler.sample with a RadFriends / SupFriends bound
// (friends_unif_kernel, see b2n_friends.cu) and the ball / cube distance it shares with the overlap query.
// Device-only: included by b2n_friends.cu and by the run-time compiled translation unit of a user likelihood
// (b2n_user_kernels.cuh).
#pragma once
#include "b2n_device.cuh"

#ifndef B2N_UNIF_MAX_DRAWS
#define B2N_UNIF_MAX_DRAWS 20000000
#endif

// distance of the transformed query xt to centre row ct (kind 0: squared Euclidean, 1: Chebyshev)
__device__ __forceinline__ double friends_dist(const double* __restrict__ ct, const double* xt, int n, int kind) {
    double s = 0.0;
    if (kind == 0) {
        for (int k = 0; k < n; k++) { const double d = ct[k] - xt[k]; s = fma(d, d, s); }
        return sqrt(s);
    }
    for (int k = 0; k < n; k++) s = fmax(s, fabs(ct[k] - xt[k]));
    return s;
}

// ---- UniformBoundSampler.sample (internal_samplers.py:243-340) with a RadFriends / SupFriends bound ----------
struct FriendsUnifParams {
    B2nModel m;
    int n, N, kind, draw_only;      // draw_only: 1 = Bound.samples (no cube test / likelihood), 3 = sample(return_q)
    const double *ctrs, *ctrs_t, *axes, *axes_inv;
    const uint32_t* dimflags;
    double loglstar;
    uint64_t seed, chain0;
    int64_t Q;
    double *u, *v, *logl;
    int *ncall, *nprop;
    uint32_t* flags;
};

template <int LIKE>
__global__ void __launch_bounds__(128) friends_unif_kernel(const FriendsUnifParams p) {
    extern __shared__ double fsm[];
    const int n = p.n, N = p.N;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
    double* uu = fsm + (size_t)warp * 5 * n;
    double* z = uu + n;
    double* xt = z + n;
    double* vv = xt + n;
    double* work = vv + n;
    const double inv_n = 1.0 / (double)n;
    for (int64_t q = (int64_t)blockIdx.x * wpb + warp; q < p.Q; q += (int64_t)gridDim.x * wpb) {
        ChainRng g;
        g.init(p.seed, p.chain0 + (uint64_t)q);
        int ncall = 0, nprop = 0;
        uint32_t fl = 0;
        double lcur = 0.0;
        bool done = false;
        while (!done) {
            if (nprop >= B2N_UNIF_MAX_DRAWS) { fl |= 0x80000000u | B2N_WARN_UNIF_INEFFICIENT; break; }
            if (nprop == 10000) fl |= B2N_WARN_UNIF_INEFFICIENT;
            int qn = 1;
            for (;;) {                                       // bound.sample(): bounding.py:797-831 / 1065-1100
                double fac = 1.0;
                if (p.kind == 0) {                           // randsphere: normal vector, then the radius uniform
                    const double ss = rng_normals_to(g, z, n, lane);
                    const double U = rng_uniform(g);
                    fac = pow(U, inv_n) / sqrt(ss);
                } else {                                     // uniform(-1, 1, size=ndim)
                    for (int e = lane; e < n; e += 32) z[e] = 2.0 * rng_uniform_elem(g, e) - 1.0;
                    g.tick++;
                }
                __syncwarp();
                int idx = 0;
                if (N > 1) {                                 // rstate.integers(nctrs): floor(U * nctrs)
                    const double U = rng_uniform(g);
                    idx = (int)(U * (double)N);
                    idx = idx < N - 1 ? idx : N - 1;
                }
                for (int j = lane; j < n; j += 32) {         // dx = ds @ axes
                    double s = 0.0;
                    for (int k = 0; k < n; k++) s = fma(z[k], __ldg(p.axes + (size_t)k * n + j), s);
                    uu[j] = fma(fac, s, p.ctrs[(size_t)idx * n + j]);
                }
                __syncwarp();
                if (N == 1) { qn = 1; break; }
                for (int j = lane; j < n; j += 32) {
                    double s = 0.0;
                    for (int k = 0; k < n; k++) s = fma(uu[k], __ldg(p.axes_inv + (size_t)k * n + j), s);
                    xt[j] = s;
                }
                __syncwarp();
                int c = 0;
                for (int i = lane; i < N; i += 32) c += friends_dist(p.ctrs_t + (size_t)i * n, xt, n, p.kind) <= 1.0 ? 1 : 0;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(B2N_FULL, c, o);
                qn = c;
                __syncwarp();
                if (qn == 1 || (p.draw_only & 2)) break;
                // (qn == 0 cannot happen mathematically -- the draw lies in the ball of centre idx -- but the two
                //  evaluation orders differ in the last bit for a point on the rim: treat it as q = 1)
                if (qn == 0) { qn = 1; break; }
                if (rng_uniform(g) < 1.0 / (double)qn) break;
            }
            nprop++;
            if (p.draw_only) {
                for (int i = lane; i < n; i += 32) vv[i] = uu[i];
                ncall = qn;
                break;
            }
            bool ok = true;
            for (int i = lane; i < n; i += 32) ok = ok && in_cube(uu[i], p.dimflags ? p.dimflags[i] : 0u);
            ok = __all_sync(B2N_FULL, ok);
            if (!ok) continue;
            for (int i = lane; i < n; i += 32) vv[i] = prior_1d(p.m, i, uu[i]);
            __syncwarp();
#ifdef B2N_USER_PRIOR
            if (p.m.prior_kind == B2N_PRIOR_USER) user_prior_warp(p.m, uu, vv, work, lane);
#endif
            lcur = warp_loglike<LIKE>(p.m, p.m.lmat, vv, work, lane);
            ncall++;
            if (lcur > p.loglstar) done = true;
        }
        __syncwarp();
        for (int i = lane; i < n; i += 32) { p.u[q * n + i] = uu[i]; p.v[q * n + i] = vv[i]; }
        if (lane == 0) { p.logl[q] = lcur; p.ncall[q] = ncall; p.nprop[q] = nprop; p.flags[q] = fl; }
        __syncwarp();
    }
}

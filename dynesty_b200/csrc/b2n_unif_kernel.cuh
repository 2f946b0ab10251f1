// b2n_unif_kernel.cuh -- uniform sampling within the resident ellipsoid bound (unif_kernel) and within the
// unit cube (unitcube_kernel), with their launch parameters.  Device-only: included by b2n_unif.cu and by the
// run-time compiled translation unit of a user likelihood (b2n_user_kernels.cuh).
#pragma once
#include "b2n_device.cuh"

#ifndef B2N_UNIF_MAX_DRAWS
#define B2N_UNIF_MAX_DRAWS 20000000
#endif

struct UnifParams {
    B2nModel m;
    int n, nc, K, draw_only;
    const double* ctrs;     // K x nc
    const double* ams;      // K x nc x nc
    const double* axesT;    // K x nc x nc (transposed)
    const double* cum;      // K cumulative volume fractions
    const uint32_t* dimflags;
    double loglstar;
    uint64_t seed, chain0;
    int64_t Q;
    double *u, *v, *logl;
    int *ncall, *nprop;
    uint32_t* flags;
    PeerSet peer;          // fused multi-GPU gather of the outputs (b2n_peer.cu)
    const B2nDyn* dyn;     // device-paced launch (b2n_ns.cu): threshold / chain ids in HBM
};

template <int LIKE>
__global__ void __launch_bounds__(256) unif_kernel(const UnifParams p) {
    extern __shared__ double sm[];
    const int n = p.n, nc = p.nc, K = p.K;
    double loglstar_ = p.loglstar;
    unsigned long long chain0_ = p.chain0;
    if (p.dyn) {
        if (p.dyn->skip) return;
        loglstar_ = p.dyn->loglstar; chain0_ = p.dyn->chain0;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
    double* uu = sm + (size_t)warp * 5 * n;   // candidate point (n)
    double* z = uu + n;                        // unit-ball draw (nc)
    double* dl = z + n;                        // delta (nc)
    double* vv = dl + n;                       // v (n)
    double* work = vv + n;                     // likelihood scratch (n)
    const double inv_nc = 1.0 / (double)nc;
    for (int64_t q = (int64_t)blockIdx.x * wpb + warp; q < p.Q; q += (int64_t)gridDim.x * wpb) {
        ChainRng g;
        g.init(p.seed, chain0_ + (uint64_t)q);
        int ncall = 0, nprop = 0;
        uint32_t fl = 0;
        double lcur = 0.0;
        bool done = false;
        while (!done) {
            if (nprop >= B2N_UNIF_MAX_DRAWS) { fl |= 0x80000000u | B2N_WARN_UNIF_INEFFICIENT; break; }
            if (nprop == 10000) fl |= B2N_WARN_UNIF_INEFFICIENT;        // :316-320
            // ---- bound.samples(1): a point uniform in the union of ellipsoids
            int idx = 0;
            for (;;) {
                if (K > 1) {                                             // rand_choice
                    const double xr = rng_uniform(g);
                    int lo = 0;
                    while (lo < K - 1 && p.cum[lo] < xr) lo++;           // searchsorted(left), clamped
                    idx = lo;
                }
                const double ss = rng_normals_to(g, z, nc, lane);
                const double U = rng_uniform(g);
                const double fac = pow(U, inv_nc) / sqrt(ss);
                __syncwarp();
                const double* A = p.axesT + (size_t)idx * nc * nc;
                for (int base = 0; base < nc; base += 64) {
                    double y0, y1;
                    warp_matvec2(A, nc, nc, z, base + lane, nc, y0, y1);
                    const int i0 = base + lane, i1 = i0 + 32;
                    if (i0 < nc) uu[i0] = fma(fac, y0, p.ctrs[(size_t)idx * nc + i0]);
                    if (i1 < nc) uu[i1] = fma(fac, y1, p.ctrs[(size_t)idx * nc + i1]);
                }
                __syncwarp();
                if (K == 1) { if (p.draw_only & 2) ncall = 1; break; }   // bounding.py:543-550
                int qn = 0, qslack = 0;
                for (int k = 0; k < K; k++) {
                    for (int i = lane; i < nc; i += 32) dl[i] = uu[i] - p.ctrs[(size_t)k * nc + i];
                    __syncwarp();
                    const double* AM = p.ams + (size_t)k * nc * nc;
                    double s = 0.0;
                    for (int base = 0; base < nc; base += 64) {
                        double y0, y1;
                        warp_matvec2(AM, nc, nc, dl, base + lane, nc, y0, y1);
                        if (base + lane < nc) s = fma(dl[base + lane], y0, s);
                        if (base + lane + 32 < nc) s = fma(dl[base + lane + 32], y1, s);
                    }
                    s = warp_sum(s);
                    qn += (s < 1.0) ? 1 : 0;
                    qslack += (s <= 1.0 + 1e-3) ? 1 : 0;
                    __syncwarp();
                }
                if (qn == 0) {                                           // :565-579
                    qn = qslack;
                    if (qn == 0) { fl |= 0x40000000u; done = true; break; }
                    fl |= B2N_WARN_Q0_SLACK;
                }
                if (p.draw_only & 2) { ncall = qn; break; }                // sample(return_q=True): no 1/q test
                if (qn == 1) break;
                if (rng_uniform(g) < 1.0 / (double)qn) break;            // :589
            }
            if (done) break;
            nprop++;
            if (p.draw_only) {           // Bound.samples(): no cube test, no likelihood (bounding.py:592-606)
                for (int i = lane; i < n; i += 32) vv[i] = uu[i];
                break;
            }
            // ---- unit-cube check on the clustered dims (internal_samplers.py:314)
            bool ok = true;
            for (int i = lane; i < nc; i += 32) ok = ok && in_cube(uu[i], p.dimflags ? p.dimflags[i] : 0u);
            ok = __all_sync(B2N_FULL, ok);
            if (!ok) continue;
            if (n > nc) {                                                // :325-327
                for (int e = lane; e < n - nc; e += 32) uu[nc + e] = rng_uniform_elem(g, e);
                g.tick++;
            }
            __syncwarp();
            for (int i = lane; i < n; i += 32) vv[i] = prior_1d(p.m, i, uu[i]);
            __syncwarp();
#ifdef B2N_USER_PRIOR
            if (p.m.prior_kind == B2N_PRIOR_USER) user_prior_warp(p.m, uu, vv, work, lane);
#endif
            lcur = warp_loglike<LIKE>(p.m, p.m.lmat, vv, work, lane);
            ncall++;
            if (lcur > loglstar_) done = true;
        }
        __syncwarp();
        for (int i = lane; i < n; i += 32) {
            peer_put(p.peer, &p.u[q * n + i], uu[i]);
            peer_put(p.peer, &p.v[q * n + i], vv[i]);
        }
        if (lane == 0) {
            peer_put(p.peer, &p.logl[q], lcur);
            peer_put(p.peer, &p.ncall[q], ncall);
            peer_put(p.peer, &p.nprop[q], nprop);
            peer_put(p.peer, &p.flags[q], fl);
        }
        __syncwarp();
    }
    peer_finish(p.peer);
}

// ---- UnitCubeSampler.sample (internal_samplers.py:343-441) for a queue of chains: draw u ~ U(0,1)^n (one
// uniform vector event per draw), v = prior_transform(u), until loglikelihood(v) > loglstar.  This is what the
// reference runs before the first bound exists (sampler.py:407-409, 625-674).  One warp per chain.
struct CubeParams {
    B2nModel m;
    int n;
    double loglstar;
    uint64_t seed, chain0;
    int64_t Q;
    double *u, *v, *logl;
    int* ncall;
    uint32_t* flags;
    PeerSet peer;
    const B2nDyn* dyn;
};

template <int LIKE>
__global__ void __launch_bounds__(128) unitcube_kernel(const CubeParams p) {
    extern __shared__ double sm[];
    const int n = p.n;
    double loglstar_ = p.loglstar;
    unsigned long long chain0_ = p.chain0;
    if (p.dyn) {
        if (p.dyn->skip) return;
        loglstar_ = p.dyn->loglstar; chain0_ = p.dyn->chain0;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
    double* uu = sm + (size_t)warp * 3 * n;
    double* vv = uu + n;
    double* work = vv + n;
    for (int64_t q = (int64_t)blockIdx.x * wpb + warp; q < p.Q; q += (int64_t)gridDim.x * wpb) {
        ChainRng g;
        g.init(p.seed, chain0_ + (uint64_t)q);
        int ncall = 0;
        uint32_t fl = 0;
        double lcur = 0.0;
        for (;;) {
            if (ncall >= B2N_UNIF_MAX_DRAWS) { fl |= 0x80000000u; break; }
            for (int e = lane; e < n; e += 32) {
                const double t = rng_uniform_elem(g, e);
                uu[e] = t;
                vv[e] = prior_1d(p.m, e, t);
            }
            g.tick++;
            __syncwarp();
#ifdef B2N_USER_PRIOR
            if (p.m.prior_kind == B2N_PRIOR_USER) user_prior_warp(p.m, uu, vv, work, lane);
#endif
            lcur = warp_loglike<LIKE>(p.m, p.m.lmat, vv, work, lane);
            ncall++;
            if (lcur > loglstar_) break;
            __syncwarp();
        }
        __syncwarp();
        for (int i = lane; i < n; i += 32) {
            peer_put(p.peer, &p.u[q * n + i], uu[i]);
            peer_put(p.peer, &p.v[q * n + i], vv[i]);
        }
        if (lane == 0) {
            peer_put(p.peer, &p.logl[q], lcur);
            peer_put(p.peer, &p.ncall[q], ncall);
            if (p.flags) peer_put(p.peer, &p.flags[q], fl);
        }
        __syncwarp();
    }
    peer_finish(p.peer);
}

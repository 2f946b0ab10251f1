// b2n_device.cuh -- device-side pieces shared by the proposal kernels:
//   * the B2N Philox stream (layout documented in oracle/philox.py)
//   * the prior-transform / log-likelihood registry ("device callback")
//   * unit-cube boundary handling (utils.py:1036-1078 of the reference)
#pragma once
#include "b2n_common.cuh"
#include <curand_philox4x32_x.h>   // curand_Philox4x32_10 (cuRAND device API)

// ---- RNG ---------------------------------------------------------------------------
struct ChainRng {
    uint2 key;
    uint32_t c2, c3;   // chain id
    uint32_t tick;     // next draw event
    __device__ __forceinline__ void init(uint64_t seed, uint64_t chain) {
        key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
        c2 = (uint32_t)chain;
        c3 = (uint32_t)(chain >> 32);
        tick = 0;
    }
    __device__ __forceinline__ uint4 block(uint32_t blk) const {
        return curand_Philox4x32_10(make_uint4(blk, tick, c2, c3), key);
    }
};

__device__ __forceinline__ double b2n_u52(uint32_t a, uint32_t b) {
    return ((double)(a >> 6) * 67108864.0 + (double)(b >> 6) + 0.5) * 0x1p-52;
}
// element e of a uniform vector event
__device__ __forceinline__ double rng_uniform_elem(const ChainRng& g, int e) {
    uint4 r = g.block((uint32_t)(e >> 1));
    return (e & 1) ? b2n_u52(r.z, r.w) : b2n_u52(r.x, r.y);
}
// scalar uniform event (all lanes compute the same value); advances the tick
__device__ __forceinline__ double rng_uniform(ChainRng& g) {
    uint4 r = g.block(0);
    g.tick++;
    return b2n_u52(r.x, r.y);
}
// Box-Muller pair of block b of a normal vector event
__device__ __forceinline__ void rng_normal_pair(const ChainRng& g, int b, double& z0, double& z1) {
    uint4 r = g.block((uint32_t)b);
    const double u0 = b2n_u52(r.x, r.y), u1 = b2n_u52(r.z, r.w);
    const double rad = sqrt(-2.0 * log(u0));
    double s, c;
    sincospi(2.0 * u1, &s, &c);
    z0 = rad * c;
    z1 = rad * s;
}
// normal vector event of size m into warp-private shared x[0..m); returns sum of squares
__device__ __forceinline__ double rng_normals_to(ChainRng& g, double* x, int m, int lane) {
    double ss = 0.0;
    const int nb = (m + 1) >> 1;
    for (int b = lane; b < nb; b += 32) {
        double z0, z1;
        rng_normal_pair(g, b, z0, z1);
        x[2 * b] = z0;
        ss = fma(z0, z0, ss);
        if (2 * b + 1 < m) { x[2 * b + 1] = z1; ss = fma(z1, z1, ss); }
    }
    g.tick++;
    return warp_sum(ss);
}

// ---- boundary handling ----------------------------------------------------------------
// np.mod(x, 1) for finite x
__device__ __forceinline__ double mod1(double x) { return x - floor(x); }
// apply_reflect (utils.py:1053-1078)
__device__ __forceinline__ double reflect1(double x) {
    const double m2 = x - 2.0 * floor(x * 0.5);   // np.mod(x, 2)
    return (m2 < 1.0) ? mod1(x) : 1.0 - mod1(x);
}
// one component of unitcheck (utils.py:1036-1050): strict inequalities
__device__ __forceinline__ bool in_cube(double x, uint32_t flag) {
    return flag ? (x > -0.5 && x < 1.5) : (x > 0.0 && x < 1.0);
}

// ---- prior transform ---------------------------------------------------------------------
__device__ __forceinline__ double prior_1d(const B2nModel& m, int i, double u) {
    switch (m.prior_kind) {
        case B2N_PRIOR_UNIFORM: return fma(m.pp1[i], u, m.pp0[i]);
        case B2N_PRIOR_NORMAL_PPF: return fma(m.pp1[i], normcdfinv(u), m.pp0[i]);
        default: return u;
    }
}

// the 2-D constraint regions of the reference's uniformity harness (tests/test_sampling.py:8-23)
__device__ __forceinline__ double region2d_logl(double shape, double x, double y) {
    const double ninf = __longlong_as_double(0xfff0000000000000LL);
    if (shape == 0.0) {                                   // diamond_logl
        const double x1 = fabs(x - 0.5), y1 = fabs(y - 0.5);
        if (fmin(x, y) < 0.0 || fmax(x, y) > 1.0) return ninf;
        const double D2 = (x1 - 0.5) * (x1 - 0.5) + (y1 - 0.5) * (y1 - 0.5);
        return D2 > 0.25 ? D2 - 0.25 : ninf;
    }
    const double mult = 16.0 * 2.0 * 3.14159265358979323846;         // checker_logl
    if (!(x >= 0.0 && x <= 1.0 && y >= 0.0 && y < 1.0)) return ninf;
    return sin(x * mult) * sin(y * mult);
}

#ifdef B2N_USER_MODEL
// the user likelihood of a run-time compiled model (contract: include/b200nest.h, b2n_model_create_user),
// defined after b2n_user_kernels.cuh in the same NVRTC program
__device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane);
#endif

#ifdef B2N_USER_BLOB
// the derived quantities of a point (contract: include/b200nest.h, b2n_model_blob), defined in the user's source;
// only b2n_user_blob_kernel (b2n_user_kernels.cuh) calls it
__device__ void b2n_user_blob(const double* v, double* work, int n, const double* p, int lane, double* blob,
                              int nblob);
#endif

#ifdef B2N_USER_PRIOR
// the user prior transform of a run-time compiled model (B2N_PRIOR_USER; contract: include/b200nest.h,
// b2n_model_create_user_ex), defined after b2n_user_kernels.cuh in the same NVRTC program
__device__ void b2n_user_prior(const double* u, double* v, double* work, int n, const double* p, int lane);

// v = prior_transform(u) as ONE warp-cooperative call (a joint prior reads every component of u).  The per-element
// prior_1d / prior_sm of the callers write u itself as a placeholder for B2N_PRIOR_USER; this overwrites it.
__device__ __forceinline__ void user_prior_warp(const B2nModel& m, const double* u, double* v, double* work,
                                                int lane) {
    __syncwarp();
    b2n_user_prior(u, v, work, m.ndim, m.pp0, lane);
    __syncwarp();
}
#endif

// ---- log-likelihood, evaluated cooperatively by one warp ---------------------------
// v: warp-private shared vector (n).  work: warp-private shared scratch (n).
// lmat: pointer to the n x n matrix for GAUSS_PREC (shared or global).
template <int LIKE>
__device__ __forceinline__ double warp_loglike(const B2nModel& m, const double* __restrict__ lmat,
                                               const double* v, double* work, int lane) {
    const int n = m.ndim;
    if (LIKE == B2N_LIKE_GAUSS_PREC) {
        for (int i = lane; i < n; i += 32) work[i] = v[i] - m.lv0[i];
        __syncwarp();
        double s = 0.0;
        for (int base = 0; base < n; base += 64) {
            double y0, y1;
            warp_matvec2(lmat, n, n, work, base + lane, n, y0, y1);
            if (base + lane < n) s = fma(work[base + lane], y0, s);
            if (base + lane + 32 < n) s = fma(work[base + lane + 32], y1, s);
        }
        s = warp_sum(s);
        __syncwarp();
        return fma(-0.5, s, m.s0);
    } else if (LIKE == B2N_LIKE_GAUSS_DIAG) {
        double s = 0.0;
        for (int i = lane; i < n; i += 32) {
            const double d = v[i] - m.lv0[i];
            s = fma(m.lv1[i] * d, d, s);
        }
        s = warp_sum(s);
        return fma(-0.5, s, m.s0);
    } else if (LIKE == B2N_LIKE_EGGBOX) {
        double p = 1.0;
        for (int i = lane; i < n; i += 32) {
            const double t = 2.0 * m.s0 * v[i] - m.s0;
            p *= cos(t * 0.5);
        }
        p = warp_prod(p);
        return pow(2.0 + p, m.s1);
    } else if (LIKE == B2N_LIKE_REGION2D) {
        return region2d_logl(m.s0, v[0], v[1]);
#ifdef B2N_USER_MODEL
    } else if (LIKE == B2N_LIKE_USER) {
        return b2n_user_loglike(v, work, n, m.lv0, lane);
#endif
    } else {  // SHELLS
        double a = 0.0, b = 0.0;
        for (int i = lane; i < n; i += 32) {
            const double d1 = v[i] - m.lv0[i], d2 = v[i] - m.lv1[i];
            a = fma(d1, d1, a);
            b = fma(d2, d2, b);
        }
        a = sqrt(warp_sum(a));
        b = sqrt(warp_sum(b));
        const double r = m.s0, w = m.s1;
        const double cst = log(1.0 / sqrt(2.0 * 3.14159265358979323846 * w * w));
        const double l1 = cst - (a - r) * (a - r) / (2.0 * w * w);
        const double l2 = cst - (b - r) * (b - r) / (2.0 * w * w);
        const double hi = fmax(l1, l2), lo = fmin(l1, l2);
        return hi + log1p(exp(lo - hi));    // np.logaddexp
    }
}

// kernel dispatch on the likelihood kind (B2N_LIKE_USER never reaches it: its kernels are loaded at run time and
// launched through b2n_user_launch)
#define B2N_DISPATCH_LIKE(kind, CALL)                                   \
    switch (kind) {                                                     \
        case B2N_LIKE_GAUSS_PREC: { CALL(B2N_LIKE_GAUSS_PREC); } break; \
        case B2N_LIKE_GAUSS_DIAG: { CALL(B2N_LIKE_GAUSS_DIAG); } break; \
        case B2N_LIKE_EGGBOX: { CALL(B2N_LIKE_EGGBOX); } break;         \
        case B2N_LIKE_REGION2D: { CALL(B2N_LIKE_REGION2D); } break;     \
        default: { CALL(B2N_LIKE_SHELLS); } break;                      \
    }

// ---- fused exchange of finished chains (b2n_peer.cu) ---------------------------------------
// peer_put: store an output element into the own array AND at the same window offset of every
// peer (NVLink peer stores).  With the exchange off (world <= 1) it is a plain store.
template <class T>
__device__ __forceinline__ void peer_put(const PeerSet& ps, T* local, T val) {
    *local = val;
    if (ps.world > 1) {
        const ptrdiff_t off = reinterpret_cast<char*>(local) - ps.base[ps.rank];
        for (int w = 0; w < ps.world; w++)
            if (w != ps.rank) *reinterpret_cast<T*>(ps.base[w] + off) = val;
    }
}

__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// peer_finish: called by EVERY thread at the end of a chain kernel.  The last CTA of the grid
// (threadFenceReduction pattern on the window's `done` word) bumps the arrive counter of every
// rank with system-scope atomics and then waits until all `world` ranks have bumped its own:
// when the kernel completes, every rank's rows are in this rank's window.  The wait is bounded
// (~10 s of SM clocks): a missing peer sets the window's err word instead of hanging the GPU.
__device__ __forceinline__ void peer_finish(const PeerSet& ps) {
    if (ps.world == 0) return;
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        char* own = ps.base[ps.rank];
        unsigned int* done = reinterpret_cast<unsigned int*>(own + 64);
        __threadfence_system();
        const unsigned int prev = atomicAdd(done, 1u);
        if (prev == gridDim.x * gridDim.y - 1) {
            atomicExch(done, 0u);
            __threadfence_system();
            for (int w = 0; w < ps.world; w++)
                atomicAdd_system(reinterpret_cast<unsigned long long*>(ps.base[w]), 1ULL);
            const long long t0 = clock64();
            while (ld_acquire_sys_u64(reinterpret_cast<unsigned long long*>(own)) < ps.target) {
                if (clock64() - t0 > 20000000000LL) {
                    *reinterpret_cast<volatile unsigned int*>(own + 8) = 1u;
                    break;
                }
                __nanosleep(200);
            }
        }
    }
}

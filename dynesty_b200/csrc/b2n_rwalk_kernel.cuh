// b2n_rwalk_kernel.cuh -- the warp-per-chain random-walk kernel (rwalk_kernel, mapping described in
// b2n_rwalk.cu) and its launch parameters.  Device-only: included by b2n_rwalk.cu and by the run-time compiled
// translation unit of a user likelihood (b2n_user_kernels.cuh).
#pragma once
#include "b2n_chain.cuh"

struct RwalkParams {
    B2nModel m;
    int n, nc, walks;
    int ldA, ldP;          // leading dims of axes^T / precision as seen by the kernel
    const double* u0;
    const int* start;      // optional: chain q starts from row start[q] of u0 (b2n_set_start_rows); NULL: row q
    const int* order;      // chains grouped by ellipsoid
    const int3* cta;       // (first, count, ell) per CTA
    const double* axesT;   // K x nc x nc, transposed (column-major axes)
    const uint32_t* dimflags;
    double loglstar, scale;
    uint64_t seed, chain0;
    double *u, *v, *logl;
    int *nacc, *nrej, *ncall;
    PeerSet peer;          // fused multi-GPU gather of the outputs (b2n_peer.cu); world == 0: off
    const B2nDyn* dyn;     // device-paced launch (b2n_ns.cu): threshold / scale / chain ids / CTA count in HBM
};

// Per-launch scalars: kernel arguments, or -- device-paced -- the B2nDyn the previous kernel on
// the stream wrote (a skipped round or a CTA beyond the round's worklist returns at once).
#define B2N_DYN_PROLOGUE(p)                                                                  \
    double loglstar_ = (p).loglstar, scale_ = (p).scale;                                     \
    unsigned long long chain0_ = (p).chain0;                                                 \
    if ((p).dyn) {                                                                           \
        if ((p).dyn->skip || (int)blockIdx.x >= (p).dyn->ncta) return;                       \
        loglstar_ = (p).dyn->loglstar; scale_ = (p).dyn->scale; chain0_ = (p).dyn->chain0;   \
    }

template <int LIKE, bool AX_SMEM, bool PREC_SMEM>
__global__ void __launch_bounds__(512, 1) rwalk_kernel(const RwalkParams p) {
    const int n = p.n, nc = p.nc;
    const int npad = (n + 1) & ~1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    B2N_DYN_PROLOGUE(p)
    const int3 cd = p.cta[blockIdx.x];
    // ---- shared-memory plan (all offsets in doubles, all even)
    int off = 0;
    const double* Ag = p.axesT + (size_t)cd.z * nc * nc;
    int offA = 0, ldA = nc;
    if (AX_SMEM) {
        offA = off; ldA = p.ldA;
        for (int e = threadIdx.x; e < nc * nc; e += blockDim.x) {
            const int j = e / nc, i = e - j * nc;
            b2n_sm[offA + j * ldA + i] = Ag[e];
        }
        off += nc * ldA;
    }
    const double* Pg = p.m.lmat;
    int offP = 0, ldP = n;
    if (LIKE == B2N_LIKE_GAUSS_PREC && PREC_SMEM) {
        offP = off; ldP = p.ldP;
        for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
            const int j = e / n, i = e - j * n;
            b2n_sm[offP + j * ldP + i] = Pg[e];
        }
        off += n * ldP;
    }
    const ModelSm ms = stage_model(p.m, off, n, npad);     // prior p0/p1, likelihood vec0/vec1
    const int op0 = ms.op0, op1 = ms.op1, omu = ms.olv0;
    off += 4 * npad;
    uint32_t* fl = reinterpret_cast<uint32_t*>(&b2n_sm[off]);
    for (int i = threadIdx.x; i < n; i += blockDim.x) fl[i] = p.dimflags ? p.dimflags[i] : 0u;
    off += ((n + 3) >> 2) << 1;
    __syncthreads();

    int oucur = off + warp * 6 * npad;
    int ouprop = oucur + npad;
    int ovcur = ouprop + npad;
    int ovprop = ovcur + npad;
    const int ox = ovprop + npad;       // direction vector
    const int od = ox + npad;           // v - mean (GAUSS_PREC) / likelihood scratch
    const double inv_nc = 1.0 / (double)nc;
    const int pk = p.m.prior_kind;

    for (int c = warp; c < cd.y; c += nwarps) {
        const int q = p.order[cd.x + c];
        ChainRng g;
        g.init(p.seed, chain0_ + (uint64_t)q);
        for (int i = lane; i < n; i += 32) b2n_sm[oucur + i] = p.u0[(size_t)(p.start ? p.start[q] : q) * n + i];
        __syncwarp();
        int nacc = 0, nrej = 0;
        double lcur = 0.0;
        for (int step = 0; step < p.walks; step++) {
            // (the previous step's likelihood READ the delta vector that the loops below rewrite: order the two --
            //  warp shuffles converge the lanes but are not a memory barrier; compute-sanitizer racecheck, round 2)
            __syncwarp();
            // (1) non-clustered dims: one vector uniform event (only if there are any)
            if (n > nc) {
                for (int e = lane; e < n - nc; e += 32) {
                    const double t = rng_uniform_elem(g, e);
                    const double vi = prior_sm(pk, op0, op1, nc + e, t);
                    b2n_sm[ouprop + nc + e] = t;
                    b2n_sm[ovprop + nc + e] = vi;
                    b2n_sm[od + nc + e] = vi - b2n_sm[omu + nc + e];
                }
                g.tick++;
            }
            // (2) uniform point in the unit nc-ball
            const double fac = scale_ * ball_direction(g, ox, nc, lane, inv_nc);
            __syncwarp();
            // (3) u' = u + fac * axes @ z on the clustered dims, (4) wrap / reflect / cube test,
            //     and (speculatively) the prior transform of the rows this lane owns
            bool ok = true;
            for (int base = 0; base < nc; base += 64) {
                double y0, y1;
                matvec2o<AX_SMEM>(Ag, offA, ldA, nc, ox, base + lane, nc, y0, y1);
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int i = base + lane + 32 * h;
                    if (i < nc) {
                        double t = fma(fac, h ? y1 : y0, b2n_sm[oucur + i]);
                        const uint32_t f = fl[i];
                        if (f & B2N_DIM_PERIODIC) t = mod1(t);
                        if (f & B2N_DIM_REFLECTIVE) t = reflect1(t);
                        ok = ok && in_cube(t, f);
                        const double vi = prior_sm(pk, op0, op1, i, t);
                        b2n_sm[ouprop + i] = t;
                        b2n_sm[ovprop + i] = vi;
                        b2n_sm[od + i] = vi - b2n_sm[omu + i];
                    }
                }
            }
            ok = __all_sync(B2N_FULL, ok);       // also orders the shared-memory writes above
            if (!ok) { nrej++; continue; }
#ifdef B2N_USER_PRIOR
            // a user prior maps the whole proposal at once, clustered and non-clustered dims, with the likelihood
            // scratch as its work (a rejected proposal needs no v: it consumes no random numbers either way)
            if (pk == B2N_PRIOR_USER) user_prior_warp(p.m, &b2n_sm[ouprop], &b2n_sm[ovprop], &b2n_sm[od], lane);
#endif
            // (5) likelihood
            double l;
            if (LIKE == B2N_LIKE_GAUSS_PREC) {
                l = fma(-0.5, quadform_full<PREC_SMEM>(Pg, offP, ldP, n, od, lane), p.m.s0);
            } else {
                l = loglike_sm<LIKE, PREC_SMEM>(p.m, ms, Pg, offP, ldP, n, ovprop, od, lane);
            }
            if (l > loglstar_) {
                int t = oucur; oucur = ouprop; ouprop = t;
                t = ovcur; ovcur = ovprop; ovprop = t;
                lcur = l;
                nacc++;
            } else {
                nrej++;
            }
        }
        if (nacc == 0) {       // recompute (v, logl) of the start point (:970-975)
            for (int i = lane; i < n; i += 32) {
                const double vi = prior_sm(pk, op0, op1, i, b2n_sm[oucur + i]);
                b2n_sm[ovcur + i] = vi;
                b2n_sm[od + i] = vi - b2n_sm[omu + i];
            }
            __syncwarp();
#ifdef B2N_USER_PRIOR
            if (pk == B2N_PRIOR_USER) user_prior_warp(p.m, &b2n_sm[oucur], &b2n_sm[ovcur], &b2n_sm[od], lane);
#endif
            if (LIKE == B2N_LIKE_GAUSS_PREC) {
                lcur = fma(-0.5, quadform_full<PREC_SMEM>(Pg, offP, ldP, n, od, lane), p.m.s0);
            } else {
                lcur = loglike_sm<LIKE, PREC_SMEM>(p.m, ms, Pg, offP, ldP, n, ovcur, od, lane);
            }
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
        __syncwarp();
    }
    peer_finish(p.peer);
}

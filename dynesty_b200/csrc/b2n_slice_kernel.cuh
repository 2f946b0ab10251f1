// b2n_slice_kernel.cuh -- the slice / rslice chain kernel (slice_kernel), its step helpers and launch
// parameters.  Device-only: included by b2n_slice.cu and by the run-time compiled translation unit of a user
// likelihood (b2n_user_kernels.cuh).
#pragma once
#include "b2n_chain.cuh"

#define B2N_MAX_EXPAND 4000000      // hard stop against a runaway stepping-out loop
#define B2N_EXPAND_SAT 0x7fffffff   // a chain's n_expand saturates here instead of wrapping

struct SliceParams {
    B2nModel m;
    int n, slices, doubling;
    int ldA, ldP;
    const double* u0;
    const int* order;
    const int3* cta;
    const double* axesT;
    double loglstar, scale;
    uint64_t seed, chain0;
    double *u, *v, *logl;
    int *nexp, *ncon, *ncall;
    uint32_t* flags;
    PeerSet peer;          // fused multi-GPU gather of the outputs (b2n_peer.cu)
    const B2nDyn* dyn;     // device-paced launch (b2n_ns.cu)
};

// F(x) of generic_slice_step (:1112-1123): logl(u + x d) or -inf outside the unit cube.
template <int LIKE, bool PREC_SMEM>
struct SliceEval {
    const B2nModel& m;
    const ModelSm& ms;
    const double* Pg;
    int offP, ldP;
    int ou, odir, oun, ovn, owork;
    int lane, n, pk;
    int nc;
    __device__ __forceinline__ double operator()(double x) {
        bool ok = true;
        for (int i = lane; i < n; i += 32) {
            const double t = fma(x, b2n_sm[odir + i], b2n_sm[ou + i]);
            b2n_sm[oun + i] = t;
            b2n_sm[ovn + i] = prior_sm(pk, ms.op0, ms.op1, i, t);
            ok = ok && (t > 0.0 && t < 1.0);
        }
        nc++;
        ok = __all_sync(B2N_FULL, ok);          // also orders the writes above
        if (!ok) return -INFINITY;
#ifdef B2N_USER_PRIOR
        if (pk == B2N_PRIOR_USER) user_prior_warp(m, &b2n_sm[oun], &b2n_sm[ovn], &b2n_sm[owork], lane);
#endif
        return loglike_sm<LIKE, PREC_SMEM>(m, ms, Pg, offP, ldP, n, ovn, owork, lane);
    }
};

template <class EVAL>
__device__ bool doubling_accept(EVAL& F, double x1, double loglstar, double L, double R, double fL, double fR) {
    double lhat = L, rhat = R, fl = fL, fr = fR;
    bool D = false;
    while (rhat - lhat > 1.1) {
        const double M = (lhat + rhat) / 2.0;
        if ((0.0 < M && M <= x1) || (x1 < M && M <= 0.0)) D = true;
        if (x1 < M) { rhat = M; fr = F(rhat); }
        else { lhat = M; fl = F(lhat); }
        if (D && loglstar >= fl && loglstar >= fr) return false;
    }
    return true;
}

// one generic_slice_step along b2n_sm[odir..] (already scaled, not yet length-capped).  On
// success the new point is left in b2n_sm[F.oun..] and its logl returned.  D doublings count 2^D - 1 expansions
// (a tiny scale takes 40 or more).  The reference counts in Python ints; here the step's count and n_expand, the
// chain's total, saturate at B2N_EXPAND_SAT (INT32_MAX) instead of wrapping.
template <class EVAL>
__device__ double slice_step(EVAL& F, ChainRng& g, double loglstar, bool doubling, int& n_expand, int& n_contract,
                             bool& expansion_warning, int& err) {
    const int n = F.n, lane = F.lane, odir = F.odir;
    const double rand0 = rng_uniform(g);                        // :1099
    double ss = 0.0;
    for (int i = lane; i < n; i += 32) ss = fma(b2n_sm[odir + i], b2n_sm[odir + i], ss);
    const double dirlen = sqrt(warp_sum(ss));
    const double maxlen = sqrt((double)n) / 2.0;
    if (dirlen > maxlen) {                                      // :1103-1108
        const double dn = dirlen / maxlen;
        for (int i = lane; i < n; i += 32) b2n_sm[odir + i] = b2n_sm[odir + i] / dn;
    }
    __syncwarp();
    double xl = -rand0, xr = 1.0 - rand0;                       // :1126-1127
    double fl = F(xl), fr = F(xr);
    double L = 0, R = 0, fL = 0, fR = 0;
    int nexp = 0;
    expansion_warning = false;
    if (!doubling) {
        while (fl > loglstar) {                                 // :1134-1137
            xl -= 1.0; fl = F(xl); nexp++;
            if (nexp > B2N_MAX_EXPAND) { err = B2N_ERR_SLICE_FAIL; break; }
        }
        while (fr > loglstar && !err) {
            xr += 1.0; fr = F(xr); nexp++;
            if (nexp > B2N_MAX_EXPAND) { err = B2N_ERR_SLICE_FAIL; break; }
        }
        if (nexp > 1000) expansion_warning = true;              // :1142-1145
    } else {
        int D = 0;                                              // :1149-1163 (n_expand += K, K *= 2)
        while (fl > loglstar || fr > loglstar) {
            const double V = rng_uniform(g);
            if (V < 0.5) { xl -= (xr - xl); fl = F(xl); }
            else { xr += (xr - xl); fr = F(xr); }
            D++;
        }
        nexp = D < 31 ? (1 << D) - 1 : B2N_EXPAND_SAT;
        L = xl; R = xr; fL = fl; fR = fr;
    }
    n_expand = (int)min((long long)n_expand + nexp, (long long)B2N_EXPAND_SAT);
    double lp = -INFINITY;
    for (int it = 0; !err; it++) {                              // :1168-1203
        const double xp = xl + rng_uniform(g) * (xr - xl);
        lp = F(xp);
        n_contract++;
        if (lp > loglstar && (!doubling || doubling_accept(F, xp, loglstar, L, R, fL, fR))) {
            if (doubling) {   // the acceptance test moved F's scratch point: restore the accepted one
                lp = F(xp);
                F.nc--;
            }
            break;
        }
        if (xp < 0.0) xl = xp;
        else if (xp > 0.0) xr = xp;
        else err = B2N_ERR_SLICE_FAIL;                          // :1191-1203
        if (it > 100000) err = B2N_ERR_SLICE_FAIL;
    }
    return lp;
}

template <int LIKE, bool RANDOM_DIR, bool AX_SMEM, bool PREC_SMEM>
__global__ void __launch_bounds__(512, 1) slice_kernel(const SliceParams p) {
    const int n = p.n;
    const int npad = (n + 1) & ~1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    double loglstar_ = p.loglstar, scale_ = p.scale;
    unsigned long long chain0_ = p.chain0;
    int doubling_ = p.doubling;
    if (p.dyn) {      // device-paced: scalars written by the previous kernel on the stream
        if (p.dyn->skip || (int)blockIdx.x >= p.dyn->ncta) return;
        loglstar_ = p.dyn->loglstar; scale_ = p.dyn->scale; chain0_ = p.dyn->chain0; doubling_ = p.dyn->doubling;
    }
    const int3 cd = p.cta[blockIdx.x];
    int off = 0;
    const double* Ag = p.axesT + (size_t)cd.z * n * n;
    int offA = 0, ldA = n;
    if (AX_SMEM) {
        offA = off; ldA = p.ldA;
        stage_matrix(Ag, offA, n, ldA);
        off += n * ldA;
    }
    const double* Pg = p.m.lmat;
    int offP = 0, ldP = n;
    if (LIKE == B2N_LIKE_GAUSS_PREC && PREC_SMEM) {
        offP = off; ldP = p.ldP;
        stage_matrix(Pg, offP, n, ldP);
        off += n * ldP;
    }
    const ModelSm ms = stage_model(p.m, off, n, npad);
    off += 4 * npad;
    __syncthreads();
    const int ou = off + warp * 6 * npad;
    const int odir = ou + npad, oun = odir + npad, ovn = oun + npad, owork = ovn + npad;
    int* idxs = reinterpret_cast<int*>(&b2n_sm[owork + npad]);   // permutation (n ints)
    const int pk = p.m.prior_kind;

    for (int c = warp; c < cd.y; c += nwarps) {
        const int q = p.order[cd.x + c];
        ChainRng g;
        g.init(p.seed, chain0_ + (uint64_t)q);
        for (int i = lane; i < n; i += 32) b2n_sm[ou + i] = p.u0[(size_t)q * n + i];
        __syncwarp();
        SliceEval<LIKE, PREC_SMEM> F{p.m, ms, Pg, offP, ldP, ou, odir, oun, ovn, owork, lane, n, pk, 0};
        int nexp = 0, ncon = 0, err = 0;
        bool doubling = doubling_ != 0, warned = false;
        double lcur = 0.0;
        for (int sl = 0; sl < p.slices && !err; sl++) {
            const int nsub = RANDOM_DIR ? 1 : n;
            if (!RANDOM_DIR && n > 1) {
                // rstate.shuffle(idxs) (:673-674): argsort (stable) of one uniform vector event
                for (int e = lane; e < n; e += 32) b2n_sm[owork + e] = rng_uniform_elem(g, e);
                g.tick++;
                __syncwarp();
                for (int e = lane; e < n; e += 32) {
                    const double ve = b2n_sm[owork + e];
                    int rk = 0;
                    for (int f = 0; f < n; f++) {
                        const double vf = b2n_sm[owork + f];
                        rk += (vf < ve || (vf == ve && f < e)) ? 1 : 0;
                    }
                    idxs[rk] = e;
                }
                __syncwarp();
            } else if (!RANDOM_DIR) {
                if (lane == 0) idxs[0] = 0;
                __syncwarp();
            }
            for (int sub = 0; sub < nsub && !err; sub++) {
                if (RANDOM_DIR) {
                    // drhat = z / |z| ; direction = axes @ drhat * scale (:820-824)
                    const double ssq = normals_sm(g, owork, n, lane);
                    const double fac = scale_ / sqrt(ssq);
                    __syncwarp();
                    for (int base = 0; base < n; base += 64) {
                        double y0, y1;
                        matvec2o<AX_SMEM>(Ag, offA, ldA, n, owork, base + lane, n, y0, y1);
                        if (base + lane < n) b2n_sm[odir + base + lane] = y0 * fac;
                        if (base + lane + 32 < n) b2n_sm[odir + base + lane + 32] = y1 * fac;
                    }
                } else {
                    // axes = scale * axes.T ; axis = axes[idx] (:665, 680) = column idx of the axes matrix
                    const int idx = idxs[sub];
                    for (int i = lane; i < n; i += 32) b2n_sm[odir + i] = scale_ * mat_ld<AX_SMEM>(Ag, offA + idx * ldA + i);
                }
                __syncwarp();
                bool ew = false;
                const double l = slice_step(F, g, loglstar_, doubling, nexp, ncon, ew, err);
                if (err) break;
                lcur = l;
                for (int i = lane; i < n; i += 32) b2n_sm[ou + i] = b2n_sm[oun + i];     // u = u_prop
                __syncwarp();
                if (ew && !doubling) { doubling = true; warned = true; }   // :689-693, 836-838
            }
        }
        // v_prop = prior_transform(u_prop) (:1204)
#ifdef B2N_USER_PRIOR
        if (pk == B2N_PRIOR_USER) {
            user_prior_warp(p.m, &b2n_sm[ou], &b2n_sm[ovn], &b2n_sm[owork], lane);
            for (int i = lane; i < n; i += 32) {
                peer_put(p.peer, &p.u[(size_t)q * n + i], b2n_sm[ou + i]);
                peer_put(p.peer, &p.v[(size_t)q * n + i], b2n_sm[ovn + i]);
            }
        } else
#endif
        for (int i = lane; i < n; i += 32) {
            const double ui = b2n_sm[ou + i];
            peer_put(p.peer, &p.u[(size_t)q * n + i], ui);
            peer_put(p.peer, &p.v[(size_t)q * n + i], prior_sm(pk, ms.op0, ms.op1, i, ui));
        }
        if (lane == 0) {
            peer_put(p.peer, &p.logl[q], lcur);
            peer_put(p.peer, &p.nexp[q], nexp);
            peer_put(p.peer, &p.ncon[q], ncon);
            peer_put(p.peer, &p.ncall[q], (int)F.nc);
            peer_put(p.peer, &p.flags[q], (warned ? B2N_WARN_DOUBLING : 0u) | (err ? 0x80000000u : 0u));
        }
        __syncwarp();
    }
    peer_finish(p.peer);
}

// b2n_chain.cuh -- warp-level building blocks shared by the proposal-chain kernels
// (rwalk, rslice, slice).  Every per-chain vector and every staged matrix lives in the CTA's
// dynamic shared memory and is addressed as b2n_sm[offset]: the compiler sees plain
// shared-space accesses with immediate offsets (no generic-address fix-ups, no 64-bit index
// math), which removes a large share of the instruction count of these kernels.
#pragma once
#include "b2n_device.cuh"
#include "b2n_fastmath.cuh"

extern __shared__ __align__(16) double b2n_sm[];

// Element `idx` of a column-major matrix that lives either in dynamic shared memory (index
// into b2n_sm) or in global memory (read-only path, L2 resident).
template <bool SMEM>
__device__ __forceinline__ double mat_ld(const double* __restrict__ g, int idx) {
    return SMEM ? b2n_sm[idx] : __ldg(g + idx);
}

// y_i = sum_j M[j*ld + i] x_j for rows i0 and i0+32.  x = b2n_sm[offx..] (16-byte aligned,
// read as one 16-byte broadcast per two columns); four columns per trip with eight
// independent accumulators so that consecutive DFMAs never wait on each other.
template <bool SMEM>
__device__ __forceinline__ void matvec2o(const double* __restrict__ g, int offM, int ld, int ncols, int offx,
                                         int i0, int nrows, double& y0, double& y1) {
    const bool r0 = i0 < nrows, r1 = i0 + 32 < nrows;
    // idle lanes re-read the LAST row (same 128-byte segment as their active neighbours: a
    // broadcast), not row 0 -- row 0 sits in the same banks as row 32 and cost an extra wavefront
    const int c0 = offM + (r0 ? i0 : nrows - 1), c1 = offM + (r1 ? i0 + 32 : nrows - 1);
    double a0 = 0, a1 = 0, b0 = 0, b1 = 0, e0 = 0, e1 = 0, f0 = 0, f1 = 0;
    int j = 0, o = 0;
    for (; j + 3 < ncols; j += 4, o += 4 * ld) {
        const double2 xa = *reinterpret_cast<const double2*>(&b2n_sm[offx + j]);
        const double2 xb = *reinterpret_cast<const double2*>(&b2n_sm[offx + j + 2]);
        a0 = fma(mat_ld<SMEM>(g, c0 + o), xa.x, a0);
        a1 = fma(mat_ld<SMEM>(g, c1 + o), xa.x, a1);
        b0 = fma(mat_ld<SMEM>(g, c0 + o + ld), xa.y, b0);
        b1 = fma(mat_ld<SMEM>(g, c1 + o + ld), xa.y, b1);
        e0 = fma(mat_ld<SMEM>(g, c0 + o + 2 * ld), xb.x, e0);
        e1 = fma(mat_ld<SMEM>(g, c1 + o + 2 * ld), xb.x, e1);
        f0 = fma(mat_ld<SMEM>(g, c0 + o + 3 * ld), xb.y, f0);
        f1 = fma(mat_ld<SMEM>(g, c1 + o + 3 * ld), xb.y, f1);
    }
    for (; j < ncols; j++, o += ld) {
        const double xj = b2n_sm[offx + j];
        a0 = fma(mat_ld<SMEM>(g, c0 + o), xj, a0);
        a1 = fma(mat_ld<SMEM>(g, c1 + o), xj, a1);
    }
    y0 = r0 ? (a0 + b0) + (e0 + f0) : 0.0;
    y1 = r1 ? (a1 + b1) + (e1 + f1) : 0.0;
}

// d^T P d = sum_i d_i (P d)_i with the full mat-vec, d = b2n_sm[od..].  (A strict-upper-
// triangle variant that halves the shared-memory wavefronts through predicated loads is not
// used: the predicated diagonal block costs more issue slots than the saved wavefronts buy.)
template <bool SMEM>
__device__ __forceinline__ double quadform_full(const double* __restrict__ g, int offP, int ld, int n, int od,
                                                int lane) {
    double sacc = 0.0;
    for (int base = 0; base < n; base += 64) {
        double y0, y1;
        matvec2o<SMEM>(g, offP, ld, n, od, base + lane, n, y0, y1);
        const int i0 = base + lane, i1 = i0 + 32;
        if (i0 < n) sacc = fma(b2n_sm[od + i0], y0, sacc);
        if (i1 < n) sacc = fma(b2n_sm[od + i1], y1, sacc);
    }
    return warp_sum(sacc);
}

// prior transform of one component; prior vectors p0/p1 staged at b2n_sm[op0..], [op1..]
__device__ __forceinline__ double prior_sm(int kind, int op0, int op1, int i, double u) {
    switch (kind) {
        case B2N_PRIOR_UNIFORM: return fma(b2n_sm[op1 + i], u, b2n_sm[op0 + i]);
        case B2N_PRIOR_NORMAL_PPF: return fma(b2n_sm[op1 + i], normcdfinv(u), b2n_sm[op0 + i]);
        default: return u;
    }
}

// Model vectors staged once per CTA: [op0 | op1 | olv0 | olv1], each npad doubles.
struct ModelSm {
    int op0, op1, olv0, olv1;
};
__device__ __forceinline__ ModelSm stage_model(const B2nModel& m, int off, int n, int npad) {
    ModelSm s{off, off + npad, off + 2 * npad, off + 3 * npad};
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        b2n_sm[s.op0 + i] = m.pp0 ? m.pp0[i] : 0.0;
        b2n_sm[s.op1 + i] = m.pp1 ? m.pp1[i] : 1.0;
        b2n_sm[s.olv0 + i] = m.lv0 ? m.lv0[i] : 0.0;
        b2n_sm[s.olv1 + i] = m.lv1 ? m.lv1[i] : 0.0;
    }
    return s;
}

// log-likelihood of the point v = b2n_sm[ov..] (warp-cooperative; scratch d = b2n_sm[od..]).
template <int LIKE, bool PREC_SMEM>
__device__ __forceinline__ double loglike_sm(const B2nModel& m, const ModelSm& ms, const double* __restrict__ Pg,
                                             int offP, int ldP, int n, int ov, int od, int lane) {
    if (LIKE == B2N_LIKE_GAUSS_PREC) {
        for (int i = lane; i < n; i += 32) b2n_sm[od + i] = b2n_sm[ov + i] - b2n_sm[ms.olv0 + i];
        __syncwarp();
        const double q = quadform_full<PREC_SMEM>(Pg, offP, ldP, n, od, lane);
        __syncwarp();
        return fma(-0.5, q, m.s0);
    } else if (LIKE == B2N_LIKE_GAUSS_DIAG) {
        double s = 0.0;
        for (int i = lane; i < n; i += 32) {
            const double d = b2n_sm[ov + i] - b2n_sm[ms.olv0 + i];
            s = fma(b2n_sm[ms.olv1 + i] * d, d, s);
        }
        return fma(-0.5, warp_sum(s), m.s0);
    } else if (LIKE == B2N_LIKE_EGGBOX) {
        double pr = 1.0;
        for (int i = lane; i < n; i += 32) {
            const double t = 2.0 * m.s0 * b2n_sm[ov + i] - m.s0;
            pr *= cos(t * 0.5);
        }
        return pow(2.0 + warp_prod(pr), m.s1);
    } else if (LIKE == B2N_LIKE_REGION2D) {
        return region2d_logl(m.s0, b2n_sm[ov], b2n_sm[ov + 1]);
#ifdef B2N_USER_MODEL
    } else if (LIKE == B2N_LIKE_USER) {
        return b2n_user_loglike(&b2n_sm[ov], &b2n_sm[od], n, m.lv0, lane);
#endif
    } else {  // SHELLS
        double a = 0.0, b = 0.0;
        for (int i = lane; i < n; i += 32) {
            const double vi = b2n_sm[ov + i];
            const double d1 = vi - b2n_sm[ms.olv0 + i], d2 = vi - b2n_sm[ms.olv1 + i];
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

// Standard-normal vector event of size m into b2n_sm[offx..]; returns sum of squares.
__device__ __forceinline__ double normals_sm(ChainRng& g, int offx, int m, int lane) {
    double ss = 0.0;
    const int nb = (m + 1) >> 1;
    for (int b = lane; b < nb; b += 32) {
        double z0, z1;
        rng_normal_pair(g, b, z0, z1);
        ss = fma(z0, z0, ss);
        if (2 * b + 1 < m) {
            *reinterpret_cast<double2*>(&b2n_sm[offx + 2 * b]) = make_double2(z0, z1);
            ss = fma(z1, z1, ss);
        } else {
            b2n_sm[offx + 2 * b] = z0;
        }
    }
    g.tick++;
    return warp_sum(ss);
}

// Uniform direction in the unit nc-ball (bounding.py:1288-1297): writes z to b2n_sm[offx..]
// and returns U^(1/nc) / |z|.  Two draw events (normal vector, then the radius uniform).
// When the normal vector needs < 32 Philox blocks the otherwise idle lane 31 generates the
// radius block in the same instruction stream (different counter), so one Philox + one log
// serve both events.
__device__ __forceinline__ double ball_direction(ChainRng& g, int offx, int nc, int lane, double inv_nc) {
    const int nb = (nc + 1) >> 1;
    if (nb <= 31) {
        const bool isr = lane == 31;
        const uint4 r = curand_Philox4x32_10(
            make_uint4(isr ? 0u : (uint32_t)lane, g.tick + (isr ? 1u : 0u), g.c2, g.c3), g.key);
        g.tick += 2;
        const double u0 = b2n_u52(r.x, r.y), u1 = b2n_u52(r.z, r.w);
        const double lg = log(u0);
        const double rad = sqrt(-2.0 * lg);
        double sn, cs;
        sincospi(2.0 * u1, &sn, &cs);
        const double z0 = rad * cs, z1 = rad * sn;
        double ss = 0.0;
        if (lane < nb) {
            ss = z0 * z0;
            if (2 * lane + 1 < nc) {
                *reinterpret_cast<double2*>(&b2n_sm[offx + 2 * lane]) = make_double2(z0, z1);
                ss = fma(z1, z1, ss);
            } else {
                b2n_sm[offx + 2 * lane] = z0;
            }
        }
        ss = warp_sum(ss);
        const double lgU = __shfl_sync(B2N_FULL, lg, 31);
        return exp(lgU * inv_nc) / sqrt(ss);
    }
    const double ss = normals_sm(g, offx, nc, lane);
    const double U = rng_uniform(g);
    return pow(U, inv_nc) / sqrt(ss);
}

// Two directions at once with the BRANCH-FREE math of b2n_fastmath.cuh (nc <= 62): same draw events and ticks
// as two calls of ball_direction(), but the two Philox -> log -> sqrt -> sincos dependency chains contain no
// control flow and are written side by side, so the instruction scheduler overlaps their latencies -- which it
// cannot do for libdevice's log / sqrt / sincospi (slow-path branches keep the calls in separate basic blocks).  `two` = false generates only the first (the second result is then meaningless).
__device__ __forceinline__ void ball_direction_pair_fast(const ChainRng& ga, const ChainRng& gb, int offa, int offb,
                                                         bool two, int nc, int lane, double inv_nc, double& fa,
                                                         double& fb) {
    const int nb = (nc + 1) >> 1;
    const bool isr = lane == 31;
    const uint32_t blk = isr ? 0u : (uint32_t)lane, dt = isr ? 1u : 0u;
    const uint4 ra = curand_Philox4x32_10(make_uint4(blk, ga.tick + dt, ga.c2, ga.c3), ga.key);
    const uint4 rb = curand_Philox4x32_10(make_uint4(blk, gb.tick + dt, gb.c2, gb.c3), gb.key);
    const double lga = b2n_log(b2n_u52(ra.x, ra.y)), lgb = b2n_log(b2n_u52(rb.x, rb.y));
    const double rada = b2n_sqrt(-2.0 * lga), radb = b2n_sqrt(-2.0 * lgb);
    double sa, ca, sb, cb;
    b2n_sincos2pi(b2n_u52(ra.z, ra.w), &sa, &ca);
    b2n_sincos2pi(b2n_u52(rb.z, rb.w), &sb, &cb);
    const double z0a = rada * ca, z1a = rada * sa, z0b = radb * cb, z1b = radb * sb;
    double ssa = 0.0, ssb = 0.0;
    if (lane < nb) {
        const bool full = 2 * lane + 1 < nc;
        ssa = full ? fma(z1a, z1a, z0a * z0a) : z0a * z0a;
        ssb = full ? fma(z1b, z1b, z0b * z0b) : z0b * z0b;
        if (full) {
            *reinterpret_cast<double2*>(&b2n_sm[offa + 2 * lane]) = make_double2(z0a, z1a);
            if (two) *reinterpret_cast<double2*>(&b2n_sm[offb + 2 * lane]) = make_double2(z0b, z1b);
        } else {
            b2n_sm[offa + 2 * lane] = z0a;
            if (two) b2n_sm[offb + 2 * lane] = z0b;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        ssa += __shfl_xor_sync(B2N_FULL, ssa, o);
        ssb += __shfl_xor_sync(B2N_FULL, ssb, o);
    }
    const double la = __shfl_sync(B2N_FULL, lga, 31), lb = __shfl_sync(B2N_FULL, lgb, 31);
    fa = b2n_div(exp(la * inv_nc), b2n_sqrt(ssa));
    fb = b2n_div(exp(lb * inv_nc), b2n_sqrt(two ? ssb : 1.0));
}

// ONE Philox block of a direction draw with the branch-free math, for callers that deal the blocks of many directions
// over the lanes (the draw warps of rwalk_mmaws_kernel).  j < nb = (nc + 1) / 2: Box-Muller block j of the normal
// vector event -> z[2j], z[2j + 1] at b2n_sm[off + 2j..], and its share of |z|^2 (the expression ball_direction's
// lane j forms) -> b2n_sm[osc].  j == nb: the block of the radius uniform (the one ball_direction's lane 31 draws)
// -> log U at b2n_sm[osc]; it runs the same straight-line code and stores only the log.  Nothing is stored unless `store`.
__device__ __forceinline__ void ball_block_fast(const ChainRng& g, int j, int nc, int off, int osc, bool store) {
    const int nb = (nc + 1) >> 1;
    const bool isr = j == nb;
    const uint4 r = curand_Philox4x32_10(make_uint4(isr ? 0u : (uint32_t)j, g.tick + (isr ? 1u : 0u), g.c2, g.c3),
                                         g.key);
    const double lg = b2n_log(b2n_u52(r.x, r.y));
    const double rad = b2n_sqrt(-2.0 * lg);
    double sn, cs;
    b2n_sincos2pi(b2n_u52(r.z, r.w), &sn, &cs);
    const double z0 = rad * cs, z1 = rad * sn;
    if (store) {
        const bool full = 2 * j + 1 < nc;
        if (isr) {
            b2n_sm[osc] = lg;
        } else if (full) {
            *reinterpret_cast<double2*>(&b2n_sm[off + 2 * j]) = make_double2(z0, z1);
            b2n_sm[osc] = fma(z1, z1, z0 * z0);
        } else {
            b2n_sm[off + 2 * j] = z0;
            b2n_sm[osc] = z0 * z0;
        }
    }
}

// |z|^2 from the per-block shares s[j] = b2n_sm[o + j], j < nb (<= 31), on ONE lane, summed in the association of the
// 32-lane butterfly `for (o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(.., s, o)` over lanes holding s[lane] (0.0 from
// lane nb on): node(a, m) = node(a, 2m) + node(a + m, 2m), leaves s[a] + s[a + 16].  Floating-point addition is
// commutative, so every lane of that butterfly holds exactly this value.
template <int M>
__device__ __forceinline__ double ss_butterfly(int o, int nb, int a) {
    if constexpr (M == 16) {
        const double lo = a < nb ? b2n_sm[o + a] : 0.0, hi = a + 16 < nb ? b2n_sm[o + a + 16] : 0.0;
        return lo + hi;
    } else {
        return ss_butterfly<2 * M>(o, nb, a) + ss_butterfly<2 * M>(o, nb, a + M);
    }
}

// Stage a column-major matrix (n x n, ld = n in global) into b2n_sm with padded leading dim.
__device__ __forceinline__ void stage_matrix(const double* __restrict__ g, int off, int n, int ldp) {
    for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
        const int j = e / n, i = e - j * n;
        b2n_sm[off + j * ldp + i] = g[e];
    }
}

#ifndef __CUDACC_RTC__
// shared by the chain entry points (defined in b2n_rwalk.cu)
int b2n_build_worklist(b2n_ctx* ctx, int64_t Q, const int32_t* ell, int K, int chains_per_cta,
                       std::vector<int>& order, std::vector<int3>& cta);
void b2n_chain_grid(const b2n_ctx* ctx, int64_t Q, int max_warps, int& chains_per_cta, int& warps);
// worklist on the device: cached for the single-ellipsoid case, else built on the host and uploaded
int b2n_worklist_dev(b2n_ctx* ctx, int64_t Q, const int32_t* ell, int K, int chains_per_cta, const void** dorder,
                     const void** dcta, unsigned* ncta);
#endif

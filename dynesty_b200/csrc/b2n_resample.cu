// b2n_resample.cu -- R bootstrap realisations of one strand-labelled record (resample_run / kld_error(error=
// 'resample') of the reference, utils.py:1495-1660, 1932-1997), all in FP64.  Contract: include/b200nest.h,
// b2n_resample_runs; restated in numpy in oracle/resample.py.
//
// Two launches:
//   resample_mult_kernel   (elements x R)  the strand draws of every realisation -> m[r][s] with integer atomics
//                                          (order-independent, so deterministic)
//   resample_scan_kernel   (R)             one CTA per realisation walks the record in tiles of RS_TILE samples,
//                                          twice: sweep 1 gives logz[-1]; sweep 2 the KL divergence, h and logzvar,
//                                          which need it.  Per tile, block scans with a fixed association give
//                                          the live count (scan of the piece differences), the last sample present
//                                          in the realisation (its logl is the previous copy's), ln X and logz
//                                          before each sample; a thread then walks the m copies of its sample.
// Nothing R x N is stored; a realisation never reads another's data, so it does not depend on R.
//
// Host side: b2n_resample_produce checks and stages a record and enqueues the two launches, for b2n_resample_runs
// (below) and for b2n_resample_posterior (b2n_posterior.cu, with the weights); the entry points stage their outputs
// through B2nOutStage (b2n_common.cuh).  The block scan and its operators are b2n_scan.cuh's.
#include "b2n_device.cuh"
#include "b2n_scan.cuh"

#include <algorithm>
#include <math.h>

namespace {

constexpr int RS_BLOCK = 256;
constexpr int RS_TILE = 1024;       // samples per tile (RS_TILE / RS_BLOCK per thread)
constexpr double RS_LOWL = -1e300;  // the logl before the first sample (nested._integrate)

struct RArgs {
    const double* logl;
    const double* wref;          // input run's logwt, or NULL
    const int32_t* strand;       // N
    const int64_t* pptr;         // N + 1
    const int32_t* pstrand;      // pieces starting at each sample
    const uint8_t* end;          // N, or NULL
    const int32_t* base_ids;     // nbase, then the nadd add-on strands
    int64_t N;
    int S, nbase, nadd;
    double zref;
    uint64_t seed, chain0;
    int32_t* mult;               // R x S
    double *out_logz, *out_logzerr, *out_h, *out_kld;
    int R;
    double* w;                   // N x R (sample-major): W = sum over a sample's copies of exp(logwt - logz[-1]),
                                 // -0.0 for a sample not drawn (resample_weights_kernel only)
    double* w2;                  // R: sum over the copies of exp(logwt - logz[-1])^2 (resample_weights_kernel only)
    const double* lrw;           // N: log-reweight added to the logwt of every copy (the _rw kernels only), else NULL
};

__global__ void __launch_bounds__(RS_BLOCK) resample_mult_kernel(RArgs A) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = blockIdx.y;
    ChainRng g;
    g.init(A.seed, A.chain0 + (uint64_t)r);
    int32_t* m = A.mult + (size_t)r * A.S;
    if (e < A.nbase) {                                          // tick 0: the base strands
        const int k = min((int)(rng_uniform_elem(g, e) * (double)A.nbase), A.nbase - 1);
        atomicAdd(m + A.base_ids[k], 1);
    }
    if (e < A.nadd) {                                           // tick 1: the add-on strands
        g.tick = 1;
        const int k = min((int)(rng_uniform_elem(g, e) * (double)A.nadd), A.nadd - 1);
        atomicAdd(m + A.base_ids[A.nbase + k], 1);
    }
}

// ln(c / (c + 1)) of copy k of a sample with live count n and m copies
__device__ __forceinline__ double copy_dlv(double n, int k, bool is_end) {
    const double c = is_end ? n - k : n;
    return log(c / (c + 1.0));
}

// WOUT: also the weights w / w2 (b2n_resample_posterior); resample_scan_kernel, without them, compiles to the code it
// had before they existed.  RW: lrw of the sample is added to the logwt of each of its copies (the h increments keep the
// unreweighted L and ldv2, as compute_integrals(reweight=) does); a KL term of zero weight is 0.
template <bool WOUT, bool RW = false>
__device__ __forceinline__ void resample_scan(const RArgs& A) {
    __shared__ double xc[RS_TILE], xp[RS_TILE], xv[RS_TILE], xz[RS_TILE], wsum[32];
    const int r = blockIdx.x;
    const int32_t* m = A.mult + (size_t)r * A.S;
    const double ln_half = -0.69314718055994530942;
    double zmax = 0.0;
    double sA = 0.0, sC = 0.0, sK = 0.0;                        // sweep 2: sums of a, dh * dlogvol, KL terms
    double sW2 = 0.0;                                           // sweep 2 (WOUT): sum of w^2 over the copies
    for (int sweep = 1; sweep <= 2; sweep++) {
        double c_cnt = 0.0, c_prev = -1.0, c_lv = 0.0, c_z = -INFINITY;   // carries across tiles
        for (int64_t t0 = 0; t0 < A.N; t0 += RS_TILE) {
            const int L = (int)min((int64_t)RS_TILE, A.N - t0);
            // live-count differences and the index of every present sample
            for (int q = threadIdx.x; q < L; q += blockDim.x) {
                const int64_t i = t0 + q;
                double d = 0.0;
                for (int64_t p = A.pptr[i]; p < A.pptr[i + 1]; p++) d += (double)m[A.pstrand[p]];
                if (i > 0) d -= (double)m[A.strand[i - 1]];
                xc[q] = d;
                xp[q] = m[A.strand[i]] > 0 ? (double)i : -1.0;
            }
            __syncthreads();
            const double tc = block_scan(xc, L, wsum, OpSum());
            const double tp = block_scan(xp, L, wsum, OpMax());
            // ln X increment of each sample's copies
            for (int q = threadIdx.x; q < L; q += blockDim.x) {
                const int64_t i = t0 + q;
                const int mi = m[A.strand[i]];
                const bool ie = A.end && A.end[i];
                const double n = c_cnt + xc[q];
                double dv = 0.0;
                for (int k = 0; k < mi; k++) dv += copy_dlv(n, k, ie);
                xv[q] = dv;
            }
            __syncthreads();
            const double tv = block_scan(xv, L, wsum, OpSum());
            // weights of the copies (logsumexp per sample); thread-private copy walk
            for (int q = threadIdx.x; q < L; q += blockDim.x) {
                const int64_t i = t0 + q;
                const int mi = m[A.strand[i]];
                double E = -INFINITY;
                if (mi > 0) {
                    const bool ie = A.end && A.end[i];
                    const double n = c_cnt + xc[q];
                    const double pidx = fmax(c_prev, q > 0 ? xp[q - 1] : -1.0);
                    const double l = A.logl[i];
                    double lp = pidx >= 0.0 ? A.logl[(int64_t)pidx] : RS_LOWL;
                    double lv = c_lv + (q > 0 ? xv[q - 1] : 0.0);
                    for (int k = 0; k < mi; k++) {
                        const double d = copy_dlv(n, k, ie);
                        double w = lae(l, lp) + lv + log1p(-exp(d)) + ln_half;
                        if (RW) w += A.lrw[i];
                        E = lae(E, w);
                        lv += d;
                        lp = l;
                    }
                }
                xz[q] = E;
            }
            __syncthreads();
            const double tz = block_scan(xz, L, wsum, OpLae());
            if (sweep == 2) {
                double a_t = 0.0, c_t = 0.0, k_t = 0.0, w2_t = 0.0;
                for (int q = threadIdx.x; q < L; q += blockDim.x) {
                    const int64_t i = t0 + q;
                    const int mi = m[A.strand[i]];
                    if (WOUT && mi == 0) A.w[(size_t)i * A.R + r] = -0.0;
                    if (mi == 0) continue;
                    double W = 0.0;
                    const bool ie = A.end && A.end[i];
                    const double n = c_cnt + xc[q];
                    const double pidx = fmax(c_prev, q > 0 ? xp[q - 1] : -1.0);
                    const double l = A.logl[i];
                    const double lp2 = A.wref ? A.wref[i] - A.zref : 0.0;
                    double lp = pidx >= 0.0 ? A.logl[(int64_t)pidx] : RS_LOWL;
                    double lv = c_lv + (q > 0 ? xv[q - 1] : 0.0);
                    double z = lae(c_z, q > 0 ? xz[q - 1] : -INFINITY);
                    for (int k = 0; k < mi; k++) {
                        const double d = copy_dlv(n, k, ie);
                        const double ldv2 = lv + log1p(-exp(d)) + ln_half;
                        double w = lae(l, lp) + ldv2;
                        if (RW) w += A.lrw[i];
                        const double zn = lae(z, w);
                        const double a = exp(l - zmax + ldv2) * l + exp(lp - zmax + ldv2) * lp;
                        const double dh = a - zmax * (exp(zn - zmax) - exp(z - zmax));
                        a_t += a;
                        c_t += dh * -d;
                        if (A.wref) {
                            const double lp1 = w - zmax;
                            if (!RW || w != -INFINITY) k_t += exp(lp1) * (lp1 - lp2);
                        }
                        if (WOUT) {
                            const double wc = exp(w - zmax);
                            W += wc;
                            w2_t += wc * wc;
                        }
                        z = zn;
                        lv += d;
                        lp = l;
                    }
                    if (WOUT) A.w[(size_t)i * A.R + r] = W;
                }
                // block sums (fixed association: one value per thread, then block_scan's order)
                __syncthreads();
                xc[threadIdx.x] = a_t; xp[threadIdx.x] = c_t; xv[threadIdx.x] = k_t;
                __syncthreads();
                sA += block_scan(xc, RS_BLOCK, wsum, OpSum());
                sC += block_scan(xp, RS_BLOCK, wsum, OpSum());
                sK += block_scan(xv, RS_BLOCK, wsum, OpSum());
                if (WOUT) {
                    xc[threadIdx.x] = w2_t;
                    __syncthreads();
                    sW2 += block_scan(xc, RS_BLOCK, wsum, OpSum());
                }
            }
            c_cnt += tc;
            c_prev = fmax(c_prev, tp);
            c_lv += tv;
            c_z = lae(c_z, tz);
            __syncthreads();
        }
        if (sweep == 1) zmax = c_z;
    }
    if (threadIdx.x != 0) return;
    if (A.out_logz) A.out_logz[r] = zmax;
    if (A.out_logzerr) A.out_logzerr[r] = sqrt(fabs(sC));       // logzvar = |cumsum(dh * dlogvol)|
    if (A.out_h) A.out_h[r] = sA - zmax;                        // h1[-1] - zmax * exp(logz[-1] - zmax)
    if (A.out_kld) A.out_kld[r] = sK;
    if (WOUT) A.w2[r] = sW2;
}

__global__ void __launch_bounds__(RS_BLOCK) resample_scan_kernel(RArgs A) { resample_scan<false>(A); }
__global__ void __launch_bounds__(RS_BLOCK) resample_weights_kernel(RArgs A) { resample_scan<true>(A); }
__global__ void __launch_bounds__(RS_BLOCK) resample_scan_rw_kernel(RArgs A) { resample_scan<false, true>(A); }
__global__ void __launch_bounds__(RS_BLOCK) resample_weights_rw_kernel(RArgs A) { resample_scan<true, true>(A); }

}  // namespace

int b2n_resample_produce(b2n_ctx* ctx, const double* logl, const int32_t* strand, int64_t N, int32_t S,
                         const uint8_t* base, const int64_t* piece_ptr, const int32_t* piece_strand, const uint8_t* end,
                         const double* logwt_ref, double logz_ref, int32_t R, uint64_t seed, uint64_t chain0,
                         const double* logrwt, double* const sum[4], int32_t* mult, double* w, const double** w2,
                         int64_t* nw2, const double** wref) {
    if (piece_ptr[0] != 0 || piece_ptr[N] < 0 || (piece_ptr[N] > 0 && !piece_strand)) return B2N_ERR_ARG;
    for (int64_t i = 0; i < N; i++)
        if (strand[i] < 0 || strand[i] >= S || piece_ptr[i + 1] < piece_ptr[i]) return B2N_ERR_ARG;
    for (int64_t p = 0; p < piece_ptr[N]; p++)
        if (piece_strand[p] < 0 || piece_strand[p] >= S) return B2N_ERR_ARG;
    std::vector<int32_t> ids;                                   // base strands, then add-on strands, increasing
    for (int s = 0; s < S; s++) if (base[s]) ids.push_back(s);
    const int nbase = (int)ids.size();
    for (int s = 0; s < S; s++) if (!base[s]) ids.push_back(s);
    const int nadd = S - nbase;
    if (nbase == 0) return b2n_fail(ctx, B2N_ERR_ARG, "b2n_resample_runs: the record has no base strand");

    RArgs A;
    memset(&A, 0, sizeof(A));
    const void* p;
    B2N_TRY(b2n_in(ctx, ctx->in0, logl, (size_t)N * sizeof(double), &p));
    A.logl = (const double*)p;
    B2N_TRY(b2n_in(ctx, ctx->in1, logwt_ref, logwt_ref ? (size_t)N * sizeof(double) : 0, &p));
    A.wref = (const double*)p;
    B2N_TRY(b2n_in(ctx, ctx->work1, logrwt, logrwt ? (size_t)N * sizeof(double) : 0, &p));
    A.lrw = (const double*)p;
    B2N_TRY(b2n_in_host(ctx, ctx->in2, strand, (size_t)N * sizeof(int32_t), &p));
    A.strand = (const int32_t*)p;
    B2N_TRY(b2n_in_host(ctx, ctx->in3, piece_ptr, (size_t)(N + 1) * sizeof(int64_t), &p));
    A.pptr = (const int64_t*)p;
    B2N_TRY(b2n_in_host(ctx, ctx->scratch0, piece_strand, (size_t)piece_ptr[N] * sizeof(int32_t), &p));
    A.pstrand = (const int32_t*)p;
    B2N_TRY(b2n_in_host(ctx, ctx->scratch2, end, end ? (size_t)N : 0, &p));
    A.end = (const uint8_t*)p;
    B2N_TRY(b2n_in_host(ctx, ctx->scratch3, ids.data(), ids.size() * sizeof(int32_t), &p));
    A.base_ids = (const int32_t*)p;
    A.N = N; A.S = S; A.nbase = nbase; A.nadd = nadd; A.zref = logz_ref; A.seed = seed; A.chain0 = chain0; A.R = R;
    // the multiplicities in `mult` or in scratch1, followed there by the R w^2 sums when the weights are asked for
    const size_t msz = (size_t)R * S * sizeof(int32_t), mpad = (msz + 255) / 256 * 256;
    if (mult) {
        A.mult = mult;
        if (w) {
            B2N_CUDA(ctx, ctx->scratch1.ensure((size_t)R * sizeof(double)));
            A.w2 = ctx->scratch1.as<double>();
        }
    } else {
        B2N_CUDA(ctx, ctx->scratch1.ensure(w ? mpad + (size_t)R * sizeof(double) : msz));
        A.mult = ctx->scratch1.as<int32_t>();
        if (w) A.w2 = (double*)((char*)ctx->scratch1.p + mpad);
    }
    A.out_logz = sum[0]; A.out_logzerr = sum[1]; A.out_h = sum[2]; A.out_kld = sum[3];
    A.w = w;
    if (w) { *w2 = A.w2; *nw2 = 1; *wref = A.wref; }

    B2N_TIME_BEGIN(ctx);
    B2N_CUDA(ctx, cudaMemsetAsync(A.mult, 0, msz, ctx->stream));
    const dim3 grid((unsigned)((std::max(A.nbase, A.nadd) + RS_BLOCK - 1) / RS_BLOCK), (unsigned)R);
    resample_mult_kernel<<<grid, RS_BLOCK, 0, ctx->stream>>>(A);
    B2N_LAUNCH_CHECK(ctx);
    if (w) (A.lrw ? resample_weights_rw_kernel : resample_weights_kernel)<<<R, RS_BLOCK, 0, ctx->stream>>>(A);
    else (A.lrw ? resample_scan_rw_kernel : resample_scan_kernel)<<<R, RS_BLOCK, 0, ctx->stream>>>(A);
    B2N_LAUNCH_CHECK(ctx);
    return B2N_OK;
}

extern "C" int b2n_resample_runs(b2n_ctx* ctx, const double* logl, const int32_t* strand, int64_t N, int32_t S,
                                 const uint8_t* base, const int64_t* piece_ptr, const int32_t* piece_strand,
                                 const uint8_t* end, const double* logwt_ref, double logz_ref, int32_t R,
                                 uint64_t seed, uint64_t chain0, double* logz, double* logzerr, double* h,
                                 double* kld, int32_t* mult) {
    if (!ctx) return B2N_ERR_ARG;
    const double* logrwt;
    B2N_TRY(b2n_take_reweight(ctx, N, &logrwt));
    if (!logl || !strand || !base || !piece_ptr || N < 1 || S < 1 || R < 1 || R > 65535) return B2N_ERR_ARG;
    if (!logwt_ref && kld) return B2N_ERR_ARG;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t rb = (size_t)R * sizeof(double);
    B2nOutStage<5> O{{logz, logzerr, h, kld, mult}, {rb, rb, rb, rb, (size_t)R * S * sizeof(int32_t)}};
    B2N_TRY(O.bind(ctx));
    double* const d[4] = {(double*)O.dev[0], (double*)O.dev[1], (double*)O.dev[2], (double*)O.dev[3]};
    B2N_TRY(b2n_resample_produce(ctx, logl, strand, N, S, base, piece_ptr, piece_strand, end, logwt_ref, logz_ref, R,
                                 seed, chain0, logrwt, d, (int32_t*)O.dev[4], nullptr, nullptr, nullptr, nullptr));
    B2N_TIME_END(ctx);
    B2N_TRY(O.done(ctx));
    return b2n_finish(ctx);
}

// b2n_equal.cu -- equal-weight posterior draws of R weight vectors over one set of N samples (the reference's
// resample_equal / Results.samples_equal, utils.py:895-903, 1120-1187), in FP64 with the reference's rounding; contract
// and semantics: include/b200nest.h (b2n_resample_equal, b2n_jitter_equal, b2n_resample_equal_runs), DESIGN.md 15.5.
//
// The weights are read as w[i * si + r * sr]: the caller's R x N rows (b2n_resample_equal) or the producers' N x R
// sample-major buffer (b2n_jitter_produce / b2n_resample_produce), where a warp's 32 vectors read one sample together.
//
//   cumsum_kernel   (R / 128)       one thread per vector, serial over N: c = cumsum(w) in np.cumsum's order (N x R),
//                                   wsum = c[N-1], u = the vector's tick-0 uniform; flags a vector it must refuse
//   counts_kernel   (N x R)         counts only: count_j = F(C_j) - F(C_{j-1}), F(C) = #{i : pos_i < C} = the first i
//                                   with pos_i >= C, from the estimate ceil(C M - u) corrected with the exact pos_i
//   draw_kernel     (R x M)         position i: the smallest j with pos_i < C_j by bisection over c (C_j = c_j / wsum
//                                   formed per probe, the bits of the reference's c /= c[-1]); and the sort key of
//                                   element i of tick 1
//   CUB segmented radix sort        the keys of each vector (stable: ties keep the index order, np.argsort's stable)
//   gather_kernel   (R x M)         idx[t] = draw[perm[t]], and the rows x[idx[t]]
// pos_i = fl(fl(u + i) / M) is non-decreasing in i, so F is a count and the draws of sample j are the positions
// [F(C_{j-1}), F(C_j)): counts and draws agree bit for bit.  Every thread writes one output element, so one sample
// holding almost all the weight costs no more than any other.  No float atomics; vector r reads only its own column.
#include "b2n_device.cuh"

#include <cub/device/device_segmented_radix_sort.cuh>

#include <math.h>
#include <vector>

namespace {

constexpr int EQ_THREADS = 256;
constexpr int EQ_CS_THREADS = 128;      // vectors per cumsum CTA
constexpr int EQ_KEY_BITS = 52;         // a uniform's random bits (oracle/philox.py, u53)
constexpr unsigned EQ_MAX_GRID = 1u << 16;     // CTAs of a grid-stride launch: 64 waves of 256 threads per SM

struct EqArgs {
    const double* w;        // w[i * si + r * sr]
    int64_t si, sr;
    int64_t N, M;
    int R;
    uint64_t seed, chain0;
    const double* x;        // N x k, may be NULL
    int k;
    double* c;              // N x R: the cumsum before the division
    double* ws;             // R: wsum
    double* u;              // R: tick 0
    int* bad;               // set when a vector is refused
    double* wsum;           // R, may be NULL
    int32_t* counts;        // R x N, may be NULL
    int32_t* draw;          // R x M: the draws in position order
    uint64_t* keys;         // R x M
    int32_t* vals;          // R x M
    const int32_t* perm;    // R x M: the sorted vals
    int32_t* idx;           // R x M
    double* xout;           // R x M x k, may be NULL
};

// The position of draw i, as the reference forms it: (u + arange(M)) / M.
__device__ __forceinline__ double eq_pos(double u, int64_t i, double Md) { return (u + (double)i) / Md; }

// #{i < M : pos_i < C}, i.e. the first i with pos_i >= C (M if none).  The estimate is within one position of the
// answer (the rounding of pos_i moves it by far less than 1 / M); the loops make it exact.  NaN stays in range.
__device__ __forceinline__ int64_t eq_first_at(double C, double u, int64_t M) {
    const double Md = (double)M;
    int64_t i = (int64_t)fmin(fmax(ceil(C * Md - u), 0.0), Md);
    while (i > 0 && eq_pos(u, i - 1, Md) >= C) i--;
    while (i < M && eq_pos(u, i, Md) < C) i++;
    return i;
}

__global__ void __launch_bounds__(EQ_CS_THREADS) cumsum_kernel(EqArgs A) {
    const int r = blockIdx.x * EQ_CS_THREADS + threadIdx.x;
    if (r >= A.R) return;
    const double* __restrict__ w = A.w + r * A.sr;
    double* __restrict__ c = A.c + r;
    const int64_t N = A.N, si = A.si, R = A.R;
    double s = 0.0;
    bool ok = true;
    int64_t i = 0;
    for (; i + 8 <= N; i += 8) {            // the loads of 8 samples ahead of their dependent adds
        double v[8];
#pragma unroll
        for (int t = 0; t < 8; t++) v[t] = w[(i + t) * si];
#pragma unroll
        for (int t = 0; t < 8; t++) {
            ok &= v[t] >= 0.0 && v[t] < INFINITY;
            s += v[t];
            c[(i + t) * R] = s;
        }
    }
    for (; i < N; i++) {
        const double v = w[i * si];
        ok &= v >= 0.0 && v < INFINITY;
        s += v;
        c[i * R] = s;
    }
    ok &= s > 0.0 && s < INFINITY;
    A.ws[r] = s;
    if (A.wsum) A.wsum[r] = s;
    ChainRng g;
    g.init(A.seed, A.chain0 + (uint64_t)r);
    A.u[r] = rng_uniform(g);
    if (!ok) *A.bad = 1;
}

__global__ void __launch_bounds__(EQ_THREADS) counts_kernel(EqArgs A) {
    const int64_t total = A.N * A.R;
    for (int64_t t = (int64_t)blockIdx.x * EQ_THREADS + threadIdx.x; t < total; t += (int64_t)gridDim.x * EQ_THREADS) {
        const int64_t j = t / A.R;
        const int r = (int)(t - j * A.R);
        const double ws = A.ws[r], u = A.u[r];
        const int64_t lo = j == 0 ? 0 : eq_first_at(A.c[t - A.R] / ws, u, A.M);
        const int64_t hi = j == A.N - 1 ? A.M : eq_first_at(A.c[t] / ws, u, A.M);   // the last sample takes pos >= 1
        A.counts[(int64_t)r * A.N + j] = (int32_t)(hi - lo);
    }
}

__global__ void __launch_bounds__(EQ_THREADS) draw_kernel(EqArgs A) {
    const int64_t total = A.M * A.R;
    const double Md = (double)A.M;
    for (int64_t t = (int64_t)blockIdx.x * EQ_THREADS + threadIdx.x; t < total; t += (int64_t)gridDim.x * EQ_THREADS) {
        const int r = (int)(t / A.M);
        const int64_t i = t - (int64_t)r * A.M;
        const double ws = A.ws[r], pos = eq_pos(A.u[r], i, Md);
        int64_t lo = 0, hi = A.N - 1;       // the answer lies in [lo, hi]; none below 1.0: N - 1
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (pos < A.c[mid * A.R + r] / ws) hi = mid;
            else lo = mid + 1;
        }
        A.draw[t] = (int32_t)lo;
        // element i of the uniform vector event at tick 1; its 52 random bits order as the uniforms do
        ChainRng g;
        g.init(A.seed, A.chain0 + (uint64_t)r);
        g.tick = 1;
        const uint4 b = g.block((uint32_t)(i >> 1));
        const uint32_t hi32 = (i & 1) ? b.z : b.x, lo32 = (i & 1) ? b.w : b.y;
        A.keys[t] = ((uint64_t)(hi32 >> 6) << 26) | (uint64_t)(lo32 >> 6);
        A.vals[t] = (int32_t)i;
    }
}

__global__ void __launch_bounds__(EQ_THREADS) gather_kernel(EqArgs A) {
    const int64_t total = A.M * A.R;
    for (int64_t t = (int64_t)blockIdx.x * EQ_THREADS + threadIdx.x; t < total; t += (int64_t)gridDim.x * EQ_THREADS) {
        const int64_t r = t / A.M;
        const int32_t j = A.draw[r * A.M + A.perm[t]];
        A.idx[t] = j;
        if (A.xout)
            for (int q = 0; q < A.k; q++) A.xout[t * A.k + q] = A.x[(int64_t)j * A.k + q];
    }
}

unsigned eq_grid(int64_t threads) {
    const int64_t b = (threads + EQ_THREADS - 1) / EQ_THREADS;
    return (unsigned)(b < (int64_t)EQ_MAX_GRID ? b : EQ_MAX_GRID);
}

struct EqWork {
    double *c, *ws, *u;
    int* bad;
    int32_t* draw;
    uint64_t *keys_in, *keys_out;
    int32_t *vals_in, *vals_out;
    int* offs;
    void* cub_tmp;
    size_t cub_bytes;
};

int eq_layout(b2n_ctx* ctx, int64_t N, int R, int64_t M, Bump& b, EqWork& w) {
    const size_t rm = (size_t)R * M;
    memset(&w, 0, sizeof(w));
    w.c = b.take<double>((size_t)N * R);
    w.ws = b.take<double>(R);
    w.u = b.take<double>(R);
    w.bad = b.take<int>(1);
    w.draw = b.take<int32_t>(rm);
    w.keys_in = b.take<uint64_t>(rm);
    w.keys_out = b.take<uint64_t>(rm);
    w.vals_in = b.take<int32_t>(rm);
    w.vals_out = b.take<int32_t>(rm);
    w.offs = b.take<int>(R + 1);
    B2N_CUDA(ctx, (cub::DeviceSegmentedRadixSort::SortPairs(nullptr, w.cub_bytes, w.keys_in, w.keys_out, w.vals_in,
                                                            w.vals_out, (int)rm, R, w.offs, w.offs + 1, 0, EQ_KEY_BITS,
                                                            ctx->stream)));
    w.cub_tmp = b.take<char>(w.cub_bytes);
    return B2N_OK;
}

// The draws of R vectors whose weights are on the device (w[i * si + r * sr]), enqueued on the stream.  idx, counts,
// wsum, xout: device (counts / wsum / xout may be NULL).  *bad: the device flag of the weight check (eq_checked).
// Uses ctx->scratch5.
int eq_launch(b2n_ctx* ctx, const double* w, int64_t si, int64_t sr, int64_t N, int R, int64_t M, uint64_t seed,
              uint64_t chain0, const double* x, int k, int32_t* idx, int32_t* counts, double* wsum, double* xout,
              const int** bad) {
    Bump b0{nullptr};
    EqWork W;
    B2N_TRY(eq_layout(ctx, N, R, M, b0, W));
    B2N_CUDA(ctx, ctx->scratch5.ensure(b0.off + 256));
    Bump b{ctx->scratch5.as<char>()};
    B2N_TRY(eq_layout(ctx, N, R, M, b, W));
    std::vector<int> offs(R + 1);
    for (int r = 0; r <= R; r++) offs[r] = (int)(r * M);
    B2N_CUDA(ctx, cudaMemcpyAsync(W.offs, offs.data(), (R + 1) * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    B2N_CUDA(ctx, cudaMemsetAsync(W.bad, 0, sizeof(int), ctx->stream));
    *bad = W.bad;
    EqArgs A{w, si, sr, N, M, R, seed, chain0, x, k, W.c, W.ws, W.u, W.bad, wsum, counts, W.draw, W.keys_in,
             W.vals_in, W.vals_out, idx, xout};
    cumsum_kernel<<<(R + EQ_CS_THREADS - 1) / EQ_CS_THREADS, EQ_CS_THREADS, 0, ctx->stream>>>(A);
    B2N_LAUNCH_CHECK(ctx);
    if (counts) {
        counts_kernel<<<eq_grid(N * R), EQ_THREADS, 0, ctx->stream>>>(A);
        B2N_LAUNCH_CHECK(ctx);
    }
    draw_kernel<<<eq_grid(M * R), EQ_THREADS, 0, ctx->stream>>>(A);
    B2N_LAUNCH_CHECK(ctx);
    B2N_CUDA(ctx, (cub::DeviceSegmentedRadixSort::SortPairs(W.cub_tmp, W.cub_bytes, W.keys_in, W.keys_out, W.vals_in,
                                                            W.vals_out, (int)(R * M), R, W.offs, W.offs + 1, 0,
                                                            EQ_KEY_BITS, ctx->stream)));
    ctx->launches++;
    gather_kernel<<<eq_grid(M * R), EQ_THREADS, 0, ctx->stream>>>(A);
    B2N_LAUNCH_CHECK(ctx);
    return B2N_OK;
}

// The end of an entry point: the outputs back to the caller, then the weight check read (this synchronises).
template <int K>
int eq_finish(b2n_ctx* ctx, const B2nOutStage<K>& O, const int* bad) {
    B2N_TRY(O.done(ctx));
    int h = 0;
    B2N_CUDA(ctx, b2n_copy_sync(ctx, &h, bad, sizeof(int), cudaMemcpyDeviceToHost));
    if (h) return b2n_fail(ctx, B2N_ERR_ARG, "a weight is negative, NaN or inf, or a weight vector sums to 0 or inf");
    return B2N_OK;
}

int eq_check(int64_t N, int R, int64_t M, const double* x, int k, const int32_t* idx, const double* xout) {
    if (N < 1 || N > INT32_MAX || M < 1 || M > INT32_MAX || R < 1 || R > 65535 || !idx || k < 0) return B2N_ERR_ARG;
    if ((int64_t)R * M > INT32_MAX) return B2N_ERR_ARG;
    if ((xout || k > 0) && (!x || k < 1)) return B2N_ERR_ARG;
    return B2N_OK;
}

}  // namespace

extern "C" int b2n_resample_equal(b2n_ctx* ctx, const double* w, int64_t N, int32_t R, int64_t M, uint64_t seed,
                                  uint64_t chain0, const double* x, int32_t k, int32_t* idx, int32_t* counts,
                                  double* wsum, double* xout) {
    if (!ctx) return B2N_ERR_ARG;
    B2N_TRY(b2n_refuse_reweight(ctx, "b2n_resample_equal"));
    if (!w) return B2N_ERR_ARG;
    B2N_TRY(eq_check(N, R, M, x, k, idx, xout));
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    const void* p;
    B2N_TRY(b2n_in(ctx, ctx->in0, w, (size_t)R * N * sizeof(double), &p));
    const double* wd = (const double*)p;
    B2N_TRY(b2n_in(ctx, ctx->scratch4, xout ? x : nullptr, (size_t)N * k * sizeof(double), &p));
    const double* xd = (const double*)p;
    const size_t rm = (size_t)R * M;
    B2nOutStage<4> O{{idx, counts, wsum, xout}, {rm * 4, (size_t)R * N * 4, (size_t)R * 8, rm * k * 8}};
    B2N_TRY(O.bind(ctx));
    const int* bad;
    B2N_TIME_BEGIN(ctx);
    B2N_TRY(eq_launch(ctx, wd, 1, N, N, R, M, seed, chain0, xd, k, (int32_t*)O.dev[0], (int32_t*)O.dev[1],
                      (double*)O.dev[2], (double*)O.dev[3], &bad));
    B2N_TIME_END(ctx);
    return eq_finish(ctx, O, bad);
}

namespace {
// The realisation entries: x staged, outputs staged; `produce` stages the record, starts the timer and enqueues the
// producer that fills the N x R weights and the summaries.
template <class Producer>
int eq_realisations(b2n_ctx* ctx, int64_t N, int32_t R, uint64_t seed, uint64_t chain0, int64_t M, const double* x,
                    int32_t k, double* logz, double* logzerr, double* h, double* kld, int32_t* idx, int32_t* counts,
                    double* wsum, double* xout, Producer produce) {
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    const void* p;
    B2N_TRY(b2n_in(ctx, ctx->scratch4, xout ? x : nullptr, (size_t)N * k * sizeof(double), &p));
    const double* xd = (const double*)p;
    B2N_CUDA(ctx, ctx->work0.ensure((size_t)N * R * sizeof(double)));
    double* Wt = ctx->work0.as<double>();
    const size_t rb = (size_t)R * sizeof(double), rm = (size_t)R * M;
    B2nOutStage<8> O{{logz, logzerr, h, kld, idx, counts, wsum, xout},
                     {rb, rb, rb, rb, rm * 4, (size_t)R * N * 4, rb, rm * k * 8}};
    B2N_TRY(O.bind(ctx));
    double* const sum[4] = {(double*)O.dev[0], (double*)O.dev[1], (double*)O.dev[2], (double*)O.dev[3]};
    B2N_TRY(produce(sum, Wt));
    const int* bad;
    B2N_TRY(eq_launch(ctx, Wt, R, 1, N, R, M, seed, B2N_EQUAL_CHAIN0 + chain0, xd, k, (int32_t*)O.dev[4],
                      (int32_t*)O.dev[5], (double*)O.dev[6], (double*)O.dev[7], &bad));
    B2N_TIME_END(ctx);
    return eq_finish(ctx, O, bad);
}
}  // namespace

extern "C" int b2n_jitter_equal(b2n_ctx* ctx, const double* logl, const int64_t* samples_n, int64_t N,
                                const double* logwt_ref, double logz_ref, int32_t approx, int32_t R, uint64_t seed,
                                uint64_t chain0, int64_t M, const double* x, int32_t k, double* logz, double* logzerr,
                                double* h, double* kld, int32_t* idx, int32_t* counts, double* wsum, double* xout) {
    if (!ctx) return B2N_ERR_ARG;
    const double* logrwt;
    B2N_TRY(b2n_take_reweight(ctx, N, &logrwt));
    if (!logl || !samples_n || !logwt_ref) return B2N_ERR_ARG;
    B2N_TRY(eq_check(N, R, M, x, k, idx, xout));
    return eq_realisations(ctx, N, R, seed, chain0, M, x, k, logz, logzerr, h, kld, idx, counts, wsum, xout,
                           [&](double* const sum[4], double* W) {
                               const double* w2;
                               const double* wref;
                               int64_t nw2;
                               return b2n_jitter_produce(ctx, logl, samples_n, N, logwt_ref, logz_ref, approx, R, seed,
                                                         chain0, logrwt, sum, nullptr, W, &w2, &nw2, &wref);
                           });
}

extern "C" int b2n_resample_equal_runs(b2n_ctx* ctx, const double* logl, const int32_t* strand, int64_t N, int32_t S,
                                       const uint8_t* base, const int64_t* piece_ptr, const int32_t* piece_strand,
                                       const uint8_t* end, const double* logwt_ref, double logz_ref, int32_t R,
                                       uint64_t seed, uint64_t chain0, int64_t M, const double* x, int32_t k,
                                       double* logz, double* logzerr, double* h, double* kld, int32_t* idx,
                                       int32_t* counts, double* wsum, double* xout) {
    if (!ctx) return B2N_ERR_ARG;
    const double* logrwt;
    B2N_TRY(b2n_take_reweight(ctx, N, &logrwt));
    if (!logl || !strand || !base || !piece_ptr || !logwt_ref || S < 1) return B2N_ERR_ARG;
    B2N_TRY(eq_check(N, R, M, x, k, idx, xout));
    return eq_realisations(ctx, N, R, seed, chain0, M, x, k, logz, logzerr, h, kld, idx, counts, wsum, xout,
                           [&](double* const sum[4], double* W) {
                               const double* w2;
                               const double* wref;
                               int64_t nw2;
                               return b2n_resample_produce(ctx, logl, strand, N, S, base, piece_ptr, piece_strand, end,
                                                           logwt_ref, logz_ref, R, seed, chain0, logrwt, sum, nullptr,
                                                           W, &w2, &nw2, &wref);
                           });
}

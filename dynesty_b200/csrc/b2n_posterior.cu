// b2n_posterior.cu -- posterior means, covariances and weighted quantiles of R weight vectors over one set of N
// samples (the reference's mean_and_cov / quantile, utils.py:1081-1117, 1196-1233), in FP64; contract and
// semantics: include/b200nest.h (b2n_weighted_stats, b2n_jitter_posterior, b2n_resample_posterior), DESIGN.md 15.3.
//
// The weights live on the device sample-major, W[i * R + r] (N x R): the producers (b2n_jitter.cu pass 2,
// b2n_resample.cu sweep 2) write them there, so that the quantile scans read 32 realisations of one sample per warp
// load.  A sample absent from a realisation (a resampled strand drawn 0 times) has W = -0.0: the sign bit is the node
// membership flag, and -0.0 adds nothing to the moments.
//
//   shift_kernel          (ceil(n/32))                 c = the record's own weighted mean (realisation entries only)
//   moments_gemm_kernel   (R/64, P/64, N/PM_KCH)       DMMA m8n8k4: W^T times [1, x - c, triu((x - c)(x - c)^T)],
//                                                      the feature tile built in shared memory from a tile of x;
//                                                      one partial per K chunk
//   moments_finish_kernel (R)                          the chunks summed in order, mean and the mirrored covariance
//   sort_keys_kernel + CUB segmented radix sort        every coordinate sorted once (stable: ties keep record order)
//   quant_chunk_kernel    (N/QC, R/32, n)              per chunk of a sorted order: sum of the present weights and
//                                                      the sum before the chunk's last present node
//   quant_lookup_kernel   (N/QC, R/32, n)              the cdf of the chunk's nodes; each quantile is written by the
//                                                      chunk holding the last node whose cdf is <= q
// Every split is over N in pieces whose bounds depend on N only, every reduction runs in a fixed order and realisation
// r reads only its own column of W: no float atomics, the same bits every call, and row r does not depend on R.
//
// The realisation entries take their weights from the producers b2n_jitter_produce / b2n_resample_produce
// (b2n_common.cuh); every entry point stages its outputs (summaries, mean, cov, quantiles) through B2nOutStage.
#include "b2n_device.cuh"

#include <cub/device/device_segmented_radix_sort.cuh>

#include <math.h>
#include <vector>

namespace {

constexpr int PM_BM = 64;           // realisations per CTA tile
constexpr int PM_BN = 64;           // moment columns per CTA tile
constexpr int PM_BK = 16;           // samples per shared-memory stage
constexpr int PM_LDS = PM_BM + 4;   // row stride of the A / B stages (== 4 mod 16: conflict-free fragment loads)
constexpr int PM_KCH = 2048;        // samples per K chunk (one partial each)
constexpr int PM_THREADS = 128;     // 4 warps, 2 x 2, each 32 x 32
constexpr int QC = 1024;            // samples per quantile chunk
constexpr int PM_NMAX = 1024;       // dimensions

__device__ __forceinline__ void dmma(double (&d)[2], double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(d[0]), "+d"(d[1])
                 : "d"(a), "d"(b));
}

struct MArgs {
    const double* W;        // N x R
    const double* x;        // N x n
    const double* c;        // n
    const int2* feat;       // P: (-1, -1) the constant, (j, -1) x_j - c_j, (a, b) (x_a - c_a)(x_b - c_b), a <= b
    int64_t N;
    int R, n, P;
    double* part;           // nchunk x R x P
};

// Partial moments of chunk blockIdx.z: part[z][r][p] = sum over its samples of W[i][r] F[i][p].
__global__ void __launch_bounds__(PM_THREADS) moments_gemm_kernel(MArgs A) {
    extern __shared__ double sm[];
    double* As = sm;                        // [PM_BK][PM_LDS]: As[k][m] = W of sample k0 + k, realisation m0 + m
    double* Bs = As + PM_BK * PM_LDS;       // [PM_BK][PM_LDS]: Bs[k][p] = feature p0 + p of sample k0 + k
    double* d = Bs + PM_BK * PM_LDS;        // [PM_BK][n]: x - c
    __shared__ int2 fp[PM_BN];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
    const int m0 = blockIdx.x * PM_BM, p0 = blockIdx.y * PM_BN, n = A.n, R = A.R;
    const int64_t kb = (int64_t)blockIdx.z * PM_KCH, ke = min(A.N, kb + PM_KCH);
    for (int p = tid; p < PM_BN; p += PM_THREADS) fp[p] = p0 + p < A.P ? A.feat[p0 + p] : make_int2(-2, -2);
    double acc[4][4][2];
#pragma unroll
    for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) acc[a][b][0] = acc[a][b][1] = 0.0;
    for (int64_t k0 = kb; k0 < ke; k0 += PM_BK) {
        for (int e = tid; e < PM_BK * PM_BM; e += PM_THREADS) {
            const int k = e / PM_BM, m = e % PM_BM;
            const int64_t i = k0 + k;
            As[k * PM_LDS + m] = (i < ke && m0 + m < R) ? A.W[i * R + m0 + m] : 0.0;
        }
        for (int e = tid; e < PM_BK * n; e += PM_THREADS) {
            const int k = e / n, j = e - k * n;
            const int64_t i = k0 + k;
            d[e] = i < ke ? A.x[i * n + j] - A.c[j] : 0.0;
        }
        __syncthreads();
        for (int e = tid; e < PM_BK * PM_BN; e += PM_THREADS) {
            const int k = e / PM_BN, p = e % PM_BN;
            const int2 f = fp[p];
            const double* dk = d + k * n;
            Bs[k * PM_LDS + p] = f.x == -1 ? 1.0 : f.x < 0 ? 0.0 : (f.y < 0 ? dk[f.x] : dk[f.x] * dk[f.y]);
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < PM_BK; kk += 4) {
            const int row = (kk + (lane & 3)) * PM_LDS + (lane >> 2);
            double a[4], b[4];
#pragma unroll
            for (int t = 0; t < 4; t++) {
                a[t] = As[row + wm + t * 8];
                b[t] = Bs[row + wn + t * 8];
            }
#pragma unroll
            for (int ti = 0; ti < 4; ti++)
#pragma unroll
                for (int tj = 0; tj < 4; tj++) dmma(acc[ti][tj], a[ti], b[tj]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int ti = 0; ti < 4; ti++)
#pragma unroll
        for (int tj = 0; tj < 4; tj++)
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int r = m0 + wm + ti * 8 + (lane >> 2), p = p0 + wn + tj * 8 + 2 * (lane & 3) + h;
                if (r < R && p < A.P) A.part[((size_t)blockIdx.z * R + r) * A.P + p] = acc[ti][tj][h];
            }
}

struct FArgs {
    const double* part;     // nchunk x R x P
    const double* w2;       // R x nw2
    const double* c;        // n
    const int2* feat;
    int nchunk, R, n, P;
    int64_t nw2;
    double* mean;           // R x n, may be NULL
    double* cov;            // R x n x n, may be NULL
};

// mean = c + M1 / M0, cov = M0 / (M0^2 - w2sum) (M2 - M1 M1^T / M0), the chunk partials summed in chunk order.
__global__ void __launch_bounds__(256) moments_finish_kernel(FArgs A) {
    extern __shared__ double m1[];          // n
    __shared__ double s_m0, s_w2;
    const int r = blockIdx.x, n = A.n;
    auto sum = [&](int p) {
        double s = 0.0;
        for (int ch = 0; ch < A.nchunk; ch++) s += A.part[((size_t)ch * A.R + r) * A.P + p];
        return s;
    };
    if (threadIdx.x == 0) {
        s_m0 = sum(0);
        double w2 = 0.0;
        for (int64_t s = 0; s < A.nw2; s++) w2 += A.w2[r * A.nw2 + s];
        s_w2 = w2;
    }
    for (int j = threadIdx.x; j < n; j += blockDim.x) m1[j] = sum(1 + j);
    __syncthreads();
    const double m0 = s_m0;
    if (A.mean)
        for (int j = threadIdx.x; j < n; j += blockDim.x) A.mean[(size_t)r * n + j] = A.c[j] + m1[j] / m0;
    if (!A.cov) return;
    const double f = m0 / (m0 * m0 - s_w2);
    for (int t = threadIdx.x; t < A.P - 1 - n; t += blockDim.x) {
        const int2 ab = A.feat[1 + n + t];
        const double v = f * (sum(1 + n + t) - m1[ab.x] * m1[ab.y] / m0);
        A.cov[((size_t)r * n + ab.x) * n + ab.y] = v;
        A.cov[((size_t)r * n + ab.y) * n + ab.x] = v;
    }
}

// w2[r] = sum of W[i][r]^2 (b2n_weighted_stats): warp g of the CTA sums samples [g N / 8, (g + 1) N / 8) in order.
__global__ void __launch_bounds__(256) wsq_kernel(const double* __restrict__ W, int64_t N, int R, double* w2) {
    __shared__ double part[8][32];
    const int lane = threadIdx.x & 31, g = threadIdx.x >> 5, r = blockIdx.x * 32 + lane;
    double s = 0.0;
    if (r < R)
        for (int64_t i = N * g / 8; i < N * (g + 1) / 8; i++) {
            const double w = W[i * R + r];
            s += w * w;
        }
    part[g][lane] = s;
    __syncthreads();
    if (g == 0 && r < R) {
        double t = 0.0;
        for (int k = 0; k < 8; k++) t += part[k][lane];
        w2[r] = t;
    }
}

// c = sum_i exp(logwt_i - max) x_i / sum_i exp(logwt_i - max): warp g of the CTA sums samples [g N / 16, ..) in order.
__global__ void __launch_bounds__(512) shift_kernel(const double* __restrict__ logwt, const double* __restrict__ x,
                                                    int64_t N, int n, double* c) {
    __shared__ double part[16][33], wpart[16][33], red[16];
    const int lane = threadIdx.x & 31, g = threadIdx.x >> 5, j = blockIdx.x * 32 + lane;
    double mx = -INFINITY;
    for (int64_t i = threadIdx.x; i < N; i += blockDim.x) mx = fmax(mx, logwt[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(B2N_FULL, mx, o));
    if (lane == 0) red[g] = mx;
    __syncthreads();
    mx = red[0];
    for (int k = 1; k < 16; k++) mx = fmax(mx, red[k]);
    double s = 0.0, e = 0.0;
#pragma unroll 1
    for (int64_t i = N * g / 16; i < N * (g + 1) / 16; i++) {
        const double wi = exp(logwt[i] - mx);
        e += wi;
        if (j < n) s += wi * x[i * n + j];
    }
    part[g][lane] = s;
    wpart[g][lane] = e;
    __syncthreads();
    if (g == 0 && j < n) {
        double ts = 0.0, te = 0.0;
        for (int k = 0; k < 16; k++) { ts += part[k][lane]; te += wpart[k][lane]; }
        c[j] = ts / te;
    }
}

// W (R x N, b2n_weighted_stats' layout) -> N x R
__global__ void transpose_kernel(const double* __restrict__ w, int64_t N, int R, double* __restrict__ W) {
    __shared__ double t[32][33];
    const int64_t i0 = (int64_t)blockIdx.x * 32;
    const int r0 = blockIdx.y * 32;
    for (int y = threadIdx.y; y < 32; y += blockDim.y) {
        const int r = r0 + y;
        const int64_t i = i0 + threadIdx.x;
        if (r < R && i < N) t[y][threadIdx.x] = w[(size_t)r * N + i];
    }
    __syncthreads();
    for (int y = threadIdx.y; y < 32; y += blockDim.y) {
        const int64_t i = i0 + y;
        const int r = r0 + threadIdx.x;
        if (r < R && i < N) W[i * R + r] = t[threadIdx.x][y];
    }
}

// keys[j][i] = x[i][j] (+ 0.0: -0.0 sorts as 0.0, as numpy's argsort has it), vals[j][i] = i
__global__ void sort_keys_kernel(const double* __restrict__ x, int64_t N, int n, double* keys, int32_t* vals) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= N * n) return;
    const int j = (int)(e / N);
    const int64_t i = e - (int64_t)j * N;
    keys[e] = x[i * n + j] + 0.0;
    vals[e] = (int32_t)i;
}

struct QArgs {
    const double* W;        // N x R
    const double* xs;       // n x N: every coordinate sorted
    const int32_t* perm;    // n x N: the record index of every sorted position
    const double* q;        // nq
    int64_t N;
    int R, n, nq, nqc;
    double* st;             // n x R x nqc x 2: chunk sum, sum before the chunk's last present node (-1: none)
    double* quant;          // R x n x nq
};

// One warp per (chunk, 32 realisations, coordinate); lane = realisation.
__global__ void __launch_bounds__(32) quant_chunk_kernel(QArgs A) {
    const int c = blockIdx.x, r = blockIdx.y * 32 + threadIdx.x, j = blockIdx.z;
    if (r >= A.R) return;
    const int32_t* perm = A.perm + (size_t)j * A.N;
    const int64_t k1 = min(A.N, (int64_t)(c + 1) * QC);
    double s = 0.0, before = -1.0;
    for (int64_t k = (int64_t)c * QC; k < k1; k++) {
        const double w = A.W[(int64_t)perm[k] * A.R + r];
        if (signbit(w)) continue;
        before = s;
        s += w;
    }
    double* st = A.st + (((size_t)j * A.R + r) * A.nqc + c) * 2;
    st[0] = s;
    st[1] = before;
}

// Node k of the sorted order (present ones only) has cum_k = fl(prefix(chunk) + local sum before k), prefix = the
// chunk sums before it added in order, and C_k = cum_k / S with S = cum of the last node: the same bits whichever
// chunk computes them, and non-decreasing, so every q has exactly one last node p with C_p <= q and one writer.
__global__ void __launch_bounds__(32) quant_lookup_kernel(QArgs A) {
    const int c = blockIdx.x, r = blockIdx.y * 32 + threadIdx.x, j = blockIdx.z;
    if (r >= A.R) return;
    const double* st = A.st + ((size_t)j * A.R + r) * A.nqc * 2;
    double pre = 0.0, mypre = 0.0, S = NAN;
    for (int cc = 0; cc < A.nqc; cc++) {
        if (cc == c) mypre = pre;
        if (st[2 * cc + 1] >= 0.0) S = pre + st[2 * cc + 1];
        pre += st[2 * cc];
    }
    const int32_t* perm = A.perm + (size_t)j * A.N;
    const double* xs = A.xs + (size_t)j * A.N;
    double* out = A.quant + ((size_t)r * A.n + j) * A.nq;
    // q in [C_p, C_k): x_p at q == C_p, else np.interp's line from node p to node k
    auto emit = [&](double xp, double Cp, double xk, double Ck) {
        for (int t = 0; t < A.nq; t++) {
            const double q = A.q[t];
            if (Cp <= q && q < Ck) out[t] = q == Cp ? xp : (xk - xp) / (Ck - Cp) * (q - Cp) + xp;
        }
    };
    const int64_t k1 = min(A.N, (int64_t)(c + 1) * QC);
    double s = 0.0, xp = 0.0, Cp = 0.0;
    bool have = false;
    for (int64_t k = (int64_t)c * QC; k < k1; k++) {
        const double w = A.W[(int64_t)perm[k] * A.R + r];
        if (signbit(w)) continue;
        const double C = (mypre + s) / S, xk = xs[k];
        if (have) emit(xp, Cp, xk, C);
        xp = xk; Cp = C; have = true;
        s += w;
    }
    if (!have) return;
    for (int64_t k = k1; k < A.N; k++) {        // the next present node, in a later chunk
        if (signbit(A.W[(int64_t)perm[k] * A.R + r])) continue;
        emit(xp, Cp, xs[k], (mypre + s) / S);
        return;
    }
    for (int t = 0; t < A.nq; t++)              // the last node
        if (Cp <= A.q[t]) out[t] = xp;
}

struct PostJob {
    int64_t N;
    int n, R, nq;
    const double* W;        // device, N x R
    const double* w2;       // device, R x nw2
    int64_t nw2;
    const double* x;        // device, N x n
    const double* c;        // device, n
    const double* q;        // device, nq
    double *mean, *cov, *quant;     // device, each may be NULL
};

// Device workspace of post_launch: carved from ctx->scratch5 (host data copied in first).
struct PostWork {
    int2* feat;
    double* part;
    double *keys_in, *keys_out;
    int32_t *vals_in, *vals_out;
    int* offs;
    void* cub_tmp;
    size_t cub_bytes;
    double* st;
};

int post_layout(b2n_ctx* ctx, int64_t N, int n, int R, bool moments, bool quant, Bump& b, PostWork& w) {
    const int P = 1 + n + n * (n + 1) / 2;
    const int64_t nchunk = (N + PM_KCH - 1) / PM_KCH, nqc = (N + QC - 1) / QC;
    memset(&w, 0, sizeof(w));
    if (moments) {
        w.feat = b.take<int2>(P);
        w.part = b.take<double>((size_t)nchunk * R * P);
    }
    if (quant) {
        const size_t nn = (size_t)N * n;
        w.keys_in = b.take<double>(nn);
        w.keys_out = b.take<double>(nn);
        w.vals_in = b.take<int32_t>(nn);
        w.vals_out = b.take<int32_t>(nn);
        w.offs = b.take<int>(n + 1);
        B2N_CUDA(ctx, (cub::DeviceSegmentedRadixSort::SortPairs(nullptr, w.cub_bytes, w.keys_in, w.keys_out, w.vals_in,
                                                                w.vals_out, (int)nn, n, w.offs, w.offs + 1, 0, 64,
                                                                ctx->stream)));
        w.cub_tmp = b.take<char>(w.cub_bytes);
        w.st = b.take<double>((size_t)n * R * nqc * 2);
    }
    return B2N_OK;
}

// The stats of one job on the stream: moments (2 launches), sort (1 + CUB's), quantiles (2 + a memset).
int post_launch(b2n_ctx* ctx, const PostJob& J) {
    const bool moments = J.mean || J.cov, quant = J.quant && J.nq > 0;
    const int n = J.n, P = 1 + n + n * (n + 1) / 2;
    const int64_t N = J.N, nchunk = (N + PM_KCH - 1) / PM_KCH, nqc = (N + QC - 1) / QC;
    Bump b0{nullptr};
    PostWork w;
    B2N_TRY(post_layout(ctx, N, n, J.R, moments, quant, b0, w));
    B2N_CUDA(ctx, ctx->scratch5.ensure(b0.off + 256));
    Bump b{ctx->scratch5.as<char>()};
    B2N_TRY(post_layout(ctx, N, n, J.R, moments, quant, b, w));
    if (moments) {
        std::vector<int2> feat;
        feat.reserve(P);
        feat.push_back(make_int2(-1, -1));
        for (int j = 0; j < n; j++) feat.push_back(make_int2(j, -1));
        for (int a = 0; a < n; a++)
            for (int c = a; c < n; c++) feat.push_back(make_int2(a, c));
        B2N_CUDA(ctx, cudaMemcpyAsync(w.feat, feat.data(), P * sizeof(int2), cudaMemcpyHostToDevice, ctx->stream));
        MArgs M{J.W, J.x, J.c, w.feat, N, J.R, n, P, w.part};
        const size_t smem = (size_t)(2 * PM_BK * PM_LDS + PM_BK * n) * sizeof(double);
        B2N_TRY(b2n_func_smem(ctx, (const void*)moments_gemm_kernel, smem));
        const dim3 grid((unsigned)((J.R + PM_BM - 1) / PM_BM), (unsigned)((P + PM_BN - 1) / PM_BN), (unsigned)nchunk);
        moments_gemm_kernel<<<grid, PM_THREADS, smem, ctx->stream>>>(M);
        B2N_LAUNCH_CHECK(ctx);
        FArgs F{w.part, J.w2, J.c, w.feat, (int)nchunk, J.R, n, P, J.nw2, J.mean, J.cov};
        moments_finish_kernel<<<J.R, 256, n * sizeof(double), ctx->stream>>>(F);
        B2N_LAUNCH_CHECK(ctx);
    }
    if (quant) {
        std::vector<int> offs(n + 1);
        for (int j = 0; j <= n; j++) offs[j] = (int)(j * N);
        B2N_CUDA(ctx, cudaMemcpyAsync(w.offs, offs.data(), (n + 1) * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
        const int64_t nn = N * n;
        sort_keys_kernel<<<(unsigned)((nn + 255) / 256), 256, 0, ctx->stream>>>(J.x, N, n, w.keys_in, w.vals_in);
        B2N_LAUNCH_CHECK(ctx);
        B2N_CUDA(ctx, (cub::DeviceSegmentedRadixSort::SortPairs(w.cub_tmp, w.cub_bytes, w.keys_in, w.keys_out,
                                                                w.vals_in, w.vals_out, (int)nn, n, w.offs, w.offs + 1,
                                                                0, 64, ctx->stream)));
        ctx->launches++;
        B2N_CUDA(ctx, cudaMemsetAsync(J.quant, 0xff, (size_t)J.R * n * J.nq * sizeof(double), ctx->stream));   // NaN
        QArgs Q{J.W, w.keys_out, w.vals_out, J.q, N, J.R, n, J.nq, (int)nqc, w.st, J.quant};
        const dim3 grid((unsigned)nqc, (unsigned)((J.R + 31) / 32), (unsigned)n);
        quant_chunk_kernel<<<grid, 32, 0, ctx->stream>>>(Q);
        B2N_LAUNCH_CHECK(ctx);
        quant_lookup_kernel<<<grid, 32, 0, ctx->stream>>>(Q);
        B2N_LAUNCH_CHECK(ctx);
    }
    return B2N_OK;
}

int post_check(int64_t N, int n, int R, const double* x, int nq, const double* q, double* quant) {
    if (N < 1 || n < 1 || n > PM_NMAX || R < 1 || R > 65535 || !x || nq < 0) return B2N_ERR_ARG;
    if (quant && (nq < 1 || !q)) return B2N_ERR_ARG;
    if (N * (int64_t)n > INT32_MAX) return B2N_ERR_ARG;
    return B2N_OK;
}

}  // namespace

extern "C" int b2n_weighted_stats(b2n_ctx* ctx, const double* x, int64_t N, int32_t n, const double* w, int32_t R,
                                  const double* shift, const double* q, int32_t nq, double* mean, double* cov,
                                  double* quant) {
    if (!ctx) return B2N_ERR_ARG;
    B2N_TRY(b2n_refuse_reweight(ctx, "b2n_weighted_stats"));
    if (!w || !shift) return B2N_ERR_ARG;
    B2N_TRY(post_check(N, n, R, x, nq, q, quant));
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    PostJob J;
    memset(&J, 0, sizeof(J));
    J.N = N; J.n = n; J.R = R; J.nq = quant ? nq : 0;
    const void* p;
    B2N_TRY(b2n_in(ctx, ctx->scratch4, x, (size_t)N * n * sizeof(double), &p));
    J.x = (const double*)p;
    B2N_TRY(b2n_in(ctx, ctx->in0, w, (size_t)R * N * sizeof(double), &p));
    const double* wr = (const double*)p;
    B2N_TRY(b2n_in(ctx, ctx->in1, shift, (size_t)n * sizeof(double), &p));
    J.c = (const double*)p;
    B2N_TRY(b2n_in(ctx, ctx->in2, quant ? q : nullptr, (size_t)nq * sizeof(double), &p));
    J.q = (const double*)p;
    B2N_CUDA(ctx, ctx->work0.ensure(((size_t)N * R + R) * sizeof(double)));
    double* Wt = ctx->work0.as<double>();
    double* w2 = Wt + (size_t)N * R;
    J.W = Wt; J.w2 = w2; J.nw2 = 1;
    const size_t rn = (size_t)R * n * sizeof(double);
    B2nOutStage<3> O{{mean, cov, quant}, {rn, rn * n, rn * nq}};
    B2N_TRY(O.bind(ctx));
    J.mean = (double*)O.dev[0]; J.cov = (double*)O.dev[1]; J.quant = (double*)O.dev[2];

    B2N_TIME_BEGIN(ctx);
    transpose_kernel<<<dim3((unsigned)((N + 31) / 32), (unsigned)((R + 31) / 32)), dim3(32, 8), 0, ctx->stream>>>(
        wr, N, R, Wt);
    B2N_LAUNCH_CHECK(ctx);
    wsq_kernel<<<(R + 31) / 32, 256, 0, ctx->stream>>>(Wt, N, R, w2);
    B2N_LAUNCH_CHECK(ctx);
    B2N_TRY(post_launch(ctx, J));
    B2N_TIME_END(ctx);

    B2N_TRY(O.done(ctx));
    return b2n_finish(ctx);
}

namespace {
// The common part of the realisation entries: x staged, outputs staged, shift from logwt_ref; `produce` stages the
// record, starts the timer and enqueues the producer that fills J.W / J.w2 / J.nw2 and the summaries, and returns the
// record's logwt on the device.
template <class Producer>
int post_realisations(b2n_ctx* ctx, int64_t N, const double* x, int32_t n, int32_t R, const double* q, int32_t nq,
                      double* logz, double* logzerr, double* h, double* kld, double* mean, double* cov, double* quant,
                      Producer produce) {
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    PostJob J;
    memset(&J, 0, sizeof(J));
    J.N = N; J.n = n; J.R = R; J.nq = quant ? nq : 0;
    const void* p;
    B2N_TRY(b2n_in(ctx, ctx->scratch4, x, (size_t)N * n * sizeof(double), &p));
    J.x = (const double*)p;
    // the shift and q after the x stage, in work0 behind W
    B2N_CUDA(ctx, ctx->work0.ensure(((size_t)N * R + n + (size_t)(quant ? nq : 0)) * sizeof(double)));
    double* Wt = ctx->work0.as<double>();
    double* c = Wt + (size_t)N * R;
    J.W = Wt; J.c = c;
    if (quant) {
        if (ctx->ptr_mode == B2N_PTR_DEVICE) J.q = q;
        else {
            B2N_CUDA(ctx, cudaMemcpyAsync(c + n, q, nq * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
            J.q = c + n;
        }
    }
    const size_t rb = (size_t)R * sizeof(double), rn = rb * n;
    B2nOutStage<7> O{{logz, logzerr, h, kld, mean, cov, quant}, {rb, rb, rb, rb, rn, rn * n, rn * nq}};
    B2N_TRY(O.bind(ctx));
    double* const sum[4] = {(double*)O.dev[0], (double*)O.dev[1], (double*)O.dev[2], (double*)O.dev[3]};
    J.mean = (double*)O.dev[4]; J.cov = (double*)O.dev[5]; J.quant = (double*)O.dev[6];

    const double* wref = nullptr;
    B2N_TRY(produce(sum, Wt, &J.w2, &J.nw2, &wref));
    shift_kernel<<<(n + 31) / 32, 512, 0, ctx->stream>>>(wref, J.x, N, n, c);
    B2N_LAUNCH_CHECK(ctx);
    B2N_TRY(post_launch(ctx, J));
    B2N_TIME_END(ctx);

    B2N_TRY(O.done(ctx));
    return b2n_finish(ctx);
}
}  // namespace

extern "C" int b2n_jitter_posterior(b2n_ctx* ctx, const double* logl, const int64_t* samples_n, int64_t N,
                                    const double* logwt_ref, double logz_ref, int32_t approx, int32_t R, uint64_t seed,
                                    uint64_t chain0, const double* x, int32_t n, const double* q, int32_t nq,
                                    double* logz, double* logzerr, double* h, double* kld, double* mean, double* cov,
                                    double* quant) {
    if (!ctx) return B2N_ERR_ARG;
    const double* logrwt;
    B2N_TRY(b2n_take_reweight(ctx, N, &logrwt));
    if (!logl || !samples_n || !logwt_ref) return B2N_ERR_ARG;
    B2N_TRY(post_check(N, n, R, x, nq, q, quant));
    return post_realisations(ctx, N, x, n, R, q, nq, logz, logzerr, h, kld, mean, cov, quant,
                             [&](double* const sum[4], double* W, const double** w2, int64_t* nw2, const double** wref) {
                                 return b2n_jitter_produce(ctx, logl, samples_n, N, logwt_ref, logz_ref, approx, R,
                                                           seed, chain0, logrwt, sum, nullptr, W, w2, nw2, wref);
                             });
}

extern "C" int b2n_resample_posterior(b2n_ctx* ctx, const double* logl, const int32_t* strand, int64_t N, int32_t S,
                                      const uint8_t* base, const int64_t* piece_ptr, const int32_t* piece_strand,
                                      const uint8_t* end, const double* logwt_ref, double logz_ref, int32_t R,
                                      uint64_t seed, uint64_t chain0, const double* x, int32_t n, const double* q,
                                      int32_t nq, double* logz, double* logzerr, double* h, double* kld, double* mean,
                                      double* cov, double* quant) {
    if (!ctx) return B2N_ERR_ARG;
    const double* logrwt;
    B2N_TRY(b2n_take_reweight(ctx, N, &logrwt));
    if (!logl || !strand || !base || !piece_ptr || !logwt_ref || S < 1) return B2N_ERR_ARG;
    B2N_TRY(post_check(N, n, R, x, nq, q, quant));
    return post_realisations(ctx, N, x, n, R, q, nq, logz, logzerr, h, kld, mean, cov, quant,
                             [&](double* const sum[4], double* W, const double** w2, int64_t* nw2, const double** wref) {
                                 return b2n_resample_produce(ctx, logl, strand, N, S, base, piece_ptr, piece_strand,
                                                             end, logwt_ref, logz_ref, R, seed, chain0, logrwt, sum,
                                                             nullptr, W, w2, nw2, wref);
                             });
}

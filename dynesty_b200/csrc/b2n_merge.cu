// b2n_merge.cu -- merge_runs (utils.py:1817-1900, _merge_two :2045-2225 of the reference): R dead-point records merged
// into one, in FP64 / int64, without atomics (bit-reproducible from call to call).
//
// One primitive, a two-run merge step (_merge_two's walk): every element of side A finds its rank in side B by binary
// search and the reverse.  A's element i lands at i + #{b < a}, B's element j at j + #{a <= b} (the base side first on
// a tie), and each writes its source index, its logl and its live count: its own plus the other side's count at the
// other side's pointer, with _merge_two's low-edge rule (an exhausted side reads as logl = +inf, count 0).
//
//   init      copies the input (logl, n, source index) into both ping-pong buffers
//   step      base group: one launch per level of the pairwise tree, all pairs of the level at once (an odd node is
//             copied); add-on runs: one launch each, onto the accumulated record
//   lnt       ln t per merged sample: ln(n / (n + 1)), or inside a group of equal logl whose first point has count n,
//             ln((n - k) / (n - k + 1)) for its k-th point (the reference's plateau mode)
//   then the passes of b2n_jitter.cu in their deterministic mode (b2n_integrate_lnt): logvol, logwt, logz, logzvar, h.
//
// The node tables of every launch are built on the host from run_ptr / nbase / lowedge and uploaded once, so the
// launches follow each other on the stream without a host round trip.  The f64 outputs are staged through
// B2nOutStage (b2n_common.cuh); perm and samples_n are copied out of the last ping-pong buffer.
#include "b2n_device.cuh"

#include <algorithm>
#include <math.h>
#include <vector>

namespace {

constexpr int MG_BLOCK = 256;

struct MBuf {
    double* logl;
    int64_t* n;
    int64_t* src;
};

// One launch: nn nodes covering [0, off[nn]); nodes (0, 1), (2, 3), .. merge, an odd last node is copied.
struct MStep {
    const int64_t* off;      // nn + 1
    const double* lowedge;   // nn
    int nn;
};

__device__ __forceinline__ int64_t merged_count(double lb, int64_t nb, double ln, int64_t nn, double eb, double en) {
    if (lb > en && ln > eb) return nb + nn;      // both runs past the other's low edge
    if (lb <= en) return nb;                      // the base side is below the new run's low edge
    return nn;
}

// #{x[0, len) < v} (strict) or #{x[0, len) <= v}; x ascending
template <bool STRICT>
__device__ __forceinline__ int64_t rank_in(const double* __restrict__ x, int64_t len, double v) {
    int64_t lo = 0, hi = len;
    while (lo < hi) {
        const int64_t mid = lo + ((hi - lo) >> 1);
        if (STRICT ? x[mid] < v : x[mid] <= v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(MG_BLOCK) merge_init_kernel(const double* __restrict__ logl,
                                                              const int64_t* __restrict__ n, int64_t N, MBuf b0,
                                                              MBuf b1) {
    const int64_t g = (int64_t)blockIdx.x * MG_BLOCK + threadIdx.x;
    if (g >= N) return;
    const double l = logl[g];
    const int64_t c = n[g];
    b0.logl[g] = l; b0.n[g] = c; b0.src[g] = g;
    b1.logl[g] = l; b1.n[g] = c; b1.src[g] = g;
}

__global__ void __launch_bounds__(MG_BLOCK) merge_step_kernel(MBuf in, MBuf out, MStep st) {
    const int64_t g = (int64_t)blockIdx.x * MG_BLOCK + threadIdx.x;
    if (g >= st.off[st.nn]) return;
    int lo = 0, hi = st.nn;                        // the node k with off[k] <= g < off[k + 1]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (st.off[mid] <= g) lo = mid;
        else hi = mid;
    }
    const int k = lo;
    const double l = in.logl[g];
    const int64_t c = in.n[g];
    if ((k | 1) >= st.nn) {                        // the odd node out
        out.logl[g] = l; out.n[g] = c; out.src[g] = in.src[g];
        return;
    }
    const int a = k & ~1;
    const int64_t oa = st.off[a], ob = st.off[a + 1], oe = st.off[a + 2];
    const double ea = st.lowedge[a], eb = st.lowedge[a + 1];
    int64_t pos, cnt;
    if (k == a) {                                  // base side: the new run's pointer = #{b < l}
        const int64_t j = rank_in<true>(in.logl + ob, oe - ob, l);
        const bool live = ob + j < oe;
        cnt = merged_count(l, c, live ? in.logl[ob + j] : INFINITY, live ? in.n[ob + j] : 0, ea, eb);
        pos = g + j;
    } else {                                       // new side: the base run's pointer = #{a <= l}
        const int64_t i = rank_in<false>(in.logl + oa, ob - oa, l);
        const bool live = oa + i < ob;
        cnt = merged_count(live ? in.logl[oa + i] : INFINITY, live ? in.n[oa + i] : 0, l, c, ea, eb);
        pos = oa + i + (g - ob);
    }
    out.logl[pos] = l; out.n[pos] = cnt; out.src[pos] = in.src[g];
}

// ln t per merged sample (the ln X recursion of _merge_two, :2159-2187): k = distance to the first sample of its group
// of equal logl (a group may span any number of blocks), n = the count of that first sample.
__global__ void __launch_bounds__(MG_BLOCK) merge_lnt_kernel(const double* __restrict__ logl,
                                                             const int64_t* __restrict__ n, int64_t N,
                                                             double* __restrict__ lnt) {
    const int64_t g = (int64_t)blockIdx.x * MG_BLOCK + threadIdx.x;
    if (g >= N) return;
    const double l = logl[g];
    const int64_t s = (g == 0 || logl[g - 1] != l) ? g : rank_in<true>(logl, g, l);
    lnt[g] = -log1p(1.0 / (double)(n[s] - (g - s)));
}

inline unsigned blocks(int64_t n) { return (unsigned)((n + MG_BLOCK - 1) / MG_BLOCK); }

}  // namespace

extern "C" int b2n_merge_runs(b2n_ctx* ctx, const double* logl, const int64_t* samples_n, const int64_t* run_ptr,
                              int32_t R, int32_t nbase, const double* lowedge, int64_t* perm, int64_t* samples_n_out,
                              double* last3, double* logvol, double* logwt, double* logz, double* logzvar, double* h) {
    if (!ctx) return B2N_ERR_ARG;
    B2N_TRY(b2n_refuse_reweight(ctx, "b2n_merge_runs"));
    if (!logl || !samples_n || !run_ptr || R < 1 || nbase < 1 || nbase > R) return B2N_ERR_ARG;
    if (run_ptr[0] != 0) return B2N_ERR_ARG;
    for (int32_t r = 0; r < R; r++) {
        if (run_ptr[r + 1] <= run_ptr[r]) return B2N_ERR_ARG;            // every run holds a sample
        if (lowedge && isnan(lowedge[r])) return B2N_ERR_ARG;
    }
    const int64_t N = run_ptr[R];
    if (N > ((int64_t)UINT32_MAX - 1) * MG_BLOCK) return B2N_ERR_ARG;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));

    // node tables of every launch, concatenated: (offsets, low edges) per step
    std::vector<int64_t> offs;
    std::vector<double> edges;
    std::vector<std::pair<size_t, int>> steps;     // (first offset / edge index, nodes)
    std::vector<int64_t> o(run_ptr, run_ptr + nbase + 1);
    std::vector<double> e(nbase);
    for (int32_t r = 0; r < nbase; r++) e[r] = lowedge ? lowedge[r] : -INFINITY;
    while (e.size() > 1) {
        const int nn = (int)e.size();
        steps.push_back({edges.size(), nn});
        // a step's offsets are nn + 1 long, its edges are padded to that length: one index serves both tables
        offs.insert(offs.end(), o.begin(), o.end());
        edges.insert(edges.end(), e.begin(), e.end());
        edges.push_back(0.0);
        std::vector<int64_t> o2;
        std::vector<double> e2;
        for (int k = 0; k < nn; k += 2) {
            o2.push_back(o[k]);
            e2.push_back(k + 1 < nn ? std::min(e[k], e[k + 1]) : e[k]);
        }
        o2.push_back(o[nn]);
        o.swap(o2);
        e.swap(e2);
    }
    double acc = e[0];
    for (int32_t r = nbase; r < R; r++) {
        const double er = lowedge ? lowedge[r] : -INFINITY;
        steps.push_back({edges.size(), 2});
        offs.insert(offs.end(), {0, run_ptr[r], run_ptr[r + 1]});
        edges.insert(edges.end(), {acc, er, 0.0});
        acc = std::min(acc, er);
    }

    const void* p;
    B2N_TRY(b2n_in(ctx, ctx->in0, logl, (size_t)N * sizeof(double), &p));
    const double* d_logl = (const double*)p;
    B2N_TRY(b2n_in(ctx, ctx->in1, samples_n, (size_t)N * sizeof(int64_t), &p));
    const int64_t* d_n = (const int64_t*)p;
    B2N_TRY(b2n_in_host(ctx, ctx->scratch2, offs.data(), offs.size() * sizeof(int64_t), &p));
    const int64_t* d_offs = (const int64_t*)p;
    B2N_TRY(b2n_in_host(ctx, ctx->scratch3, edges.data(), edges.size() * sizeof(double), &p));
    const double* d_edges = (const double*)p;
    // two ping-pong buffers of (logl, n, src), then ln t
    B2N_CUDA(ctx, ctx->work0.ensure((size_t)N * 3 * 8));
    B2N_CUDA(ctx, ctx->work1.ensure((size_t)N * 4 * 8));
    MBuf b[2];
    for (int k = 0; k < 2; k++) {
        char* w = (char*)(k ? ctx->work1.p : ctx->work0.p);
        b[k] = MBuf{(double*)w, (int64_t*)(w + (size_t)N * 8), (int64_t*)(w + (size_t)N * 16)};
    }
    double* d_lnt = (double*)((char*)ctx->work1.p + (size_t)N * 24);

    const size_t nb = (size_t)N * sizeof(double);
    B2nOutStage<6> O{{last3, logvol, logwt, logz, logzvar, h}, {3 * sizeof(double), nb, nb, nb, nb, nb}};
    B2N_TRY(O.bind(ctx));
    double* fd[6];
    for (int k = 0; k < 6; k++) fd[k] = (double*)O.dev[k];

    B2N_TIME_BEGIN(ctx);
    merge_init_kernel<<<blocks(N), MG_BLOCK, 0, ctx->stream>>>(d_logl, d_n, N, b[0], b[1]);
    B2N_LAUNCH_CHECK(ctx);
    int cur = 0;
    for (const auto& s : steps) {
        const MStep st{d_offs + s.first, d_edges + s.first, s.second};
        merge_step_kernel<<<blocks(offs[s.first + s.second]), MG_BLOCK, 0, ctx->stream>>>(b[cur], b[cur ^ 1], st);
        B2N_LAUNCH_CHECK(ctx);
        cur ^= 1;
    }
    const MBuf m = b[cur];
    merge_lnt_kernel<<<blocks(N), MG_BLOCK, 0, ctx->stream>>>(m.logl, m.n, N, d_lnt);
    B2N_LAUNCH_CHECK(ctx);
    B2N_TRY(b2n_integrate_lnt(ctx, m.logl, d_lnt, nullptr, N, fd[0], fd[1], fd[2], fd[3], fd[4], fd[5]));
    B2N_TIME_END(ctx);

    const cudaMemcpyKind kind = ctx->ptr_mode == B2N_PTR_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    if (perm) B2N_CUDA(ctx, cudaMemcpyAsync(perm, m.src, (size_t)N * sizeof(int64_t), kind, ctx->stream));
    if (samples_n_out) B2N_CUDA(ctx, cudaMemcpyAsync(samples_n_out, m.n, (size_t)N * sizeof(int64_t), kind, ctx->stream));
    B2N_TRY(O.done(ctx));
    return b2n_finish(ctx);
}

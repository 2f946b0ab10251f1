// b2n_multi.cu -- MultiEllipsoid decomposition: level-synchronous version of the
// recursive 2-means split _bounding_ellipsoids (reference bounding.py:1464-1563),
// MultiEllipsoid.update's containment check (:683-685) and the bootstrap expansion
// factor (:1593-1648).
//
// The reference recursion ALWAYS expands both children before applying its two volume
// tests (:1548-1560), so the tree of candidate ellipsoids does not depend on the tests:
// we expand it breadth-first -- all siblings of a level share one k-means launch, one
// partition launch and one batch of bounding-ellipsoid launches -- and then evaluate the
// accept/reject logic bottom-up on the host from the per-node log-volumes.
#include "b2n_bounding.cuh"
#include <cooperative_groups.h>
#include <algorithm>
#include <cmath>
#include <vector>


// ---- root std (ddof = 0) from the raw covariance diagonal: points.std(axis=0) (:1504)
__global__ void root_scale_kernel(NodeArrays na, int node, int count, double* __restrict__ scale) {
    const int n = na.n;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const double v = na.covraw[(size_t)node * n * n + (size_t)i * n + i];
        scale[i] = sqrt(v * (double)(count - 1) / (double)count);
    }
}

// obs = points / scale (bounding.py:1510), computed ONCE per update: IEEE division like numpy,
// and the ten Lloyd iterations of every level then read the scaled copy.
__global__ void scale_points_kernel(const double* __restrict__ P, int64_t total, int n,
                                    const double* __restrict__ scale, double* __restrict__ out) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x)
        out[e] = P[e] / scale[e % n];
}

// ---- 2-means, scipy.cluster.vq.kmeans2(minit='matrix', iter=10) semantics (:1510-1514):
// one CTA per node; centres start at the major-axis end points (:1500-1501, 278-284) in the
// std-scaled space; 10 x { assign to the nearest centre (ties -> cluster 0), centroid =
// member mean, an empty cluster keeps its centre }; the labels returned are those of the
// last assignment (before the last centroid update).
//
// GPU mapping (sm_90 thread-block clusters): each node is handled by a THREAD-BLOCK CLUSTER of 8 CTAs (8 SMs): CTA r
// walks the r-th eighth of the node's points, reduces its per-warp partial sums in its own
// shared memory, and after a cluster barrier every CTA reads the 8 partials through
// distributed shared memory (fixed rank order -> every CTA derives bit-identical centroids,
// run-to-run reproducible, no atomics).  Two cluster barriers per Lloyd iteration.
#define KM_CLUSTER 8
__global__ void __cluster_dims__(KM_CLUSTER, 1, 1) __launch_bounds__(512)
    kmeans2_kernel(const double* __restrict__ P, const int* __restrict__ perm, NodeArrays na,
                   const NodeRef* __restrict__ refs, const double* __restrict__ scale,
                   unsigned char* __restrict__ labels, int* __restrict__ counts, int stage_cap) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ double sm[];
    const int n = na.n;
    const int nodei = blockIdx.x / KM_CLUSTER, rank = (int)cluster.block_rank();
    const NodeRef nr = refs[nodei];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    double* c = sm;                        // 2 x n centres (scaled space)
    double* part0 = c + 2 * n;             // 2 x (2 x n) partial sums of this CTA (read by the peers), by iteration parity
    double* acc = part0 + 4 * n;           // nw x 2 x n
    int* cnt = reinterpret_cast<int*>(acc + (size_t)nw * 2 * n);   // nw x 2
    // the first `stage_cap` rows of this CTA's share of the node, staged ONCE: the ten Lloyd iterations used to
    // re-read every row through perm[] from L2 -- two dependent long-latency loads per trip, 15 us per iteration
    // at 250 rows per CTA; rows beyond the capacity (large nodes) keep coming from L2
    double* stg = reinterpret_cast<double*>(cnt + (size_t)nw * 2 + ((nw * 2) & 1));
    const int ns = n | 1;                  // odd row stride: a thread per row walks the columns bank-conflict free
    unsigned char* slab = reinterpret_cast<unsigned char*>(stg + (size_t)stage_cap * ns);   // labels of the staged rows
    __shared__ int pcnt2[2][2];            // this CTA's member counts (read by the peers), by iteration parity
    __shared__ int tot[2];
    const int lo = nr.start + (int)((long long)nr.count * rank / KM_CLUSTER);
    const int hi = nr.start + (int)((long long)nr.count * (rank + 1) / KM_CLUSTER);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const double ctr = na.mean[(size_t)nr.node * n + i];
        const double v = na.axes[(size_t)nr.node * n * n + (size_t)i * n + (n - 1)];   // largest eigenvalue = last column
        c[i] = (ctr - v) / scale[i];
        c[n + i] = (ctr + v) / scale[i];
    }
    const int nst = min(hi - lo, stage_cap);
    // (row indices first, one coalesced load per 32 rows of the warp: a row's loads then do not wait for its
    //  perm[] entry, and the rows of a warp are in flight together instead of one dependent pair after another)
    for (int r0 = warp; r0 < nst; r0 += 32 * nw) {
        const int mine = r0 + lane * nw;
        const int idx = mine < nst ? perm[lo + mine] : 0;
        const int cntw = min(32, (nst - r0 + nw - 1) / nw);
#pragma unroll 4
        for (int t = 0; t < cntw; t++) {
            const size_t row = (size_t)__shfl_sync(B2N_FULL, idx, t) * n;
            const int r = r0 + t * nw;
            for (int i = lane; i < n; i += 32) stg[(size_t)r * ns + i] = P[row + i];
        }
    }
    __syncthreads();
    // Every row of this CTA staged (the usual case): the THREAD-PER-ROW form of the Lloyd iteration.  The
    // warp-per-row form below spends ~400 instructions per pair of rows, most of them shuffles and addressing, and
    // is issue bound (ncu: 4.1e6 warp instructions per launch at 2000 x 50, 43 % of the issue slots with 4 warps
    // per scheduler).  Here two adjacent lanes own a row (half of the columns each, one shuffle to combine), the
    // distances are sequential sums with no reduction tree, and the centroid sums are formed by (chunk, cluster,
    // column) threads walking the staged rows -- ~20 x fewer instructions per iteration.  Same barriers, same
    // DSMEM exchange, same scipy semantics as below; all sums in a fixed order.
    if (nst == hi - lo) {
        const int rows = nst, T = blockDim.x, tid = threadIdx.x;
        const int nh = (n + 1) >> 1;
        const int CH = max(1, min(nw, T / (2 * n)));            // row chunks of the centroid pass (acc holds nw x 2n)
        for (int it = 0; it < 10; it++) {
            for (int base = 0; base < rows; base += T >> 1) {
                const int r = base + (tid >> 1), h = tid & 1;
                const bool valid = r < rows;
                double d0 = 0.0, d1 = 0.0;
                if (valid) {
                    const double* pr = stg + (size_t)r * ns;
                    const int i1 = min(n, (h + 1) * nh);
                    for (int i = h * nh; i < i1; i++) {
                        const double o = pr[i];
                        const double a = o - c[i], b = o - c[n + i];
                        d0 = fma(a, a, d0);
                        d1 = fma(b, b, d1);
                    }
                }
                const double q0 = __shfl_xor_sync(B2N_FULL, d0, 1), q1 = __shfl_xor_sync(B2N_FULL, d1, 1);
                if (valid && h == 0) {
                    const int lab = ((d1 + q1) < (d0 + q0)) ? 1 : 0;       // lower half + upper half, ties -> cluster 0
                    slab[r] = (unsigned char)lab;
                    labels[lo + r] = (unsigned char)lab;
                }
            }
            __syncthreads();
            for (int e = tid; e < CH * 2 * n; e += T) {
                const int ch = e / (2 * n), f = e - ch * 2 * n, k = f / n, i = f - k * n;
                const int r0 = (int)((long long)rows * ch / CH), r1 = (int)((long long)rows * (ch + 1) / CH);
                double sacc = 0.0;
                int m = 0;
                for (int r = r0; r < r1; r++)
                    if (slab[r] == k) { sacc += stg[(size_t)r * ns + i]; m++; }
                acc[(size_t)ch * 2 * n + f] = sacc;
                if (i == 0) cnt[ch * 2 + k] = m;
            }
            __syncthreads();
            // the partials alternate between two buffers: a peer reads buffer (it & 1) between the cluster barriers
            // of iterations it and it + 1, and this CTA writes it again only after the barrier of it + 1 -- ONE
            // cluster barrier per Lloyd iteration instead of two
            double* part = part0 + (it & 1) * 2 * n;
            int* pcnt = pcnt2[it & 1];
            for (int e = tid; e < 2 * n; e += T) {
                double t = 0.0;
                for (int ch = 0; ch < CH; ch++) t += acc[(size_t)ch * 2 * n + e];
                part[e] = t;
            }
            if (tid < 2) {
                int t = 0;
                for (int ch = 0; ch < CH; ch++) t += cnt[ch * 2 + tid];
                pcnt[tid] = t;
            }
            cluster.sync();
            if (tid < 2) {
                int t = 0;
                for (int rk = 0; rk < KM_CLUSTER; rk++) t += *cluster.map_shared_rank(&pcnt[tid], rk);
                tot[tid] = t;
            }
            __syncthreads();
            for (int e = tid; e < 2 * n; e += T) {
                const int cl = e / n;
                if (tot[cl] > 0) {
                    double t = 0.0;
                    for (int rk = 0; rk < KM_CLUSTER; rk++) t += cluster.map_shared_rank(part, rk)[e];
                    c[e] = t / (double)tot[cl];
                }
            }
            __syncthreads();
        }
        if (rank == 0 && tid < 2) counts[nodei * 2 + tid] = tot[tid];
        cluster.sync();          // no CTA leaves while a peer may still read its partials
        return;
    }
    for (int it = 0; it < 10; it++) {
        for (int i = lane; i < 2 * n; i += 32) acc[(size_t)warp * 2 * n + i] = 0.0;
        if (lane < 2) cnt[warp * 2 + lane] = 0;
        __syncwarp();
        // two points per trip: their row loads and shuffle reductions overlap
        for (int r = lo + warp; r < hi; r += 2 * nw) {
            const int r2 = r + nw;
            const bool two = r2 < hi;
            // P = points / scale (scaled once per update); a staged row is the same doubles from shared memory
            const double* p1 = (r - lo < nst) ? stg + (size_t)(r - lo) * ns : P + (size_t)perm[r] * n;
            const double* p2 = !two ? p1 : ((r2 - lo < nst) ? stg + (size_t)(r2 - lo) * ns : P + (size_t)perm[r2] * n);
            double d0 = 0.0, d1 = 0.0, e0 = 0.0, e1 = 0.0;
            for (int i = lane; i < n; i += 32) {
                const double o = p1[i];
                const double o2 = p2[i];
                const double a = o - c[i], b = o - c[n + i];
                const double a2 = o2 - c[i], b2 = o2 - c[n + i];
                d0 = fma(a, a, d0);
                d1 = fma(b, b, d1);
                e0 = fma(a2, a2, e0);
                e1 = fma(b2, b2, e1);
            }
            d0 = warp_sum(d0);
            d1 = warp_sum(d1);
            e0 = warp_sum(e0);
            e1 = warp_sum(e1);
            const int lab = (d1 < d0) ? 1 : 0;
            const int lab2 = (e1 < e0) ? 1 : 0;
            double* dst = acc + (size_t)warp * 2 * n + (size_t)lab * n;
            for (int i = lane; i < n; i += 32) dst[i] += p1[i];
            if (lane == 0) { cnt[warp * 2 + lab]++; labels[r] = (unsigned char)lab; }
            if (two) {
                double* dst2 = acc + (size_t)warp * 2 * n + (size_t)lab2 * n;
                for (int i = lane; i < n; i += 32) dst2[i] += p2[i];
                if (lane == 0) { cnt[warp * 2 + lab2]++; labels[r2] = (unsigned char)lab2; }
            }
        }
        __syncthreads();
        // CTA partials (fixed warp order)
        double* part = part0 + (it & 1) * 2 * n;       // alternating buffers: one cluster barrier per iteration (see above)
        int* pcnt = pcnt2[it & 1];
        for (int e = threadIdx.x; e < 2 * n; e += blockDim.x) {
            double s = 0.0;
            for (int w = 0; w < nw; w++) s += acc[(size_t)w * 2 * n + e];
            part[e] = s;
        }
        if (threadIdx.x < 2) {
            int t = 0;
            for (int w = 0; w < nw; w++) t += cnt[w * 2 + threadIdx.x];
            pcnt[threadIdx.x] = t;
        }
        cluster.sync();
        // cluster totals through distributed shared memory (fixed rank order)
        if (threadIdx.x < 2) {
            int t = 0;
            for (int rk = 0; rk < KM_CLUSTER; rk++) t += *cluster.map_shared_rank(&pcnt[threadIdx.x], rk);
            tot[threadIdx.x] = t;
        }
        __syncthreads();
        for (int e = threadIdx.x; e < 2 * n; e += blockDim.x) {
            const int cl = e / n;
            if (tot[cl] > 0) {
                double s = 0.0;
                for (int rk = 0; rk < KM_CLUSTER; rk++) s += cluster.map_shared_rank(part, rk)[e];
                c[e] = s / (double)tot[cl];
            }
        }
        __syncthreads();
    }
    if (rank == 0 && threadIdx.x < 2) counts[nodei * 2 + threadIdx.x] = tot[threadIdx.x];
    cluster.sync();          // no CTA leaves while a peer may still read its partials
}

// ---- stable partition of a node's segment by label: [label 0 ..., label 1 ...]
// (points[labels == k] keeps the original order, :1518)
__global__ void __launch_bounds__(256) partition_kernel(const int* __restrict__ perm_in, int* __restrict__ perm_out,
                                                        const NodeRef* __restrict__ refs,
                                                        const unsigned char* __restrict__ labels,
                                                        const int* __restrict__ counts) {
    __shared__ int wsum[8];
    __shared__ int base0, base1;
    const NodeRef nr = refs[blockIdx.x];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) { base0 = nr.start; base1 = nr.start + counts[blockIdx.x * 2]; }
    __syncthreads();
    for (int off = 0; off < nr.count; off += 256) {
        const int r = nr.start + off + threadIdx.x;
        const bool valid = off + threadIdx.x < nr.count;
        const int lab = valid ? labels[r] : 1;
        const bool is0 = valid && lab == 0;
        const unsigned b0 = __ballot_sync(B2N_FULL, is0);
        const unsigned bv = __ballot_sync(B2N_FULL, valid);
        if (lane == 0) wsum[warp] = __popc(b0);
        __syncthreads();
        int pre0 = 0, chunk0 = 0;
        for (int w = 0; w < 8; w++) { if (w < warp) pre0 += wsum[w]; chunk0 += wsum[w]; }
        const int before0 = pre0 + __popc(b0 & ((1u << lane) - 1));
        const int before_valid = warp * 32 + __popc(bv & ((1u << lane) - 1));   // chunk is dense until the tail
        if (valid) {
            const int v = perm_in[r];
            if (is0) perm_out[base0 + before0] = v;
            else perm_out[base1 + (before_valid - before0)] = v;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            const int nvalid = min(256, nr.count - off);
            base0 += chunk0;
            base1 += nvalid - chunk0;
        }
        __syncthreads();
    }
}

__global__ void scatter_labels_kernel(const int* __restrict__ perm, int start, int count, int leaf, int* __restrict__ labels) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < count) labels[perm[start + r]] = leaf;
}

// ---- host-side tree --------------------------------------------------------------------------
struct HNode {
    int start, count, level;
    int child[2];
    int split[2];         // the two cluster sizes of the node's k-means split, -1 if none was attempted
    double logvol;
};

static double logaddexp(double a, double b) {
    const double hi = std::max(a, b), lo = std::min(a, b);
    return hi + log1p(exp(lo - hi));
}
static double logsumexp(const std::vector<double>& v) {
    double hi = -INFINITY;
    for (double x : v) hi = std::max(hi, x);
    double s = 0.0;
    for (double x : v) s += exp(x - hi);
    return hi + log(s);
}

// the accept / reject logic of _bounding_ellipsoids, bottom-up (:1541-1563)
static void resolve(const std::vector<HNode>& t, int id, int n, std::vector<int>& out) {
    const HNode& nd = t[id];
    if (nd.child[0] < 0) { out.push_back(id); return; }
    std::vector<int> sub;
    resolve(t, nd.child[0], n, sub);
    resolve(t, nd.child[1], n, sub);
    const double nparam = (double)((n * (n + 3)) / 2);
    const double dec = nparam * log((double)nd.count) / (double)nd.count;
    bool ok = logaddexp(t[nd.child[0]].logvol, t[nd.child[1]].logvol) - nd.logvol < -dec;
    if (!ok) {
        std::vector<double> lv;
        for (int s : sub) lv.push_back(t[s].logvol);
        ok = logsumexp(lv) - nd.logvol < -dec * ((double)sub.size() - 1.0);
    }
    if (ok) out.insert(out.end(), sub.begin(), sub.end());
    else out.push_back(id);
}

// Decompose the node (level 0 of w.perm, segment [0, count)) -> final leaves.
// Leaves' arrays stay in w.na; returns node ids + final perm buffer index.
#define B2N_RETRY_FULL (-1000)    // internal: a candidate node could not be certified, redo with the eigen path

// fast = true: candidates of the tree go through the Cholesky path (chol_node_kernel), only the accepted
// leaves are fitted with the eigen path; returns B2N_RETRY_FULL if a candidate cannot be certified.
static int decompose(BoundWork& w, int count, std::vector<HNode>& tree, std::vector<int>& leaves, int& final_level,
                     uint32_t* warn, bool fast = false) {
    b2n_ctx* ctx = w.ctx;
    const int n = w.n;
    cudaStream_t st = ctx->stream;
    tree.clear();
    HNode root;
    root.start = 0; root.count = count; root.level = 0; root.child[0] = root.child[1] = -1; root.split[0] = root.split[1] = -1; root.logvol = 0;
    tree.push_back(root);
    const std::vector<NodeRef> refs(1, b2n_node_ref(0, 0, count, 0));
    std::vector<NodeStat> hs;
    // fast: the candidates' stats are read ONCE, after the expansion (nothing on the host needs them earlier:
    // the k-means start centres, the partitions and the children's fits read the node arrays on the device) --
    // a level's launches queue behind the previous level's without a host round trip
    if (fast) {
        B2N_TRY(b2n_fit_candidates(w, refs));
    } else {
        B2N_TRY(b2n_fit_nodes(w, refs, hs));
        if (hs[0].fallback && warn) *warn |= B2N_WARN_IDENTITY_FALLBACK;
        if (hs[0].error) return hs[0].error;
        tree[0].logvol = hs[0].logvol;
    }
    // the root's full (eigen) fit, speculatively, on the side stream while the tree is expanded (b2n_bounding.cu);
    // whatever way this function is left, the side stream has drained first
    struct SpecScope {
        b2n_ctx* c; SpecRoot sp;
        explicit SpecScope(b2n_ctx* ctx) : c(ctx) {}
        ~SpecScope() { b2n_spec_root_wait(c, sp); }
    } spec(ctx);
    if (fast && count >= 4 * n && count == (int)w.N) B2N_TRY(b2n_spec_root_launch(w, count, spec.sp));

    // scale = std of the ROOT points, reused at every depth (:1503-1504, 1548-1549)
    B2N_CUDA(ctx, ctx->work1.ensure((size_t)n * sizeof(double)));
    double* scale = ctx->work1.as<double>();
    root_scale_kernel<<<1, 128, 0, st>>>(w.na, 0, count, scale);
    B2N_LAUNCH_CHECK(ctx);
    const double* Pscaled = w.P;
    if (count >= 4 * n) {      // something will be split: scaled copy of the point block
        B2N_CUDA(ctx, ctx->in2.ensure((size_t)w.N * n * sizeof(double)));
        const int64_t total = w.N * (int64_t)n;
        scale_points_kernel<<<(unsigned)std::min<int64_t>((total + 255) / 256, (int64_t)ctx->sm_count * 8), 256, 0, st>>>(
            w.P, total, n, scale, ctx->in2.as<double>());
        B2N_LAUNCH_CHECK(ctx);
        Pscaled = ctx->in2.as<double>();
    }

    DevBuf& labbuf = ctx->out7;          // per-position labels (N bytes) + counts
    B2N_CUDA(ctx, labbuf.ensure((size_t)w.N + (size_t)w.cap * 2 * sizeof(int) + 64));
    unsigned char* dlab = labbuf.as<unsigned char>();
    int* dcounts = reinterpret_cast<int*>(dlab + ((w.N + 15) & ~(int64_t)15));

    std::vector<int> frontier(1, 0);
    int cur = 0;
    const int min_size = 2 * n;
    int nwarps = 16;
    while ((size_t)(6 * n + (size_t)nwarps * 2 * n) * sizeof(double) + nwarps * 2 * sizeof(int) > (size_t)ctx->max_smem_optin && nwarps > 1)
        nwarps >>= 1;
    const size_t km_base = (size_t)(6 * n + (size_t)nwarps * 2 * n) * sizeof(double) + (size_t)(nwarps * 2 + 2) * sizeof(int);
    if (km_base > (size_t)ctx->max_smem_optin) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "ndim too large for k-means kernel");
    // rows a CTA may stage in shared memory (its eighth of the largest node of a level), within half an SM's
    // shared memory so that the chain kernels of other replicas keep their place next to it
    const size_t km_room = std::min((size_t)ctx->max_smem_optin, (size_t)120 * 1024);
    const int km_stage_max = km_room > km_base ? (int)((km_room - km_base) / ((size_t)(n | 1) * sizeof(double) + 1)) : 0;

    while (!frontier.empty()) {
        std::vector<int> split;
        for (int id : frontier)
            if (tree[id].count >= 2 * min_size) split.push_back(id);      // :1493
        if (split.empty()) break;
        std::vector<NodeRef> srefs;
        for (int id : split) srefs.push_back(b2n_node_ref(id, tree[id].start, tree[id].count, cur));
        const void* drefs;
        B2N_TRY(b2n_in_host(ctx, ctx->scratch5, srefs.data(), srefs.size() * sizeof(NodeRef), &drefs));
        const int* pin = w.perm + (size_t)cur * w.N;
        int* pout = w.perm + (size_t)(1 - cur) * w.N;
        int maxcount = 0;
        for (int id : split) maxcount = std::max(maxcount, tree[id].count);
        const int stage_cap = std::min(km_stage_max, (maxcount + KM_CLUSTER - 1) / KM_CLUSTER + 1);
        const size_t km_smem = km_base + (size_t)stage_cap * (n | 1) * sizeof(double) + (((size_t)stage_cap + 15) & ~(size_t)15);
        B2N_TRY(b2n_func_smem(ctx, (const void*)(kmeans2_kernel), km_smem));
        kmeans2_kernel<<<(unsigned)split.size() * KM_CLUSTER, nwarps * 32, km_smem, st>>>(Pscaled, pin, w.na, (const NodeRef*)drefs, scale,
                                                                           dlab, dcounts, stage_cap);
        B2N_LAUNCH_CHECK(ctx);
        // carry every segment forward, then overwrite the split ones with their partition
        B2N_CUDA(ctx, cudaMemcpyAsync(pout, pin, (size_t)w.N * sizeof(int), cudaMemcpyDeviceToDevice, st));
        partition_kernel<<<(unsigned)split.size(), 256, 0, st>>>(pin, pout, (const NodeRef*)drefs, dlab, dcounts);
        B2N_LAUNCH_CHECK(ctx);
        std::vector<int> hc(split.size() * 2);
        B2N_CUDA(ctx, cudaMemcpyAsync(hc.data(), dcounts, hc.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
        B2N_CUDA(ctx, cudaStreamSynchronize(st));
        cur = 1 - cur;
        std::vector<int> next;
        std::vector<NodeRef> crefs;
        for (size_t i = 0; i < split.size(); i++) {
            const int c0 = hc[2 * i], c1 = hc[2 * i + 1];
            const int id = split[i];
            tree[id].split[0] = c0; tree[id].split[1] = c1;
            if (std::min(c0, c1) < min_size) continue;                    // :1521-1522
            if ((int)tree.size() + 2 > w.cap) return b2n_fail(ctx, B2N_ERR_TOO_MANY_ELLS, "node capacity exceeded");
            for (int k = 0; k < 2; k++) {
                HNode ch;
                ch.start = tree[id].start + (k ? c0 : 0);
                ch.count = k ? c1 : c0;
                ch.level = cur; ch.child[0] = ch.child[1] = -1; ch.split[0] = ch.split[1] = -1; ch.logvol = 0;
                tree[id].child[k] = (int)tree.size();
                crefs.push_back(b2n_node_ref((int)tree.size(), ch.start, ch.count, cur));
                next.push_back((int)tree.size());
                tree.push_back(ch);
            }
        }
        if (fast) {
            B2N_TRY(b2n_fit_candidates(w, crefs));
        } else if (!crefs.empty()) {
            B2N_TRY(b2n_fit_nodes(w, crefs, hs));
            for (size_t i = 0; i < crefs.size(); i++) {
                if (hs[i].fallback && warn) *warn |= B2N_WARN_IDENTITY_FALLBACK;
                if (hs[i].error) return hs[i].error;
                tree[crefs[i].node].logvol = hs[i].logvol;
            }
        }
        frontier = next;
    }
    if (fast) {
        std::vector<NodeStat> all;
        B2N_TRY(b2n_read_stats(w, all));
        for (size_t id = 0; id < tree.size(); id++) {
            if (all[id].suspect || all[id].pad || all[id].error) return B2N_RETRY_FULL;
            tree[id].logvol = all[id].logvol;
        }
    }
    leaves.clear();
    resolve(tree, 0, n, leaves);
    final_level = cur;
    bool adopted = false;
    if (fast && leaves.size() == 1 && leaves[0] == 0) {
        // nothing was split for good: the root's speculative fit is the result
        NodeStat rs;
        B2N_TRY(b2n_spec_root_adopt(w, spec.sp, &rs, &adopted));
        if (adopted) tree[0].logvol = rs.logvol;
    }
    if (fast && !adopted) {
        // the accepted leaves get the full fit (eigen-decomposition: axes, axlens, and the reference's exact
        // ladder / rescale); a leaf's points are the segment [start, start+count) of EITHER index buffer as a
        // set (partitions only permute inside segments), so the last buffer serves all of them
        std::vector<NodeRef> lrefs;
        for (int id : leaves) lrefs.push_back(b2n_node_ref(id, tree[id].start, tree[id].count, cur));
        B2N_TRY(b2n_fit_nodes(w, lrefs, hs));
        for (size_t k = 0; k < leaves.size(); k++) {
            if (hs[k].fallback && warn) *warn |= B2N_WARN_IDENTITY_FALLBACK;
            if (hs[k].error) return hs[k].error;
            tree[leaves[k]].logvol = hs[k].logvol;
        }
    }
    return B2N_OK;
}

// gather the leaf ellipsoids into contiguous device arrays (for membership checks)
static int gather_leaves(BoundWork& w, const std::vector<int>& leaves, double** dctrs, double** dams) {
    b2n_ctx* ctx = w.ctx;
    const size_t n = w.n, nn = n * n, K = leaves.size();
    B2N_CUDA(ctx, ctx->scratch2.ensure(K * (n + nn) * sizeof(double)));
    double* c = ctx->scratch2.as<double>();
    double* a = c + K * n;
    for (size_t k = 0; k < K; k++) {
        B2N_CUDA(ctx, cudaMemcpyAsync(c + k * n, w.na.mean + (size_t)leaves[k] * n, n * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
        B2N_CUDA(ctx, cudaMemcpyAsync(a + k * nn, w.na.am + (size_t)leaves[k] * nn, nn * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    }
    *dctrs = c;
    *dams = a;
    return B2N_OK;
}

// The decomposition of b2n_multi_decompose and b2n_multi_tree: the points uploaded, the candidate path chosen, the
// tree expanded and resolved, and redone with the eigen path if a candidate could not be certified.  *fast_used:
// the tree returned is the one of the Cholesky candidates.
static int multi_run(b2n_ctx* ctx, const double* points, int64_t N, int n, BoundWork& w, const void** dP,
                     std::vector<HNode>& tree, std::vector<int>& leaves, int& level, uint32_t* warn, bool* fast_used) {
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    if (warn) *warn = 0;
    B2N_TRY(b2n_in(ctx, ctx->in0, points, (size_t)N * n * sizeof(double), dP));
    const int cap = (int)std::max<int64_t>(3, N / std::max(n, 1) + 3);
    B2N_TRY(b2n_boundwork_init(ctx, w, (const double*)*dP, N, n, cap));
    B2N_TRY(b2n_init_identity_perm(w));
    level = 0;
    // candidates through the Cholesky path when the two work matrices fit in shared memory (n <= ~117)
    // and the path has not just failed to certify a node of this problem (ctx->bound_fast_skip)
    const char* fenv = getenv("B2N_BOUND_FAST");
    const int ldw = n | 1;
    bool fast = !(fenv && !strcmp(fenv, "0")) && N >= 4 * (int64_t)n &&
                (size_t)(2 * n * ldw + 3 * n + 32 + 2 * (n + 2)) * sizeof(double) <= (size_t)ctx->max_smem_optin;
    if (fast && ctx->bound_fast_skip > 0 && !(fenv && fenv[0] == '1')) { ctx->bound_fast_skip--; fast = false; }   // "1" forces the attempt
    *fast_used = fast;
    int dst = decompose(w, (int)N, tree, leaves, level, warn, fast);
    if (dst == B2N_RETRY_FULL) {
        ctx->bound_fast_skip = 16;
        *fast_used = false;
        if (warn) *warn = 0;
        B2N_TRY(b2n_init_identity_perm(w));
        dst = decompose(w, (int)N, tree, leaves, level, warn, false);
    }
    return dst;
}

extern "C" int b2n_multi_decompose(b2n_ctx* ctx, const double* points, int64_t N, int32_t n, int32_t max_ells,
                                   int32_t* nells, int32_t* labels, double* ctrs, double* covs, double* ams,
                                   double* axes, double* axlens, double* logvols, uint32_t* warn) {
    if (!ctx || !points || N < 1 || n < 1 || max_ells < 1 || !nells) return B2N_ERR_ARG;
    if (N == 1) return B2N_ERR_SINGLE_POINT;
    const void* dP;
    BoundWork w;
    std::vector<HNode> tree;
    std::vector<int> leaves;
    int level = 0;
    bool fast_used = false;
    const int dst = multi_run(ctx, points, N, n, w, &dP, tree, leaves, level, warn, &fast_used);
    if (dst != B2N_OK) return dst;
    const int K = (int)leaves.size();
    *nells = K;
    if (K > max_ells) return B2N_ERR_TOO_MANY_ELLS;
    // sanity check: every point inside some ellipsoid (:683-685)
    double *dc, *da;
    B2N_TRY(gather_leaves(w, leaves, &dc, &da));
    B2N_CUDA(ctx, ctx->out6.ensure((size_t)N * sizeof(int)));
    int* dq = ctx->out6.as<int>();
    B2N_TRY(b2n_membership_dev(ctx, (const double*)dP, N, n, dc, da, K, 1, nullptr, dq, nullptr));
    std::vector<int> hq(N);
    B2N_CUDA(ctx, cudaMemcpyAsync(hq.data(), dq, (size_t)N * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int64_t i = 0; i < N; i++)
        if (hq[i] < 1) return B2N_ERR_INVALID_REGION;
    // outputs
    std::vector<double> lv(K);
    for (int k = 0; k < K; k++) {
        B2N_TRY(b2n_emit_node(w, leaves[k], k, ctrs, covs, ams, axes, axlens));
        lv[k] = tree[leaves[k]].logvol;
    }
    if (logvols) {
        if (ctx->ptr_mode == B2N_PTR_DEVICE)
            B2N_CUDA(ctx, cudaMemcpyAsync(logvols, lv.data(), K * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        else
            memcpy(logvols, lv.data(), K * sizeof(double));
    }
    if (labels) {
        void* dl;
        B2N_TRY(b2n_out(ctx, ctx->out5, labels, (size_t)N * sizeof(int), &dl));
        const int* pm = w.perm + (size_t)level * N;
        for (int k = 0; k < K; k++) {
            const HNode& nd = tree[leaves[k]];
            scatter_labels_kernel<<<(nd.count + 255) / 256, 256, 0, ctx->stream>>>(pm, nd.start, nd.count, k, (int*)dl);
            B2N_LAUNCH_CHECK(ctx);
        }
        B2N_TRY(b2n_out_done(ctx, labels, dl, (size_t)N * sizeof(int)));
    }
    B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B2N_OK;
}

extern "C" int b2n_multi_tree(b2n_ctx* ctx, const double* points, int64_t N, int32_t n, int32_t max_nodes,
                              int32_t* nnodes, int32_t* nodes, double* logvols, int32_t* perm, int32_t* path) {
    if (!ctx || !points || N < 1 || n < 1 || max_nodes < 1 || !nnodes || !nodes || !logvols || !perm || !path)
        return B2N_ERR_ARG;
    if (N == 1) return B2N_ERR_SINGLE_POINT;
    const void* dP;
    BoundWork w;
    std::vector<HNode> tree;
    std::vector<int> leaves;
    int level = 0;
    bool fast_used = false;
    B2N_TRY(multi_run(ctx, points, N, n, w, &dP, tree, leaves, level, nullptr, &fast_used));
    const int T = (int)tree.size();
    *nnodes = T;
    if (T > max_nodes) return B2N_ERR_TOO_MANY_ELLS;
    std::vector<int> accepted(T, 0);
    for (int id : leaves) accepted[id] = 1;
    for (int i = 0; i < T; i++) {
        const HNode& nd = tree[i];
        const int row[7] = {nd.start, nd.count, nd.child[0], nd.child[1], nd.split[0], nd.split[1], accepted[i]};
        memcpy(nodes + (size_t)7 * i, row, sizeof(row));
        logvols[i] = nd.logvol;
    }
    B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    B2N_CUDA(ctx, b2n_copy_sync(ctx, perm, w.perm + (size_t)level * N, (size_t)N * sizeof(int), cudaMemcpyDeviceToHost));
    *path = fast_used ? 1 : 0;
    return B2N_OK;
}

// ---- bootstrap -------------------------------------------------------------------------------
// host Philox4x32-10 for the resampling indices (B2N stream: one uniform vector event,
// element e -> floor(U_e * N); see oracle/philox.py for the layout)
static inline void philox_block(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1,
                                uint32_t out[4]) {
    for (int r = 0; r < 10; r++) {
        const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n1 = (uint32_t)p1;
        const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1, n3 = (uint32_t)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
static inline double u52(uint32_t a, uint32_t b) {
    return ((double)(a >> 6) * 67108864.0 + (double)(b >> 6) + 0.5) * 0x1p-52;
}

__global__ void min_dist_kernel(const double* __restrict__ d2, int M, int K, double* __restrict__ out) {
    // out[0] = max_m min_k sqrt(d2[m,k])   (single block, deterministic)
    __shared__ double red[32];
    double best = -INFINITY;
    for (int m = threadIdx.x; m < M; m += blockDim.x) {
        double mn = INFINITY;
        for (int k = 0; k < K; k++) mn = fmin(mn, d2[(size_t)m * K + k]);
        best = fmax(best, sqrt(mn));
    }
    best = warp_max(best);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        double b = red[0];
        for (int w = 1; w < (int)(blockDim.x >> 5); w++) b = fmax(b, red[w]);
        out[0] = b;
    }
}

extern "C" int b2n_bootstrap_expand(b2n_ctx* ctx, const double* points, int64_t N, int32_t n, int32_t multi,
                                    int32_t nboot, uint64_t seed, uint64_t chain0, double* expands) {
    if (!ctx || !points || N < 2 || n < 1 || nboot < 0 || !expands) return B2N_ERR_ARG;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    const void* dP;
    B2N_TRY(b2n_in(ctx, ctx->in0, points, (size_t)N * n * sizeof(double), &dP));
    BoundWork w;
    const int cap = (int)std::max<int64_t>(3, N / std::max(n, 1) + 3);
    B2N_TRY(b2n_boundwork_init(ctx, w, (const double*)dP, N, n, cap));
    std::vector<int> perm(N);
    std::vector<char> sel(N);
    for (int rep = 0; rep < nboot; rep++) {
        // _bootstrap_points (:1593-1616)
        std::fill(sel.begin(), sel.end(), 0);
        const uint64_t chain = chain0 + (uint64_t)rep;
        for (int64_t b = 0; b < (N + 1) / 2; b++) {
            uint32_t r[4];
            philox_block((uint32_t)b, 0u, (uint32_t)chain, (uint32_t)(chain >> 32), (uint32_t)seed, (uint32_t)(seed >> 32), r);
            const double u[2] = {u52(r[0], r[1]), u52(r[2], r[3])};
            for (int s = 0; s < 2 && 2 * b + s < N; s++) {
                int64_t idx = (int64_t)(u[s] * (double)N);
                if (idx > N - 1) idx = N - 1;
                sel[idx] = 1;
            }
        }
        int64_t n_in = 0;
        for (int64_t i = 0; i < N; i++) n_in += sel[i];
        if (n_in < 2) sel[0] = sel[1] = 1;
        if (n_in > N - 1) sel[0] = 0;
        int64_t a = 0, z = N;
        for (int64_t i = 0; i < N; i++) if (sel[i]) perm[a++] = (int)i;
        for (int64_t i = N - 1; i >= 0; i--) if (!sel[i]) perm[--z] = (int)i;     // out-of-bag at the tail
        n_in = a;
        const int64_t n_out = N - n_in;
        B2N_CUDA(ctx, cudaMemcpyAsync(w.perm, perm.data(), (size_t)N * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
        std::vector<HNode> tree;
        std::vector<int> leaves;
        int level = 0;
        if (multi) {
            B2N_TRY(decompose(w, (int)n_in, tree, leaves, level, nullptr));
        } else {
            std::vector<NodeStat> hs;
            if (n_in == 1) return B2N_ERR_SINGLE_POINT;
            B2N_TRY(b2n_fit_nodes(w, std::vector<NodeRef>(1, b2n_node_ref(0, 0, (int)n_in, 0)), hs));
            if (hs[0].error) return hs[0].error;
            leaves.assign(1, 0);
        }
        // distances of the out-of-bag points (:1636-1646); gather them contiguously first
        const int K = (int)leaves.size();
        double *dc, *da;
        B2N_TRY(gather_leaves(w, leaves, &dc, &da));
        std::vector<double> hout((size_t)n_out * n);
        // (host mode keeps a host copy of the points; device mode reads them back once)
        const double* hp = points;
        std::vector<double> hp_copy;
        if (ctx->ptr_mode == B2N_PTR_DEVICE) {
            hp_copy.resize((size_t)N * n);
            B2N_CUDA(ctx, cudaMemcpyAsync(hp_copy.data(), dP, (size_t)N * n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
            B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            hp = hp_copy.data();
        }
        for (int64_t i = 0; i < n_out; i++)
            memcpy(&hout[(size_t)i * n], hp + (size_t)perm[n_in + i] * n, (size_t)n * sizeof(double));
        B2N_CUDA(ctx, ctx->in1.ensure(hout.size() * sizeof(double) + 8));
        B2N_CUDA(ctx, cudaMemcpyAsync(ctx->in1.p, hout.data(), hout.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        B2N_CUDA(ctx, ctx->out6.ensure((size_t)n_out * K * sizeof(double) + 64));
        double* dd2 = ctx->out6.as<double>();
        B2N_TRY(b2n_membership_dev(ctx, ctx->in1.as<double>(), n_out, n, dc, da, K, 1, nullptr, nullptr, dd2));
        B2N_CUDA(ctx, ctx->out5.ensure(64));
        min_dist_kernel<<<1, 256, 0, ctx->stream>>>(dd2, (int)n_out, K, ctx->out5.as<double>());
        B2N_LAUNCH_CHECK(ctx);
        double mx = 0.0;
        B2N_CUDA(ctx, cudaMemcpyAsync(&mx, ctx->out5.p, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        expands[rep] = std::max(1.0, mx);
    }
    return B2N_OK;
}

// b2n_jitter.cu -- R prior-volume realisations of one dead-point record (utils.py:1273-1467 jitter_run /
// compute_integrals, :1932-1997 kld_error of the reference), all in FP64.
//
// Random streams (B2N layout, oracle/philox.py; restated in oracle/jitter.py): realisation r is the chain
// (seed, chain0 + r).  Tick 0 is one uniform vector event over the F samples with nlive_flag set; the e-th of them
// gets ln t = ln(U_e) / n.  Decreasing stretch s (the reference's _find_decrease) is tick s + 1: nstart_s + 1
// uniforms, y = -ln U, C = prefix sums of y, and its j-th sample gets ln t = ln(C[k_j] / C[k_{j-1}]) with
// k_j = samples_n[j] - 1 and k_{-1} = nstart_s.
//
// The record is cut into SEGMENTS on the host: pieces of at most TILE samples that are either a run of flagged
// samples outside every stretch (their t come from tick 0) or a piece of one stretch.  A stretch piece only needs
// C up to the largest index it reads (k of the sample before it, or nstart), so a long stretch (the add_live tail)
// splits into pieces that each rescan a prefix of its exponentials.  Nothing R x N is stored unless the full arrays
// are asked for: the two per-segment passes regenerate ln t from the counter-based stream.
//
//   pass 1   (segments x R)  ln t, local prefix of ln t (sum D), local log-sum-exp of the weights (E)
//   scan 1   (R)             logvol and logz at every segment start, logz[-1]
//   pass 2   (segments x R)  logvol, logwt, logz per sample; segment sums of the h increments (A), of dh * dlogvol (C)
//                            and of the KL terms (K); the full arrays when asked for
//   scan 2   (R)             logzerr[-1], h[-1], kld[-1]; the kld prefix at every segment start
//   offsets  (segments x R)  adds that prefix to the full kld array (only when it is asked for), and the prefixes of
//                            A and C to the full h and logzvar arrays (b2n_integrate_lnt only)
//
// b2n_integrate_lnt (below, for b2n_merge.cu) runs the same passes in a deterministic mode: one realisation whose ln t
// per sample is read from an array (segment_lnt<true>), over a plan of tick-0 segments only; b2n_compute_integrals
// (below) runs that mode on ln t = diff(logvol).  With a log-reweight (A.lrw, b2n_set_reweight) the passes run their
// _rw instantiations, which add it to every logwt.
//
// Host side: b2n_jitter_produce stages a record and enqueues the passes, for b2n_jitter_runs (below) and for
// b2n_jitter_posterior (b2n_posterior.cu, with the weights of pass 2); the entry points stage their outputs through
// B2nOutStage (b2n_common.cuh).  The block scan and its operators are b2n_scan.cuh's.
#include "b2n_device.cuh"
#include "b2n_scan.cuh"

#include <algorithm>
#include <math.h>

namespace {

constexpr int JT_BLOCK = 256;
constexpr int JT_TILE = 1024;       // samples per segment
constexpr int JT_CHUNK = 2048;      // exponentials scanned per step

struct JSeg {
    int64_t a;       // first sample
    int32_t len;     // samples
    int32_t tick;    // 0: flagged samples (tick-0 draws); s + 1: piece of stretch s
    int64_t kprev;   // stretch piece: the C index its first ratio divides by (= the scan length - 1)
};

struct JArgs {
    const double* logl;
    const double* wref;      // input run's logwt, or NULL (no KL divergence)
    const int32_t* nlive;    // samples_n
    const int32_t* aux;      // flagged sample: its element of the tick-0 event; stretch sample: k = samples_n - 1
    const JSeg* seg;
    const double* lnt;       // given ln t per sample (b2n_integrate_lnt), else NULL
    int64_t N, nseg;
    int R;
    double zref;
    uint64_t seed, chain0;
    double* sD; double* sE; double* sV; double* sZ; double* sA; double* sC; double* sK;   // R x nseg each
    double* zend;            // R: logz[-1]
    double* out_logz; double* out_logzerr; double* out_h; double* out_kld;                // R each, may be NULL
    double* f_logvol; double* f_logwt; double* f_logz; double* f_kld;                     // R x N, may be NULL
    double* f_h; double* f_logzvar;                      // N, may be NULL (b2n_integrate_lnt only)
    double* f_w;             // N x R (sample-major): w = exp(logwt - logz[-1]) (jitter_weights_kernel only)
    double* s_w2;            // R x nseg: segment sums of w^2 (jitter_weights_kernel only)
    const double* lrw;       // N: log-reweight added to every logwt (the _rw kernels only), else NULL
};

// ln t of the segment's samples into lt[0, len)
template <bool GIVEN>
__device__ void segment_lnt(const JArgs& A, const JSeg& s, int r, double* lt, double* cap, double* buf, double* wsum) {
    if (GIVEN) {
        for (int i = threadIdx.x; i < s.len; i += blockDim.x) lt[i] = A.lnt[s.a + i];
        __syncthreads();
        return;
    }
    ChainRng g;
    g.init(A.seed, A.chain0 + (uint64_t)r);
    const int L = s.len;
    if (s.tick == 0) {
        for (int i = threadIdx.x; i < L; i += blockDim.x)
            lt[i] = log(rng_uniform_elem(g, A.aux[s.a + i])) / (double)A.nlive[s.a + i];
        __syncthreads();
        return;
    }
    g.tick = (uint32_t)s.tick;
    // cap[0] = C[kprev], cap[1 + i] = C[k of sample a + i]
    double carry = 0.0;
    for (int64_t c0 = 0; c0 <= s.kprev; c0 += JT_CHUNK) {
        const int m = (int)min((int64_t)JT_CHUNK, s.kprev + 1 - c0);
        for (int e = threadIdx.x; e < m; e += blockDim.x) buf[e] = -log(rng_uniform_elem(g, (int)(c0 + e)));
        __syncthreads();
        const double tot = block_scan(buf, m, wsum, OpSum());
        for (int q = threadIdx.x; q <= L; q += blockDim.x) {
            const int64_t k = q == 0 ? s.kprev : (int64_t)A.aux[s.a + q - 1];
            if (k >= c0 && k < c0 + m) cap[q] = carry + buf[k - c0];
        }
        carry += tot;
        __syncthreads();
    }
    for (int i = threadIdx.x; i < L; i += blockDim.x) lt[i] = log(cap[i + 1] / cap[i]);
    __syncthreads();
}

// GIVEN: ln t read from A.lnt (b2n_integrate_lnt); the full h / logzvar arrays are written only in that mode, so the
// instantiations of b2n_jitter_runs compile to the code they had before it existed.  WOUT (pass 2 only): also the
// weights f_w and the segment sums of their squares s_w2 (b2n_jitter_posterior), likewise only in that mode.  RW: lrw[j]
// is added to every logwt (pass 1's local weights, pass 2's cap), so logz, the KL terms and the weights are the
// reweighted ones while the h increments keep the unreweighted L and ldv2 (compute_integrals(reweight=)); a KL term of
// zero weight is 0.  Without RW the code is the one it was before the reweight existed.
template <int PASS, bool GIVEN, bool WOUT, bool RW = false>
__device__ __forceinline__ void jitter_pass(const JArgs& A) {
    __shared__ double lt[JT_TILE], pv[JT_TILE], cap[JT_TILE + 1], buf[JT_CHUNK], wsum[32];
    const int64_t sg = blockIdx.x;
    const int r = blockIdx.y;
    const JSeg s = A.seg[sg];
    const int L = s.len;
    const int64_t so = (int64_t)r * A.nseg + sg;
    segment_lnt<GIVEN>(A, s, r, lt, cap, buf, wsum);
    for (int i = threadIdx.x; i < L; i += blockDim.x) pv[i] = lt[i];
    __syncthreads();
    const double D = block_scan(pv, L, wsum, OpSum());      // pv[i] = sum of lt[0..i]
    const double ln_half = -0.69314718055994530942;
    if (PASS == 1) {
        for (int i = threadIdx.x; i < L; i += blockDim.x) {
            const int64_t j = s.a + i;
            const double lprev = j > 0 ? A.logl[j - 1] : -1e300;
            buf[i] = (i > 0 ? pv[i - 1] : 0.0) + lae(A.logl[j], lprev) + log1p(-exp(lt[i])) + ln_half;
            if (RW) buf[i] += A.lrw[j];
        }
        __syncthreads();
        const double E = block_scan(buf, L, wsum, OpLae());
        if (threadIdx.x == 0) { A.sD[so] = D; A.sE[so] = E; }
        return;
    }
    const double V = A.sV[so], Z = A.sZ[so], zmax = A.zend[r];
    const size_t fo = (size_t)r * A.N + s.a;
    // logwt (cap), then its log-sum-exp scan (buf) -> logz
    for (int i = threadIdx.x; i < L; i += blockDim.x) {
        const int64_t j = s.a + i;
        const double lprev = j > 0 ? A.logl[j - 1] : -1e300;
        cap[i] = lae(A.logl[j], lprev) + V + (i > 0 ? pv[i - 1] : 0.0) + log1p(-exp(lt[i])) + ln_half;
        buf[i] = cap[i];
    }
    if (RW) {
        __syncthreads();
        for (int i = threadIdx.x; i < L; i += blockDim.x) buf[i] = cap[i] += A.lrw[s.a + i];
    }
    __syncthreads();
    block_scan(buf, L, wsum, OpLae());
    for (int i = threadIdx.x; i < L; i += blockDim.x) buf[i] = lae(Z, buf[i]);
    __syncthreads();
    // per sample: the increment a_i of h1 = cumsum(a), dh_i * dlogvol_i, the KL term (read-only pass; thread t owns
    // samples t + u * blockDim)
    constexpr int U = JT_TILE / JT_BLOCK;
    double* sa = buf + JT_TILE;
    double c_r[U], k_r[U], w2_r[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
        const int i = threadIdx.x + u * JT_BLOCK;
        c_r[u] = k_r[u] = w2_r[u] = 0.0;
        if (i >= L) continue;
        const int64_t j = s.a + i;
        const double l = A.logl[j], lprev = j > 0 ? A.logl[j - 1] : -1e300;
        const double ldv2 = V + (i > 0 ? pv[i - 1] : 0.0) + log1p(-exp(lt[i])) + ln_half;
        const double a = exp(l - zmax + ldv2) * l + exp(lprev - zmax + ldv2) * lprev;
        const double dh = a - zmax * (exp(buf[i] - zmax) - exp((i > 0 ? buf[i - 1] : Z) - zmax));
        sa[i] = a;
        c_r[u] = dh * -lt[i];
        if (!GIVEN && A.wref) {             // (no KL divergence against given ln t)
            const double lp1 = cap[i] - zmax;
            if (!RW || lp1 != -INFINITY) k_r[u] = exp(lp1) * (lp1 - (A.wref[j] - A.zref));
        }
        if (WOUT) {
            const double w = exp(cap[i] - zmax);
            A.f_w[(size_t)j * A.R + r] = w;
            w2_r[u] = w * w;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < L; i += blockDim.x) {
        if (A.f_logvol) A.f_logvol[fo + i] = V + pv[i];
        if (A.f_logwt) A.f_logwt[fo + i] = cap[i];
        if (A.f_logz) A.f_logz[fo + i] = buf[i];
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < U; u++) {
        const int i = threadIdx.x + u * JT_BLOCK;
        if (i < L) { lt[i] = c_r[u]; pv[i] = k_r[u]; }
        if (WOUT && i < L) cap[i] = w2_r[u];
    }
    __syncthreads();
    const double Asum = block_scan(sa, L, wsum, OpSum());
    const double Csum = block_scan(lt, L, wsum, OpSum());
    const double Ksum = block_scan(pv, L, wsum, OpSum());
    if (WOUT) {
        const double W2sum = block_scan(cap, L, wsum, OpSum());
        if (threadIdx.x == 0) A.s_w2[so] = W2sum;
    }
    if (A.f_kld)
        for (int i = threadIdx.x; i < L; i += blockDim.x) A.f_kld[fo + i] = pv[i];
    if (GIVEN) {
        // segment-local parts: h = h1 - zmax exp(logz - zmax) with h1's local prefix in sa; logzvar's local prefix
        // in lt (the offsets launch adds the prefixes of the segments before)
        if (A.f_h)
            for (int i = threadIdx.x; i < L; i += blockDim.x) A.f_h[fo + i] = sa[i] - zmax * exp(buf[i] - zmax);
        if (A.f_logzvar)
            for (int i = threadIdx.x; i < L; i += blockDim.x) A.f_logzvar[fo + i] = lt[i];
    }
    if (threadIdx.x == 0) { A.sA[so] = Asum; A.sC[so] = Csum; A.sK[so] = Ksum; }
}

template <int PASS, bool GIVEN>
__global__ void __launch_bounds__(JT_BLOCK) jitter_pass_kernel(JArgs A) { jitter_pass<PASS, GIVEN, false>(A); }

// Pass 2 of b2n_jitter_posterior: jitter_pass_kernel<2, false> plus the weights.
__global__ void __launch_bounds__(JT_BLOCK) jitter_weights_kernel(JArgs A) { jitter_pass<2, false, true>(A); }

// The same two with the log-reweight A.lrw (b2n_set_reweight, b2n_compute_integrals).
template <int PASS, bool GIVEN>
__global__ void __launch_bounds__(JT_BLOCK) jitter_pass_rw_kernel(JArgs A) { jitter_pass<PASS, GIVEN, false, true>(A); }
__global__ void __launch_bounds__(JT_BLOCK) jitter_weights_rw_kernel(JArgs A) { jitter_pass<2, false, true, true>(A); }

// One realisation per block: running scans over its segments in chunks of JT_TILE.
// PASS 1: logvol (sV) and logz (sZ) before every segment, zend = logz[-1].
// PASS 2: the summaries; the kld prefix before every segment into sK (in place) when the full kld array is wanted,
// likewise the h1 prefix into sA and the logzvar prefix into sC when the full h / logzvar arrays are.
template <int PASS>
__global__ void __launch_bounds__(JT_BLOCK) jitter_scan_kernel(JArgs A) {
    __shared__ double x[JT_TILE], y[JT_TILE], z[JT_TILE], wsum[32];
    const int r = blockIdx.x;
    const int64_t base = (int64_t)r * A.nseg;
    double c0 = 0.0, c1 = PASS == 1 ? -INFINITY : 0.0, c2 = 0.0;
    for (int64_t g0 = 0; g0 < A.nseg; g0 += JT_TILE) {
        const int m = (int)min((int64_t)JT_TILE, A.nseg - g0);
        if (PASS == 1) {
            for (int i = threadIdx.x; i < m; i += blockDim.x) x[i] = A.sD[base + g0 + i];
            __syncthreads();
            const double td = block_scan(x, m, wsum, OpSum());
            for (int i = threadIdx.x; i < m; i += blockDim.x) {
                const double v = i > 0 ? c0 + x[i - 1] : c0;
                y[i] = v;
                z[i] = v + A.sE[base + g0 + i];
            }
            __syncthreads();
            const double tz = block_scan(z, m, wsum, OpLae());
            for (int i = threadIdx.x; i < m; i += blockDim.x) {
                A.sV[base + g0 + i] = y[i];
                A.sZ[base + g0 + i] = i > 0 ? lae(c1, z[i - 1]) : c1;
            }
            c0 += td;
            c1 = lae(c1, tz);
        } else {
            for (int i = threadIdx.x; i < m; i += blockDim.x) {
                x[i] = A.sA[base + g0 + i];
                y[i] = A.sC[base + g0 + i];
                z[i] = A.sK[base + g0 + i];
            }
            __syncthreads();
            const double ta = block_scan(x, m, wsum, OpSum());
            const double tc = block_scan(y, m, wsum, OpSum());
            const double tk = block_scan(z, m, wsum, OpSum());
            if (A.f_kld)
                for (int i = threadIdx.x; i < m; i += blockDim.x) A.sK[base + g0 + i] = i > 0 ? c2 + z[i - 1] : c2;
            if (A.f_h)
                for (int i = threadIdx.x; i < m; i += blockDim.x) A.sA[base + g0 + i] = i > 0 ? c0 + x[i - 1] : c0;
            if (A.f_logzvar)
                for (int i = threadIdx.x; i < m; i += blockDim.x) A.sC[base + g0 + i] = i > 0 ? c1 + y[i - 1] : c1;
            c0 += ta;
            c1 += tc;
            c2 += tk;
        }
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    if (PASS == 1) {
        A.zend[r] = c1;
        if (A.out_logz) A.out_logz[r] = c1;
    } else {
        const double zmax = A.zend[r];
        if (A.out_logzerr) A.out_logzerr[r] = sqrt(fabs(c1));       // logzvar = |cumsum(dh * dlogvol)|
        if (A.out_h) A.out_h[r] = c0 - zmax;                        // h1[-1] - zmax * exp(logz[-1] - zmax)
        if (A.out_kld) A.out_kld[r] = c2;
    }
}

// The prefixes scan 2 left in sK / sA / sC added to the segment-local full kld / h / logzvar arrays.
__global__ void __launch_bounds__(JT_BLOCK) jitter_offsets_kernel(JArgs A) {
    const int64_t sg = blockIdx.x;
    const int r = blockIdx.y;
    const JSeg s = A.seg[sg];
    const int64_t so = (int64_t)r * A.nseg + sg;
    const size_t fo = (size_t)r * A.N + s.a;
    if (A.f_kld) {
        const double off = A.sK[so];
        for (int i = threadIdx.x; i < s.len; i += blockDim.x) A.f_kld[fo + i] += off;
    }
    if (A.f_h) {
        const double off = A.sA[so];
        for (int i = threadIdx.x; i < s.len; i += blockDim.x) A.f_h[fo + i] += off;
    }
    if (A.f_logzvar) {                      // logzvar = |cumsum(dh * dlogvol)|
        const double off = A.sC[so];
        for (int i = threadIdx.x; i < s.len; i += blockDim.x) A.f_logzvar[fo + i] = fabs(A.f_logzvar[fo + i] + off);
    }
}

// The passes on the stream for a prepared JArgs (seg, nseg, N, R and the scratch pointers set).
int jitter_launch(b2n_ctx* ctx, const JArgs& A, bool given) {
    const dim3 grid((unsigned)A.nseg, (unsigned)A.R);
    const bool rw = A.lrw != nullptr;
    if (given) (rw ? jitter_pass_rw_kernel<1, true> : jitter_pass_kernel<1, true>)<<<grid, JT_BLOCK, 0, ctx->stream>>>(A);
    else (rw ? jitter_pass_rw_kernel<1, false> : jitter_pass_kernel<1, false>)<<<grid, JT_BLOCK, 0, ctx->stream>>>(A);
    B2N_LAUNCH_CHECK(ctx);
    jitter_scan_kernel<1><<<A.R, JT_BLOCK, 0, ctx->stream>>>(A);
    B2N_LAUNCH_CHECK(ctx);
    if (given) (rw ? jitter_pass_rw_kernel<2, true> : jitter_pass_kernel<2, true>)<<<grid, JT_BLOCK, 0, ctx->stream>>>(A);
    else if (A.f_w) (rw ? jitter_weights_rw_kernel : jitter_weights_kernel)<<<grid, JT_BLOCK, 0, ctx->stream>>>(A);
    else (rw ? jitter_pass_rw_kernel<2, false> : jitter_pass_kernel<2, false>)<<<grid, JT_BLOCK, 0, ctx->stream>>>(A);
    B2N_LAUNCH_CHECK(ctx);
    jitter_scan_kernel<2><<<A.R, JT_BLOCK, 0, ctx->stream>>>(A);
    B2N_LAUNCH_CHECK(ctx);
    if (A.f_kld || A.f_h || A.f_logzvar) {
        jitter_offsets_kernel<<<grid, JT_BLOCK, 0, ctx->stream>>>(A);
        B2N_LAUNCH_CHECK(ctx);
    }
    return B2N_OK;
}

// Per-(realisation, segment) scratch: 7 x R x nseg (8 with the w^2 sums), + logz[-1] per realisation.
int jitter_scratch(b2n_ctx* ctx, JArgs& A, bool w2 = false) {
    const size_t rs = (size_t)A.R * A.nseg;
    B2N_CUDA(ctx, ctx->scratch1.ensure(((w2 ? 8 : 7) * rs + A.R) * sizeof(double)));
    double* sp = ctx->scratch1.as<double>();
    A.sD = sp; A.sE = sp + rs; A.sV = sp + 2 * rs; A.sZ = sp + 3 * rs;
    A.sA = sp + 4 * rs; A.sC = sp + 5 * rs; A.sK = sp + 6 * rs; A.zend = sp + 7 * rs;
    if (w2) A.s_w2 = sp + 7 * rs + A.R;
    return B2N_OK;
}

// The segment table and the per-sample aux words (the stretch plan; depends on samples_n only).  O(N), one pass.
int jitter_plan(const int64_t* n, int64_t N, int approx, std::vector<JSeg>& seg, std::vector<int32_t>& aux) {
    seg.clear();
    aux.assign(N, 0);
    int64_t rank = 0;                  // tick-0 elements handed out so far
    int64_t nstretch = 0;
    auto dec = [&](int64_t i) { return !approx && i > 0 && i < N && n[i] < n[i - 1]; };
    JSeg open{0, 0, 0, 0};
    auto flush = [&]() { if (open.len > 0) seg.push_back(open); open.len = 0; };
    int64_t i = 0;
    while (i < N) {
        if (n[i] < 1 || n[i] > INT32_MAX) return B2N_ERR_ARG;
        if (dec(i + 1)) {              // sample i opens a decreasing stretch [i, j)
            flush();
            int64_t j = i + 1;
            while (j < N && dec(j)) j++;
            rank++;                    // the stretch's first sample still takes its tick-0 element
            const int64_t nstart = n[i];
            nstretch++;
            if (nstretch >= (int64_t)UINT32_MAX) return B2N_ERR_ARG;
            for (int64_t m = i; m < j; m++) {
                if (n[m] < 1) return B2N_ERR_ARG;
                aux[m] = (int32_t)(n[m] - 1);
            }
            for (int64_t a = i; a < j; a += JT_TILE) {
                const int64_t kprev = a == i ? nstart : n[a - 1] - 1;
                seg.push_back(JSeg{a, (int32_t)std::min<int64_t>(JT_TILE, j - a), (int32_t)nstretch, kprev});
            }
            i = j;
            continue;
        }
        if (rank > INT32_MAX) return B2N_ERR_ARG;
        if (open.len == 0) open = JSeg{i, 0, 0, 0};
        aux[i] = (int32_t)rank++;
        if (++open.len == JT_TILE) flush();
        i++;
    }
    flush();
    return B2N_OK;
}

}  // namespace

int b2n_jitter_produce(b2n_ctx* ctx, const double* logl, const int64_t* samples_n, int64_t N, const double* logwt_ref,
                       double logz_ref, int32_t approx, int32_t R, uint64_t seed, uint64_t chain0, const double* logrwt,
                       double* const sum[4], double* const full[4], double* w, const double** w2, int64_t* nw2,
                       const double** wref) {
    std::vector<JSeg> seg;
    std::vector<int32_t> aux;
    B2N_TRY(jitter_plan(samples_n, N, approx, seg, aux));
    std::vector<int32_t> nl(N);
    for (int64_t i = 0; i < N; i++) nl[i] = (int32_t)samples_n[i];
    const int64_t nseg = (int64_t)seg.size();
    if (nseg > INT32_MAX) return B2N_ERR_ARG;

    JArgs A;
    memset(&A, 0, sizeof(A));
    const void* p;
    B2N_TRY(b2n_in(ctx, ctx->in0, logl, (size_t)N * sizeof(double), &p));
    A.logl = (const double*)p;
    B2N_TRY(b2n_in(ctx, ctx->in1, logwt_ref, logwt_ref ? (size_t)N * sizeof(double) : 0, &p));
    A.wref = (const double*)p;
    B2N_TRY(b2n_in(ctx, ctx->work1, logrwt, logrwt ? (size_t)N * sizeof(double) : 0, &p));
    A.lrw = (const double*)p;
    B2N_TRY(b2n_in_host(ctx, ctx->in2, nl.data(), (size_t)N * sizeof(int32_t), &p));
    A.nlive = (const int32_t*)p;
    B2N_TRY(b2n_in_host(ctx, ctx->in3, aux.data(), (size_t)N * sizeof(int32_t), &p));
    A.aux = (const int32_t*)p;
    B2N_TRY(b2n_in_host(ctx, ctx->scratch0, seg.data(), seg.size() * sizeof(JSeg), &p));
    A.seg = (const JSeg*)p;
    A.N = N; A.nseg = nseg; A.R = R; A.zref = logz_ref; A.seed = seed; A.chain0 = chain0;
    B2N_TRY(jitter_scratch(ctx, A, w != nullptr));
    A.out_logz = sum[0]; A.out_logzerr = sum[1]; A.out_h = sum[2]; A.out_kld = sum[3];
    if (full) { A.f_logvol = full[0]; A.f_logwt = full[1]; A.f_logz = full[2]; A.f_kld = full[3]; }
    A.f_w = w;
    if (w) { *w2 = A.s_w2; *nw2 = A.nseg; *wref = A.wref; }

    B2N_TIME_BEGIN(ctx);
    return jitter_launch(ctx, A, false);
}

extern "C" int b2n_jitter_runs(b2n_ctx* ctx, const double* logl, const int64_t* samples_n, int64_t N,
                               const double* logwt_ref, double logz_ref, int32_t approx, int32_t R, uint64_t seed,
                               uint64_t chain0, double* logz, double* logzerr, double* h, double* kld,
                               double* logvol_full, double* logwt_full, double* logz_full, double* kld_full) {
    if (!ctx) return B2N_ERR_ARG;
    const double* logrwt;
    B2N_TRY(b2n_take_reweight(ctx, N, &logrwt));
    if (!logl || !samples_n || N < 1 || R < 1 || R > 65535) return B2N_ERR_ARG;
    if (!logwt_ref && (kld || kld_full)) return B2N_ERR_ARG;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t rb = (size_t)R * sizeof(double), fb = rb * N;
    B2nOutStage<8> O{{logz, logzerr, h, kld, logvol_full, logwt_full, logz_full, kld_full},
                     {rb, rb, rb, rb, fb, fb, fb, fb}};
    B2N_TRY(O.bind(ctx));
    double* d[8];
    for (int k = 0; k < 8; k++) d[k] = (double*)O.dev[k];
    B2N_TRY(b2n_jitter_produce(ctx, logl, samples_n, N, logwt_ref, logz_ref, approx, R, seed, chain0, logrwt, d, d + 4,
                               nullptr, nullptr, nullptr, nullptr));
    B2N_TIME_END(ctx);
    B2N_TRY(O.done(ctx));
    return b2n_finish(ctx);
}

// compute_integrals (utils.py:1411-1467) of one record whose ln t per sample is given: logvol = cumsum(lnt), then the
// quadrature of the passes above, with the log-reweight lrw (N, or NULL) added to every logwt.  Every pointer is a
// device pointer; the outputs may be NULL.  last3 (3 doubles): logz[-1], logzerr[-1] = sqrt(|logzvar[-1]|), h[-1].
// Enqueues on the context's stream and does not synchronise; uses ctx->scratch0 and ctx->scratch1.
int b2n_integrate_lnt(b2n_ctx* ctx, const double* logl, const double* lnt, const double* lrw, int64_t N, double* last3,
                      double* logvol, double* logwt, double* logz, double* logzvar, double* h) {
    std::vector<JSeg> seg;
    for (int64_t a = 0; a < N; a += JT_TILE) seg.push_back(JSeg{a, (int32_t)std::min<int64_t>(JT_TILE, N - a), 0, 0});
    if ((int64_t)seg.size() > INT32_MAX) return B2N_ERR_ARG;
    JArgs A;
    memset(&A, 0, sizeof(A));
    const void* p;
    B2N_TRY(b2n_in_host(ctx, ctx->scratch0, seg.data(), seg.size() * sizeof(JSeg), &p));
    A.seg = (const JSeg*)p;
    A.logl = logl; A.lnt = lnt; A.lrw = lrw;
    A.N = N; A.nseg = (int64_t)seg.size(); A.R = 1;
    B2N_TRY(jitter_scratch(ctx, A));
    if (last3) { A.out_logz = last3; A.out_logzerr = last3 + 1; A.out_h = last3 + 2; }
    A.f_logvol = logvol; A.f_logwt = logwt; A.f_logz = logz; A.f_logzvar = logzvar; A.f_h = h;
    return jitter_launch(ctx, A, true);
}

namespace {
// ln t = diff(logvol, prepend=0): the volumes of compute_integrals as the deterministic passes read them
__global__ void __launch_bounds__(JT_BLOCK) logvol_diff_kernel(const double* logvol, int64_t N, double* lnt) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) lnt[i] = i > 0 ? logvol[i] - logvol[i - 1] : logvol[0];
}
}  // namespace

extern "C" int b2n_compute_integrals(b2n_ctx* ctx, const double* logl, const double* logvol, const double* logrwt,
                                     int64_t N, double* last3, double* logwt, double* logz, double* logzvar,
                                     double* h) {
    if (!ctx) return B2N_ERR_ARG;
    B2N_TRY(b2n_refuse_reweight(ctx, "b2n_compute_integrals"));
    if (!logl || !logvol || N < 1 || (N + JT_BLOCK - 1) / JT_BLOCK > INT32_MAX) return B2N_ERR_ARG;
    B2N_TRY(b2n_reweight_check(ctx, logrwt, N));
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t nb = (size_t)N * sizeof(double);
    B2nOutStage<5> O{{last3, logwt, logz, logzvar, h}, {3 * sizeof(double), nb, nb, nb, nb}};
    B2N_TRY(O.bind(ctx));
    const void *dl, *dv, *dr;
    B2N_TRY(b2n_in(ctx, ctx->in0, logl, nb, &dl));
    B2N_TRY(b2n_in(ctx, ctx->in1, logvol, nb, &dv));
    B2N_TRY(b2n_in(ctx, ctx->work1, logrwt, logrwt ? nb : 0, &dr));
    B2N_CUDA(ctx, ctx->in2.ensure(nb));
    double* lnt = ctx->in2.as<double>();
    B2N_TIME_BEGIN(ctx);
    logvol_diff_kernel<<<(unsigned)((N + JT_BLOCK - 1) / JT_BLOCK), JT_BLOCK, 0, ctx->stream>>>((const double*)dv, N, lnt);
    B2N_LAUNCH_CHECK(ctx);
    B2N_TRY(b2n_integrate_lnt(ctx, (const double*)dl, lnt, (const double*)dr, N, (double*)O.dev[0], nullptr,
                              (double*)O.dev[1], (double*)O.dev[2], (double*)O.dev[3], (double*)O.dev[4]));
    B2N_TIME_END(ctx);
    B2N_TRY(O.done(ctx));
    return b2n_finish(ctx);
}

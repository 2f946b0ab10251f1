// b2n_bounding.cu -- bounding-ellipsoid construction kernels + entry points.
//
//   moments      : mean and ddof=1 covariance of each node (np.mean / np.cov, reference
//                  bounding.py:1410-1411), two-pass (centered) and deterministic:
//                  per-job partials reduced in a fixed order, no atomics.
//   eig_ladder   : parallel cyclic Jacobi eigen-decomposition of the n x n covariance in
//                  shared memory + the improve_covar_mat repair ladder (:1311-1384) +
//                  am = V diag(1/l) V^T and axes = V sqrt(l)                (:1353, 1381)
//   fmax / scale : max_i d_i^T am d_i (:1438) and the (1 - 1e-3) safety rescale (:1444-1450),
//                  then the Ellipsoid constructor quantities axlens / logvol (:212-217).
// LAPACK's ?syevr (what scipy.linalg.eigh calls in the reference) is a third-party
// dependency; Jacobi is used here because it maps onto one CTA with the matrix resident
// in shared memory and is at least as accurate for SPD matrices.  Eigenvalues come out
// in ascending order like LAPACK; eigenvector SIGNS are not defined by either.
#include "b2n_bounding.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

// ------------------------------------------------------------------ moments
#define B2N_FMAX_SUB 4     // CTAs per 128-row job in the fmax scan


__global__ void __launch_bounds__(256) colsum_partial_kernel(const double* __restrict__ P, const int* __restrict__ perm,
                                                             int64_t N, int n, const JobL* __restrict__ jobs,
                                                             double* __restrict__ partial) {
    extern __shared__ double sm[];   // 8 x n
    const JobL jb = jobs[blockIdx.x];
    const int* pm = perm + (size_t)jb.level * N;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int i = tx; i < n; i += 32) {
        double s = 0.0;
        for (int r = jb.r0 + ty; r < jb.r1; r += 8) s += P[(size_t)pm[r] * n + i];
        sm[ty * n + i] = s;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        double s = 0.0;
        for (int g = 0; g < 8; g++) s += sm[g * n + i];
        partial[(size_t)jb.slot * n + i] = s;
    }
}

__global__ void mean_finalize_kernel(const NodeRef* __restrict__ refs, int n, const double* __restrict__ partial,
                                     double* __restrict__ mean) {
    const NodeRef nr = refs[blockIdx.x];
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        double s = 0.0;
        for (int k = 0; k < nr.nslots; k++) s += partial[(size_t)(nr.slot0 + k) * n + i];
        mean[(size_t)nr.node * n + i] = s / (double)nr.count;
    }
}

// C_partial[slot] = sum_{r in job} d_r d_r^T on one 64x64 output tile; 16x16 threads, 4x4
// register tile each; centred rows staged through shared memory 16 at a time.
__global__ void __launch_bounds__(256) cov_partial_kernel(const double* __restrict__ P, const int* __restrict__ perm,
                                                          int64_t N, int n, const JobL* __restrict__ jobs,
                                                          const double* __restrict__ mean,
                                                          double* __restrict__ partial, int ntile) {
    __shared__ double As[B2N_TK][B2N_TILE + 1];
    __shared__ double Bs[B2N_TK][B2N_TILE + 1];
    const JobL jb = jobs[blockIdx.x];
    const int* pm = perm + (size_t)jb.level * N;
    const double* mu = mean + (size_t)jb.node * n;
    int ib = 0, jt = blockIdx.y;          // decode upper-triangular tile index
    while (jt >= ntile - ib) { jt -= ntile - ib; ib++; }
    const int jbk = ib + jt;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    double acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) acc[a][b] = 0.0;
    for (int k0 = jb.r0; k0 < jb.r1; k0 += B2N_TK) {
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const int idx = threadIdx.x + e * 256;
            const int kk = idx >> 6, c = idx & 63;
            const int r = k0 + kk;
            double a = 0.0, b = 0.0;
            if (r < jb.r1) {
                const size_t row = (size_t)pm[r] * n;
                const int ca = ib * B2N_TILE + c, cb = jbk * B2N_TILE + c;
                if (ca < n) a = P[row + ca] - mu[ca];
                if (cb < n) b = P[row + cb] - mu[cb];
            }
            As[kk][c] = a;
            Bs[kk][c] = b;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < B2N_TK; kk++) {
            double a[4], b[4];
#pragma unroll
            for (int t = 0; t < 4; t++) { a[t] = As[kk][ty * 4 + t]; b[t] = Bs[kk][tx * 4 + t]; }
#pragma unroll
            for (int x = 0; x < 4; x++)
#pragma unroll
                for (int y = 0; y < 4; y++) acc[x][y] = fma(a[x], b[y], acc[x][y]);
        }
        __syncthreads();
    }
    double* out = partial + (size_t)jb.slot * n * n;
#pragma unroll
    for (int x = 0; x < 4; x++)
#pragma unroll
        for (int y = 0; y < 4; y++) {
            const int i = ib * B2N_TILE + ty * 4 + x, j = jbk * B2N_TILE + tx * 4 + y;
            if (i < n && j < n) {
                out[(size_t)i * n + j] = acc[x][y];
                if (ib != jbk) out[(size_t)j * n + i] = acc[x][y];
            }
        }
}

__global__ void cov_finalize_kernel(const NodeRef* __restrict__ refs, int n, const double* __restrict__ partial,
                                    double* __restrict__ covraw) {
    const NodeRef nr = refs[blockIdx.x];
    const size_t nn = (size_t)n * n;
    const double inv = 1.0 / (double)(nr.count - 1);
    for (size_t e = (size_t)blockIdx.y * blockDim.x + threadIdx.x; e < nn; e += (size_t)gridDim.y * blockDim.x) {
        double s = 0.0;
        for (int k = 0; k < nr.nslots; k++) s += partial[(size_t)(nr.slot0 + k) * nn + e];
        covraw[(size_t)nr.node * nn + e] = s * inv;
    }
}

#include "b2n_jacobi.cuh"

// improve_covar_mat (bounding.py:1311-1384) for one node per CTA.
// pass 0: input = covraw ; pass 1: input = current cov (after the pass-0 rescale).
// SMEM: the two work matrices live in the CTA's shared memory (every n the single-CTA path takes in practice) and are
// addressed as such -- through the generic pointer of the global-memory fallback a third of the instructions of a
// Jacobi round were 64-bit address arithmetic.
template <bool SMEM>
__global__ void __launch_bounds__(1024) eig_ladder_kernel(NodeArrays na, const int* __restrict__ nodelist, int pass,
                                                         double* __restrict__ gwork) {
    extern __shared__ double sm[];
    const int n = na.n, ld = na.ld, tid = threadIdx.x, T = blockDim.x;
    const int node = nodelist[blockIdx.x];
    const size_t nn = (size_t)n * n;
    double* small = sm;                       // cc[half] ss[half] lamv[n] rank/tmp[n] red[32]
    const int half = ((n + 1) & ~1) >> 1;
    double* cc = small;
    double* ss = cc + half;
    double* lamv = ss + half;
    double* tmpv = lamv + n;
    double* red = tmpv + n;
    double* A = SMEM ? red + 32 : gwork + (size_t)blockIdx.x * 2 * n * ld;
    double* VT = A + (size_t)n * ld;
    __shared__ int s_failed, s_sweeps;
    __shared__ double s_mx;

    double* Cm = na.cov + (size_t)node * nn;
    if (pass == 0) {
        const double* src = na.covraw + (size_t)node * nn;
        for (size_t e = tid; e < nn; e += T) Cm[e] = src[e];
    }
    __syncthreads();
    int failed = 0, trial = 0;
    for (trial = 0; trial < 100; trial++) {
        for (size_t e = tid; e < nn; e += T) {
            const int i = (int)(e / n), j = (int)(e - (size_t)i * n);
            A[(size_t)i * ld + j] = Cm[e];
            VT[(size_t)i * ld + j] = (i == j) ? 1.0 : 0.0;
        }
        __syncthreads();
        const int sw = jacobi_eig(A, VT, n, ld, cc, ss, red);
        for (int k = tid; k < n; k += T) lamv[k] = A[(size_t)k * ld + k];
        __syncthreads();
        if (tid == 0) {
            bool fin = true;
            double mx = -INFINITY, mn = INFINITY;
            for (int k = 0; k < n; k++) {
                const double l = lamv[k];
                fin = fin && (l == l) && (fabs(l) < INFINITY);
                mx = fmax(mx, l);
                mn = fmin(mn, l);
            }
            int f = 0;
            if (!fin) f = 2;
            else if (mx <= 0) f = 2;
            else if (mn < mx / 1e12) f = 1;
            s_failed = f;
            s_mx = mx;
            s_sweeps = sw;
        }
        __syncthreads();
        failed = s_failed;
        if (failed == 0) break;
        if (failed == 1) {
            const double floorv = 10.0 * s_mx / 1e12;
            for (int k = tid; k < n; k += T) tmpv[k] = fmax(lamv[k], floorv);
            __syncthreads();
            for (size_t e = tid; e < nn; e += T) {
                const int i = (int)(e / n), j = (int)(e - (size_t)i * n);
                double s = 0.0;
                for (int k = 0; k < n; k++) s = fma(VT[(size_t)k * ld + i] * tmpv[k], VT[(size_t)k * ld + j], s);
                Cm[e] = s;
            }
        } else {
            const double coeff = 1e-10 * pow(1e10, (double)trial / 99.0);
            for (size_t e = tid; e < nn; e += T) {
                const int i = (int)(e / n), j = (int)(e - (size_t)i * n);
                Cm[e] = (1.0 - coeff) * Cm[e] + ((i == j) ? coeff : 0.0);
            }
        }
        __syncthreads();
    }
    double* AM = na.am + (size_t)node * nn;
    double* AX = na.axes + (size_t)node * nn;
    double* LM = na.lam + (size_t)node * n;
    NodeStat* st = na.stat + node;
    if (failed > 0) {               // identity fallback (:1373-1378)
        for (size_t e = tid; e < nn; e += T) {
            const int i = (int)(e / n), j = (int)(e - (size_t)i * n);
            const double v = (i == j) ? 1.0 : 0.0;
            Cm[e] = v; AM[e] = v; AX[e] = v;
        }
        for (int k = tid; k < n; k += T) LM[k] = 1.0;
        if (tid == 0) { st->good = 0; st->fallback = 1; st->sweeps = s_sweeps; st->retry = 0; }
        return;
    }
    // rank-sort eigenvalues ascending (LAPACK order); tmpv[k] = rank of eigenpair k
    for (int k = tid; k < n; k += T) {
        const double l = lamv[k];
        int rk = 0;
        for (int j = 0; j < n; j++) rk += (lamv[j] < l || (lamv[j] == l && j < k)) ? 1 : 0;
        tmpv[k] = (double)rk;
        LM[rk] = l;
        cc[k] = 1.0 / l;          // cc|ss (2*half >= n doubles) are free after the decomposition
    }
    __syncthreads();
    for (size_t e = tid; e < nn; e += T) {
        const int i = (int)(e / n), j = (int)(e - (size_t)i * n);
        double s = 0.0;
        // am = (V * (1/l)) @ V^T, the reciprocal taken once per eigenvalue as in bounding.py:1381
        for (int k = 0; k < n; k++) s = fma(VT[(size_t)k * ld + i] * cc[k], VT[(size_t)k * ld + j], s);
        AM[e] = s;
        // here j plays the role of the eigen index: axes[i][rank_j] = V[i][j] sqrt(l_j)
        AX[(size_t)i * n + (int)tmpv[j]] = VT[(size_t)j * ld + i] * sqrt(lamv[j]);
    }
    if (tid == 0) {
        if (pass == 0) st->good = (trial == 0) ? 1 : 0;
        st->fallback = 0;
        st->sweeps = s_sweeps;
        st->retry = 0;
    }
}

// ------------------------------------------------------------------ symmetric sweeps in registers
// cov^-1 and the Cholesky pivots of an n x n SPD matrix by n symmetric SWEEPS: sweeping pivot k,
//     A_ij -= A_ik A_kj / d  (i, j != k),   A_ik = A_ki = A_ik / d,   A_kk = -1 / d,   d = A_kk,
// leaves the Schur complement of the swept block in the rest (d is the k-th Cholesky pivot L_kk^2: same positivity
// test, ln det = sum ln d) and after n sweeps A = -cov^-1.  The matrix lives in REGISTERS for all n sweeps: 512
// threads, warp w owns rows w, w + 16, ... (R of them), lane l the columns l, l + 32, ... (C of them).  A sweep
// needs only the pivot column -- published to shared memory by its owners (double buffered) -- so it costs ONE
// barrier, no matrix traffic, no integer division.  (i, j) and (j, i) see the same operands in the same order: the
// matrix stays symmetric to the bit.  Also returns |cov|_inf and |cov^-1|_inf (row sums = warp reductions).
template <int R, int C>
static __device__ __forceinline__ bool sweep_inverse_regs(const double* __restrict__ src, double* __restrict__ Cm,
                                                          double* __restrict__ AM, int n, double* ybuf, double* dg,
                                                          double* red, int* s_bad, double& cnorm, double& anorm) {
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;        // blockDim.x == 512
    const int npad = (n + 1) & ~1;
    double v[R][C];
#pragma unroll
    for (int a = 0; a < R; a++)
#pragma unroll
        for (int b = 0; b < C; b++) {
            const int i = w + 16 * a, j = lane + 32 * b;
            double c = 0.0;
            if (i < n && j < n) { c = src[(size_t)i * n + j]; Cm[(size_t)i * n + j] = c; }
            v[a][b] = c;
        }
    double rmax = 0.0;
#pragma unroll
    for (int a = 0; a < R; a++) {
        double t = 0.0;
#pragma unroll
        for (int b = 0; b < C; b++) t += fabs(v[a][b]);
        rmax = fmax(rmax, warp_sum(t));
    }
    if (lane == 0) red[w] = rmax;
    if (lane == 0) {                                   // column 0
#pragma unroll
        for (int a = 0; a < R; a++) if (w + 16 * a < n) ybuf[w + 16 * a] = v[a][0];
    }
    __syncthreads();
    cnorm = 0.0;
    for (int q = 0; q < 16; q++) cnorm = fmax(cnorm, red[q]);
    for (int k = 0; k < n; k++) {
        const double* cur = ybuf + (k & 1) * npad;
        double* nxt = ybuf + ((k + 1) & 1) * npad;
        const double d = cur[k];
        if (!(d > 0.0) || !(d < INFINITY)) {           // the same value in every thread: uniform exit
            if (tid == 0) *s_bad = 1;
            break;
        }
        if (tid == 0) dg[k] = d;
        const double rinv = 1.0 / d;
        double yj[C];
#pragma unroll
        for (int b = 0; b < C; b++) yj[b] = (lane + 32 * b < n) ? cur[lane + 32 * b] : 0.0;
        const int bsel = (k + 1) >> 5;
        const bool pub = (k + 1 < n) && (lane == ((k + 1) & 31));
#pragma unroll
        for (int a = 0; a < R; a++) {
            const int i = w + 16 * a;
            if (i < n) {
                const double yi = cur[i];
#pragma unroll
                for (int b = 0; b < C; b++) {
                    const int j = lane + 32 * b;
                    double x;
                    if (i == k) x = (j == k) ? -rinv : yj[b] * rinv;
                    else if (j == k) x = yi * rinv;
                    else x = fma(-(yi * yj[b]), rinv, v[a][b]);
                    v[a][b] = x;
                    if (pub && b == bsel) nxt[i] = x;          // column k + 1 as the next sweep needs it
                }
            }
        }
        __syncthreads();
    }
    __syncthreads();
    if (*s_bad) return false;
    rmax = 0.0;
#pragma unroll
    for (int a = 0; a < R; a++) {
        double t = 0.0;
#pragma unroll
        for (int b = 0; b < C; b++) {
            const int i = w + 16 * a, j = lane + 32 * b;
            if (i < n && j < n) AM[(size_t)i * n + j] = -v[a][b]; else v[a][b] = 0.0;
            t += fabs(v[a][b]);
        }
        rmax = fmax(rmax, warp_sum(t));
    }
    if (lane == 0) red[w] = rmax;
    __syncthreads();
    anorm = 0.0;
    for (int q = 0; q < 16; q++) anorm = fmax(anorm, red[q]);
    __syncthreads();
    return true;
}

// ------------------------------------------------------------------ candidate nodes: Cholesky path
// _bounding_ellipsoids (bounding.py:1464-1563) fits an ellipsoid to EVERY node of the candidate tree --
// it always recurses into both children before its two volume tests -- but returns only the accepted
// leaves (one, for a unimodal live set).  What the recursion needs from a candidate is (i) its
// log-volume, (ii) its precision matrix (for the fmax rescale, :1438-1450) and (iii) its major axis
// (k-means start centres, :278-284, 1500-1501); none of that needs the full eigen-decomposition, which
// is the latency-bound part of a bound update (0.66 ms per tree level at n = 50).  For a candidate:
//   symmetric sweeps of cov (the Cholesky pivots d_k = L_kk^2 without the factor)  ->  ln det = sum ln d_k,
//   am = -(swept matrix);
//   improve_covar_mat's test (all eigenvalues finite, max > 0, min >= max/1e12, :1343-1352) is certified
//   by cond_2 <= |cov|_inf |am|_inf < 1e10 (a sufficient condition: then the ladder is a no-op);
//   major axis by power iteration to 1e-13, written as the LAST column of `axes` (largest eigenvalue).
// The pivots d_k are stored where the eigenvalues go (`lam`): scale_finish_kernel's sum of logs is then
// ln det, and its rescale / singularity test apply unchanged.  A node that cannot be certified (Cholesky
// break-down, condition bound, slow power iteration: near-degenerate leading eigenvalues) is flagged
// `suspect` and the caller redoes the whole update with the eigen path.  Accepted leaves are always
// re-fitted with the eigen path (they need axes / axlens), so outputs never come from this kernel.
// The fit is two INDEPENDENT latency chains that both start from the raw covariance -- (1) Cholesky -> L^-1 -> am,
// pivots, conditioning; (2) repeated squaring -> major axis -- run as two launches on two streams (PART 1 on the main
// stream, PART 2 on a side stream; they write disjoint outputs and disjoint words of the node's NodeStat:
// `suspect` / `pad`), b2n_fit_candidates.
template <int PART>
__global__ void __launch_bounds__(512) chol_node_kernel(NodeArrays na, const int* __restrict__ nodelist) {
    extern __shared__ double sm[];
    const int n = na.n, ld = na.ld, tid = threadIdx.x, T = blockDim.x;
    const int node = nodelist[blockIdx.x];
    const size_t nn = (size_t)n * n;
    double* L = sm;                          // n x ld: the matrix being swept (-> -cov^-1); then squaring workspace
    double* Li = L + (size_t)n * ld;         // n x ld: squaring workspace
    double* dg = Li + (size_t)n * ld;        // n: pivots d_k = L_kk^2 of the sweeps
    double* v = dg + n;                      // n: power-iteration vector
    double* y = v + n;                       // n
    double* red = y + n;                     // 32
    double* ybuf = red + 32;                 // 2 x (n + 2): pivot columns of the sweeps (double buffered)
    __shared__ int s_bad, s_it;
    __shared__ double s_lam, s_diff;
    const double* src = na.covraw + (size_t)node * nn;
    double* Cm = na.cov + (size_t)node * nn;
    NodeStat* st = na.stat + node;
    if (tid == 0) { s_bad = 0; s_it = 0; }
    if (PART == 1) {
    // ---- precision matrix, pivots, |cov|_inf |am|_inf: symmetric sweeps on a register-resident matrix
    //      (sweep_inverse_regs above)
    double cnorm = 0.0, anorm = 0.0;
    double* AM = na.am + (size_t)node * nn;
    __syncthreads();
    const bool okA = (n <= 64) ? sweep_inverse_regs<4, 2>(src, Cm, AM, n, ybuf, dg, red, &s_bad, cnorm, anorm)
                               : sweep_inverse_regs<8, 4>(src, Cm, AM, n, ybuf, dg, red, &s_bad, cnorm, anorm);
    if (!okA) {
        if (tid == 0) { st->suspect = 1; st->good = 1; st->fallback = 0; st->retry = 0; }
        for (int k = tid; k < n; k += T) na.lam[(size_t)node * n + k] = 1.0;
        return;
    }
    for (int k = tid; k < n; k += T) na.lam[(size_t)node * n + k] = dg[k];
    if (tid == 0) { st->suspect = (cnorm * anorm < 1e10) ? 0 : 1; st->good = 1; st->fallback = 0; st->retry = 0; }
    return;
    }   // PART == 1
    __syncthreads();
    // ---- major axis.  Plain power iteration stalls on the deep nodes of the tree (a half of a half of a
    //      Gaussian cloud has a leading eigenvalue within a few % of the next ones), so the dominant
    //      eigenvector is extracted by REPEATED SQUARING: M <- M^2 / |M^2|_F, 18 times = the 2^18-th power of
    //      cov in 18 small matrix products (the two Cholesky work matrices are free now).  M converges to
    //      v1 v1^T (|.|_F = 1, trace 1); a gap below ~1e-4 leaves trace(M) != 1 and is flagged suspect.
    double* A = L;
    double* B = Li;
    {
        double ss = 0.0;
        for (size_t e = tid; e < nn; e += T) { const double c = src[e]; ss = fma(c, c, ss); }
        const double inv = rsqrt(block_sum(ss, red));
        for (size_t e = tid; e < nn; e += T) {
            const int i = (int)(e / n), j = (int)(e - (size_t)i * n);
            A[(size_t)i * ld + j] = src[e] * inv;
        }
        __syncthreads();
    }
    // One squaring = n^2/2 dot products of length n out of shared memory on ONE SM: bandwidth bound, so each
    // thread owns a 2 x 2 tile {ti, ti+nt} x {tj, tj+nt} (rows a tile-stride apart: consecutive threads read
    // consecutive rows, conflict free with the odd leading dimension) -- one load per FMA instead of two --
    // and the loop stops as soon as M is a projector to round-off (trace(M) = |M|_F = 1).
    const int nt = (n + 1) >> 1;
    for (int sq = 0; sq < 18; sq++) {
        double ss = 0.0;
        for (int e = tid; e < nt * nt; e += T) {
            const int ti = e / nt, tj = e - ti * nt;
            if (tj > ti) continue;
            const int i0 = ti, i1 = ti + nt, j0 = tj, j1 = tj + nt;
            const bool vi = i1 < n, vj = j1 < n;
            const double* r0 = A + (size_t)i0 * ld;
            const double* r1 = A + (size_t)(vi ? i1 : i0) * ld;
            const double* c0 = A + (size_t)j0 * ld;
            const double* c1 = A + (size_t)(vj ? j1 : j0) * ld;
            double a00 = 0.0, a01 = 0.0, a10 = 0.0, a11 = 0.0;
            for (int m = 0; m < n; m++) {
                const double x0 = r0[m], x1 = r1[m], y0 = c0[m], y1 = c1[m];
                a00 = fma(x0, y0, a00);
                a01 = fma(x0, y1, a01);
                a10 = fma(x1, y0, a10);
                a11 = fma(x1, y1, a11);
            }
            const double wgt = (ti == tj) ? 1.0 : 2.0;           // off-diagonal tiles are mirrored
            B[(size_t)i0 * ld + j0] = a00; B[(size_t)j0 * ld + i0] = a00;
            ss = fma(wgt * a00, a00, ss);
            if (vj) { B[(size_t)i0 * ld + j1] = a01; B[(size_t)j1 * ld + i0] = a01; ss = fma(wgt * a01, a01, ss); }
            if (vi) { B[(size_t)i1 * ld + j0] = a10; B[(size_t)j0 * ld + i1] = a10; ss = fma(wgt * a10, a10, ss); }
            if (vi && vj) { B[(size_t)i1 * ld + j1] = a11; B[(size_t)j1 * ld + i1] = a11; ss = fma(wgt * a11, a11, ss); }
        }
        const double inv = rsqrt(block_sum(ss, red));
        double tr = 0.0;
        for (size_t e = tid; e < nn; e += T) {
            const int i = (int)(e / n), j = (int)(e - (size_t)i * n);
            const double bv = B[(size_t)i * ld + j] * inv;
            B[(size_t)i * ld + j] = bv;
            if (i == j) tr += bv;
        }
        tr = block_sum(tr, red);
        __syncthreads();
        double* t = A; A = B; B = t;
        if (fabs(tr - 1.0) < 1e-13) break;                       // uniform: every thread holds the same sum
    }
    // trace test + the column of the largest diagonal entry as the start of two clean-up power steps on cov
    if (tid == 0) {
        double tr = 0.0;
        int jm = 0;
        for (int i = 0; i < n; i++) {
            tr += A[(size_t)i * ld + i];
            if (A[(size_t)i * ld + i] > A[(size_t)jm * ld + jm]) jm = i;
        }
        s_diff = fabs(tr - 1.0);
        s_it = jm;
    }
    __syncthreads();
    const double trdev = s_diff;
    {
        const int jm = s_it;
        double ss = 0.0;
        for (int i = tid; i < n; i += T) { const double c = A[(size_t)i * ld + jm]; ss = fma(c, c, ss); }
        const double inv = rsqrt(block_sum(ss, red));
        for (int i = tid; i < n; i += T) v[i] = A[(size_t)i * ld + jm] * inv;
        __syncthreads();
    }
    double lam = 0.0;
    bool conv = false;
    int it = 0;
    for (; it < 3; it++) {
        for (int i = tid; i < n; i += T) {
            double a0 = 0.0, a1 = 0.0;
            const double* row = src + (size_t)i * n;
            int j = 0;
            for (; j + 1 < n; j += 2) { a0 = fma(row[j], v[j], a0); a1 = fma(row[j + 1], v[j + 1], a1); }
            if (j < n) a0 = fma(row[j], v[j], a0);
            y[i] = a0 + a1;
        }
        __syncthreads();
        if (tid < 32) {
            double ss = 0.0;
            for (int i = tid; i < n; i += 32) ss = fma(y[i], y[i], ss);
            ss = warp_sum(ss);
            const double nrm = sqrt(ss), inv = 1.0 / nrm;
            double df = 0.0;
            for (int i = tid; i < n; i += 32) {
                const double nv = y[i] * inv;
                df = fmax(df, fabs(nv - v[i]));
                v[i] = nv;
            }
            df = warp_max(df);
            if (tid == 0) { s_lam = nrm; s_diff = df; }
        }
        __syncthreads();
        lam = s_lam;
        conv = s_diff < 1e-11 && trdev < 1e-6;
    }
    // sign convention: the component of largest magnitude is positive.  (Own shared word + a barrier first:
    // compute-sanitizer racecheck flagged the earlier version, which reused s_lam here while slower threads could
    // still be reading the eigenvalue from it.)
    __shared__ double s_sgn;
    __syncthreads();
    if (tid == 0) {
        int im = 0;
        for (int i = 1; i < n; i++) if (fabs(v[i]) > fabs(v[im])) im = i;
        s_sgn = v[im] < 0.0 ? -1.0 : 1.0;
    }
    __syncthreads();
    const double sgn = s_sgn, ax = sqrt(lam);
    double* AX = na.axes + (size_t)node * nn;
    for (size_t e = tid; e < nn; e += T) {
        const int i = (int)(e / n), j = (int)(e - (size_t)i * n);
        AX[e] = (j == n - 1) ? sgn * v[i] * ax : 0.0;
    }
    if (tid == 0) {                 // the major-axis half reports through its own word
        st->pad = (conv && lam > 0.0) ? 0 : 1;
        st->sweeps = it;
    }
}

// ------------------------------------------------------------------ fmax + rescale + finish
__global__ void __launch_bounds__(256) fmax_partial_kernel(const double* __restrict__ P, const int* __restrict__ perm,
                                                           int64_t N, NodeArrays na, const JobL* __restrict__ jobs,
                                                           double* __restrict__ partial) {
    extern __shared__ double sm[];     // 8 warps x n
    __shared__ double wmax[8];
    const int n = na.n;
    const JobL jb = jobs[blockIdx.x];
    const int* pm = perm + (size_t)jb.level * N;
    const double* mu = na.mean + (size_t)jb.node * n;
    const double* AM = na.am + (size_t)jb.node * n * n;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* d = sm + (size_t)warp * n;
    double best = -INFINITY;
    // a job's rows are dealt over gridDim.y CTAs (a 2000-point node is only 16 jobs: too few CTAs otherwise)
    const int chunk = (jb.r1 - jb.r0 + (int)gridDim.y - 1) / (int)gridDim.y;
    const int rb = jb.r0 + (int)blockIdx.y * chunk, re = min(rb + chunk, jb.r1);
    for (int r = rb + warp; r < re; r += 8) {
        const size_t row = (size_t)pm[r] * n;
        __syncwarp();
        for (int i = lane; i < n; i += 32) d[i] = P[row + i] - mu[i];
        __syncwarp();
        double s = 0.0;
        for (int base = 0; base < n; base += 64) {
            double y0, y1;
            warp_matvec2(AM, n, n, d, base + lane, n, y0, y1);
            if (base + lane < n) s = fma(d[base + lane], y0, s);
            if (base + lane + 32 < n) s = fma(d[base + lane + 32], y1, s);
        }
        s = warp_sum(s);
        best = fmax(best, s);
    }
    if (lane == 0) wmax[warp] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        double b = wmax[0];
        for (int w = 1; w < 8; w++) b = fmax(b, wmax[w]);
        partial[(size_t)jb.slot * gridDim.y + blockIdx.y] = b;
    }
}

__global__ void __launch_bounds__(1024) scale_finish_kernel(NodeArrays na, const NodeRef* __restrict__ refs,
                                                           const double* __restrict__ partial, int pass,
                                                           double logvol_pref, int nsub) {
    __shared__ double s_mult;
    __shared__ double red[32];
    const int n = na.n, tid = threadIdx.x, T = blockDim.x;
    const NodeRef nr = refs[blockIdx.x];
    const size_t nn = (size_t)n * n;
    NodeStat* st = na.stat + nr.node;
    if (st->retry) return;          // covariance still being repaired: decomposed again first
    // max over the node's job partials: all threads, then one warp (a maximum does not depend on the order)
    {
        double m = -INFINITY;
        for (int k = tid; k < nr.nslots * nsub; k += T) m = fmax(m, partial[(size_t)nr.slot0 * nsub + k]);
        m = warp_max(m);
        if ((tid & 31) == 0) red[tid >> 5] = m;
        __syncthreads();
    }
    if (tid == 0) {
        double fm = -INFINITY;
        for (int k = 0; k < ((T + 31) >> 5); k++) fm = fmax(fm, red[k]);
        st->fmax = fm;
        double mult = 1.0;
        if (pass == 0) {
            if (fm > 1.0 - 1e-3) mult = fm / (1.0 - 1e-3);
            st->mult = mult;
            st->error = 0;
        } else if (fm >= 1.0) {
            st->error = B2N_ERR_ELL_INIT;
        }
        s_mult = mult;
    }
    __syncthreads();
    const double mult = s_mult;
    double* Cm = na.cov + (size_t)nr.node * nn;
    double* AM = na.am + (size_t)nr.node * nn;
    double* AX = na.axes + (size_t)nr.node * nn;
    double* LM = na.lam + (size_t)nr.node * n;
    if (mult != 1.0) {
        const double sq = sqrt(mult);
        for (size_t e = tid; e < nn; e += T) { Cm[e] *= mult; AM[e] /= mult; AX[e] *= sq; }
        for (int k = tid; k < n; k += T) LM[k] *= mult;
    }
    __syncthreads();
    // Ellipsoid.__init__ (:212-222): axlens, logvol, singularity check
    double part = 0.0;
    int bad = 0;
    for (int k = tid; k < n; k += T) {
        const double l = LM[k];
        if (!(l > 0.0) || !(l < INFINITY)) bad = 1;
        na.axlens[(size_t)nr.node * n + k] = sqrt(l);
        part += log(l);
    }
    const double tot = block_sum(part, red);
    const double nbad = block_sum((double)bad, red);
    if (tid == 0) {
        st->logvol = logvol_pref + 0.5 * tot;
        if (nbad > 0 && st->error == 0) st->error = B2N_ERR_SINGULAR;
    }
}

// ------------------------------------------------------------------ host orchestration

static double logvol_prefactor(int n) {   // bounding.py:1271-1285 (p = 2)
    return n * log(2.0) + n * lgamma(1.5) - lgamma(n / 2.0 + 1.0);
}

static size_t align8(size_t x) { return (x + 7) & ~(size_t)7; }

int b2n_boundwork_init(b2n_ctx* ctx, BoundWork& w, const double* dP, int64_t N, int n, int cap) {
    w.ctx = ctx; w.P = dP; w.N = N; w.n = n; w.cap = cap;
    w.logvol_pref = logvol_prefactor(n);
    const size_t nn = (size_t)n * n;
    size_t bytes = 0;
    const size_t o_mean = bytes; bytes += align8((size_t)cap * n * sizeof(double));
    const size_t o_covraw = bytes; bytes += (size_t)cap * nn * sizeof(double);
    const size_t o_cov = bytes; bytes += (size_t)cap * nn * sizeof(double);
    const size_t o_am = bytes; bytes += (size_t)cap * nn * sizeof(double);
    const size_t o_axes = bytes; bytes += (size_t)cap * nn * sizeof(double);
    const size_t o_lam = bytes; bytes += align8((size_t)cap * n * sizeof(double));
    const size_t o_axl = bytes; bytes += align8((size_t)cap * n * sizeof(double));
    const size_t o_stat = bytes; bytes += align8((size_t)cap * sizeof(NodeStat));
    B2N_CUDA(ctx, ctx->scratch0.ensure(bytes));
    char* b = ctx->scratch0.as<char>();
    w.na.n = n;
    w.na.ld = n | 1;
    w.na.mean = (double*)(b + o_mean); w.na.covraw = (double*)(b + o_covraw);
    w.na.cov = (double*)(b + o_cov); w.na.am = (double*)(b + o_am); w.na.axes = (double*)(b + o_axes);
    w.na.lam = (double*)(b + o_lam); w.na.axlens = (double*)(b + o_axl); w.na.stat = (NodeStat*)(b + o_stat);
    B2N_CUDA(ctx, ctx->scratch3.ensure((size_t)2 * N * sizeof(int)));
    w.perm = ctx->scratch3.as<int>();
    return B2N_OK;
}

// the jobs of a batch of nodes (b2n_rows_per_job rows each, slots numbered from 0); sets each ref's slot0 / nslots
static std::vector<JobL> node_jobs(std::vector<NodeRef>& refs, int64_t N) {
    const int rows = b2n_rows_per_job(N);
    std::vector<JobL> jobs;
    for (NodeRef& r : refs) {
        r.slot0 = (int)jobs.size();
        for (int a = r.start; a < r.start + r.count; a += rows)
            jobs.push_back(JobL{r.node, a, std::min(a + rows, r.start + r.count), (int)jobs.size(), r.level, 0, 0, 0});
        r.nslots = (int)jobs.size() - r.slot0;
    }
    return jobs;
}

// a batch of nodes on the device: its jobs (ctx->scratch4), refs (scratch5) and node ids (work0)
struct NodeBatch {
    int nnodes, njobs;
    const JobL* jobs;
    const NodeRef* refs;
    const int* list;
};

static int stage_nodes(BoundWork& w, std::vector<NodeRef> refs, NodeBatch& b) {
    b2n_ctx* ctx = w.ctx;
    const std::vector<JobL> jobs = node_jobs(refs, w.N);
    std::vector<int> list;
    for (const NodeRef& r : refs) list.push_back(r.node);
    const void *djobs, *drefs, *dlist;
    B2N_TRY(b2n_in_host(ctx, ctx->scratch4, jobs.data(), jobs.size() * sizeof(JobL), &djobs));
    B2N_TRY(b2n_in_host(ctx, ctx->scratch5, refs.data(), refs.size() * sizeof(NodeRef), &drefs));
    B2N_TRY(b2n_in_host(ctx, ctx->work0, list.data(), list.size() * sizeof(int), &dlist));
    b = NodeBatch{(int)refs.size(), (int)jobs.size(), (const JobL*)djobs, (const NodeRef*)drefs, (const int*)dlist};
    return B2N_OK;
}

// mean and sample covariance of every node of the batch -> na.mean / na.covraw; the per-job partials go to
// ctx->scratch1, which the fmax scan reuses
static int launch_moments(BoundWork& w, const NodeBatch& b) {
    b2n_ctx* ctx = w.ctx;
    const int n = w.n;
    const size_t nn = (size_t)n * n;
    B2N_CUDA(ctx, ctx->scratch1.ensure((size_t)b.njobs * std::max(nn, (size_t)n) * sizeof(double)));
    double* partial = ctx->scratch1.as<double>();
    cudaStream_t st = ctx->stream;
    colsum_partial_kernel<<<b.njobs, 256, (size_t)8 * n * sizeof(double), st>>>(w.P, w.perm, w.N, n, b.jobs, partial);
    B2N_LAUNCH_CHECK(ctx);
    mean_finalize_kernel<<<b.nnodes, 128, 0, st>>>(b.refs, n, partial, w.na.mean);
    B2N_LAUNCH_CHECK(ctx);
    const int ntile = (n + B2N_TILE - 1) / B2N_TILE;
    cov_partial_kernel<<<dim3(b.njobs, ntile * (ntile + 1) / 2), 256, 0, st>>>(w.P, w.perm, w.N, n, b.jobs, w.na.mean,
                                                                              partial, ntile);
    B2N_LAUNCH_CHECK(ctx);
    cov_finalize_kernel<<<dim3(b.nnodes, (unsigned)std::min<size_t>((nn + 255) / 256, 64)), 256, 0, st>>>(
        b.refs, n, partial, w.na.covraw);
    B2N_LAUNCH_CHECK(ctx);
    return B2N_OK;
}

// fmax scan of the batch's rows, then rescale + volume of its nodes; `wait`: an event the finish waits for
static int launch_fmax_finish(BoundWork& w, const NodeBatch& b, int pass, cudaEvent_t wait = nullptr) {
    b2n_ctx* ctx = w.ctx;
    cudaStream_t st = ctx->stream;
    double* partial = ctx->scratch1.as<double>();
    fmax_partial_kernel<<<dim3(b.njobs, B2N_FMAX_SUB), 256, (size_t)8 * w.n * sizeof(double), st>>>(w.P, w.perm, w.N,
                                                                                                  w.na, b.jobs, partial);
    B2N_LAUNCH_CHECK(ctx);
    if (wait) B2N_CUDA(ctx, cudaStreamWaitEvent(st, wait, 0));
    scale_finish_kernel<<<b.nnodes, 1024, 0, st>>>(w.na, b.refs, partial, pass, w.logvol_pref, B2N_FMAX_SUB);
    B2N_LAUNCH_CHECK(ctx);
    return B2N_OK;
}

// The single-CTA eigen solve (eig_ladder_kernel): both n x ld work matrices in shared memory when they fit, else in a
// global workspace of gwork_bytes per node (used only if the sliced solver cannot take the matrix either).  One
// HALF-warp per rotation pair of a Jacobi round (n/2 pairs), at least 4 warps for the O(n^2) loops.
struct EigPlan {
    bool smem;
    size_t smem_bytes, gwork_bytes;
    int threads;
};

static EigPlan eig_plan(const BoundWork& w) {
    const int n = w.n, half = ((n + 1) & ~1) / 2;
    const size_t small_b = (size_t)(2 * half + 2 * n + 32) * sizeof(double);
    const size_t mats_b = (size_t)2 * n * w.na.ld * sizeof(double);
    const bool smem = small_b + mats_b <= (size_t)w.ctx->max_smem_optin;
    return EigPlan{smem, small_b + (smem ? mats_b : 0), mats_b, 32 * std::max(4, std::min(32, (half + 1) / 2))};
}

static int launch_eig(BoundWork& w, const EigPlan& p, const NodeArrays& na, const int* dlist, int pn, int pass,
                      double* gwork, cudaStream_t st) {
    b2n_ctx* ctx = w.ctx;
    if (p.smem) {
        B2N_TRY(b2n_func_smem(ctx, (const void*)(eig_ladder_kernel<true>), p.smem_bytes));
        eig_ladder_kernel<true><<<pn, p.threads, p.smem_bytes, st>>>(na, dlist, pass, gwork);
    } else {
        B2N_TRY(b2n_func_smem(ctx, (const void*)(eig_ladder_kernel<false>), p.smem_bytes));
        eig_ladder_kernel<false><<<pn, p.threads, p.smem_bytes, st>>>(na, dlist, pass, gwork);
    }
    B2N_LAUNCH_CHECK(ctx);
    return B2N_OK;
}

// a high-priority non-blocking stream and its two events, created on first use
static int side_stream(b2n_ctx* ctx, cudaStream_t& s, cudaEvent_t& done, cudaEvent_t& go) {
    if (s) return B2N_OK;
    int lo = 0, hi = 0;
    if (cudaDeviceGetStreamPriorityRange(&lo, &hi) != cudaSuccess) { cudaGetLastError(); hi = 0; }
    B2N_CUDA(ctx, cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, hi));
    B2N_CUDA(ctx, cudaEventCreateWithFlags(&done, cudaEventDisableTiming));
    B2N_CUDA(ctx, cudaEventCreateWithFlags(&go, cudaEventDisableTiming));
    return B2N_OK;
}

// Full bounding_ellipsoid (bounding.py:1387-1461) for every node in `refs`.
// On return `stats` holds the per-node NodeStat (host copy); the stream is synchronised.
int b2n_fit_nodes(BoundWork& w, const std::vector<NodeRef>& refs, std::vector<NodeStat>& stats) {
    b2n_ctx* ctx = w.ctx;
    const int nnodes = (int)refs.size();
    if (nnodes == 0) return B2N_OK;
    cudaStream_t st = ctx->stream;
    NodeBatch b;
    B2N_TRY(stage_nodes(w, refs, b));
    B2N_TRY(launch_moments(w, b));
    // eigen + ladder.  large n: packed-triangle / column-sliced Jacobi (b2n_eig_sliced.cu); else the single-CTA kernel
    const EigPlan ep = eig_plan(w);
    double* gwork = nullptr;
    if (!ep.smem) {
        B2N_CUDA(ctx, ctx->scratch2.ensure((size_t)nnodes * ep.gwork_bytes));
        gwork = ctx->scratch2.as<double>();
    }
    std::vector<NodeStat> hs(nnodes), all;
    std::vector<int> which(nnodes);
    for (int i = 0; i < nnodes; i++) which[i] = i;
    for (int pass = 0; pass < 2; pass++) {
        if (pass == 1) {
            // second pass only for nodes whose matrix needed repair (:1454-1457)
            std::vector<NodeRef> refs2;
            which.clear();
            for (int i = 0; i < nnodes; i++)
                if (!hs[i].good && !hs[i].error) { refs2.push_back(refs[i]); which.push_back(i); }
            if (refs2.empty()) break;
            B2N_TRY(stage_nodes(w, refs2, b));
        }
        int sliced = 0;
        if (!ep.smem) B2N_TRY(b2n_eig_sliced(w, b.list, b.nnodes, pass, 0, &sliced));
        if (!sliced) B2N_TRY(launch_eig(w, ep, w.na, b.list, b.nnodes, pass, gwork, st));
        B2N_TRY(launch_fmax_finish(w, b, pass));
        B2N_CUDA(ctx, cudaStreamSynchronize(st));
        B2N_TRY(b2n_read_stats(w, all));
        for (int i : which) hs[i] = all[refs[i].node];
        // sliced path: the repair ladder is one decomposition per launch -> re-run the nodes whose covariance was
        // modified (rare: rank-deficient / ill-conditioned clouds).  Attempt 99 is a node's 100th decomposition, at
        // which eig_check_kernel ends the ladder (identity fallback, retry cleared): no node is left to retry.
        for (int attempt = 1; sliced && attempt < 100; attempt++) {
            std::vector<NodeRef> refs3;
            std::vector<int> again;
            for (int i = 0; i < nnodes; i++)
                if (hs[i].retry) { refs3.push_back(refs[i]); again.push_back(i); }
            if (refs3.empty()) break;
            NodeBatch r;
            B2N_TRY(stage_nodes(w, refs3, r));
            int used = 0;
            B2N_TRY(b2n_eig_sliced(w, r.list, r.nnodes, pass, 1, &used));
            B2N_TRY(launch_fmax_finish(w, r, pass));
            B2N_CUDA(ctx, cudaStreamSynchronize(st));
            B2N_TRY(b2n_read_stats(w, all));
            for (int i : again) hs[i] = all[refs[i].node];
        }
    }
    stats = hs;
    return B2N_OK;
}

// The candidates of a multi-ellipsoid tree through the Cholesky path (chol_node_kernel): moments, then the two halves
// of the fit side by side -- the major axes (repeated squaring) on a side stream, Cholesky / precision matrix / fmax
// scan on the main one -- meeting before scale_finish (which rescales the axes).  Nothing on the host depends on a
// candidate's stats before the end of the expansion (a certified candidate never takes the second pass): this only
// enqueues, the caller reads them all at once (b2n_read_stats) and the next level's launches queue behind these
// without a host round trip.
int b2n_fit_candidates(BoundWork& w, const std::vector<NodeRef>& refs) {
    b2n_ctx* ctx = w.ctx;
    if (refs.empty()) return B2N_OK;
    const int n = w.n, ld = w.na.ld;
    cudaStream_t st = ctx->stream;
    NodeBatch b;
    B2N_TRY(stage_nodes(w, refs, b));
    B2N_TRY(launch_moments(w, b));
    B2N_TRY(side_stream(ctx, ctx->stream_side2, ctx->ev_side2, ctx->ev_side2_go));
    const size_t csm = (size_t)(2 * n * ld + 3 * n + 32 + 2 * (n + 2)) * sizeof(double);
    B2N_TRY(b2n_func_smem(ctx, (const void*)(chol_node_kernel<1>), csm));
    B2N_TRY(b2n_func_smem(ctx, (const void*)(chol_node_kernel<2>), csm));
    B2N_CUDA(ctx, cudaEventRecord(ctx->ev_side2_go, st));
    B2N_CUDA(ctx, cudaStreamWaitEvent(ctx->stream_side2, ctx->ev_side2_go, 0));
    chol_node_kernel<2><<<b.nnodes, 512, csm, ctx->stream_side2>>>(w.na, b.list);
    B2N_LAUNCH_CHECK(ctx);
    B2N_CUDA(ctx, cudaEventRecord(ctx->ev_side2, ctx->stream_side2));
    chol_node_kernel<1><<<b.nnodes, 512, csm, st>>>(w.na, b.list);
    B2N_LAUNCH_CHECK(ctx);
    return launch_fmax_finish(w, b, 0, ctx->ev_side2);
}

// ------------------------------------------------------------------ speculative fit of the root node
// _bounding_ellipsoids (bounding.py:1464-1563) returns the ROOT ellipsoid whenever no split of the candidate tree
// is accepted -- every update of a unimodal live set (C2).  An accepted leaf needs the full eigen fit (axes,
// axlens, the reference's repair ladder): moments + eig_ladder + fmax + finish = 0.75 ms of single-CTA latency
// at n = 50 that used to FOLLOW the ~1.9 ms of the candidate tree.  The root's fit depends on the root's moments
// only, and those exist after the first candidate launch: it is issued on a second (high-priority) stream into
// SHADOW arrays, occupies one SM while the tree is expanded on the others, and is adopted at the end if the root
// is the accepted leaf and its covariance needed no repair (otherwise the ordinary re-fit runs, as before).
// Reads shared with the main stream are read-only there (points, mean / covraw of node 0); the row order is a
// private copy of perm level 0 (the ping-pong buffer is overwritten two levels down).
int b2n_spec_root_launch(BoundWork& w, int count, SpecRoot& sp) {
    b2n_ctx* ctx = w.ctx;
    const int n = w.n;
    const size_t nn = (size_t)n * n;
    sp.launched = false;
    const EigPlan ep = eig_plan(w);
    if (!ep.smem) return B2N_OK;          // sliced solver territory: no speculation
    B2N_TRY(side_stream(ctx, ctx->stream_side, ctx->ev_side, ctx->ev_side_go));
    cudaStream_t side = ctx->stream_side;
    std::vector<NodeRef> refs(1, b2n_node_ref(0, 0, count, 0));
    sp.jobs = node_jobs(refs, w.N);
    sp.ref = refs[0];
    const int njobs = (int)sp.jobs.size();
    sp.node0 = 0;
    size_t bytes = 0;
    auto take = [&bytes](size_t b) { const size_t o = bytes; bytes += (b + 255) & ~(size_t)255; return o; };
    const size_t o_perm = take((size_t)w.N * sizeof(int));
    const size_t o_jobs = take((size_t)njobs * sizeof(JobL));
    const size_t o_ref = take(sizeof(NodeRef));
    const size_t o_list = take(sizeof(int));
    const size_t o_part = take((size_t)njobs * B2N_FMAX_SUB * sizeof(double));
    const size_t o_cov = take(nn * sizeof(double)), o_am = take(nn * sizeof(double)), o_axes = take(nn * sizeof(double));
    const size_t o_lam = take((size_t)n * sizeof(double)), o_axl = take((size_t)n * sizeof(double));
    const size_t o_stat = take(sizeof(NodeStat));
    B2N_CUDA(ctx, ctx->spec.ensure(bytes));
    char* b = ctx->spec.as<char>();
    sp.perm = (int*)(b + o_perm);
    sp.na = w.na;                          // mean / covraw: the main arrays (node 0, read-only from here on)
    sp.na.cov = (double*)(b + o_cov); sp.na.am = (double*)(b + o_am); sp.na.axes = (double*)(b + o_axes);
    sp.na.lam = (double*)(b + o_lam); sp.na.axlens = (double*)(b + o_axl); sp.na.stat = (NodeStat*)(b + o_stat);
    // the row order of the root: copied on the MAIN stream (ordered before the partitions that recycle the buffer)
    B2N_CUDA(ctx, cudaMemcpyAsync(sp.perm, w.perm, (size_t)w.N * sizeof(int), cudaMemcpyDeviceToDevice, ctx->stream));
    B2N_CUDA(ctx, cudaEventRecord(ctx->ev_side_go, ctx->stream));
    B2N_CUDA(ctx, cudaStreamWaitEvent(side, ctx->ev_side_go, 0));
    B2N_CUDA(ctx, cudaMemcpyAsync(b + o_jobs, sp.jobs.data(), (size_t)njobs * sizeof(JobL), cudaMemcpyHostToDevice, side));
    B2N_CUDA(ctx, cudaMemcpyAsync(b + o_ref, &sp.ref, sizeof(NodeRef), cudaMemcpyHostToDevice, side));
    B2N_CUDA(ctx, cudaMemcpyAsync(b + o_list, &sp.node0, sizeof(int), cudaMemcpyHostToDevice, side));
    B2N_CUDA(ctx, cudaMemsetAsync(b + o_stat, 0, sizeof(NodeStat), side));
    B2N_TRY(launch_eig(w, ep, sp.na, (const int*)(b + o_list), 1, 0, nullptr, side));
    fmax_partial_kernel<<<dim3(njobs, B2N_FMAX_SUB), 256, (size_t)8 * n * sizeof(double), side>>>(
        w.P, sp.perm, w.N, sp.na, (const JobL*)(b + o_jobs), (double*)(b + o_part));
    B2N_LAUNCH_CHECK(ctx);
    scale_finish_kernel<<<1, 1024, 0, side>>>(sp.na, (const NodeRef*)(b + o_ref), (const double*)(b + o_part), 0,
                                              w.logvol_pref, B2N_FMAX_SUB);
    B2N_LAUNCH_CHECK(ctx);
    B2N_CUDA(ctx, cudaEventRecord(ctx->ev_side, side));
    sp.launched = true;
    return B2N_OK;
}

// Wait for the speculative fit; *ok = it is the fit the ordinary path would have produced for node 0 (covariance
// accepted untouched, no error) and its arrays are now node 0's.
int b2n_spec_root_adopt(BoundWork& w, SpecRoot& sp, NodeStat* stat, bool* ok) {
    b2n_ctx* ctx = w.ctx;
    *ok = false;
    if (!sp.launched) return B2N_OK;
    B2N_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_side, 0));
    NodeStat hs;
    B2N_CUDA(ctx, b2n_copy_sync(ctx, &hs, sp.na.stat, sizeof(NodeStat), cudaMemcpyDeviceToHost));
    if (!hs.good || hs.fallback || hs.error || hs.retry) return B2N_OK;
    const size_t n = w.n, nn = n * n;
    cudaStream_t st = ctx->stream;
    B2N_CUDA(ctx, cudaMemcpyAsync(w.na.cov, sp.na.cov, nn * sizeof(double), cudaMemcpyDeviceToDevice, st));
    B2N_CUDA(ctx, cudaMemcpyAsync(w.na.am, sp.na.am, nn * sizeof(double), cudaMemcpyDeviceToDevice, st));
    B2N_CUDA(ctx, cudaMemcpyAsync(w.na.axes, sp.na.axes, nn * sizeof(double), cudaMemcpyDeviceToDevice, st));
    B2N_CUDA(ctx, cudaMemcpyAsync(w.na.lam, sp.na.lam, n * sizeof(double), cudaMemcpyDeviceToDevice, st));
    B2N_CUDA(ctx, cudaMemcpyAsync(w.na.axlens, sp.na.axlens, n * sizeof(double), cudaMemcpyDeviceToDevice, st));
    B2N_CUDA(ctx, cudaMemcpyAsync(w.na.stat, sp.na.stat, sizeof(NodeStat), cudaMemcpyDeviceToDevice, st));
    *stat = hs;
    *ok = true;
    return B2N_OK;
}

void b2n_spec_root_wait(b2n_ctx* ctx, SpecRoot& sp) {
    if (sp.launched && ctx->stream_side) cudaStreamSynchronize(ctx->stream_side);
    sp.launched = false;
}

// host copy of every node's NodeStat (the stream is synchronised on return)
int b2n_read_stats(BoundWork& w, std::vector<NodeStat>& all) {
    all.resize(w.cap);
    B2N_CUDA(w.ctx, b2n_copy_sync(w.ctx, all.data(), w.na.stat, (size_t)w.cap * sizeof(NodeStat), cudaMemcpyDeviceToHost));
    return B2N_OK;
}

// np.mean / np.cov(ddof=1) of one node (rows [0, count) of perm level 0): the moment kernels of b2n_fit_nodes
// without the eigen / fmax stages (used by b2n_friends.cu)
int b2n_node_moments(BoundWork& w, int count) {
    b2n_ctx* ctx = w.ctx;
    std::vector<NodeRef> refs(1, b2n_node_ref(0, 0, count, 0));
    const std::vector<JobL> jobs = node_jobs(refs, w.N);
    const void *djobs, *drefs;
    B2N_TRY(b2n_in_host(ctx, ctx->scratch4, jobs.data(), jobs.size() * sizeof(JobL), &djobs));
    B2N_TRY(b2n_in_host(ctx, ctx->scratch5, refs.data(), sizeof(NodeRef), &drefs));
    return launch_moments(w, NodeBatch{1, (int)jobs.size(), (const JobL*)djobs, (const NodeRef*)drefs, nullptr});
}

int b2n_init_identity_perm(BoundWork& w) {
    std::vector<int> id(w.N);
    for (int64_t i = 0; i < w.N; i++) id[i] = (int)i;
    B2N_CUDA(w.ctx, cudaMemcpyAsync(w.perm, id.data(), w.N * sizeof(int), cudaMemcpyHostToDevice, w.ctx->stream));
    return B2N_OK;
}

// copy node `node` arrays to caller outputs (device or host according to pointer mode)
int b2n_emit_node(BoundWork& w, int node, int k, double* ctr, double* cov, double* am, double* axes, double* axlens) {
    b2n_ctx* ctx = w.ctx;
    const size_t n = w.n, nn = n * n;
    const cudaMemcpyKind kind = ctx->ptr_mode == B2N_PTR_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    if (ctr) B2N_CUDA(ctx, cudaMemcpyAsync(ctr + k * n, w.na.mean + node * n, n * sizeof(double), kind, ctx->stream));
    if (cov) B2N_CUDA(ctx, cudaMemcpyAsync(cov + k * nn, w.na.cov + node * nn, nn * sizeof(double), kind, ctx->stream));
    if (am) B2N_CUDA(ctx, cudaMemcpyAsync(am + k * nn, w.na.am + node * nn, nn * sizeof(double), kind, ctx->stream));
    if (axes) B2N_CUDA(ctx, cudaMemcpyAsync(axes + k * nn, w.na.axes + node * nn, nn * sizeof(double), kind, ctx->stream));
    if (axlens) B2N_CUDA(ctx, cudaMemcpyAsync(axlens + k * n, w.na.axlens + node * n, n * sizeof(double), kind, ctx->stream));
    return B2N_OK;
}

extern "C" int b2n_bounding_ellipsoid(b2n_ctx* ctx, const double* points, int64_t N, int32_t n, double* ctr,
                                      double* cov, double* am, double* axes, double* axlens, double* logvol,
                                      uint32_t* warn) {
    if (!ctx || !points || N < 1 || n < 1) return B2N_ERR_ARG;
    if (N == 1) return B2N_ERR_SINGLE_POINT;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    const void* dP;
    B2N_TRY(b2n_in(ctx, ctx->in0, points, (size_t)N * n * sizeof(double), &dP));
    BoundWork w;
    B2N_TRY(b2n_boundwork_init(ctx, w, (const double*)dP, N, n, 1));
    B2N_TRY(b2n_init_identity_perm(w));
    std::vector<NodeStat> hs;
    B2N_TRY(b2n_fit_nodes(w, std::vector<NodeRef>(1, b2n_node_ref(0, 0, (int)N, 0)), hs));
    if (warn) *warn = hs[0].fallback ? B2N_WARN_IDENTITY_FALLBACK : 0u;
    if (hs[0].error) return hs[0].error;
    B2N_TRY(b2n_emit_node(w, 0, 0, ctr, cov, am, axes, axlens));
    if (logvol) {
        if (ctx->ptr_mode == B2N_PTR_DEVICE)
            B2N_CUDA(ctx, cudaMemcpyAsync(logvol, &hs[0].logvol, sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        else
            *logvol = hs[0].logvol;
    }
    B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B2N_OK;
}

// Moments of a block of points: count-weighted building blocks of the covariance of a row-SHARDED live set
// (SURVEY 8e: all-reduce of (count, sum x, sum x x^T) at the bound update).  mean = np.mean(points, 0),
// cov = np.cov(points, rowvar=False) (ddof = 1) of THIS block; blocks combine exactly through
//   S = sum_r [ (N_r - 1) cov_r + N_r (mean_r - mean)(mean_r - mean)^T ],  cov = S / (N - 1).
extern "C" int b2n_moments(b2n_ctx* ctx, const double* points, int64_t N, int32_t n, double* mean, double* cov) {
    if (!ctx || !points || N < 1 || n < 1 || !mean || !cov) return B2N_ERR_ARG;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    const void* dP;
    B2N_TRY(b2n_in(ctx, ctx->in0, points, (size_t)N * n * sizeof(double), &dP));
    BoundWork w;
    B2N_TRY(b2n_boundwork_init(ctx, w, (const double*)dP, N, n, 1));
    B2N_TRY(b2n_init_identity_perm(w));
    B2N_TRY(b2n_node_moments(w, (int)N));
    if (N == 1) B2N_CUDA(ctx, cudaMemsetAsync(w.na.covraw, 0, (size_t)n * n * sizeof(double), ctx->stream));   // (ddof = 1)
    B2N_TRY(b2n_emit_node(w, 0, 0, mean, nullptr, nullptr, nullptr, nullptr));
    const cudaMemcpyKind kind = ctx->ptr_mode == B2N_PTR_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    B2N_CUDA(ctx, cudaMemcpyAsync(cov, w.na.covraw, (size_t)n * n * sizeof(double), kind, ctx->stream));
    B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B2N_OK;
}

// improve_covar_mat (bounding.py:1311-1384) on a caller-supplied matrix: the repair ladder of the fit
// kernels exposed on its own (the same eig_ladder_kernel / sliced solver, fed through `covraw`).
extern "C" int b2n_improve_covar(b2n_ctx* ctx, const double* covar, int32_t n, double* cov_out, double* am,
                                 double* axes, int32_t* good, uint32_t* warn) {
    if (!ctx || !covar || n < 1) return B2N_ERR_ARG;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    BoundWork w;
    B2N_TRY(b2n_boundwork_init(ctx, w, nullptr, 1, n, 1));
    const size_t nn = (size_t)n * n;
    cudaStream_t st = ctx->stream;
    const cudaMemcpyKind in_kind = ctx->ptr_mode == B2N_PTR_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    B2N_CUDA(ctx, cudaMemcpyAsync(w.na.covraw, covar, nn * sizeof(double), in_kind, st));
    B2N_CUDA(ctx, cudaMemsetAsync(w.na.stat, 0, sizeof(NodeStat), st));
    const int zero = 0;
    const void* dlist;
    B2N_TRY(b2n_in_host(ctx, ctx->work0, &zero, sizeof(int), &dlist));
    const EigPlan ep = eig_plan(w);
    NodeStat hs;
    memset(&hs, 0, sizeof(hs));
    int sliced = 0;
    if (!ep.smem) {
        B2N_TRY(b2n_eig_sliced(w, (const int*)dlist, 1, 0, 0, &sliced));
        // one decomposition per launch; attempt 99 is the 100th, which ends the ladder (eig_check_kernel)
        for (int attempt = 1; sliced && attempt <= 100; attempt++) {
            B2N_CUDA(ctx, cudaStreamSynchronize(st));
            B2N_CUDA(ctx, b2n_copy_sync(ctx, &hs, w.na.stat, sizeof(NodeStat), cudaMemcpyDeviceToHost));
            if (!hs.retry) break;
            int used = 0;
            B2N_TRY(b2n_eig_sliced(w, (const int*)dlist, 1, 0, 1, &used));
        }
    }
    if (!sliced) {
        double* gwork = nullptr;
        if (!ep.smem) {
            B2N_CUDA(ctx, ctx->scratch2.ensure(ep.gwork_bytes));
            gwork = ctx->scratch2.as<double>();
        }
        B2N_TRY(launch_eig(w, ep, w.na, (const int*)dlist, 1, 0, gwork, st));
    }
    B2N_CUDA(ctx, cudaStreamSynchronize(st));
    B2N_CUDA(ctx, b2n_copy_sync(ctx, &hs, w.na.stat, sizeof(NodeStat), cudaMemcpyDeviceToHost));
    if (good) *good = hs.good;
    if (warn) *warn = hs.fallback ? B2N_WARN_IDENTITY_FALLBACK : 0u;
    B2N_TRY(b2n_emit_node(w, 0, 0, nullptr, cov_out, am, axes, nullptr));
    B2N_CUDA(ctx, cudaStreamSynchronize(st));
    return B2N_OK;
}

// ------------------------------------------------------------------ FP64 issue ceilings (bench.py roofline)
// What the chain kernels are made of is FP64 FMA (vector pipe) and FP64 MMA (tensor pipe, DMMA).  Both ceilings are
// MEASURED here instead of quoted: every warp runs `iters` rounds of 16 independent dependency chains (DFMA: 16
// accumulators per thread; m8n8k4: 8 accumulator pairs per warp; the m16n8 shapes: 4 accumulator quads per warp),
// 8 warps x 8 CTAs per SM.  KIND: 0 DFMA, 1 m8n8k4, 2 m16n8k4, 3 m16n8k8, 4 m16n8k16 (bench.py reports against 0, 1).
template <int KIND>
__device__ __forceinline__ void fp64_op(double* acc, double a, double b) {
    if constexpr (KIND == 0) {
        acc[0] = fma(acc[0], a, b);
    } else if constexpr (KIND == 1) {
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                     : "+d"(acc[0]), "+d"(acc[1])
                     : "d"(a), "d"(b));
    } else if constexpr (KIND == 2) {
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                     : "+d"(acc[0]), "+d"(acc[1]), "+d"(acc[2]), "+d"(acc[3])
                     : "d"(a), "d"(a), "d"(b));
    } else if constexpr (KIND == 3) {
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                     "{%0,%1,%2,%3};\n"
                     : "+d"(acc[0]), "+d"(acc[1]), "+d"(acc[2]), "+d"(acc[3])
                     : "d"(a), "d"(a), "d"(a), "d"(a), "d"(b), "d"(b));
    } else {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                     "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
                     : "+d"(acc[0]), "+d"(acc[1]), "+d"(acc[2]), "+d"(acc[3])
                     : "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(b), "d"(b), "d"(b), "d"(b));
    }
}
// accumulator doubles per lane of one instruction, flop per instruction (DFMA: per lane; MMA: per warp)
__host__ __device__ constexpr int fp64_acc(int kind) { return kind == 0 ? 1 : (kind == 1 ? 2 : 4); }
static double fp64_flop(int kind) { return kind == 0 ? 2.0 : 2.0 * (kind == 1 ? 8 : 16) * 8 * (kind <= 2 ? 4 : (kind == 3 ? 8 : 16)); }

template <int KIND>
__global__ void __launch_bounds__(256) fp64_peak_kernel(int iters, double seed, double* __restrict__ out) {
    double acc[16];
#pragma unroll
    for (int i = 0; i < 16; i++) acc[i] = seed * (double)(threadIdx.x + i + 1);
    const double a = 1.0 + 1e-9 * seed, b = 1e-9 * (double)(threadIdx.x & 3);
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < 16; i += fp64_acc(KIND)) fp64_op<KIND>(&acc[i], a, b);
    }
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 16; i++) s += acc[i];
    if (s == 123456.789) out[blockIdx.x * blockDim.x + threadIdx.x] = s;     // keeps the chains alive
}

// Dependent-issue latency: ONE warp, ONE dependency chain of `iters` instructions, timed in SM clocks.
template <int KIND>
__global__ void __launch_bounds__(32) fp64_latency_kernel(int iters, double seed, long long* __restrict__ cyc,
                                                          double* __restrict__ out) {
    double acc[4];
#pragma unroll
    for (int i = 0; i < 4; i++) acc[i] = seed * (double)(threadIdx.x + i + 1);
    const double a = 1.0 + 1e-9 * seed, b = 1e-9 * (double)(threadIdx.x & 3);
    __syncwarp();
    const long long t0 = clock64();
    for (int it = 0; it < iters; it++) fp64_op<KIND>(acc, a, b);
    const long long t1 = clock64();
    const double s = acc[0] + acc[1] + acc[2] + acc[3];
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
    if (s == 123456.789) out[threadIdx.x] = s;
}

#define B2N_FP64_KIND(K_, CALL) \
    switch (K_) { case 0: CALL(0); break; case 1: CALL(1); break; case 2: CALL(2); break; case 3: CALL(3); break; default: CALL(4); break; }

extern "C" int b2n_fp64_peak(b2n_ctx* ctx, int32_t kind, int32_t iters, double* tflops, double* ms_out) {
    if (!ctx || kind < 0 || kind > 4 || iters < 1 || !tflops) return B2N_ERR_ARG;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    const int ctas = ctx->sm_count * 8, threads = 256;
    B2N_CUDA(ctx, ctx->scratch1.ensure((size_t)ctas * threads * sizeof(double)));
    cudaEvent_t e0, e1;
    B2N_CUDA(ctx, cudaEventCreate(&e0));
    B2N_CUDA(ctx, cudaEventCreate(&e1));
    cudaStream_t st = ctx->stream;
    float best = 1e30f;
    for (int rep = 0; rep < 5; rep++) {          // rep 0 warms up; best of the rest
        cudaEventRecord(e0, st);
#define B2N_PEAK(K) fp64_peak_kernel<K><<<ctas, threads, 0, st>>>(iters, 1.0 + rep, ctx->scratch1.as<double>())
        B2N_FP64_KIND(kind, B2N_PEAK)
#undef B2N_PEAK
        cudaEventRecord(e1, st);
        ctx->launches++;
        B2N_CUDA(ctx, cudaEventSynchronize(e1));
        float ms = 0.f;
        B2N_CUDA(ctx, cudaEventElapsedTime(&ms, e0, e1));
        if (rep > 0 && ms < best) best = ms;
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    B2N_CUDA(ctx, cudaGetLastError());
    // flop: DFMA 2 per lane per instruction; DMMA m x n x k: 2 m n k per warp instruction (m8n8k4: 512)
    const double per_thread_instr = (double)iters * (16.0 / fp64_acc(kind));
    const double flops = kind == 0 ? per_thread_instr * fp64_flop(0) * (double)ctas * threads
                                   : per_thread_instr * fp64_flop(kind) * (double)ctas * (threads / 32);
    *tflops = flops / ((double)best * 1e-3) / 1e12;
    if (ms_out) *ms_out = (double)best;
    return B2N_OK;
}

extern "C" int b2n_fp64_latency(b2n_ctx* ctx, int32_t kind, int32_t iters, double* cycles) {
    if (!ctx || kind < 0 || kind > 4 || iters < 1 || !cycles) return B2N_ERR_ARG;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    B2N_CUDA(ctx, ctx->scratch1.ensure(32 * sizeof(double) + sizeof(long long)));
    double* out = ctx->scratch1.as<double>();
    long long* cyc = reinterpret_cast<long long*>(out + 32);
    cudaStream_t st = ctx->stream;
    double best = 1e30;
    for (int rep = 0; rep < 5; rep++) {          // rep 0 warms up; best of the rest
#define B2N_LAT(K) fp64_latency_kernel<K><<<1, 32, 0, st>>>(iters, 1.0 + rep, cyc, out)
        B2N_FP64_KIND(kind, B2N_LAT)
#undef B2N_LAT
        ctx->launches++;
        B2N_CUDA(ctx, cudaGetLastError());
        long long c = 0;
        B2N_CUDA(ctx, b2n_copy_sync(ctx, &c, cyc, sizeof(c), cudaMemcpyDeviceToHost));
        if (rep > 0 && (double)c < best) best = (double)c;
    }
    *cycles = best / (double)iters;
    return B2N_OK;
}
#undef B2N_FP64_KIND

// Bit-identity probe of the FP64 MMA shapes: one warp per 16 x 8 tile, A 16 x 8, B 8 x 8 (k x n), C 16 x 8, all
// row-major.  out[4][tile][16 x 8]:
//   0  m16n8k4 (k 0..3) + C
//   1  two m8n8k4 (rows 0..7, rows 8..15; k 0..3) + C
//   2  m16n8k8 (k 0..7) + C
//   3  two chained m16n8k4 (k 0..3, then k 4..7) + C
// Fragments (PTX ISA, mma .f64): g = lane / 4, t = lane % 4; A rows g / g + 8, column t (+ 4 for the k 4..7 half);
// B row t (+ 4), column g; C / D rows g / g + 8, columns 2 t, 2 t + 1.
__global__ void __launch_bounds__(32) dmma_probe_kernel(const double* __restrict__ A, const double* __restrict__ B,
                                                        const double* __restrict__ Cm, double* __restrict__ out, int ntiles) {
    const int tile = blockIdx.x, lane = threadIdx.x, g = lane >> 2, t = lane & 3;
    const double* a = A + (size_t)tile * 128;
    const double* b = B + (size_t)tile * 64;
    const double* c = Cm + (size_t)tile * 128;
    const double a00 = a[g * 8 + t], a10 = a[(g + 8) * 8 + t], a01 = a[g * 8 + t + 4], a11 = a[(g + 8) * 8 + t + 4];
    const double b0 = b[t * 8 + g], b1 = b[(t + 4) * 8 + g];
    const double c0 = c[g * 8 + 2 * t], c1 = c[g * 8 + 2 * t + 1], c2 = c[(g + 8) * 8 + 2 * t], c3 = c[(g + 8) * 8 + 2 * t + 1];
    double r[4][4];
    r[0][0] = c0; r[0][1] = c1; r[0][2] = c2; r[0][3] = c3;
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(r[0][0]), "+d"(r[0][1]), "+d"(r[0][2]), "+d"(r[0][3]) : "d"(a00), "d"(a10), "d"(b0));
    r[1][0] = c0; r[1][1] = c1; r[1][2] = c2; r[1][3] = c3;
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(r[1][0]), "+d"(r[1][1]) : "d"(a00), "d"(b0));
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(r[1][2]), "+d"(r[1][3]) : "d"(a10), "d"(b0));
    r[2][0] = c0; r[2][1] = c1; r[2][2] = c2; r[2][3] = c3;
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+d"(r[2][0]), "+d"(r[2][1]), "+d"(r[2][2]), "+d"(r[2][3])
                 : "d"(a00), "d"(a10), "d"(a01), "d"(a11), "d"(b0), "d"(b1));
    r[3][0] = c0; r[3][1] = c1; r[3][2] = c2; r[3][3] = c3;
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(r[3][0]), "+d"(r[3][1]), "+d"(r[3][2]), "+d"(r[3][3]) : "d"(a00), "d"(a10), "d"(b0));
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(r[3][0]), "+d"(r[3][1]), "+d"(r[3][2]), "+d"(r[3][3]) : "d"(a01), "d"(a11), "d"(b1));
#pragma unroll
    for (int o = 0; o < 4; o++) {
        double* d = out + ((size_t)o * ntiles + tile) * 128;
        d[g * 8 + 2 * t] = r[o][0];
        d[g * 8 + 2 * t + 1] = r[o][1];
        d[(g + 8) * 8 + 2 * t] = r[o][2];
        d[(g + 8) * 8 + 2 * t + 1] = r[o][3];
    }
}

extern "C" int b2n_dmma_probe(b2n_ctx* ctx, int32_t ntiles, const double* a, const double* b, const double* c,
                              double* out) {
    if (!ctx || ntiles < 1 || !a || !b || !c || !out) return B2N_ERR_ARG;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    const void *da, *db, *dc;
    B2N_TRY(b2n_in_host(ctx, ctx->in0, a, (size_t)ntiles * 128 * sizeof(double), &da));
    B2N_TRY(b2n_in_host(ctx, ctx->in1, b, (size_t)ntiles * 64 * sizeof(double), &db));
    B2N_TRY(b2n_in_host(ctx, ctx->in2, c, (size_t)ntiles * 128 * sizeof(double), &dc));
    const size_t ob = (size_t)4 * ntiles * 128 * sizeof(double);
    B2N_CUDA(ctx, ctx->out0.ensure(ob));
    dmma_probe_kernel<<<ntiles, 32, 0, ctx->stream>>>((const double*)da, (const double*)db, (const double*)dc,
                                                      ctx->out0.as<double>(), ntiles);
    B2N_LAUNCH_CHECK(ctx);
    B2N_CUDA(ctx, b2n_copy_sync(ctx, out, ctx->out0.p, ob, cudaMemcpyDeviceToHost));
    return B2N_OK;
}

// ------------------------------------------------------------------ scale_to_logvol
// Ellipsoid.scale_to_logvol (bounding.py:242-276); one CTA per ellipsoid.
__global__ void __launch_bounds__(1024) scale_to_logvol_kernel(int n, double* __restrict__ covs, double* __restrict__ ams,
                                                              double* __restrict__ axes, double* __restrict__ axlens,
                                                              double* __restrict__ logvols,
                                                              const double* __restrict__ targets) {
    extern __shared__ double sm[];     // fax[n], lam[n], wc[n], wa[n], order[n]
    double* fax = sm;
    double* lam = fax + n;
    double* wc = lam + n;              // per-axis weights of the rebuilt cov / am (hoisted out of the n^3 loop)
    double* wa = wc + n;
    int* order = reinterpret_cast<int*>(wa + n);
    __shared__ int s_iso;
    __shared__ double s_f;
    const int k = blockIdx.x, tid = threadIdx.x, T = blockDim.x;
    const size_t nn = (size_t)n * n;
    double* Cm = covs + k * nn;
    double* AM = ams + k * nn;
    double* AX = axes + k * nn;
    double* AL = axlens + (size_t)k * n;
    const double logf = targets[k] - logvols[k];
    const double max_log_axlen = log(sqrt((double)n) / 2.0);
    if (tid == 0) {
        double mx = -INFINITY;
        for (int i = 0; i < n; i++) mx = fmax(mx, log(AL[i]));
        s_iso = (mx < max_log_axlen - logf / n) ? 1 : 0;
        s_f = exp(logf / n);
    }
    for (int i = tid; i < n; i += T) lam[i] = AL[i] * AL[i];
    __syncthreads();
    if (s_iso) {
        const double f = s_f, f2 = f * f, if2 = 1.0 / f2;
        for (size_t e = tid; e < nn; e += T) { Cm[e] *= f2; AM[e] *= if2; AX[e] *= f; }
        for (int i = tid; i < n; i += T) AL[i] *= f;
    } else {
        // water-filling from the largest eigenvalue down (:258-275)
        for (int i = tid; i < n; i += T) {
            int rk = 0;   // rank in DESCENDING eigenvalue order (np.argsort(l)[::-1])
            for (int j = 0; j < n; j++) rk += (lam[j] > lam[i] || (lam[j] == lam[i] && j > i)) ? 1 : 0;
            order[rk] = i;
        }
        __syncthreads();
        if (tid == 0) {
            double cur = logf;
            int left = n;
            for (int r = 0; r < n; r++) {
                const int i = order[r];
                const double delta = fmax(fmin(max_log_axlen - log(AL[i]), cur / left), 0.0);
                fax[i] = exp(delta);
                cur -= delta;
                left -= 1;
            }
        }
        __syncthreads();
        for (int q = tid; q < n; q += T) {
            const double f2 = fax[q] * fax[q];
            wc[q] = f2;
            wa[q] = 1.0 / (lam[q] * lam[q] * f2);
        }
        __syncthreads();
        // cov = sum_k a_k a_k^T fax_k^2 ; am = sum_k a_k a_k^T / (lam_k^2 fax_k^2),  a_k = axes[:,k]
        for (size_t e = tid; e < nn; e += T) {
            const int i = (int)(e / n), j = (int)(e - (size_t)i * n);
            double c = 0.0, a = 0.0;
            for (int q = 0; q < n; q++) {
                const double pr = AX[(size_t)i * n + q] * AX[(size_t)j * n + q];
                c = fma(pr, wc[q], c);
                a = fma(pr, wa[q], a);
            }
            Cm[e] = c;
            AM[e] = a;
        }
        __syncthreads();
        for (size_t e = tid; e < nn; e += T) AX[e] *= fax[e % n];
        for (int i = tid; i < n; i += T) AL[i] *= fax[i];
    }
    if (tid == 0) logvols[k] = targets[k];
}

extern "C" int b2n_scale_to_logvol(b2n_ctx* ctx, int32_t K, int32_t n, double* covs, double* ams, double* axes,
                                   double* axlens, double* logvols, const double* targets) {
    if (!ctx || K < 1 || n < 1 || !covs || !ams || !axes || !axlens || !logvols || !targets) return B2N_ERR_ARG;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t nn = (size_t)n * n;
    const void *ci, *ai, *xi, *li, *vi, *ti;
    B2N_TRY(b2n_in(ctx, ctx->out0, covs, K * nn * sizeof(double), &ci));
    B2N_TRY(b2n_in(ctx, ctx->out1, ams, K * nn * sizeof(double), &ai));
    B2N_TRY(b2n_in(ctx, ctx->out2, axes, K * nn * sizeof(double), &xi));
    B2N_TRY(b2n_in(ctx, ctx->out3, axlens, (size_t)K * n * sizeof(double), &li));
    B2N_TRY(b2n_in(ctx, ctx->out4, logvols, (size_t)K * sizeof(double), &vi));
    B2N_TRY(b2n_in_host(ctx, ctx->in3, targets, (size_t)K * sizeof(double), &ti));
    const size_t smem = (size_t)(5 * n + 2) * sizeof(double);
    scale_to_logvol_kernel<<<K, 1024, smem, ctx->stream>>>(n, (double*)ci, (double*)ai, (double*)xi, (double*)li,
                                                          (double*)vi, (const double*)ti);
    B2N_LAUNCH_CHECK(ctx);
    B2N_TRY(b2n_out_done(ctx, covs, ci, K * nn * sizeof(double)));
    B2N_TRY(b2n_out_done(ctx, ams, ai, K * nn * sizeof(double)));
    B2N_TRY(b2n_out_done(ctx, axes, xi, K * nn * sizeof(double)));
    B2N_TRY(b2n_out_done(ctx, axlens, li, (size_t)K * n * sizeof(double)));
    B2N_TRY(b2n_out_done(ctx, logvols, vi, (size_t)K * sizeof(double)));
    return b2n_finish(ctx);
}

// b2n_scan.cuh -- the block scan of the run-statistics kernels (b2n_jitter.cu, b2n_resample.cu) and its operators.
#pragma once
#include "b2n_common.cuh"

#include <math.h>

__device__ __forceinline__ double lae(double a, double b) {     // np.logaddexp
    if (a == -INFINITY) return b;
    if (b == -INFINITY) return a;
    const double m = fmax(a, b);
    return m + log1p(exp(-fabs(a - b)));
}
struct OpSum {
    __device__ static double id() { return 0.0; }
    __device__ double operator()(double a, double b) const { return a + b; }
};
struct OpLae {
    __device__ static double id() { return -INFINITY; }
    __device__ double operator()(double a, double b) const { return lae(a, b); }
};
struct OpMax {                      // over sample indices: the identity -1 stands for none
    __device__ static double id() { return -1.0; }
    __device__ double operator()(double a, double b) const { return fmax(a, b); }
};

// In-place inclusive scan of x[0, n) (shared memory) with a fixed association: thread t owns a contiguous run of
// ceil(n / blockDim) elements, then warp shuffles, then the warp totals.  Any n >= 0; blockDim a multiple of 32, at
// most 1024 (wsum holds one total per warp, 32 doubles).  Returns the total (identity for n == 0) to every thread.
template <class Op>
__device__ double block_scan(double* x, int n, double* wsum, Op op) {
    const int t = threadIdx.x, lane = t & 31, w = t >> 5, nw = blockDim.x >> 5;
    const int ipt = (n + blockDim.x - 1) / blockDim.x;
    const int i0 = min(t * ipt, n), i1 = min(i0 + ipt, n);
    double acc = Op::id();
    for (int i = i0; i < i1; i++) { acc = op(acc, x[i]); x[i] = acc; }
    double v = acc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double u = __shfl_up_sync(B2N_FULL, v, o);
        if (lane >= o) v = op(u, v);
    }
    if (lane == 31) wsum[w] = v;
    __syncthreads();
    if (w == 0) {
        double s = lane < nw ? wsum[lane] : Op::id();
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double u = __shfl_up_sync(B2N_FULL, s, o);
            if (lane >= o) s = op(u, s);
        }
        if (lane < nw) wsum[lane] = s;
    }
    __syncthreads();
    double ex = __shfl_up_sync(B2N_FULL, v, 1);
    if (lane == 0) ex = Op::id();
    if (w > 0) ex = op(wsum[w - 1], ex);
    if (t > 0)
        for (int i = i0; i < i1; i++) x[i] = op(ex, x[i]);
    const double total = wsum[nw - 1];
    __syncthreads();
    return total;
}

// b2n_eval_kernel.cuh -- batched prior transform + log-likelihood (model_eval_kernel).  Device-only: included
// by b2n_ctx.cu and by the run-time compiled translation unit of a user likelihood (b2n_user_kernels.cuh).
#pragma once
#include "b2n_device.cuh"

// ---- batched model evaluation: one warp per point -------------------------------------
template <int LIKE>
__global__ void __launch_bounds__(256) model_eval_kernel(B2nModel m, const double* __restrict__ u,
                                                         int64_t M, double* __restrict__ v,
                                                         double* __restrict__ logl) {
    extern __shared__ double sm[];
    const int n = m.ndim;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    double* vv = sm + (size_t)warp * 2 * n;
    double* work = vv + n;
    for (int64_t p = (int64_t)blockIdx.x * wpb + warp; p < M; p += (int64_t)gridDim.x * wpb) {
        for (int i = lane; i < n; i += 32) {
            const double x = prior_1d(m, i, u[p * n + i]);
            vv[i] = x;
            if (v) v[p * n + i] = x;
        }
        __syncwarp();
#ifdef B2N_USER_PRIOR
        if (m.prior_kind == B2N_PRIOR_USER) {
            user_prior_warp(m, u + p * n, vv, work, lane);
            if (v)
                for (int i = lane; i < n; i += 32) v[p * n + i] = vv[i];
        }
#endif
        const double l = warp_loglike<LIKE>(m, m.lmat, vv, work, lane);
        if (lane == 0) logl[p] = l;
        __syncwarp();
    }
}

// b2n_user_kernels.cuh -- the NVRTC translation unit of a user likelihood (B2N_LIKE_USER).
//
// A run-time compiled program is this header followed by the user's source, which defines
//     __device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane);
// and, when the program is compiled with B2N_USER_PRIOR, also
//     __device__ void b2n_user_prior(const double* u, double* v, double* work, int n, const double* p, int lane);
// and, when it is compiled with B2N_USER_BLOB, also
//     __device__ void b2n_user_blob(const double* v, double* work, int n, const double* p, int lane, double* blob,
//                                   int nblob);
// (contract: include/b200nest.h, b2n_model_create_user / b2n_model_create_user_ex).  The header brings in the chain-kernel templates that
// libb200nest.so instantiates for the registry likelihoods -- the same code, with LIKE = B2N_LIKE_USER calling the
// user's function -- and the b2n_ warp reductions the user's code may call.  Which instantiations to request from
// NVRTC (one name expression per B2nUserSlot) is owned by the library: b2n_user_kernel_exprs.
#pragma once
#ifndef B2N_USER_MODEL
#define B2N_USER_MODEL
#endif
#include "b2n_eval_kernel.cuh"
#include "b2n_unif_kernel.cuh"
#include "b2n_rwalk_kernel.cuh"
#include "b2n_slice_kernel.cuh"
#include "b2n_friends_kernel.cuh"

// warp reductions for the user's code: every lane gets the reduction over the 32 lanes
__device__ __forceinline__ double b2n_warp_sum(double v) { return warp_sum(v); }
__device__ __forceinline__ double b2n_warp_prod(double v) { return warp_prod(v); }
__device__ __forceinline__ double b2n_warp_max(double v) { return warp_max(v); }
__device__ __forceinline__ double b2n_warp_min(double v) { return warp_min(v); }

#ifdef B2N_USER_PRIOR
// A program that also defines b2n_user_prior (B2N_PRIOR_USER) is compiled with B2N_USER_PRIOR, which puts the
// warp-cooperative prior call into every kernel above.  b2n_model_create_user_ex looks this symbol up before it
// accepts the image for a model with a user prior: an image compiled without it would only write the placeholders.
extern "C" __device__ const int b2n_user_prior_abi = 1;
#endif

#ifdef B2N_USER_BLOB
// The blob of M points v (M x ndim) into blob (M x nblob), both row-major: one warp per point, grid-stride loop.
// Dynamic shared memory: per warp, v (n), work (n) and the blob row (nblob) doubles.  The row starts as NaN, so an
// element the user leaves unwritten is NaN in the output.  Not a B2nUserSlot: b2n_model_create_user(_ex) looks it
// up by this name, and a model whose image lacks it has no blob.
extern "C" __global__ void __launch_bounds__(256) b2n_user_blob_kernel(B2nModel m, const double* __restrict__ v,
                                                                       int64_t M, int nblob,
                                                                       double* __restrict__ blob) {
    extern __shared__ double blob_sm[];   // (its own name: an extern "C" function gives it C linkage)
    const int n = m.ndim;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    double* vv = blob_sm + (size_t)warp * (2 * n + nblob);
    double* work = vv + n;
    double* bb = work + n;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    for (int64_t p = (int64_t)blockIdx.x * wpb + warp; p < M; p += (int64_t)gridDim.x * wpb) {
        for (int i = lane; i < n; i += 32) vv[i] = v[p * n + i];
        for (int i = lane; i < nblob; i += 32) bb[i] = nan;
        __syncwarp();
        b2n_user_blob(vv, work, n, m.lv0, lane, bb, nblob);
        __syncwarp();
        for (int i = lane; i < nblob; i += 32) blob[p * nblob + i] = bb[i];
        __syncwarp();
    }
}
#endif

// (the user's source follows)

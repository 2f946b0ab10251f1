// b2n_user_kernels.cuh -- the NVRTC translation unit of a user likelihood (B2N_LIKE_USER).
//
// A run-time compiled program is this header followed by the user's source, which defines
//     __device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane);
// and, when the program is compiled with B2N_USER_PRIOR, also
//     __device__ void b2n_user_prior(const double* u, double* v, double* work, int n, const double* p, int lane);
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

// (the user's source follows)

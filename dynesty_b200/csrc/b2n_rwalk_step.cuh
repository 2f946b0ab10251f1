// b2n_rwalk_step.cuh -- parameters and host entry of the stepped random walk (b2n_rwalk_step.cu), shared with the
// device-paced rounds (b2n_ns.cu).
#pragma once
#include "b2n_common.cuh"

struct RwalkStepParams {
    int n, nc, walks, step;
    const double* u0;       // Q x n start points (launch 0)
    const int* order;       // per-CTA worklist, as rwalk_kernel's
    const int3* cta;
    const double* axesT;    // K x nc x nc, transposed (column-major axes)
    const uint32_t* dimflags;
    double loglstar, scale;
    uint64_t seed, chain0;
    const B2nDyn* dyn;      // device-paced (b2n_ns.cu): threshold / scale / chain ids / CTA count / skip in HBM
    double *u, *v, *logl;   // chain state = the outputs of the fill
    int *nacc, *nrej, *ncall;
    uint32_t* tick;
    int* in_cube;
    double* u_prop;
    double* u_start;        // optional copy of the start rows (launch 0)
    const double *v_prop, *logl_prop, *v_start, *logl_start;
};

#ifndef __CUDACC_RTC__
// chains per CTA, warps per CTA and dynamic shared memory of a launch over Q chains of n dimensions
int b2n_rwalk_step_plan(b2n_ctx* ctx, int64_t Q, int n, int* chains_per_cta, int* warps, size_t* smem);
// enqueue one launch of rwalk_step_kernel on the ctx stream
int b2n_rwalk_step_launch(b2n_ctx* ctx, const RwalkStepParams& p, unsigned grid, int warps, size_t smem);
// check the caller's state and put it, walks and step into p
int b2n_rwalk_step_bind(b2n_ctx* ctx, int32_t walks, int32_t step, const b2n_rwalk_state* st, RwalkStepParams& p);
#endif

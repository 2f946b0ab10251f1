// b2n_rwalk_step.cu -- the random walk of rwalk_kernel (b2n_rwalk_kernel.cuh) cut into one launch per step, for
// likelihoods that cannot run inside a kernel: a batched PyTorch function (dynesty_b200.TorchModel).  Part of
// libb200nest.so (C ABI: include/b200nest.h, b2n_rwalk_step / b2n_ns_rwalk_step).
//
// A fill of Q chains x `walks` steps is walks + 1 launches of rwalk_step_kernel, with the caller's likelihood between
// them on the same stream:
//   launch 0          chain q starts at u0[q] (tick 0, no counts), and proposes step 0 -> u_prop[q], in_cube[q]
//   caller            (v_start, logl_start) of the start rows, (v_prop, logl_prop) of u_prop
//   launch s, 1..w-1  accepts step s - 1 (in the cube and logl_prop > loglstar: u, v, logl <- the proposal, nacc++;
//                     else nrej++), then proposes step s
//   caller            (v_prop, logl_prop) of u_prop
//   launch walks      accepts step walks - 1; a chain that never accepted returns its start's (v_start, logl_start)
// The chain's draws are rwalk_kernel's, event for event: same Philox stream (seed, chain0 + q), same events (the
// non-clustered uniforms, the ball direction), same arithmetic for u + fac * axes @ z, wrap / reflect and the cube
// test.  Its tick lives in HBM between launches.  An out-of-cube proposal uses up a step and no likelihood call, as in
// rwalk_kernel: its row of u_prop is the chain's current point, so that the caller only ever evaluates points of the
// cube, and the accept half ignores the row.  A NaN logl_prop is rejected (NaN > loglstar is false).
#include "b2n_rwalk_kernel.cuh"
#include "b2n_rwalk_step.cuh"


// Dynamic shared memory per warp: the direction z and the current point, npad doubles each.
__global__ void __launch_bounds__(512) rwalk_step_kernel(const RwalkStepParams p) {
    const int n = p.n, nc = p.nc, step = p.step;
    const int npad = (n + 1) & ~1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    B2N_DYN_PROLOGUE(p)
    const int3 cd = p.cta[blockIdx.x];
    const double* Ag = p.axesT + (size_t)cd.z * nc * nc;
    const int ox = warp * 2 * npad;     // direction vector
    const int ocur = ox + npad;         // current point of the chain
    const double inv_nc = 1.0 / (double)nc;
    for (int c = warp; c < cd.y; c += nwarps) {
        const int q = p.order[cd.x + c];
        const size_t row = (size_t)q * n;
        // ---- accept step - 1 (or start the chain)
        int nacc = 0, nrej = 0;
        uint32_t tick = 0;
        bool acc = false;
        const double* src = p.u0 + row;
        if (step > 0) {
            nacc = p.nacc[q]; nrej = p.nrej[q]; tick = p.tick[q];
            const double l = p.logl_prop[q];
            acc = p.in_cube[q] != 0 && l > loglstar_;
            if (acc) { nacc++; src = p.u_prop + row; if (lane == 0) p.logl[q] = l; }
            else { nrej++; src = p.u + row; }
        }
        for (int i = lane; i < n; i += 32) {
            const double x = src[i];
            b2n_sm[ocur + i] = x;
            if (step == 0) {
                p.u[row + i] = x;
                if (p.u_start) p.u_start[row + i] = x;
            } else if (acc) {
                p.u[row + i] = x;
                p.v[row + i] = p.v_prop[row + i];
            }
        }
        // (the rows of u_prop / v_prop just read are rewritten below; v_prop may BE u_prop -- an identity prior)
        __syncwarp();
        if (step < p.walks) {
            // ---- propose step `step`: rwalk_kernel's (1) - (4)
            ChainRng g;
            g.init(p.seed, chain0_ + (uint64_t)q);
            g.tick = tick;
            if (n > nc) {
                for (int e = lane; e < n - nc; e += 32) p.u_prop[row + nc + e] = rng_uniform_elem(g, e);
                g.tick++;
            }
            const double fac = scale_ * ball_direction(g, ox, nc, lane, inv_nc);
            __syncwarp();
            bool ok = true;
            for (int base = 0; base < nc; base += 64) {
                double y0, y1;
                matvec2o<false>(Ag, 0, nc, nc, ox, base + lane, nc, y0, y1);
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int i = base + lane + 32 * h;
                    if (i < nc) {
                        double x = fma(fac, h ? y1 : y0, b2n_sm[ocur + i]);
                        const uint32_t f = p.dimflags ? __ldg(p.dimflags + i) : 0u;
                        if (f & B2N_DIM_PERIODIC) x = mod1(x);
                        if (f & B2N_DIM_REFLECTIVE) x = reflect1(x);
                        ok = ok && in_cube(x, f);
                        p.u_prop[row + i] = x;
                    }
                }
            }
            ok = __all_sync(B2N_FULL, ok);
            if (!ok) {       // the callable sees the chain's current point; the accept half ignores the row
                __syncwarp();
                for (int i = lane; i < n; i += 32) p.u_prop[row + i] = b2n_sm[ocur + i];
            }
            if (lane == 0) { p.in_cube[q] = ok ? 1 : 0; p.tick[q] = g.tick; }
        } else if (nacc == 0) {
            // ---- the last launch: a chain that never moved returns its start's (v, logl), as rwalk_kernel's recompute
            for (int i = lane; i < n; i += 32) p.v[row + i] = p.v_start[row + i];
            if (lane == 0) p.logl[q] = p.logl_start[q];
        }
        if (lane == 0) {
            p.nacc[q] = nacc; p.nrej[q] = nrej;
            if (step == p.walks) p.ncall[q] = p.walks;
        }
        __syncwarp();
    }
}

// Launch geometry: the chains per CTA of rwalk_kernel's grid, warps limited by the shared memory they need.
int b2n_rwalk_step_plan(b2n_ctx* ctx, int64_t Q, int n, int* chains_per_cta, int* warps, size_t* smem) {
    const size_t per_warp = (size_t)2 * ((n + 1) & ~1) * sizeof(double);
    const int max_warps = (int)std::min<size_t>(16, (size_t)ctx->max_smem_optin / per_warp);
    if (max_warps < 1) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "ndim too large for the stepped rwalk kernel");
    b2n_chain_grid(ctx, Q, max_warps, *chains_per_cta, *warps);
    *smem = per_warp * (size_t)*warps;
    return B2N_OK;
}

// Enqueue one launch; p carries everything but the geometry.
int b2n_rwalk_step_launch(b2n_ctx* ctx, const RwalkStepParams& p, unsigned grid, int warps, size_t smem) {
    B2N_TRY(b2n_func_smem(ctx, (const void*)rwalk_step_kernel, smem));
    B2N_TIME_BEGIN(ctx);
    rwalk_step_kernel<<<grid, warps * 32, smem, ctx->stream>>>(p);
    B2N_TIME_END(ctx);
    B2N_LAUNCH_CHECK(ctx);
    return B2N_OK;
}

int b2n_rwalk_step_bind(b2n_ctx* ctx, int32_t walks, int32_t step, const b2n_rwalk_state* st, RwalkStepParams& p) {
    if (!st || walks < 1 || step < 0 || step > walks) return B2N_ERR_ARG;
    if (!st->u_prop || !st->tick || !st->in_cube) return B2N_ERR_ARG;
    if (step > 0 && (!st->v_prop || !st->logl_prop)) return b2n_fail(ctx, B2N_ERR_ARG, "stepped rwalk: step > 0 needs v_prop and logl_prop");
    if (step == walks && (!st->v_start || !st->logl_start)) return b2n_fail(ctx, B2N_ERR_ARG, "stepped rwalk: the last step needs v_start and logl_start");
    p.walks = walks; p.step = step;
    p.dimflags = st->dimflags;
    p.tick = st->tick; p.in_cube = st->in_cube; p.u_prop = st->u_prop; p.u_start = st->u_start;
    p.v_prop = st->v_prop; p.logl_prop = st->logl_prop; p.v_start = st->v_start; p.logl_start = st->logl_start;
    return B2N_OK;
}

extern "C" int b2n_rwalk_step(b2n_ctx* ctx, const b2n_chain_args* a, int32_t walks, int32_t step, b2n_rwalk_state* st,
                              double* u, double* v, double* logl, int32_t* n_accept, int32_t* n_reject, int32_t* ncall) {
    if (!ctx || !a) return B2N_ERR_ARG;
    if (ctx->ptr_mode != B2N_PTR_DEVICE) return b2n_fail(ctx, B2N_ERR_ARG, "b2n_rwalk_step takes device pointers (B2N_PTR_DEVICE)");
    if (ctx->peer.total > 0 || ctx->start_idx || ctx->dyn.active)
        return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "b2n_rwalk_step: no gather mode, start rows by index or device pacing");
    const int n = a->ndim, nc = a->ncdim;
    const int64_t Q = a->nchain;
    if (n < 1 || nc < 1 || nc > n || Q < 1 || Q > INT32_MAX || !a->u0 || !u || !v || !logl || !n_accept || !n_reject ||
        !ncall || !st->order || !st->cta)
        return B2N_ERR_ARG;
    if (ctx->bK < 1 || ctx->bn != nc) return b2n_fail(ctx, B2N_ERR_ARG, "resident bound missing or of wrong dimension (b2n_bound_set)");
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    int cpc, warps;
    size_t smem;
    B2N_TRY(b2n_rwalk_step_plan(ctx, Q, n, &cpc, &warps, &smem));
    if (step == 0) {         // the fill's worklist, into the caller's buffers (read by every later step)
        std::vector<int> order;
        std::vector<int3> cta;
        B2N_TRY(b2n_build_worklist(ctx, Q, a->ell, ctx->bK, cpc, order, cta));
        B2N_CUDA(ctx, cudaMemcpyAsync(st->order, order.data(), order.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
        B2N_CUDA(ctx, cudaMemcpyAsync(st->cta, cta.data(), cta.size() * sizeof(int3), cudaMemcpyHostToDevice, ctx->stream));
        st->ncta = (int32_t)cta.size();
    }
    if (st->ncta < 1 || st->ncta > Q) return b2n_fail(ctx, B2N_ERR_ARG, "b2n_rwalk_step: ncta not set by step 0");
    RwalkStepParams p;
    memset(&p, 0, sizeof(p));
    B2N_TRY(b2n_rwalk_step_bind(ctx, walks, step, st, p));
    p.n = n; p.nc = nc; p.u0 = a->u0;
    p.order = st->order; p.cta = reinterpret_cast<const int3*>(st->cta);
    p.axesT = ctx->b_axesT.as<double>();
    p.loglstar = a->loglstar; p.scale = a->scale; p.seed = a->seed; p.chain0 = a->chain0;
    p.u = u; p.v = v; p.logl = logl; p.nacc = n_accept; p.nrej = n_reject; p.ncall = ncall;
    return b2n_rwalk_step_launch(ctx, p, (unsigned)st->ncta, warps, smem);
}

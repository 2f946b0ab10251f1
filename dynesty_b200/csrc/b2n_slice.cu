// b2n_slice.cu -- batched slice-sampling chains (one warp per chain).
//
// Replaces RSliceSampler.sample (reference internal_samplers.py:745-855) and
// SliceSampler.sample (:593-709), both built on generic_slice_step (:1075-1206) and the
// Neal (2003) doubling acceptance test _slice_doubling_accept (:1038-1072).
//
// All control flow of a slice step (stepping out, doubling, shrinking) depends only on
// warp-uniform scalars (log-likelihood values, uniforms that every lane derives from the
// same Philox counter), so the 32 lanes of a chain stay converged while they cooperate on
// the vector work: u + x*d, the unit-cube test, the prior transform and the likelihood.
// Same layout as the rwalk kernel (b2n_chain.cuh): persistent-sized grid, one ellipsoid per
// CTA, axes^T / precision matrix staged once in shared memory with 128-byte padded columns,
// all per-chain vectors addressed as b2n_sm[offset].
// NOTE (reference behaviour kept): the slice samplers read kwargs['nonperiodic'], which
// the 3.0 sampler never sets (:654, 804), so every dimension is hard-bounded to (0, 1).
#include "b2n_slice_kernel.cuh"
#include <algorithm>
#include <vector>


template <bool RANDOM_DIR>
static int slice_batch_impl(b2n_ctx* ctx, const b2n_chain_args* a, int32_t slices, int32_t doubling, double* u,
                            double* v, double* logl, int32_t* n_expand, int32_t* n_contract, int32_t* ncall,
                            uint32_t* flags) {
    B2nModel m;
    B2N_TRY(b2n_chain_begin(ctx, a, false, &m));
    const bool gather = ctx->peer.total > 0;      // outputs may be NULL in gather mode (b2n_peer_result)
    if (!gather && (!u || !v || !logl || !n_expand || !n_contract || !ncall || !flags)) return B2N_ERR_ARG;
    const int n = a->ndim;
    const int64_t Q = a->nchain;
    if (n != m.ndim || a->ncdim != n || slices < 1 || Q < 0 || !a->u0)
        return b2n_fail(ctx, B2N_ERR_ARG, "slice samplers need ncdim == ndim (internal_samplers.py:658, 809)");
    if (ctx->bK < 1 || ctx->bn != n) return b2n_fail(ctx, B2N_ERR_ARG, "resident bound missing or of wrong dimension");
    if (Q == 0) return b2n_chain_none(ctx);
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    ZcScope zc(ctx);          // pinned caller buffers are read / written in place (host-pointer mode)
    const int npad = (n + 1) & ~1;
    const size_t per_warp = (size_t)6 * npad * sizeof(double);           // u, d, un, vn, work, idxs
    const size_t model_b = (size_t)4 * npad * sizeof(double);
    const size_t limit = (size_t)ctx->max_smem_optin;
    const int max_warps = (int)std::min<size_t>(16, (limit - model_b) / per_warp);
    if (max_warps < 1) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "ndim too large for the slice kernel");
    int chains_per_cta, warps;
    b2n_chain_grid(ctx, Q, max_warps, chains_per_cta, warps);
    const size_t fixed = per_warp * warps + model_b;
    const int ldA = (n + 15) & ~15, ldP = ldA;
    const size_t ax_b = (size_t)n * ldA * sizeof(double);
    const size_t pr_b = (m.like_kind == B2N_LIKE_GAUSS_PREC) ? ax_b : 0;
    const bool ax_s = fixed + ax_b <= limit;
    const bool pr_s = pr_b > 0 && fixed + (ax_s ? ax_b : 0) + pr_b <= limit;
    const size_t smem = fixed + (ax_s ? ax_b : 0) + (pr_s ? pr_b : 0);
    const bool dyn = ctx->dyn.active;        // device-paced launch (b2n_ns.cu)
    if (dyn) {
        B2N_TRY(b2n_chain_dyn(ctx, chains_per_cta));
        if (ctx->dyn.plan_only) return B2N_OK;
    }
    SliceParams p;
    p.dyn = dyn ? ctx->dyn.dev : nullptr;
    p.m = m; p.n = n; p.slices = slices; p.doubling = doubling; p.ldA = ldA; p.ldP = ldP;
    p.loglstar = a->loglstar; p.scale = a->scale; p.seed = a->seed; p.chain0 = a->chain0;
    p.axesT = ctx->b_axesT.as<double>();
    const void *du0, *dorder, *dcta;
    B2N_TRY(b2n_in(ctx, ctx->in0, a->u0, (size_t)Q * n * sizeof(double), &du0));
    unsigned ncta = 0;
    if (dyn) {
        dorder = ctx->dyn.order; dcta = ctx->dyn.cta;
    } else {
        B2N_TRY(b2n_worklist_dev(ctx, Q, a->ell, ctx->bK, chains_per_cta, &dorder, &dcta, &ncta));
    }
    void* const out[B2N_NSLOT] = {u, v, logl, n_expand, n_contract, ncall, flags};
    void* dev[B2N_NSLOT];
    B2N_TRY(b2n_chain_bind(ctx, n, Q, out, dev, &p.peer));
    p.u0 = (const double*)du0; p.order = (const int*)dorder; p.cta = (const int3*)dcta;
    p.u = (double*)dev[0]; p.v = (double*)dev[1]; p.logl = (double*)dev[2];
    p.nexp = (int*)dev[3]; p.ncon = (int*)dev[4]; p.ncall = (int*)dev[5]; p.flags = (uint32_t*)dev[6];
    const unsigned grid = dyn ? (unsigned)ctx->dyn.max_cta : ncta;
#define LAUNCH(L, AXS, PRS)                                                                          \
    do {                                                                                             \
        B2N_TRY(b2n_func_smem(ctx, (const void*)(slice_kernel<L, RANDOM_DIR, AXS, PRS>), (size_t)(smem))); \
        slice_kernel<L, RANDOM_DIR, AXS, PRS><<<grid, warps * 32, smem, ctx->stream>>>(p);            \
    } while (0)
#define CALL(L)                                \
    if (ax_s && pr_s) LAUNCH(L, true, true);   \
    else if (ax_s) LAUNCH(L, true, false);     \
    else if (pr_s) LAUNCH(L, false, true);     \
    else LAUNCH(L, false, false);
    B2N_TIME_BEGIN(ctx);
    if (m.like_kind == B2N_LIKE_USER) {      // (pr_s is false: no precision matrix)
        void* args[] = {(void*)&p};
        B2N_TRY(b2n_user_launch(ctx, a->model_id, B2N_US_SLICE + (RANDOM_DIR ? 2 : 0) + (ax_s ? 1 : 0), dim3(grid),
                                dim3(warps * 32), smem, args));
    } else {
        B2N_DISPATCH_LIKE(m.like_kind, CALL)
    }
    B2N_TIME_END(ctx);
#undef CALL
#undef LAUNCH
    B2N_LAUNCH_CHECK(ctx);
    if (dyn) return B2N_OK;      // device-paced: the commit kernel of the round folds the flags
    // a collapsed interval anywhere = RuntimeError in the reference
    static const B2nFlagStatus fail[] = {{0x80000000u, B2N_ERR_SLICE_FAIL, nullptr}};
    return b2n_chain_end(ctx, n, Q, out, dev, fail, 1);
}

extern "C" int b2n_rslice_batch(b2n_ctx* ctx, const b2n_chain_args* a, int32_t slices, int32_t doubling,
                                double* u, double* v, double* logl, int32_t* n_expand, int32_t* n_contract,
                                int32_t* ncall, uint32_t* flags) {
    return slice_batch_impl<true>(ctx, a, slices, doubling, u, v, logl, n_expand, n_contract, ncall, flags);
}
extern "C" int b2n_slice_batch(b2n_ctx* ctx, const b2n_chain_args* a, int32_t slices, int32_t doubling, double* u,
                               double* v, double* logl, int32_t* n_expand, int32_t* n_contract, int32_t* ncall,
                               uint32_t* flags) {
    return slice_batch_impl<false>(ctx, a, slices, doubling, u, v, logl, n_expand, n_contract, ncall, flags);
}

// b2n_unif.cu -- batched uniform sampling within the resident (multi-)ellipsoid bound.
//
// Replaces UniformBoundSampler.sample (reference internal_samplers.py:243-340) whose
// bound draw is MultiEllipsoid.sample (bounding.py:525-590) / Ellipsoid.sample
// (:307-319): pick an ellipsoid with probability proportional to its volume (rand_choice,
// :1300-1308), draw uniformly inside it (randsphere, :1288-1297), count the q ellipsoids
// containing the draw (strict <1, with the 1e-3 slack retry of :565-579) and accept with
// probability 1/q; reject draws outside the unit cube (internal_samplers.py:314-322);
// append fresh U(0,1) for the non-clustered dims (:325-327); evaluate; repeat until
// logl > loglstar.  One warp per chain.
#include "b2n_unif_kernel.cuh"
#include <vector>


extern "C" int b2n_unif_batch(b2n_ctx* ctx, const b2n_chain_args* a, double* u, double* v, double* logl,
                              int32_t* ncall, int32_t* nprop, uint32_t* flags) {
    B2nModel m;
    B2N_TRY(b2n_chain_begin(ctx, a, a && (a->reserved & B2N_OPT_DRAW_ONLY), &m));
    const int draw_only = (a->reserved & B2N_OPT_DRAW_ONLY) ? ((a->reserved & B2N_OPT_DRAW_MIXTURE) ? 3 : 1) : 0;
    const bool gather = ctx->peer.total > 0;      // outputs may be NULL in gather mode (b2n_peer_result)
    if (!gather && (!u || !v || !logl || !ncall || !nprop || !flags)) return B2N_ERR_ARG;
    const int n = a->ndim, nc = a->ncdim;
    const int64_t Q = a->nchain;
    if (n != m.ndim || nc < 1 || nc > n || Q < 0 || (draw_only && n != nc)) return B2N_ERR_ARG;
    if (ctx->bK < 1 || ctx->bn != nc || ctx->h_logvols.empty())
        return b2n_fail(ctx, B2N_ERR_ARG, "resident bound (with ctrs/ams/logvols) missing or of wrong dimension");
    if (Q == 0) return b2n_chain_none(ctx);
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    ZcScope zc(ctx);          // pinned caller buffers are written in place (host-pointer mode)
    const bool dyn = ctx->dyn.active;        // device-paced launch (b2n_ns.cu)
    if (dyn) {
        B2N_TRY(b2n_chain_dyn(ctx, 1));
        if (ctx->dyn.plan_only) return B2N_OK;
        if (draw_only) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "device-paced launch needs device pointers and no gather mode");
    }
    const int K = ctx->bK;
    // probs = exp(logvol_ells - logsumexp(logvol_ells)) ; cumsum (bounding.py:552, 1305)
    std::vector<double> cum(K);
    double hi = -INFINITY;
    for (double x : ctx->h_logvols) hi = std::max(hi, x);
    double se = 0.0;
    for (double x : ctx->h_logvols) se += exp(x - hi);
    const double lse = hi + log(se);
    double run = 0.0;
    for (int k = 0; k < K; k++) { run += exp(ctx->h_logvols[k] - lse); cum[k] = run; }
    const void *dcum, *dfl_in = nullptr;
    B2N_TRY(b2n_in_host(ctx, ctx->work0, cum.data(), cum.size() * sizeof(double), &dcum));
    std::vector<uint32_t> fl;
    if (a->dimflags) {
        fl.assign(a->dimflags, a->dimflags + n);
        B2N_TRY(b2n_in_host(ctx, ctx->in3, fl.data(), fl.size() * sizeof(uint32_t), &dfl_in));
    }
    UnifParams p;
    p.dyn = dyn ? ctx->dyn.dev : nullptr;
    p.m = m; p.n = n; p.nc = nc; p.K = K; p.Q = Q; p.draw_only = draw_only;
    p.ctrs = ctx->b_ctrs.as<double>(); p.ams = ctx->b_ams.as<double>(); p.axesT = ctx->b_axesT.as<double>();
    p.cum = (const double*)dcum; p.dimflags = (const uint32_t*)dfl_in;
    p.loglstar = a->loglstar; p.seed = a->seed; p.chain0 = a->chain0;
    void* const out[B2N_NSLOT] = {u, v, logl, ncall, nprop, nullptr, flags};
    void* dev[B2N_NSLOT];
    B2N_TRY(b2n_chain_bind(ctx, n, Q, out, dev, &p.peer));
    p.u = (double*)dev[0]; p.v = (double*)dev[1]; p.logl = (double*)dev[2];
    p.ncall = (int*)dev[3]; p.nprop = (int*)dev[4]; p.flags = (uint32_t*)dev[6];
    const int threads = 128, wpb = threads / 32;
    const size_t smem = (size_t)wpb * 5 * n * sizeof(double);
    if (smem > (size_t)ctx->max_smem_optin) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "ndim too large for the unif kernel");
    int64_t blocks = (Q + wpb - 1) / wpb;
#define CALL(L)                                                                                         \
    if (smem > 48 * 1024)                                                                               \
        B2N_TRY(b2n_func_smem(ctx, (const void*)(unif_kernel<L>), (size_t)(smem))); \
    unif_kernel<L><<<(unsigned)blocks, threads, smem, ctx->stream>>>(p);
    B2N_TIME_BEGIN(ctx);
    if (m.like_kind == B2N_LIKE_USER) {
        void* args[] = {(void*)&p};
        B2N_TRY(b2n_user_launch(ctx, a->model_id, B2N_US_UNIF, dim3((unsigned)blocks), dim3(threads), smem, args));
    } else {
        B2N_DISPATCH_LIKE(m.like_kind, CALL)
    }
    B2N_TIME_END(ctx);
#undef CALL
    B2N_LAUNCH_CHECK(ctx);
    if (dyn) return B2N_OK;      // device-paced: the commit kernel of the round folds the flags
    static const B2nFlagStatus fail[] = {
        {0x40000000u, B2N_ERR_Q0, nullptr},
        {0x80000000u, B2N_ERR_UNSUPPORTED, "uniform sampling did not find a point (bound draw limit)"}};
    return b2n_chain_end(ctx, n, Q, out, dev, fail, 2);
}


extern "C" int b2n_unitcube_batch(b2n_ctx* ctx, const b2n_chain_args* a, double* u, double* v, double* logl,
                                  int32_t* ncall, uint32_t* flags) {
    B2nModel m;
    B2N_TRY(b2n_chain_begin(ctx, a, false, &m));
    const bool gather = ctx->peer.total > 0;
    if (!gather && (!u || !v || !logl || !ncall)) return B2N_ERR_ARG;
    const int n = a->ndim;
    const int64_t Q = a->nchain;
    if (n != m.ndim || Q < 0) return B2N_ERR_ARG;
    if (Q == 0) return b2n_chain_none(ctx);
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    ZcScope zc(ctx);
    const bool dyn = ctx->dyn.active;
    if (dyn) {
        B2N_TRY(b2n_chain_dyn(ctx, 1));
        if (ctx->dyn.plan_only) return B2N_OK;
    }
    CubeParams p;
    p.dyn = dyn ? ctx->dyn.dev : nullptr;
    p.m = m; p.n = n; p.Q = Q; p.loglstar = a->loglstar; p.seed = a->seed; p.chain0 = a->chain0;
    void* const out[B2N_NSLOT] = {u, v, logl, ncall, nullptr, nullptr, flags};
    void* dev[B2N_NSLOT];
    B2N_TRY(b2n_chain_bind(ctx, n, Q, out, dev, &p.peer));
    if (!dev[B2N_SLOT_FLAGS]) {      // flags may be NULL: the draw-limit summary still reads them
        B2N_CUDA(ctx, ctx->out6.ensure((size_t)Q * sizeof(uint32_t)));
        dev[B2N_SLOT_FLAGS] = ctx->out6.p;
    }
    p.u = (double*)dev[0]; p.v = (double*)dev[1]; p.logl = (double*)dev[2]; p.ncall = (int*)dev[3]; p.flags = (uint32_t*)dev[6];
    const int threads = 128, wpb = threads / 32;
    const size_t smem = (size_t)wpb * 3 * n * sizeof(double);
    if (smem > (size_t)ctx->max_smem_optin) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "ndim too large for the unit-cube kernel");
    const int64_t blocks = (Q + wpb - 1) / wpb;
#define CALL(L)                                                                                             \
    if (smem > 48 * 1024)                                                                                   \
        B2N_TRY(b2n_func_smem(ctx, (const void*)(unitcube_kernel<L>), (size_t)(smem))); \
    unitcube_kernel<L><<<(unsigned)blocks, threads, smem, ctx->stream>>>(p);
    B2N_TIME_BEGIN(ctx);
    if (m.like_kind == B2N_LIKE_USER) {
        void* args[] = {(void*)&p};
        B2N_TRY(b2n_user_launch(ctx, a->model_id, B2N_US_UNITCUBE, dim3((unsigned)blocks), dim3(threads), smem, args));
    } else {
        B2N_DISPATCH_LIKE(m.like_kind, CALL)
    }
    B2N_TIME_END(ctx);
#undef CALL
    B2N_LAUNCH_CHECK(ctx);
    if (dyn) return B2N_OK;
    static const B2nFlagStatus fail[] = {
        {0x80000000u, B2N_ERR_UNSUPPORTED, "unit-cube sampling did not find a point above the threshold (draw limit)"}};
    return b2n_chain_end(ctx, n, Q, out, dev, fail, 1);
}

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


__global__ void unif_error_kernel(const uint32_t* flags, int64_t Q, int* out) {
    int bad = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < Q; i += (int64_t)gridDim.x * blockDim.x) {
        if (flags[i] & 0x40000000u) bad |= 1;
        if (flags[i] & 0x80000000u) bad |= 2;
    }
    if (bad) atomicOr(out, bad);
}

extern "C" int b2n_unif_batch(b2n_ctx* ctx, const b2n_chain_args* a, double* u, double* v, double* logl,
                              int32_t* ncall, int32_t* nprop, uint32_t* flags) {
    if (!ctx || !a) return B2N_ERR_ARG;
    if (ctx->start_idx) {       // b2n_set_start_rows is for the next b2n_rwalk_batch only: do not let it linger
        ctx->start_idx = nullptr; ctx->start_nrows = 0;
        return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "start rows by index (b2n_set_start_rows) are read by b2n_rwalk_batch only");
    }
    const bool gather = ctx->peer.total > 0;      // outputs may be NULL in gather mode (b2n_peer_result)
    if (!gather && (!u || !v || !logl || !ncall || !nprop || !flags)) return B2N_ERR_ARG;
    const int draw_only = (a->reserved & B2N_OPT_DRAW_ONLY) ? ((a->reserved & B2N_OPT_DRAW_MIXTURE) ? 3 : 1) : 0;
    B2nModel m;
    memset(&m, 0, sizeof(m));
    m.ndim = a->ndim;
    m.like_kind = B2N_LIKE_EGGBOX;
    if (!draw_only) {
        if (a->model_id < 0 || a->model_id >= (int)ctx->models.size()) return B2N_ERR_ARG;
        m = ctx->models[a->model_id];
    }
    const int n = a->ndim, nc = a->ncdim;
    const int64_t Q = a->nchain;
    if (n != m.ndim || nc < 1 || nc > n || Q < 0 || (draw_only && n != nc)) return B2N_ERR_ARG;
    if (ctx->bK < 1 || ctx->bn != nc || ctx->h_logvols.empty())
        return b2n_fail(ctx, B2N_ERR_ARG, "resident bound (with ctrs/ams/logvols) missing or of wrong dimension");
    if (Q == 0) return gather ? b2n_fail(ctx, B2N_ERR_ARG, "gather mode: every rank must run at least one chain") : B2N_OK;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    ZcScope zc(ctx);          // pinned caller buffers are written in place (host-pointer mode)
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
    const bool dyn = ctx->dyn.active;        // device-paced launch (b2n_ns.cu)
    if (dyn && (gather || ctx->ptr_mode != B2N_PTR_DEVICE || draw_only))
        return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "device-paced launch needs device pointers and no gather mode");
    UnifParams p;
    p.dyn = dyn ? ctx->dyn.dev : nullptr;
    p.m = m; p.n = n; p.nc = nc; p.K = K; p.Q = Q; p.draw_only = draw_only;
    p.ctrs = ctx->b_ctrs.as<double>(); p.ams = ctx->b_ams.as<double>(); p.axesT = ctx->b_axesT.as<double>();
    p.cum = (const double*)dcum; p.dimflags = (const uint32_t*)dfl_in;
    p.loglstar = a->loglstar; p.seed = a->seed; p.chain0 = a->chain0;
    void *du, *dv, *dl, *dnc, *dnp, *dfl;
    void* gdev[7];
    bool peer_on = false;
    B2N_TRY(b2n_peer_begin(ctx, n, &p.peer, gdev, &peer_on));
    if (peer_on) {
        if (ctx->peer.row0 + Q > ctx->peer.total) return b2n_fail(ctx, B2N_ERR_ARG, "gather rows out of range (b2n_peer_rows)");
        du = gdev[0]; dv = gdev[1]; dl = gdev[2]; dnc = gdev[3]; dnp = gdev[4]; dfl = gdev[6];
    } else {
        B2N_TRY(b2n_out(ctx, ctx->out0, u, (size_t)Q * n * sizeof(double), &du));
        B2N_TRY(b2n_out(ctx, ctx->out1, v, (size_t)Q * n * sizeof(double), &dv));
        B2N_TRY(b2n_out(ctx, ctx->out2, logl, (size_t)Q * sizeof(double), &dl));
        B2N_TRY(b2n_out(ctx, ctx->out3, ncall, (size_t)Q * sizeof(int), &dnc));
        B2N_TRY(b2n_out(ctx, ctx->out4, nprop, (size_t)Q * sizeof(int), &dnp));
        B2N_TRY(b2n_out(ctx, ctx->out6, flags, (size_t)Q * sizeof(uint32_t), &dfl));
    }
    p.u = (double*)du; p.v = (double*)dv; p.logl = (double*)dl;
    p.ncall = (int*)dnc; p.nprop = (int*)dnp; p.flags = (uint32_t*)dfl;
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
    int* herr = reinterpret_cast<int*>(ctx->pinned);
    *herr = 0;
    B2N_CUDA(ctx, ctx->out7.ensure(64));
    B2N_CUDA(ctx, cudaMemsetAsync(ctx->out7.p, 0, sizeof(int), ctx->stream));
    const uint32_t* eflags = peer_on ? (const uint32_t*)(ctx->peer.win + ctx->peer.off[6]) : (const uint32_t*)dfl;
    unif_error_kernel<<<64, 256, 0, ctx->stream>>>(eflags, peer_on ? ctx->peer.total : Q, ctx->out7.as<int>());
    B2N_LAUNCH_CHECK(ctx);
    B2N_CUDA(ctx, cudaMemcpyAsync(herr, ctx->out7.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    if (peer_on) {
        void* const user7[7] = {u, v, logl, ncall, nprop, nullptr, flags};
        B2N_TRY(b2n_peer_end(ctx, n, user7));
        B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (ctx->ptr_mode == B2N_PTR_HOST && *ctx->peer.err_host)
            return b2n_fail(ctx, B2N_ERR_PEER, "a peer never arrived at the exchange (timeout in the kernel)");
        if (*herr & 1) return B2N_ERR_Q0;
        if (*herr & 2) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "uniform sampling did not find a point (bound draw limit)");
        return B2N_OK;
    }
    B2N_TRY(b2n_out_done(ctx, u, du, (size_t)Q * n * sizeof(double)));
    B2N_TRY(b2n_out_done(ctx, v, dv, (size_t)Q * n * sizeof(double)));
    B2N_TRY(b2n_out_done(ctx, logl, dl, (size_t)Q * sizeof(double)));
    B2N_TRY(b2n_out_done(ctx, ncall, dnc, (size_t)Q * sizeof(int)));
    B2N_TRY(b2n_out_done(ctx, nprop, dnp, (size_t)Q * sizeof(int)));
    B2N_TRY(b2n_out_done(ctx, flags, dfl, (size_t)Q * sizeof(uint32_t)));
    B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (*herr & 1) return B2N_ERR_Q0;
    if (*herr & 2) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "uniform sampling did not find a point (bound draw limit)");
    return B2N_OK;
}


extern "C" int b2n_unitcube_batch(b2n_ctx* ctx, const b2n_chain_args* a, double* u, double* v, double* logl,
                                  int32_t* ncall, uint32_t* flags) {
    if (!ctx || !a) return B2N_ERR_ARG;
    if (ctx->start_idx) {       // b2n_set_start_rows is for the next b2n_rwalk_batch only: do not let it linger
        ctx->start_idx = nullptr; ctx->start_nrows = 0;
        return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "start rows by index (b2n_set_start_rows) are read by b2n_rwalk_batch only");
    }
    const bool gather = ctx->peer.total > 0;
    if (!gather && (!u || !v || !logl || !ncall)) return B2N_ERR_ARG;
    if (a->model_id < 0 || a->model_id >= (int)ctx->models.size()) return B2N_ERR_ARG;
    const B2nModel m = ctx->models[a->model_id];
    const int n = a->ndim;
    const int64_t Q = a->nchain;
    if (n != m.ndim || Q < 0) return B2N_ERR_ARG;
    if (Q == 0) return gather ? b2n_fail(ctx, B2N_ERR_ARG, "gather mode: every rank must run at least one chain") : B2N_OK;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    ZcScope zc(ctx);
    const bool dyn = ctx->dyn.active;
    if (dyn) {
        ctx->dyn.cpc = 1;
        if (ctx->dyn.plan_only) return B2N_OK;
        if (gather || ctx->ptr_mode != B2N_PTR_DEVICE) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "device-paced launch needs device pointers and no gather mode");
    }
    CubeParams p;
    p.dyn = dyn ? ctx->dyn.dev : nullptr;
    p.m = m; p.n = n; p.Q = Q; p.loglstar = a->loglstar; p.seed = a->seed; p.chain0 = a->chain0;
    void *du, *dv, *dl, *dnc, *dfl = nullptr;
    void* gdev[7];
    bool peer_on = false;
    B2N_TRY(b2n_peer_begin(ctx, n, &p.peer, gdev, &peer_on));
    if (peer_on) {
        if (ctx->peer.row0 + Q > ctx->peer.total) return b2n_fail(ctx, B2N_ERR_ARG, "gather rows out of range (b2n_peer_rows)");
        du = gdev[0]; dv = gdev[1]; dl = gdev[2]; dnc = gdev[3]; dfl = gdev[6];
    } else {
        B2N_TRY(b2n_out(ctx, ctx->out0, u, (size_t)Q * n * sizeof(double), &du));
        B2N_TRY(b2n_out(ctx, ctx->out1, v, (size_t)Q * n * sizeof(double), &dv));
        B2N_TRY(b2n_out(ctx, ctx->out2, logl, (size_t)Q * sizeof(double), &dl));
        B2N_TRY(b2n_out(ctx, ctx->out3, ncall, (size_t)Q * sizeof(int), &dnc));
        if (dyn) dfl = flags;
        else { B2N_CUDA(ctx, ctx->out6.ensure((size_t)Q * sizeof(uint32_t))); dfl = ctx->out6.p; }
    }
    p.u = (double*)du; p.v = (double*)dv; p.logl = (double*)dl; p.ncall = (int*)dnc; p.flags = (uint32_t*)dfl;
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
    int* herr = reinterpret_cast<int*>(ctx->pinned);
    *herr = 0;
    B2N_CUDA(ctx, ctx->out7.ensure(64));
    B2N_CUDA(ctx, cudaMemsetAsync(ctx->out7.p, 0, sizeof(int), ctx->stream));
    const uint32_t* eflags = peer_on ? (const uint32_t*)(ctx->peer.win + ctx->peer.off[6]) : (const uint32_t*)dfl;
    unif_error_kernel<<<64, 256, 0, ctx->stream>>>(eflags, peer_on ? ctx->peer.total : Q, ctx->out7.as<int>());
    B2N_LAUNCH_CHECK(ctx);
    B2N_CUDA(ctx, cudaMemcpyAsync(herr, ctx->out7.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    if (peer_on) {
        void* const user7[7] = {u, v, logl, ncall, nullptr, nullptr, flags};
        B2N_TRY(b2n_peer_end(ctx, n, user7));
        B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (ctx->ptr_mode == B2N_PTR_HOST && *ctx->peer.err_host)
            return b2n_fail(ctx, B2N_ERR_PEER, "a peer never arrived at the exchange (timeout in the kernel)");
    } else {
        B2N_TRY(b2n_out_done(ctx, u, du, (size_t)Q * n * sizeof(double)));
        B2N_TRY(b2n_out_done(ctx, v, dv, (size_t)Q * n * sizeof(double)));
        B2N_TRY(b2n_out_done(ctx, logl, dl, (size_t)Q * sizeof(double)));
        B2N_TRY(b2n_out_done(ctx, ncall, dnc, (size_t)Q * sizeof(int)));
        if (flags && ctx->ptr_mode == B2N_PTR_HOST)
            B2N_CUDA(ctx, cudaMemcpyAsync(flags, dfl, (size_t)Q * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
        B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    if (*herr & 2) return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "unit-cube sampling did not find a point above the threshold (draw limit)");
    return B2N_OK;
}

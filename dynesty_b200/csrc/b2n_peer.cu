// b2n_peer.cu -- multi-GPU exchange of finished chains over NVLink peer memory.
//
// SURVEY.md 8(e): the path shards by chains (the reference's pool.map over queue slots,
// sampler.py:717) and every rank needs every finished chain, i.e. an all-gather per queue fill.
// Here the gather is FUSED into the chain kernels: each rank owns an exchange window in its HBM,
// maps the windows of all peers (CUDA IPC; NVSwitch gives every pair full bandwidth), and the
// kernels store every finished chain into all windows (b2n_chain.cuh: peer_put).  The grid's last
// CTA then signals every peer's arrive counter and waits for its own counter to reach
// world x epoch (peer_finish), so "launch complete on this rank" implies "all rows of the fill
// are present in this rank's window" -- no collective, no extra launch, the stores overlap the
// tail of the compute.  This file is the host side: window management and the gather-mode
// plumbing of the batch entry points.
#include "b2n_common.cuh"

static inline uint64_t al256(uint64_t b) { return (b + 255) & ~(uint64_t)255; }

static uint64_t slot_bytes(int64_t R, int n) {
    uint64_t b = 0;
    for (int k = 0; k < B2N_NSLOT; k++) b += al256((uint64_t)R * b2n_slot_row_bytes(k, n));
    return b;
}

static void slot_offsets(int64_t R, int n, int slot, uint64_t off[B2N_NSLOT]) {
    uint64_t o = B2N_PEER_HDR + (uint64_t)slot * slot_bytes(R, n);
    for (int k = 0; k < B2N_NSLOT; k++) { off[k] = o; o += al256((uint64_t)R * b2n_slot_row_bytes(k, n)); }
}

void b2n_peer_release(b2n_ctx* ctx) {
    PeerState& P = ctx->peer;
    for (int w = 0; w < B2N_MAX_PEERS; w++) {
        if (P.opened[w] && P.base[w]) cudaIpcCloseMemHandle(P.base[w]);
        P.opened[w] = false;
        P.base[w] = nullptr;
    }
    if (P.win) cudaFree(P.win);
    if (P.err_host) cudaFreeHost(P.err_host);
    P = PeerState();
}

extern "C" {

uint64_t b2n_peer_window_bytes(int64_t total_rows, int32_t ndim) {
    return B2N_PEER_HDR + 2 * slot_bytes(total_rows, ndim);
}

int b2n_peer_export(b2n_ctx* ctx, uint64_t bytes, unsigned char* handle) {
    if (!ctx || !handle || bytes < B2N_PEER_HDR) return B2N_ERR_ARG;
    static_assert(sizeof(cudaIpcMemHandle_t) == B2N_PEER_HANDLE_BYTES, "IPC handle size");
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    b2n_peer_release(ctx);
    PeerState& P = ctx->peer;
    B2N_CUDA(ctx, cudaMalloc((void**)&P.win, bytes));
    P.win_bytes = bytes;
    B2N_CUDA(ctx, cudaMemsetAsync(P.win, 0, bytes, ctx->stream));
    B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    B2N_CUDA(ctx, cudaDeviceSynchronize());          // header is zero before any peer can store
    B2N_CUDA(ctx, cudaHostAlloc((void**)&P.err_host, 64, cudaHostAllocDefault));
    *P.err_host = 0;
    cudaIpcMemHandle_t h;
    B2N_CUDA(ctx, cudaIpcGetMemHandle(&h, P.win));
    memcpy(handle, &h, sizeof(h));
    return B2N_OK;
}

static int peer_common(b2n_ctx* ctx, int rank, int world) {
    if (!ctx || world < 1 || world > B2N_MAX_PEERS || rank < 0 || rank >= world) return B2N_ERR_ARG;
    if (!ctx->peer.win) return b2n_fail(ctx, B2N_ERR_PEER, "b2n_peer_export must come first");
    ctx->peer.world = world;
    ctx->peer.rank = rank;
    ctx->peer.epoch = 0;
    return B2N_OK;
}

int b2n_peer_import(b2n_ctx* ctx, int32_t rank, int32_t world, const unsigned char* handles) {
    B2N_TRY(peer_common(ctx, rank, world));
    if (!handles) return B2N_ERR_ARG;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    PeerState& P = ctx->peer;
    for (int w = 0; w < world; w++) {
        if (w == rank) { P.base[w] = P.win; continue; }
        cudaIpcMemHandle_t h;
        memcpy(&h, handles + (size_t)w * B2N_PEER_HANDLE_BYTES, sizeof(h));
        void* p = nullptr;
        B2N_CUDA(ctx, cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        P.base[w] = (char*)p;
        P.opened[w] = true;
    }
    return B2N_OK;
}

int b2n_peer_import_raw(b2n_ctx* ctx, int32_t rank, int32_t world, void* const* windows) {
    B2N_TRY(peer_common(ctx, rank, world));
    if (!windows) return B2N_ERR_ARG;
    PeerState& P = ctx->peer;
    for (int w = 0; w < world; w++) {
        if (w != rank && !windows[w]) return B2N_ERR_ARG;
        P.base[w] = (w == rank) ? P.win : (char*)windows[w];
    }
    return B2N_OK;
}

int b2n_peer_rows(b2n_ctx* ctx, int64_t row0, int64_t total_rows) {
    if (!ctx || row0 < 0 || total_rows < 0 || (total_rows > 0 && row0 >= total_rows)) return B2N_ERR_ARG;
    if (total_rows > 0 && ctx->peer.world < 1) return b2n_fail(ctx, B2N_ERR_PEER, "peer windows not imported");
    ctx->peer.row0 = row0;
    ctx->peer.total = total_rows;
    return B2N_OK;
}

int b2n_peer_result(b2n_ctx* ctx, void** window, uint64_t* offsets7) {
    if (!ctx || !ctx->peer.win) return B2N_ERR_ARG;
    if (window) *window = ctx->peer.win;
    if (offsets7) memcpy(offsets7, ctx->peer.off, sizeof(ctx->peer.off));
    return B2N_OK;
}

int b2n_peer_read(b2n_ctx* ctx, uint64_t offset, void* host_dst, uint64_t bytes) {
    if (!ctx || !ctx->peer.win || !host_dst || offset + bytes > ctx->peer.win_bytes) return B2N_ERR_ARG;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    B2N_CUDA(ctx, cudaMemcpyAsync(host_dst, ctx->peer.win + offset, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B2N_OK;
}

int b2n_peer_check(b2n_ctx* ctx) {
    if (!ctx || !ctx->peer.win) return B2N_ERR_ARG;
    B2N_CUDA(ctx, cudaSetDevice(ctx->device));
    B2N_CUDA(ctx, cudaMemcpyAsync(ctx->peer.err_host, ctx->peer.win + 8, 4, cudaMemcpyDeviceToHost, ctx->stream));
    B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (*ctx->peer.err_host) return b2n_fail(ctx, B2N_ERR_PEER, "a peer never arrived at the exchange (timeout in the kernel)");
    return B2N_OK;
}

}  // extern "C"

int b2n_chain_begin(b2n_ctx* ctx, const b2n_chain_args* a, bool draw_only, B2nModel* m) {
    if (!ctx || !a) return B2N_ERR_ARG;
    if (ctx->start_idx) {
        ctx->start_idx = nullptr; ctx->start_nrows = 0;
        return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "start rows by index (b2n_set_start_rows) are read by b2n_rwalk_batch only");
    }
    if (draw_only) {
        memset(m, 0, sizeof(*m));
        m->ndim = a->ndim;
        m->like_kind = B2N_LIKE_EGGBOX;
        return B2N_OK;
    }
    if (a->model_id < 0 || a->model_id >= (int)ctx->models.size()) return B2N_ERR_ARG;
    *m = ctx->models[a->model_id];
    return B2N_OK;
}

int b2n_chain_none(b2n_ctx* ctx) {
    return ctx->peer.total > 0 ? b2n_fail(ctx, B2N_ERR_ARG, "gather mode: every rank must run at least one chain") : B2N_OK;
}

int b2n_chain_dyn(b2n_ctx* ctx, int chains_per_cta) {
    ctx->dyn.cpc = chains_per_cta;
    if (!ctx->dyn.plan_only && (ctx->peer.total > 0 || ctx->ptr_mode != B2N_PTR_DEVICE))
        return b2n_fail(ctx, B2N_ERR_UNSUPPORTED, "device-paced launch needs device pointers and no gather mode");
    return B2N_OK;
}

int b2n_chain_bind(b2n_ctx* ctx, int n, int64_t Q, void* const* out, void** dev, PeerSet* ps) {
    PeerState& P = ctx->peer;
    *ps = PeerSet();
    if (P.total == 0) {
        DevBuf* const stage[B2N_NSLOT] = {&ctx->out0, &ctx->out1, &ctx->out2, &ctx->out3, &ctx->out4, &ctx->out5, &ctx->out6};
        for (int k = 0; k < B2N_NSLOT; k++) B2N_TRY(b2n_out(ctx, *stage[k], out[k], (size_t)Q * b2n_slot_row_bytes(k, n), &dev[k]));
        return B2N_OK;
    }
    if (b2n_peer_window_bytes(P.total, n) > P.win_bytes)
        return b2n_fail(ctx, B2N_ERR_PEER, "exchange window too small for this fill (b2n_peer_window_bytes)");
    P.epoch++;
    slot_offsets(P.total, n, (int)(P.epoch & 1), P.off);
    for (int k = 0; k < B2N_NSLOT; k++) dev[k] = P.win + P.off[k] + (uint64_t)P.row0 * b2n_slot_row_bytes(k, n);
    ps->world = P.world;
    ps->rank = P.rank;
    for (int w = 0; w < P.world; w++) ps->base[w] = P.base[w];
    ps->target = (unsigned long long)P.world * P.epoch;
    if (P.row0 + Q > P.total) return b2n_fail(ctx, B2N_ERR_ARG, "gather rows out of range (b2n_peer_rows)");
    return B2N_OK;
}

__global__ void chain_flags_kernel(const uint32_t* flags, int64_t Q, uint32_t mask, unsigned* out) {
    uint32_t bad = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < Q; i += (int64_t)gridDim.x * blockDim.x)
        bad |= flags[i] & mask;
    if (bad) atomicOr(out, bad);
}

int b2n_chain_end(b2n_ctx* ctx, int n, int64_t Q, void* const* out, void* const* dev, const B2nFlagStatus* tab,
                  int ntab) {
    PeerState& P = ctx->peer;
    const bool gather = P.total > 0;
    unsigned* hbits = reinterpret_cast<unsigned*>(ctx->pinned);
    if (ntab > 0) {
        uint32_t mask = 0;
        for (int t = 0; t < ntab; t++) mask |= tab[t].bit;
        *hbits = 0;
        B2N_CUDA(ctx, ctx->out7.ensure(64));
        B2N_CUDA(ctx, cudaMemsetAsync(ctx->out7.p, 0, sizeof(unsigned), ctx->stream));
        // (gather mode: over the rows of ALL ranks, so that every rank returns the same status)
        const uint32_t* flags = gather ? (const uint32_t*)(P.win + P.off[B2N_SLOT_FLAGS]) : (const uint32_t*)dev[B2N_SLOT_FLAGS];
        chain_flags_kernel<<<64, 256, 0, ctx->stream>>>(flags, gather ? P.total : Q, mask, ctx->out7.as<unsigned>());
        B2N_LAUNCH_CHECK(ctx);
        B2N_CUDA(ctx, cudaMemcpyAsync(hbits, ctx->out7.p, sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
    }
    if (gather) {
        const cudaMemcpyKind kind = ctx->ptr_mode == B2N_PTR_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
        for (int k = 0; k < B2N_NSLOT; k++)
            if (out[k]) B2N_CUDA(ctx, cudaMemcpyAsync(out[k], P.win + P.off[k], (size_t)P.total * b2n_slot_row_bytes(k, n), kind, ctx->stream));
        if (ctx->ptr_mode == B2N_PTR_HOST)
            B2N_CUDA(ctx, cudaMemcpyAsync(P.err_host, P.win + 8, 4, cudaMemcpyDeviceToHost, ctx->stream));
    } else {
        for (int k = 0; k < B2N_NSLOT; k++) B2N_TRY(b2n_out_done(ctx, out[k], dev[k], (size_t)Q * b2n_slot_row_bytes(k, n)));
    }
    if (ntab > 0 || ctx->ptr_mode == B2N_PTR_HOST) B2N_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (gather && ctx->ptr_mode == B2N_PTR_HOST && *P.err_host)
        return b2n_fail(ctx, B2N_ERR_PEER, "a peer never arrived at the exchange (timeout in the kernel)");
    for (int t = 0; t < ntab; t++)
        if (*hbits & tab[t].bit) return tab[t].msg ? b2n_fail(ctx, tab[t].status, tab[t].msg) : tab[t].status;
    return B2N_OK;
}

// b2n_bounding.cuh -- node-batched bounding-ellipsoid construction (shared by the
// single-ellipsoid, multi-ellipsoid and bootstrap entry points).
//
// A "node" is a subset of the live points: a contiguous segment [start, start+count)
// of an index array `perm` into the (N, n) row-major point block.  All kernels take
// a list of nodes so that the siblings of one recursion level of
// _bounding_ellipsoids (reference bounding.py:1464-1563) are processed by ONE
// launch per stage.
#pragma once
#include "b2n_device.cuh"

// rows of a node handled by one moment / fmax job: 128 for large live sets; smaller ones are cut finer so that a
// level of the tree is ~64 jobs instead of ~16 (2000 x 50 would otherwise launch 16 CTAs on a GPU of 132 SMs)
static inline int b2n_rows_per_job(long long N) {
    if (N > 8192) return 128;
    long long r = ((N + 63) / 64 + 15) / 16 * 16;
    return (int)(r < 32 ? 32 : (r > 128 ? 128 : r));
}
#define B2N_TILE 64              // covariance output tile edge
#define B2N_TK 16                // rows per shared-memory stage of the covariance kernel

struct NodeStat {
    int good;        // improve_covar_mat returned good_mat (trial == 0)   bounding.py:1382
    int fallback;    // identity fallback taken                              bounding.py:1373-1378
    int error;       // b2n_status for this node (0 ok)
    int sweeps;      // Jacobi sweeps of the last decomposition (diagnostic)
    int trial;       // repair-ladder trial counter (sliced path: one decomposition per launch)
    int retry;       // 1 = covariance was modified, decompose again (bounding.py:1362-1371)
    int suspect;     // candidate (Cholesky) path only: conditioning / convergence not certified -> the caller
                     // redoes the whole update with the full eigen path
    int pad;
    double fmax;     // max_i delta_i^T am delta_i                           bounding.py:1438
    double mult;     // covariance scaling applied after pass 0              bounding.py:1444-1450
    double logvol;
};

struct NodeRef {     // per-node view used by finalize kernels
    int node;
    int start, count;
    int slot0, nslots;
    int level;       // which perm buffer holds this node's indices
};

// Node-indexed device arrays (capacity `cap` nodes)
struct NodeArrays {
    int n, ld;               // dimension, leading dim of the eigen workspaces
    double* mean;            // cap x n
    double* covraw;          // cap x n x n   sample covariance (ddof = 1)
    double* cov;             // cap x n x n   "safe" covariance (after ladder + scaling)
    double* am;              // cap x n x n   precision
    double* axes;            // cap x n x n   axes[i][k] = V[i][k] * sqrt(lam_k), ascending lam
    double* lam;             // cap x n       eigenvalues of cov, ascending
    double* axlens;          // cap x n
    NodeStat* stat;          // cap
};

struct BoundWork {
    b2n_ctx* ctx;
    const double* P;     // device points (N x n)
    int64_t N;
    int n, cap;
    NodeArrays na;
    int* perm;           // 2 x N ping-pong index buffers ("levels" 0 / 1)
    double logvol_pref;
};
#ifdef __cplusplus
#include <vector>
static inline NodeRef b2n_node_ref(int node, int start, int count, int level) {
    return NodeRef{node, start, count, 0, 0, level};
}
int b2n_boundwork_init(b2n_ctx* ctx, BoundWork& w, const double* dP, int64_t N, int n, int cap);
// The full fit (eigen-decomposition + repair ladder) of every node; synchronises and returns the nodes' stats.
int b2n_fit_nodes(BoundWork& w, const std::vector<NodeRef>& refs, std::vector<NodeStat>& stats);
// Nodes that are only CANDIDATES of the multi-ellipsoid tree (bounding.py:1464-1563 evaluates every candidate but
// returns few): Cholesky-based precision / log-volume + major axis, see chol_node_kernel.  Enqueued only: the
// stats are read later with b2n_read_stats.
int b2n_fit_candidates(BoundWork& w, const std::vector<NodeRef>& refs);
int b2n_read_stats(BoundWork& w, std::vector<NodeStat>& all);
struct JobL {   // one CTA-sized slice of one node: rows [r0, r1) of perm level `level`, partial-result slot `slot`
    int node, r0, r1, slot, level, pad0, pad1, pad2;
};
// speculative eigen fit of the root node on the context's side stream (b2n_bounding.cu)
struct SpecRoot {
    bool launched = false;
    NodeArrays na;               // shadow arrays of node 0 (mean / covraw alias the main arrays)
    int* perm = nullptr;         // private copy of the root's row order
    std::vector<JobL> jobs;      // host copies live as long as the copies they feed
    NodeRef ref;
    int node0 = 0;
};
int b2n_spec_root_launch(BoundWork& w, int count, SpecRoot& sp);
int b2n_spec_root_adopt(BoundWork& w, SpecRoot& sp, NodeStat* stat, bool* ok);
void b2n_spec_root_wait(b2n_ctx* ctx, SpecRoot& sp);
int b2n_emit_node(BoundWork& w, int node, int k, double* ctr, double* cov, double* am, double* axes, double* axlens);
int b2n_init_identity_perm(BoundWork& w);
// mean + sample covariance (ddof = 1) of node 0 = rows [0, count) of perm level 0 -> w.na.mean / w.na.covraw
int b2n_node_moments(BoundWork& w, int count);
int b2n_eig_sliced(BoundWork& w, const int* dlist, int pn, int pass, int retry_only, int* used);
#endif

int b2n_membership_dev(b2n_ctx* ctx, const double* x, int64_t M, int n, const double* ctrs,
                       const double* ams, int K, int strict, uint8_t* mask, int* q, double* d2);

/* b200nest.h -- C ABI of libb200nest.so: the H100 (sm_90a) implementation of
 * dynesty's bounding-and-proposal hot path.
 *
 * The reference (joshspeagle/dynesty @ 99451618, pure Python) has no FFI; its
 * extension seams are three Python duck-types (SURVEY.md section 8b):
 *   bound=<Bound>            py/dynesty/bounding.py:76-122
 *   sample=<InternalSampler> py/dynesty/internal_samplers.py:36-203
 *   pool=<obj with .map>     py/dynesty/utils.py:2358-2381
 * Each entry point below replaces the numeric body of the reference function
 * cited next to it; the Python classes in dynesty_b200/ (ctypes) mirror the
 * three duck-types and call these.  INTEGRATION.md shows the binding.
 *
 * Conventions
 *   - all matrices row-major float64; u = unit-cube coordinates (N, n).
 *   - every function returns a b2n_status (0 = ok); the library never returns
 *     owned memory: the caller allocates all outputs.
 *   - pointer mode (b2n_set_pointer_mode): B2N_PTR_HOST (default) = array
 *     arguments are host pointers, the call copies in/out and synchronises
 *     before returning; B2N_PTR_DEVICE = array arguments are device pointers on
 *     the ctx device, work is enqueued on the ctx stream and NOT synchronised
 *     (functions that must return a host scalar synchronise and say so).
 *     Arguments documented "host" are host pointers in both modes.
 *     In B2N_PTR_HOST mode the chain entry points (b2n_{rwalk,rslice,slice,unif}_batch) use PINNED caller
 *     buffers in place: the kernel reads the start points and writes the finished chains through the
 *     buffers' device alias (no staging copy); pageable buffers are staged.  Same results either way.
 *   - one caller thread per ctx (the reference's master is single-threaded,
 *     calls are strictly serialised from Sampler, sampler.py:676-778).
 */
#ifndef B200NEST_H_
#define B200NEST_H_

#ifdef __CUDACC_RTC__
/* NVRTC (the run-time compiled kernels of a user likelihood) has no C library headers */
#include <cuda/std/cstdint>
typedef cuda::std::int32_t int32_t;
typedef cuda::std::int64_t int64_t;
typedef cuda::std::uint8_t uint8_t;
typedef cuda::std::uint32_t uint32_t;
typedef cuda::std::uint64_t uint64_t;
#else
#include <stddef.h>
#include <stdint.h>
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2n_ctx b2n_ctx;

/* ---- status codes; the Python layer maps them 1:1 onto the reference's
 *      exceptions (file:line of the raise in the reference) ---------------- */
typedef enum {
    B2N_OK = 0,
    B2N_ERR_CUDA = 1,            /* CUDA runtime failure (b2n_last_error)           */
    B2N_ERR_ARG = 2,             /* bad argument                                    */
    B2N_ERR_SINGLE_POINT = 3,    /* ValueError   bounding.py:1405-1407, RuntimeError :666-668 */
    B2N_ERR_SINGULAR = 4,        /* ValueError   bounding.py:218-222                */
    B2N_ERR_ELL_INIT = 5,        /* RuntimeError bounding.py:1451-1453              */
    B2N_ERR_INVALID_REGION = 6,  /* RuntimeError bounding.py:683-685                */
    B2N_ERR_Q0 = 7,              /* RuntimeError bounding.py:570-574                */
    B2N_ERR_SLICE_FAIL = 8,      /* RuntimeError internal_samplers.py:1191-1203     */
    B2N_ERR_NOMEM = 9,
    B2N_ERR_UNSUPPORTED = 10,
    B2N_ERR_TOO_MANY_ELLS = 11,  /* max_ells too small for the decomposition        */
    B2N_ERR_PEER = 12,           /* peer exchange not configured / a peer never arrived */
    B2N_ERR_PLATEAU = 13         /* RuntimeError sampler.py:473-475: no live point above loglstar   */
} b2n_status;

/* warning bits (the reference issues warnings.warn at the cited lines) */
#define B2N_WARN_IDENTITY_FALLBACK 1u /* bounding.py:1373-1378                       */
#define B2N_WARN_DOUBLING          2u /* internal_samplers.py:694, 839, 1144         */
#define B2N_WARN_Q0_SLACK          4u /* bounding.py:576-579                         */
#define B2N_WARN_UNIF_INEFFICIENT  8u /* internal_samplers.py:316-320                */

#define B2N_PTR_HOST   0
#define B2N_PTR_DEVICE 1

/* per-dimension boundary flags (utils.py:950-976 get_nonbounded) */
#define B2N_DIM_PERIODIC   1u
#define B2N_DIM_REFLECTIVE 2u

int  b2n_init(int device, b2n_ctx** ctx);
void b2n_free(b2n_ctx* ctx);
int  b2n_set_stream(b2n_ctx* ctx, void* cuda_stream);   /* cudaStream_t; NULL = own stream */
int  b2n_set_pointer_mode(b2n_ctx* ctx, int mode);
int  b2n_synchronize(b2n_ctx* ctx);
/* Chains per CTA of the chain kernels: by default a launch spreads its chains over as many CTAs as the GPU holds
 * (small launches: ONE chain per CTA, the shortest latency for a lone run).  When many contexts share the GPU
 * (replicas), packing k chains into a CTA (lock-step, k <= 8 / 16 depending on the kernel) leaves the SMs to the
 * other contexts at a small cost in per-launch latency.  Results do not depend on it. */
int  b2n_set_chain_pack(b2n_ctx* ctx, int32_t chains_per_cta);
/* Start points by INDEX for the next b2n_rwalk_batch call (one call, then reset): `u0` of that call is then the
 * whole live set, `nrows` x ndim, and chain q starts from row idx[q] -- what Sampler.propose_live / _fill_queue do
 * with `self.live_u[i, :]` (sampler.py:469-491, 708-717) moved into the kernel: the caller no longer gathers the Q
 * start rows into a contiguous block (40 us of a 0.32 ms end-to-end step at C2).  idx: nchain int32 in [0, nrows),
 * host or device memory like the other arrays of the call; NULL cancels.  Any other chain entry point called with
 * the setting pending clears it and returns B2N_ERR_UNSUPPORTED. */
int  b2n_set_start_rows(b2n_ctx* ctx, const int32_t* idx, int64_t nrows);
/* diagnostic: host microseconds per launch when `nlaunch` empty kernels are enqueued back to back on the ctx stream
 * (call it from several threads / contexts at once to see what the driver's launch path sustains) */
int  b2n_debug_launch_rate(b2n_ctx* ctx, int32_t nlaunch, double* us_per_launch);
const char* b2n_strerror(int status);
const char* b2n_last_error(b2n_ctx* ctx);
const char* b2n_version(void);
/* number of kernel launches issued through this ctx since b2n_init (bench.py gpu_launches) */
int64_t b2n_launch_count(b2n_ctx* ctx);
/* kernel timing for the roofline: when enabled, the chain entry points bracket their main
 * kernel with CUDA events on the ctx stream; b2n_last_kernel_ms waits for it and returns the
 * duration of the most recent one (ms, <0 if none). */
int  b2n_set_timing(b2n_ctx* ctx, int enabled);
double b2n_last_kernel_ms(b2n_ctx* ctx);

/* ---- device models: the "device-side likelihood callback" -----------------
 * The reference evaluates user Python callables prior_transform(u) and
 * loglikelihood(v) once per proposal (internal_samplers.py:957-958, 1116-1117,
 * 328-329).  Inside a kernel that callback is a registry of formulas, plus
 * user CUDA code compiled at run time (B2N_LIKE_USER, b2n_model_create_user): */
#define B2N_PRIOR_IDENTITY   0  /* v = u                                          */
#define B2N_PRIOR_UNIFORM    1  /* v = p0[i] + p1[i]*u   (lo, width)               */
#define B2N_PRIOR_NORMAL_PPF 2  /* v = p0[i] + p1[i]*ndtri(u)  (mu, sigma)         */
#define B2N_PRIOR_USER       3  /* user CUDA code compiled at run time: b2n_model_create_user_ex below  */
#define B2N_LIKE_GAUSS_PREC  0  /* -0.5 (v-vec0)^T mat (v-vec0) + s0              */
#define B2N_LIKE_GAUSS_DIAG  1  /* -0.5 sum vec1[i] (v-vec0)[i]^2 + s0            */
#define B2N_LIKE_EGGBOX      2  /* (2 + prod cos((2 s0 v - s0)/2))^s1  (tmax, power) */
#define B2N_LIKE_SHELLS      3  /* logaddexp of two shells: centres vec0, vec1, radius s0, width s1 */
#define B2N_LIKE_REGION2D    4  /* the hard-edged 2-D regions of the reference's sampler-uniformity harness
                                   (tests/test_sampling.py:8-23) on (v[0], v[1]), other dims free:
                                   s0 = 0: diamond_logl, s0 = 1: checker_logl; -inf outside           */
#define B2N_LIKE_USER        5  /* user CUDA code compiled at run time: b2n_model_create_user below     */

typedef struct {
    int32_t ndim;
    int32_t prior_kind;
    int32_t like_kind;
    int32_t reserved;
    const double* prior_p0;  /* host, ndim (or NULL) */
    const double* prior_p1;  /* host, ndim (or NULL) */
    const double* like_vec0; /* host, ndim (or NULL) */
    const double* like_vec1; /* host, ndim (or NULL) */
    const double* like_mat;  /* host, ndim*ndim symmetric (or NULL) */
    double like_s0, like_s1, like_s2;
} b2n_model_desc;

/* copies the parameters to the device; *model_id is a small integer handle. host args. */
int b2n_model_create(b2n_ctx* ctx, const b2n_model_desc* desc, int32_t* model_id);

/* v = prior_transform(u), logl = loglikelihood(v) for M points (u: M x ndim).
 * Replaces the pool.map of the two callables in sampler.py:148-158. v may be NULL. */
int b2n_model_eval(b2n_ctx* ctx, int32_t model_id, const double* u, int64_t M,
                   double* v, double* logl);

/* ---- user likelihoods: user CUDA code compiled into the proposal kernels at run time ----------
 * The user writes ONE warp-cooperative device function,
 *
 *     __device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane);
 *
 *   - all 32 lanes of a warp call it, lane = 0..31, and it must return the same value on every lane;
 *   - v: the prior-transformed point (n doubles, warp-private shared memory, read only);
 *   - work: n doubles of warp-private shared scratch (contents undefined on entry);
 *   - p: the model's parameter array in device memory (nparams doubles of b2n_model_create_user; NULL if none);
 *   - the warp reductions b2n_warp_sum / b2n_warp_prod / b2n_warp_max / b2n_warp_min are available; a scalar
 *     likelihood is computed on lane 0 and broadcast with __shfl_sync(0xffffffff, x, 0).
 * The prior is the registry's (B2N_PRIOR_*, per-dimension p0 / p1).  The caller compiles the chain kernels with
 * that function as the likelihood -- NVRTC, sm_90a, the program being
 *     #include "b2n_user_kernels.cuh"  followed by the user's source,
 * with one name expression per slot of b2n_user_kernel_exprs -- and hands the cubin to b2n_model_create_user.
 * Every entry point that takes a model id then launches the user's instantiation of the same kernel with the same
 * grid and shared-memory plan.  b2n_rwalk_batch runs a user model on the warp-per-chain kernel at every ndim (the
 * lock-step tensor-core kernels exist for the registry only; B2N_RWALK_IMPL=mma gives B2N_ERR_UNSUPPORTED).
 *
 * b2n_user_kernel_exprs: the NVRTC name expressions to instantiate, in slot order (host only, static strings).
 * b2n_model_create_user: desc gives ndim and the prior; desc->like_kind must be B2N_LIKE_USER (like_* ignored).
 *     image: the cubin (host, image_bytes); lowered_names: the mangled name of every slot, as NVRTC reported it
 *     for the expression of the same index.  Loads the image on the context's device (unloaded by b2n_free) and
 *     copies params (host, nparams doubles, may be NULL) to the device. */
int b2n_user_kernel_exprs(const char* const** exprs, int32_t* count);
int b2n_model_create_user(b2n_ctx* ctx, const b2n_model_desc* desc, const double* params, int64_t nparams,
                          const void* image, size_t image_bytes, const char* const* lowered_names,
                          int32_t* model_id);

/* ---- user priors: a user prior transform compiled into the same kernels ---------------------------------------
 * Beside b2n_user_loglike the user may write a second warp-cooperative device function,
 *
 *     __device__ void b2n_user_prior(const double* u, double* v, double* work, int n, const double* p, int lane);
 *
 *   - all 32 lanes of a warp call it; it writes v[0, n) from u[0, n) and may read ANY component of u, so joint
 *     (non-separable) transforms are allowed: correlated Gaussians, ordered parameters, simplex weights;
 *   - u: read only, n doubles behind a generic pointer (warp-private shared memory in the chain kernels, global
 *     memory in b2n_model_eval);
 *   - v, work: n doubles each of warp-private shared memory; the contents of work are undefined on entry;
 *   - p: the prior's own parameter array in device memory (nprior_params doubles of b2n_model_create_user_ex),
 *     or NULL if none;
 *   - the caller issues __syncwarp() before and after the call; inside it, __syncwarp() between one lane writing
 *     work (or v) and another lane reading it.  The b2n_warp_* reductions are available;
 *   - it must be deterministic: the same u gives the same bits of v.
 * The prior is applied only to proposals inside the unit cube (a random-walk proposal rejected by the cube test
 * is never transformed).  A per-dimension example (log-uniform on [p[i], p[n+i]]):
 *
 *     __device__ void b2n_user_prior(const double* u, double* v, double* work, int n, const double* p, int lane) {
 *         for (int i = lane; i < n; i += 32) v[i] = p[i] * exp(u[i] * log(p[n + i] / p[i]));
 *     }
 *
 * A joint example (correlated Gaussian v = mu + L z, z = ndtri(u), mu = p[0, n), L column-major at p + n):
 *
 *     __device__ void b2n_user_prior(const double* u, double* v, double* work, int n, const double* p, int lane) {
 *         for (int i = lane; i < n; i += 32) work[i] = normcdfinv(u[i]);
 *         __syncwarp();
 *         for (int i = lane; i < n; i += 32) {
 *             double s = p[i];
 *             for (int j = 0; j <= i; j++) s = fma(p[n + (size_t)j * n + i], work[j], s);
 *             v[i] = s;
 *         }
 *     }
 *
 * The program is then  #define B2N_USER_PRIOR, #include "b2n_user_kernels.cuh", the prior, the likelihood  (same
 * options and name expressions as above); B2N_USER_PRIOR also defines the marker b2n_user_prior_abi in the image.
 *
 * b2n_model_create_user_ex: b2n_model_create_user with the prior's parameters.
 *   - desc->prior_kind == B2N_PRIOR_USER: the image must define b2n_user_prior_abi (else B2N_ERR_ARG); prior_params
 *     (host, nprior_params doubles, may be NULL) are copied to the device; desc->prior_p0 / prior_p1 are ignored.
 *   - any other prior kind: exactly b2n_model_create_user; nprior_params must be 0.
 * b2n_model_create and b2n_model_create_user reject B2N_PRIOR_USER. */
int b2n_model_create_user_ex(b2n_ctx* ctx, const b2n_model_desc* desc, const double* params, int64_t nparams,
                             const double* prior_params, int64_t nprior_params,
                             const void* image, size_t image_bytes, const char* const* lowered_names,
                             int32_t* model_id);

/* ---- user blobs: derived quantities of a user model, saved with every sample ------------------------------------
 * The user's source may define a third warp-cooperative device function,
 *
 *     __device__ void b2n_user_blob(const double* v, double* work, int n, const double* p, int lane,
 *                                   double* blob, int nblob);
 *
 *   - all 32 lanes of a warp call it; v (n doubles, read only), work (n doubles of scratch), p (the likelihood's
 *     params, the pointer b2n_user_loglike gets) and lane are those of b2n_user_loglike, which it may call;
 *   - blob: nblob doubles of warp-private shared memory, NaN on entry; the kernel writes them to the point's output
 *     row after the call, so an element left unwritten is NaN;
 *   - the caller issues __syncwarp() before and after the call; inside it, the rule of b2n_user_prior applies;
 *   - it must be deterministic: the same v gives the same bits of the blob.
 * The chain kernels never call it.  A blob is a function of the physical point v, so the blob of a saved sample is
 * computed after the run by one b2n_model_blob over the samples, and equals what a chain carrying the blob of its
 * last accepted point would hold.
 *
 * The program is then  #define B2N_USER_BLOB  (beside B2N_USER_PRIOR when there is a user prior), #include
 * "b2n_user_kernels.cuh", the user's code (same options and name expressions as above).  B2N_USER_BLOB declares
 * b2n_user_blob and adds the kernel extern "C" b2n_user_blob_kernel, which is not a slot of b2n_user_kernel_exprs:
 * b2n_model_create_user(_ex) look it up by that name, and a model whose image lacks it has no blob.
 *
 * b2n_model_blob: blob (M x nblob) of the points v (M x ndim), both row-major, host or device pointers by the
 *     pointer mode.  One warp per point.  B2N_ERR_ARG (message in b2n_last_error) for a registry model, a user model
 *     whose image has no b2n_user_blob_kernel, nblob < 1, M < 0, or (2 ndim + nblob) doubles of staging per point
 *     above the device's opt-in shared memory per block.  M = 0: B2N_OK, no launch.  With b2n_set_timing the call's
 *     kernel time is b2n_last_kernel_ms. */
int b2n_model_blob(b2n_ctx* ctx, int32_t model_id, const double* v, int64_t M, int32_t nblob, double* blob);

/* ---- ellipsoid membership: MultiEllipsoid.within/overlap/contains
 *      (bounding.py:502-523), Ellipsoid.distance_many/contains (:286-305) ----
 * d2[m,k] = (x_m - c_k)^T A_k (x_m - c_k); mask[m,k] = d2 < 1 (strict != 0) or
 * d2 <= 1 (strict == 0); q[m] = number of ellipsoids containing x_m.
 * mask / q / d2 may each be NULL. */
int b2n_membership(b2n_ctx* ctx, const double* x, int64_t M, int32_t n,
                   const double* ctrs, const double* ams, int32_t K, int32_t strict,
                   uint8_t* mask, int32_t* q, double* d2);

/* ---- bounding construction ------------------------------------------------
 * bounding_ellipsoid (bounding.py:1387-1461) incl. improve_covar_mat
 * (:1311-1384) and the Ellipsoid constructor (:201-240).  Outputs: ctr (n),
 * cov/am/axes (n x n; axes[:,i] = i-th principal axis scaled by its length,
 * columns ordered by ascending eigenvalue), axlens (n), logvol (1).
 * *warn receives B2N_WARN_* bits (host int, may be NULL).  Synchronises. */
int b2n_bounding_ellipsoid(b2n_ctx* ctx, const double* points, int64_t N, int32_t n,
                           double* ctr, double* cov, double* am, double* axes,
                           double* axlens, double* logvol, uint32_t* warn);

/* MultiEllipsoid.update without bootstrap: bounding_ellipsoid + the recursive
 * 2-means split _bounding_ellipsoids (bounding.py:665-686, 1464-1563) + the
 * all-points-contained check (:683-685).  labels[N] = index of the leaf
 * ellipsoid each point was assigned to.  nells: host int out.  Arrays sized
 * for max_ells.  Synchronises.  Internally the update uses two more streams of the
 * context besides its own (the root's eigen fit runs speculatively beside the expansion of
 * the candidate tree, the two halves of a candidate fit run side by side);
 * they are drained before the call returns, the caller sees one synchronous call. */
int b2n_multi_decompose(b2n_ctx* ctx, const double* points, int64_t N, int32_t n,
                        int32_t max_ells, int32_t* nells, int32_t* labels,
                        double* ctrs, double* covs, double* ams, double* axes,
                        double* axlens, double* logvols, uint32_t* warn);

/* DIAGNOSTIC, not on the sampling path: the candidate tree of b2n_multi_decompose.  Runs exactly the
 * decomposition b2n_multi_decompose runs on the same points -- the same choice of the Cholesky candidate
 * path (B2N_BOUND_FAST, the context's skip count after a failed certification) and the same redo with the
 * eigen path -- and returns the tree instead of the leaves.  *nnodes (host int): nodes in the tree; the call
 * fails with B2N_ERR_TOO_MANY_ELLS if that exceeds max_nodes (N / n + 3 always suffices).  Node i (node 0
 * is the root; children follow their parent) fills nodes[7 i .. 7 i + 6] = { start, count, child 0, child 1
 * (-1: none), the two cluster sizes of its 2-means split (-1: no split attempted; a split refused by the 2n
 * minimum has sizes but no children), 1 if it is an accepted leaf } and logvols[i] = its log-volume: the
 * candidate fit's, or the final eigen fit's for an accepted leaf.  The node's points are the rows
 * perm[start .. start + count) as a SET (perm[N]: the row order the last partition left).  *path = 1 if the
 * tree came from the Cholesky candidates, 0 from the eigen path.  nodes, logvols, perm and path are host
 * arrays in either pointer mode.  Synchronises. */
int b2n_multi_tree(b2n_ctx* ctx, const double* points, int64_t N, int32_t n, int32_t max_nodes,
                   int32_t* nnodes, int32_t* nodes, double* logvols, int32_t* perm, int32_t* path);

/* Block moments for a row-SHARDED live set (SURVEY.md 8e): mean (n) and sample covariance (n x n, ddof = 1; zeros
 * for a single row) of `points` (N x n) -- np.mean / np.cov of bounding.py:1410-1412 for one shard.  Shards combine
 * exactly: S = sum_r [(N_r - 1) cov_r + N_r (mean_r - mean)(mean_r - mean)^T], cov = S / (N - 1); the ellipsoid then
 * follows from b2n_improve_covar on the combined covariance and an all-reduce(max) of the shard-local
 * max_i delta_i^T am delta_i (b2n_membership's d2).  Synchronises. */
int b2n_moments(b2n_ctx* ctx, const double* points, int64_t N, int32_t n, double* mean, double* cov);

/* improve_covar_mat (bounding.py:1311-1384) on its own: the <= 100-trial repair ladder (eigenvalue clamp at
 * 10 max/1e12, then the identity blend, then the identity fallback) applied to `covar` (n x n).  Outputs:
 * the repaired covariance, its inverse `am`, `axes` = V sqrt(lambda) (columns, ascending eigenvalue);
 * *good = 1 iff the input passed untouched (host int), *warn = B2N_WARN_IDENTITY_FALLBACK bit.  Synchronises. */
int b2n_improve_covar(b2n_ctx* ctx, const double* covar, int32_t n, double* cov_out, double* am,
                      double* axes, int32_t* good, uint32_t* warn);

/* Measured FP64 issue ceilings of this GPU for bench.py's roofline: kind 0 = FP64 FMA (vector pipe),
 * kind 1 = FP64 m8n8k4 MMA (tensor pipe), kinds 2, 3, 4 = the m16n8k4, m16n8k8, m16n8k16 MMA shapes;
 * `iters` rounds of 16 independent accumulator chains per thread, all SMs.
 * *tflops, *ms (best of 4 timed launches, CUDA events): host outputs.  Synchronises. */
int b2n_fp64_peak(b2n_ctx* ctx, int32_t kind, int32_t iters, double* tflops, double* ms);

/* Dependent-issue latency of the instruction of b2n_fp64_peak's `kind`: one warp, one chain of `iters`
 * instructions, SM clocks per instruction (best of 4 launches) in *cycles (host).  Synchronises. */
int b2n_fp64_latency(b2n_ctx* ctx, int32_t kind, int32_t iters, double* cycles);

/* Bit-identity probe of the FP64 MMA shapes on `ntiles` tiles (host arrays, row-major): a[ntiles][16][8],
 * b[ntiles][8][8] (k x n), c[ntiles][16][8].  out[4][ntiles][16][8]: 0 = one m16n8k4 (k 0..3) + c,
 * 1 = two m8n8k4 (rows 0..7 and 8..15, k 0..3) + c, 2 = one m16n8k8 + c, 3 = two chained m16n8k4
 * (k 0..3, then k 4..7) + c.  Synchronises. */
int b2n_dmma_probe(b2n_ctx* ctx, int32_t ntiles, const double* a, const double* b, const double* c, double* out);

/* Ellipsoid.scale_to_logvol for K ellipsoids (bounding.py:242-276, 478-495).
 * target_logvols: host, K.  covs/ams/axes/axlens/logvols updated in place. */
int b2n_scale_to_logvol(b2n_ctx* ctx, int32_t K, int32_t n, double* covs, double* ams,
                        double* axes, double* axlens, double* logvols,
                        const double* target_logvols);

/* _ellipsoid_bootstrap_expand for nboot replicas (bounding.py:1593-1648):
 * replica r resamples with the B2N stream (seed, chain0 + r) (one integers
 * event, oracle/philox.py), fits in-bag, expand[r] = max(1, max out-of-bag
 * min-over-ellipsoids distance).  expands: host, nboot.  Synchronises. */
int b2n_bootstrap_expand(b2n_ctx* ctx, const double* points, int64_t N, int32_t n,
                         int32_t multi, int32_t nboot, uint64_t seed, uint64_t chain0,
                         double* expands);

/* ---- run uncertainties: prior-volume realisations (utils.py:1273-1467 jitter_run, :1932-1997 kld_error) ------
 * R realisations of one dead-point record of N samples (logl ascending, samples_n = live points at each sample).
 * Realisation r draws from the B2N stream (seed, chain0 + r) in the reference's own call order, so the unmodified
 * reference driven by oracle.jitter.ScriptedJitterGenerator(seed, chain0 + r) consumes the same numbers:
 *   tick 0      one uniform vector event over the F samples whose nlive_flag is set (_find_decrease, :1273-1314;
 *               approx != 0: every sample, F = N).  The e-th flagged sample gets ln t = ln(U_e) / samples_n
 *               (rstate.beta(a=samples_n[flag], b=1), :1368).  A flagged sample that opens a decreasing stretch
 *               still takes its element; its t is then replaced by the stretch's.
 *   tick s + 1  decreasing stretch s (samples [b0, b1), nstart = samples_n[b0]): nstart + 1 uniforms, y = -ln U
 *               (rstate.exponential(size=nstart+1), :1384), C = prefix sums of y; sample b0 + j gets
 *               ln t = ln(C[k_j] / C[k_{j-1}]), k_j = samples_n[b0 + j] - 1, k_{-1} = nstart (:1385-1389).
 * Then logvol = cumsum(ln t), the trapezoid integrals of compute_integrals (:1411-1467) give logwt, logz, logzvar
 * and h, and kld = cumsum(p1 (ln p1 - ln p2)) with ln p1 = logwt - logz[-1], ln p2 = logwt_ref - logz_ref (the
 * input run's weights, :1976-1992).  logwt_ref NULL: no KL divergence (kld and kld_full must then be NULL).
 * All arithmetic is FP64; the sums are reassociated (block scans), so values agree with the sequential numpy
 * formulas to rounding, and realisation r does not depend on R.
 * samples_n: HOST, N (the stretch plan is built from it on the host).  logl, logwt_ref: N.
 * Summary outputs, R each, each may be NULL: logz[-1], logzerr[-1] = sqrt(|logzvar[-1]|), h[-1], kld[-1].
 * Full outputs, R x N row-major, each may be NULL: logvol, logwt, logz, kld.  Without them no R x N buffer is
 * allocated.  A fixed number of kernel launches (4, 5 with kld_full), whatever R, N or the number of stretches;
 * R <= 65535.  Synchronises in host-pointer mode. */
int b2n_jitter_runs(b2n_ctx* ctx, const double* logl, const int64_t* samples_n, int64_t N,
                    const double* logwt_ref, double logz_ref, int32_t approx, int32_t R, uint64_t seed,
                    uint64_t chain0, double* logz, double* logzerr, double* h, double* kld,
                    double* logvol_full, double* logwt_full, double* logz_full, double* kld_full);

/* ---- run uncertainties: resample_run (utils.py:1495-1660 of the reference) ----------------------------------------
 * R bootstrap realisations of one record of N samples (logl ascending) made of S strands (strand[i] in 0..S-1, the
 * compacted samples_id).  Strand s is a BASE strand when base[s] != 0 (one of its samples belongs to a batch whose
 * lower bound is -inf), else an add-on strand.  Realisation r draws from the B2N stream (seed, chain0 + r) in the
 * reference's call order, so the unmodified reference driven by oracle.resample.ScriptedResampleGenerator(seed,
 * chain0 + r) consumes the same numbers:
 *   tick 0   one uniform vector event of nbase elements; element e picks base strand
 *            base_ids[min(floor(U_e * nbase), nbase - 1)], base_ids = the base strands in increasing order
 *   tick 1   the same over the nadd add-on strands, present only when nadd > 0.
 * m[s] = the times strand s is drawn.  Sample i appears m[strand[i]] times in the realisation.
 * Live counts (the strand rule): sample p is one PIECE of its strand, live on (birth_p, logl_p]; birth_p is the
 * threshold p entered the live set above.  The piece plan is built on the host: piece_ptr (N + 1) and piece_strand
 * form a CSR of the pieces whose first covered sample is i (a piece covers samples first..p); pieces of live points
 * that were never recorded (a record without its final live points) are listed with their strand and never end.
 * The count at sample i is n_i = sum over the pieces covering it of m of their strand.  Its m copies get ln X
 * increments ln(n/(n+1)) each, except at a strand's last sample when end[i] != 0 (a final live point): there the
 * copies get n, n-1, .., n-m+1 live points, a total increment of ln((n-m+1)/(n+1)).
 * Then the trapezoid integrals of compute_integrals (:1411-1467) over the copies give logz, logzvar and h, and
 * kld = sum of p1 (ln p1 - ln p2), ln p1 = logwt - logz[-1], ln p2 = logwt_ref - logz_ref of the copy's sample
 * (kld_error, :1976-1992).  logwt_ref NULL: no KL divergence (kld must then be NULL).
 * FP64; one CTA per realisation scans the record, so realisation r does not depend on R (R <= 65535).
 * strand, base, piece_ptr, piece_strand, end: HOST.  logl, logwt_ref: N.  end may be NULL (no strand ends).
 * Summary outputs, R each, each may be NULL: logz[-1], logzerr[-1] = sqrt(|logzvar[-1]|), h[-1], kld[-1].
 * mult: R x S row-major int32 (m of every strand), may be NULL.  Two kernel launches whatever R, N or S.
 * Synchronises in host-pointer mode. */
int b2n_resample_runs(b2n_ctx* ctx, const double* logl, const int32_t* strand, int64_t N, int32_t S,
                      const uint8_t* base, const int64_t* piece_ptr, const int32_t* piece_strand, const uint8_t* end,
                      const double* logwt_ref, double logz_ref, int32_t R, uint64_t seed, uint64_t chain0,
                      double* logz, double* logzerr, double* h, double* kld, int32_t* mult);

/* ---- posterior summaries of weighted sample sets (utils.py:1081-1117 mean_and_cov, :1196-1233 quantile) ----------
 * R weight vectors over one set of N samples x (N x n, row-major).  For each realisation r (DESIGN.md section 15.3):
 *   mean_r = sum_i w_ri x_i / wsum,  cov_r = wsum / (wsum^2 - w2sum) sum_i w_ri (x_i - mean_r)(x_i - mean_r)^T,
 * wsum = sum_i w_ri and w2sum = sum of the squares of the weights (of the copies, on the resample path).  The second
 * moments are accumulated about a shift c (n) that is the same for every realisation of a call, then corrected:
 * sum w (x - mean)(x - mean)^T = sum w (x - c)(x - c)^T - wsum (mean - c)(mean - c)^T.
 * quant_r[j][t]: the weighted quantile q[t] of coordinate j.  Nodes: the samples present in realisation r, sorted
 * stably by (x_ij, i); a node carries its weight (on the resample path, the sum over the sample's copies).  Node k has
 * cdf C_k = sum_{l<k} w_l / sum_{l<M-1} w_l (M nodes, so the last node's own weight never enters); for q, take p = the
 * largest k with C_k <= q: the result is x_p if q == C_p or p is the last node, else the linear interpolation from
 * (C_p, x_p) towards (C_{p+1}, x_{p+1}) -- np.interp's rule with repeated cdf values.  A node of weight 0 is a node; a
 * weight of -0.0 (the sign bit set) marks a sample ABSENT from the realisation.  A set whose sum_{l<M-1} w_l is 0 (one
 * node, or all the weight on the last node) gives NaN; with one sample present wsum^2 == w2sum and cov is undefined,
 * as in the reference.  q must lie in [0, 1]; 1 <= n <= 1024, N * n < 2^31.
 * All FP64.  Sums over N are split in pieces whose bounds depend on N only and reduced in a fixed order, without float
 * atomics: the same bits every call, and realisation r's outputs do not depend on R or on the other realisations.
 * Outputs, each may be NULL: mean (R x n), cov (R x n x n), quant (R x n x nq), row-major.  A fixed number of kernel
 * launches (plus those of one CUB segmented radix sort of the n coordinates when quant is asked for), whatever R, N or
 * n; R <= 65535.  Synchronises in host-pointer mode.
 *
 * b2n_weighted_stats: the weights given, w (R x N, >= 0), and the shift given, shift (n); x, w, shift, q host or device
 * like the other arrays of the call. */
int b2n_weighted_stats(b2n_ctx* ctx, const double* x, int64_t N, int32_t n, const double* w, int32_t R,
                       const double* shift, const double* q, int32_t nq, double* mean, double* cov, double* quant);

/* b2n_jitter_posterior / b2n_resample_posterior: the realisations of b2n_jitter_runs / b2n_resample_runs (same
 * arguments, streams and summaries logz, logzerr, h, kld -- bit for bit), together with the posterior summaries above of
 * each realisation over the record's sample positions x (N x n, in record order):
 *   jitter     w_ri = exp(logwt_ri - logz_r[-1]), every sample present;
 *   resample   W_ri = the sum over sample i's copies of exp(logwt_copy - logz_r[-1]), w2sum over the copies; a sample
 *              drawn 0 times is absent.
 * logwt_ref is required: the shift is the record's own weighted mean, sum exp(logwt_ref) x / sum exp(logwt_ref),
 * computed on the device.  The weights stay on the device (an N x R buffer). */
int b2n_jitter_posterior(b2n_ctx* ctx, const double* logl, const int64_t* samples_n, int64_t N,
                         const double* logwt_ref, double logz_ref, int32_t approx, int32_t R, uint64_t seed,
                         uint64_t chain0, const double* x, int32_t n, const double* q, int32_t nq, double* logz,
                         double* logzerr, double* h, double* kld, double* mean, double* cov, double* quant);
int b2n_resample_posterior(b2n_ctx* ctx, const double* logl, const int32_t* strand, int64_t N, int32_t S,
                           const uint8_t* base, const int64_t* piece_ptr, const int32_t* piece_strand,
                           const uint8_t* end, const double* logwt_ref, double logz_ref, int32_t R, uint64_t seed,
                           uint64_t chain0, const double* x, int32_t n, const double* q, int32_t nq, double* logz,
                           double* logzerr, double* h, double* kld, double* mean, double* cov, double* quant);

/* ---- equal-weight posterior samples (utils.py:895-903 samples_equal, :1120-1187 resample_equal) ------------------
 * R weight vectors over one set of N samples, each turned into M equal-weight draws by the reference's systematic
 * resampling, with its rounding (DESIGN.md section 15.5).  For vector r, on the B2N stream (seed, chain):
 *   tick 0   one uniform u (rstate.random());
 *   c        the SEQUENTIAL left-to-right FP64 cumsum of w (np.cumsum's order), wsum = c[N-1], C_j = c_j / wsum;
 *   pos_i    = (u + i) / M, that add then that divide, i = 0..M-1;
 *   draw_i   = the smallest j with pos_i < C_j.  A position that rounds to 1.0 (possible only when u + M - 1 rounds
 *              up to M) takes N - 1, where the reference raises IndexError;
 *   tick 1   one uniform vector event of M elements; perm = its stable argsort (rstate.permutation: ties, of
 *            probability ~2^-53, by index; no event is drawn for M == 1 in the oracle, and none is needed);
 *   idx[t]   = draw[perm[t]].
 * counts[j] = the times sample j is drawn: floor(M w_j / wsum) or its ceiling.  A sample of weight 0 is never drawn
 * (a weight of -0.0 counts as 0).  idx points at rows of the record; xout[t] = x[idx[t]] (k values a row).
 * The cumsum runs one thread per vector over N (the N x R weights are read coalesced across vectors); counts come
 * from an estimate of each boundary's first position, corrected with the same pos_i; each position finds its sample by
 * bisection.  No float atomics; vector r's outputs do not depend on R.  A fixed number of kernel launches (3, 4 with
 * counts, plus those of one CUB segmented radix sort) whatever N, M or R.
 * Refused with B2N_ERR_ARG: N or M < 1 or >= 2^31, R < 1 or > 65535, R * M >= 2^31, x NULL with k > 0 or xout
 * given, k < 0; and, after the device has checked the weights (these calls therefore synchronise), a weight that
 * is negative, NaN or inf, or a vector whose sum is 0 or inf.
 * Outputs: idx (R x M int32), counts (R x N int32, may be NULL), wsum (R, may be NULL), xout (R x M x k, may be
 * NULL), row-major.
 *
 * b2n_resample_equal: the weights given, w (R x N, row-major); vector r uses the stream (seed, chain0 + r).  w and x
 * host or device like the outputs. */
int b2n_resample_equal(b2n_ctx* ctx, const double* w, int64_t N, int32_t R, int64_t M, uint64_t seed, uint64_t chain0,
                       const double* x, int32_t k, int32_t* idx, int32_t* counts, double* wsum, double* xout);
/* b2n_jitter_equal / b2n_resample_equal_runs: the realisations of b2n_jitter_runs / b2n_resample_runs (same record
 * arguments and streams, summaries logz, logzerr, h, kld bit for bit, and a pending b2n_set_reweight read the same
 * way), each turned into M equal-weight draws over the record's rows as above.  The weights are those of
 * b2n_jitter_posterior / b2n_resample_posterior: w_ri = exp(logwt_ri - logz_r[-1]); on the resample path the sum over
 * sample i's copies (a sample drawn 0 times has weight -0.0).  So the resample path draws record rows, where the
 * reference's resample_run(res).samples_equal() draws over the copies as rows of their own: the same distribution,
 * not the same bits.  Realisation r's draw uses the stream (seed, B2N_EQUAL_CHAIN0 + chain0 + r), disjoint from the
 * realisation's own (seed, chain0 + r).  logwt_ref is required (kld). */
#define B2N_EQUAL_CHAIN0 (1ull << 62)
int b2n_jitter_equal(b2n_ctx* ctx, const double* logl, const int64_t* samples_n, int64_t N, const double* logwt_ref,
                     double logz_ref, int32_t approx, int32_t R, uint64_t seed, uint64_t chain0, int64_t M,
                     const double* x, int32_t k, double* logz, double* logzerr, double* h, double* kld, int32_t* idx,
                     int32_t* counts, double* wsum, double* xout);
int b2n_resample_equal_runs(b2n_ctx* ctx, const double* logl, const int32_t* strand, int64_t N, int32_t S,
                            const uint8_t* base, const int64_t* piece_ptr, const int32_t* piece_strand,
                            const uint8_t* end, const double* logwt_ref, double logz_ref, int32_t R, uint64_t seed,
                            uint64_t chain0, int64_t M, const double* x, int32_t k, double* logz, double* logzerr,
                            double* h, double* kld, int32_t* idx, int32_t* counts, double* wsum, double* xout);

/* ---- merge_runs (utils.py:1817-1900, _merge_two :2045-2225 of the reference) ---------------------------------------
 * R dead-point records of N samples in all, concatenated: run r is samples [run_ptr[r], run_ptr[r + 1]), its logl
 * ascending and free of NaN (assumed, not checked), samples_n its live count at every sample (>= 1).  The first nbase
 * runs are the BASE group, merged as the reference's pairwise tree: (0, 1), (2, 3), .. per level, an odd run passes to
 * the next level.  Runs nbase..R-1 are ADD-ON runs, merged onto the result one at a time in that order.
 * Each merge of two runs is _merge_two's walk: the base side's point goes first on a tie; the merged point's count is
 * the sum of both runs' counts at their current points (an exhausted run: logl +inf, count 0), except that only the
 * base's count applies while the base's current logl <= the new run's low edge, and otherwise only the new run's while
 * the new run's current logl <= the base's low edge.  lowedge[r]: run r's low edge, the least lower bound of the
 * batches its samples belong to (-inf for a run started from the prior; NULL: -inf for every run); a merged run's is
 * the lesser of its two.
 * Then ln X (:2159-2187): ln t = ln(n / (n + 1)) per merged sample, except inside a group of m >= 2 equal logl whose
 * first point has count n, where the k-th point (k = 0..m-1) gets ln((n - k) / (n - k + 1)) (a group longer than n + 1
 * gives non-finite volumes); logvol = cumsum(ln t), and the trapezoid integrals of compute_integrals (:1411-1467).
 * run_ptr (R + 1, run_ptr[0] = 0, every run non-empty) and lowedge (R): HOST.  logl, samples_n (int64): N.
 * Outputs, each may be NULL: perm (N, int64): the index in the concatenation of every merged sample; samples_n_out
 * (N, int64): the merged counts; last3 (3): logz[-1], logzerr[-1] = sqrt(|logzvar[-1]|), h[-1]; logvol, logwt, logz,
 * logzvar, h (N each): the full arrays of compute_integrals.
 * FP64 / int64, no atomics: the outputs are the same bits from call to call.  1 + ceil(log2 nbase) + (R - nbase) + 1
 * merge launches, then the 4 or 5 of the quadrature, with no host round trip.  1 <= nbase <= R <= 2^31 - 1, N >= 1.
 * Synchronises in host-pointer mode. */
int b2n_merge_runs(b2n_ctx* ctx, const double* logl, const int64_t* samples_n, const int64_t* run_ptr, int32_t R,
                   int32_t nbase, const double* lowedge, int64_t* perm, int64_t* samples_n_out, double* last3,
                   double* logvol, double* logwt, double* logz, double* logzvar, double* h);

/* ---- importance reweighting (reweight_run, utils.py:1663-1708; compute_integrals(reweight=), :1411-1467) ----------
 * A log-reweight logrwt_i = logp_new_i - logp_old_i per sample changes one thing in the quadrature: for every sample,
 * or every copy of a sample in a resample realisation,
 *   logwt_i = logaddexp(L_i, L_{i-1}) + logdvol2_i + logrwt_i.
 * logz, the importance weights exp(logwt - logz[-1]) and the KL terms p1 (ln p1 - ln p2), ln p1 = logwt - logz[-1],
 * follow from it.  The h increments exp(L - zmax + logdvol2) L + .. keep the UNREWEIGHTED L and logdvol2, normalised by
 * the reweighted zmax = logz[-1], so h and logzvar are those of the reference's compute_integrals(reweight=).  Entries
 * may be -inf (zero weight: a KL term of zero weight is 0, where the reference would compute 0 * -inf = NaN); NaN and
 * +inf are refused in host-pointer mode and undefined in device-pointer mode.
 *
 * b2n_compute_integrals: compute_integrals(logl, logvol, reweight=logrwt) of one record on the deterministic passes of
 * b2n_jitter_runs (ln t = diff(logvol, prepend=0)).  logrwt may be NULL (no reweight).  logl, logvol, logrwt: N, host
 * or device like the outputs.  Outputs, each may be NULL: last3 (3): logz[-1], logzerr[-1] = sqrt(|logzvar[-1]|),
 * h[-1]; logwt, logz, logzvar, h (N each).  FP64, sums reassociated (block scans).  5 or 6 kernel launches (6 when
 * logzvar or h is asked for).  Synchronises in host-pointer mode. */
int b2n_compute_integrals(b2n_ctx* ctx, const double* logl, const double* logvol, const double* logrwt, int64_t N,
                          double* last3, double* logwt, double* logz, double* logzvar, double* h);
/* b2n_set_reweight: the log-reweight (N, host or device like the arrays of the call) for the NEXT b2n_jitter_runs /
 * b2n_resample_runs / b2n_jitter_posterior / b2n_resample_posterior / b2n_jitter_equal / b2n_resample_equal_runs
 * call, whose realisations then carry it as above
 * (one call, then reset, however that call ends; the array must stay valid until then).  That call needs the same N,
 * else it fails with B2N_ERR_ARG.  b2n_merge_runs, b2n_weighted_stats, b2n_resample_equal and b2n_compute_integrals
 * called with a
 * reweight pending clear it and return B2N_ERR_UNSUPPORTED.  NULL cancels.  The realisation entry points keep their
 * launch counts; with the reweight they run the _rw instantiations of the same passes. */
int b2n_set_reweight(b2n_ctx* ctx, const double* logrwt, int64_t N);

/* ---- resident bound for the proposal kernels --------------------------------
 * Uploads K ellipsoids of dimension ncdim (what Sampler ships to every task as
 * `axes` / kwargs['bound'], sampler.py:708-717, internal_samplers.py:229-233).
 * host pointers in both modes.  ctrs/ams/logvols may be NULL if only
 * rwalk/slice are used. */
int b2n_bound_set(b2n_ctx* ctx, int32_t K, int32_t ncdim, const double* ctrs,
                  const double* ams, const double* axes, const double* logvols);

/* b2n_unif_batch only: draw from the bound without the unit-cube test and without
 * evaluating a model (Bound.samples, bounding.py:321-334, 592-606); needs ndim == ncdim,
 * model_id ignored. */
#define B2N_OPT_DRAW_ONLY 1
/* with DRAW_ONLY: MultiEllipsoid.sample(return_q=True) semantics (bounding.py:580-584): the
 * draw is returned WITHOUT the 1/q acceptance test and ncall[q] receives q (the number of
 * ellipsoids containing it) -- the input of monte_carlo_logvol (:608-630). */
#define B2N_OPT_DRAW_MIXTURE 2

/* ---- proposal chains ----------------------------------------------------------
 * One chain per queue slot (sampler.py:690-717).  Chain q consumes the B2N
 * Philox stream (seed, chain0 + q) -- see oracle/philox.py for the layout. */
typedef struct {
    int64_t nchain;          /* Q                                                   */
    int32_t ndim;            /* n                                                   */
    int32_t ncdim;           /* clustered dims (axes are ncdim x ncdim)              */
    int32_t model_id;
    int32_t reserved;        /* option bits: B2N_OPT_*                               */
    const double* u0;        /* Q x ndim start points (live points with logl > loglstar) */
    const int32_t* ell;      /* HOST, Q: index into the resident bound of the axes of
                                each chain (get_random_axes, bounding.py:726-731); NULL = 0 */
    const uint8_t* dimflags; /* HOST, ndim B2N_DIM_* flags or NULL                      */
    double loglstar;
    double scale;
    uint64_t seed;
    uint64_t chain0;
} b2n_chain_args;

/* RWalkSampler.sample -> generic_random_walk (internal_samplers.py:505-561,
 * 866-986, propose_ball_point :989-1035): exactly `walks` proposals per chain.
 * Outputs per chain: u, v (Q x ndim), logl, n_accept, n_reject, ncall (Q). */
int b2n_rwalk_batch(b2n_ctx* ctx, const b2n_chain_args* a, int32_t walks,
                    double* u, double* v, double* logl,
                    int32_t* n_accept, int32_t* n_reject, int32_t* ncall);

/* ---- stepped random walk: the walk of b2n_rwalk_batch, one launch per step, for a likelihood that runs OUTSIDE the
 * library between the launches (a batched PyTorch function on the same stream, dynesty_b200.TorchModel).
 * A fill of Q chains is walks + 1 calls, step = 0 .. walks, each enqueuing one launch and no synchronisation:
 *   step 0        chain q starts at u0[q] (u written, u_start[q] too when given) and proposes step 0
 *   step s        accepts step s - 1 -- inside the cube and logl_prop[q] > loglstar: u, v, logl <- the proposal and
 *                 n_accept + 1, else n_reject + 1 (a NaN logl_prop is rejected) -- then proposes step s
 *   step walks    accepts step walks - 1; a chain that never accepted gets v_start / logl_start; ncall = walks
 * A proposal writes u_prop[q] and in_cube[q]; an out-of-cube proposal's row of u_prop is the chain's current u, so
 * that the caller only ever evaluates points of the cube.  Between step s and s + 1 the caller puts the prior
 * transform of u_prop in v_prop and its log-likelihood in logl_prop; before step `walks` the same for the start rows
 * in v_start / logl_start.  Chain q draws from the B2N stream (seed, chain0 + q) exactly as in b2n_rwalk_batch, so
 * a likelihood that returns the bits the in-kernel one does gives bit-identical chains.  Every pointer is a device
 * pointer, and the fields are re-read at every call (the caller may point v_prop at a new buffer each step). */
typedef struct {
    double*         u_prop;      /* Q x ndim, out                                                       */
    const double*   v_prop;      /* Q x ndim, in (steps >= 1): prior transform of u_prop                */
    const double*   logl_prop;   /* Q, in (steps >= 1)                                                  */
    double*         u_start;     /* Q x ndim, out at step 0 (a copy of the start rows), may be NULL     */
    const double*   v_start;     /* Q x ndim, in (step walks): prior transform of the start rows        */
    const double*   logl_start;  /* Q, in (step walks)                                                  */
    uint32_t*       tick;        /* Q: next draw event of every chain                                   */
    int32_t*        in_cube;     /* Q: the last proposal lies inside the cube                           */
    const uint32_t* dimflags;    /* ndim B2N_DIM_* flags (device, uint32) or NULL; b2n_chain_args.dimflags is not read */
    int32_t*        order;       /* Q, written at step 0 (b2n_rwalk_step): the chains grouped by ellipsoid */
    int32_t*        cta;         /* 3 x Q, written at step 0 (b2n_rwalk_step): (first, count, ellipsoid) per CTA */
    int32_t         ncta;        /* out at step 0 (b2n_rwalk_step), in at later steps                   */
    int32_t         reserved;
} b2n_rwalk_state;

/* One step of a host fill: a = the fill's chains as for b2n_rwalk_batch (u0 a device pointer; ell read at step 0
 * only), outputs as b2n_rwalk_batch's, which also hold the chains' state between the calls.  Needs
 * B2N_PTR_DEVICE, the resident bound, no gather mode and no pending b2n_set_start_rows. */
int b2n_rwalk_step(b2n_ctx* ctx, const b2n_chain_args* a, int32_t walks, int32_t step, b2n_rwalk_state* st,
                   double* u, double* v, double* logl, int32_t* n_accept, int32_t* n_reject, int32_t* ncall);

/* RSliceSampler.sample (internal_samplers.py:745-855) / SliceSampler.sample
 * (:593-709) -> generic_slice_step (:1075-1206).  flags[q]: B2N_WARN_DOUBLING if
 * the chain switched to doubling; status B2N_ERR_SLICE_FAIL if any chain's
 * interval collapsed or stepped out more than 4e6 times.  n_expand[q] saturates at
 * INT32_MAX (a step with D doublings counts 2^D - 1, and a tiny scale takes 31 or
 * more), where the reference's count keeps growing. */
int b2n_rslice_batch(b2n_ctx* ctx, const b2n_chain_args* a, int32_t slices,
                     int32_t doubling, double* u, double* v, double* logl,
                     int32_t* n_expand, int32_t* n_contract, int32_t* ncall,
                     uint32_t* flags);
int b2n_slice_batch(b2n_ctx* ctx, const b2n_chain_args* a, int32_t slices,
                    int32_t doubling, double* u, double* v, double* logl,
                    int32_t* n_expand, int32_t* n_contract, int32_t* ncall,
                    uint32_t* flags);

/* UnitCubeSampler.sample (internal_samplers.py:343-441) for a queue: every chain draws u ~ U(0,1)^ndim (one
 * uniform vector event per draw of its B2N stream) until loglikelihood(prior_transform(u)) > loglstar; ncall[q] =
 * number of draws.  u0 / ell / scale / ncdim unused, no resident bound needed.  flags may be NULL. */
int b2n_unitcube_batch(b2n_ctx* ctx, const b2n_chain_args* a, double* u, double* v, double* logl,
                       int32_t* ncall, uint32_t* flags);

/* UniformBoundSampler.sample (internal_samplers.py:243-340) with
 * MultiEllipsoid.sample (bounding.py:525-590) as the bound draw; u0/ell/scale
 * unused.  nprop[q] = draws from the bound incl. out-of-cube ones. */
int b2n_unif_batch(b2n_ctx* ctx, const b2n_chain_args* a, double* u, double* v,
                   double* logl, int32_t* ncall, int32_t* nprop, uint32_t* flags);

/* ---- RadFriends / SupFriends: one ball / cube per live point (bounding.py:734-996, 999-1263) ------------------
 * kind: 0 = balls (RadFriends, Euclidean norm), 1 = cubes (SupFriends, Chebyshev norm).
 * b2n_friends_update  = RadFriends.update / SupFriends.update (:874-958 / 1142-1226): covariance from the clusters
 *     of the single-linkage tree cut at Mahalanobis distance 1 under the CURRENT metric am_prev (use_clustering;
 *     :966-993), am = pinvh(cov), axes = sqrtm(cov), axes_inv = pinvh(axes), radius = leave-one-out nearest-neighbour
 *     distance (nboot = 0; :1683-1705) or the bootstrap radius over nboot realisations (:1651-1680; realisation b
 *     resamples with the B2N stream (seed, chain0 + b), one integers event), everything rescaled by the radius,
 *     logvol = prefactor - slogdet(am) / 2.  Outputs (n x n each, logvol / radius / nclusters host scalars); the
 *     caller keeps `ctrs = points` (:950, sampler.py:481).  Synchronises.
 * b2n_friends_set     makes (ctrs, axes, axes_inv) the resident friends bound of the ctx.
 * b2n_friends_overlap = overlap(x) (:785-790 / 1052-1057) for M query points: q[m] = number of balls / cubes
 *     containing x_m (contains = q > 0, within = the indices).
 * b2n_friends_unif_batch = UniformBoundSampler.sample (internal_samplers.py:243-340) with the bound's own
 *     sample() (:797-831 / 1065-1100: random centre + random offset, accepted with probability 1/q) as the draw;
 *     a->reserved = B2N_OPT_DRAW_ONLY: Bound.samples (no cube test / likelihood), | B2N_OPT_DRAW_MIXTURE:
 *     sample(return_q=True), ncall[q] = q. */
int b2n_friends_update(b2n_ctx* ctx, const double* points, int64_t N, int32_t n, int32_t kind, int32_t use_clustering,
                       const double* am_prev, int32_t nboot, uint64_t seed, uint64_t chain0, double* cov, double* am,
                       double* axes, double* axes_inv, double* logvol, double* radius, int32_t* nclusters);
int b2n_friends_set(b2n_ctx* ctx, int32_t kind, const double* ctrs, int64_t N, int32_t n, const double* axes,
                    const double* axes_inv);
int b2n_friends_overlap(b2n_ctx* ctx, const double* x, int64_t M, int32_t n, int32_t* q);
int b2n_friends_unif_batch(b2n_ctx* ctx, const b2n_chain_args* a, double* u, double* v, double* logl, int32_t* ncall,
                           int32_t* nprop, uint32_t* flags);

/* ---- multi-GPU exchange over NVLink peer memory (SURVEY.md 8e) ------------------------------
 * The path shards by CHAINS: rank r of W runs rows [row0, row0 + nchain) of a `total_rows`-chain
 * queue fill (the reference's pool.map over queue slots, sampler.py:717, one slot = one chain).
 * Every rank needs every finished chain (replicated live set), which is an all-gather.  Instead
 * of a collective after the kernel, the chain kernels themselves store each finished chain into
 * the exchange WINDOW of every rank (peer stores over NVLink/NVSwitch), and the last CTA of the
 * grid runs a cross-GPU arrive/wait on counters in the windows: when a b2n_*_batch launch has
 * completed on a rank, all `total_rows` rows are present in that rank's window.
 *
 *   b2n_peer_export   allocate this rank's window, return its 64-byte CUDA IPC handle
 *   (exchange the handles of all ranks with any host transport, e.g. torch.distributed)
 *   b2n_peer_import   map the windows of all ranks (one process per GPU)
 *   b2n_peer_import_raw  same for ranks living in THIS process (device pointers of the windows)
 *   b2n_peer_rows     switch the following b2n_{rwalk,rslice,slice,unif}_batch calls to gather
 *                     mode: a->nchain local chains are rows [row0, row0+nchain) of total_rows;
 *                     output pointers then receive ALL total_rows rows (they may be NULL in
 *                     device-pointer mode: read the window through b2n_peer_result instead).
 *                     total_rows = 0 switches gather mode off.  All ranks must issue the same
 *                     sequence of gather-mode calls.
 *   b2n_peer_result   window pointer + byte offsets {u, v, logl, int0, int1, int2, flags} of the
 *                     last gather-mode call.  int0..int2 hold the call's int32 counters in argument
 *                     order, flags its uint32 flags: rwalk n_accept, n_reject, ncall; slice
 *                     n_expand, n_contract, ncall, flags; unif ncall, nprop, -, flags; unitcube
 *                     ncall, -, -, flags.
 *   b2n_peer_read     synchronise and copy `bytes` at byte `offset` of the own window to HOST memory
 *   b2n_peer_check    synchronise and report B2N_ERR_PEER if a peer never arrived (device mode;
 *                     host-pointer mode checks on return of every call).
 * Windows are double-buffered by call parity, so a rank may consume the rows of call k on its
 * stream while faster peers already store the rows of call k+1. */
#define B2N_PEER_HANDLE_BYTES 64
#define B2N_MAX_PEERS 8
int b2n_peer_export(b2n_ctx* ctx, uint64_t bytes, unsigned char* handle);
int b2n_peer_import(b2n_ctx* ctx, int32_t rank, int32_t world, const unsigned char* handles);
int b2n_peer_import_raw(b2n_ctx* ctx, int32_t rank, int32_t world, void* const* windows);
int b2n_peer_rows(b2n_ctx* ctx, int64_t row0, int64_t total_rows);
int b2n_peer_result(b2n_ctx* ctx, void** window, uint64_t* offsets7);
int b2n_peer_read(b2n_ctx* ctx, uint64_t offset, void* host_dst, uint64_t bytes);
int b2n_peer_check(b2n_ctx* ctx);
/* bytes a window needs for gather-mode calls of total_rows x ndim */
uint64_t b2n_peer_window_bytes(int64_t total_rows, int32_t ndim);

/* ---- device-resident nested-sampling rounds (SURVEY.md 8f-1: "replace K worst points per launch") ----
 * Replaces the reference's per-iteration master loop for the bounded phase of a run: the
 * worst-point search and evidence update of Sampler.sample (sampler.py:1040-1212,
 * utils.py:1470-1492 progress_integration), propose_live (:469-491), _fill_queue / _new_point
 * (:676-778) and the samplers' tune() (internal_samplers.py:460-493, 1209-1239).
 *
 * One ROUND removes the `batch` lowest live points at once (threshold L* = the batch-th lowest
 * logl), evolves `batch` chains from uniformly chosen survivors at L* against the resident bound
 * and writes every chain end point into a freed slot.  Unlike the reference's queue (an entry
 * evolved at an older threshold is kept only if it beats the current one -- a filter that
 * selects the offspring of the best live points when chains stay correlated with their starts,
 * DESIGN.md 9.4) no chain is ever discarded, so there is no selection effect; the live-point
 * count N, N-1, .., N-batch+1 seen by the removed points enters the quadrature the way the
 * reference treats a shrinking live set (ln X -= ln((m+1)/m) at a point with m live points).
 * Tuning (internal_samplers.py:460-493, 1209-1239) happens once per round; for rwalk the update is the product of the
 * `batch` per-iteration updates the reference would have made at that scale, exp(min(batch, ncdim) (abar - facc) /
 * (ncdim facc)) -- batch = 1 is the reference's rule.
 * Launches of R rounds: propose | chains | commit+propose | chains | ... | commit (R chain launches and R + 1
 * single-CTA step launches), no host synchronisation in between;
 * b2n_ns_run enqueues rounds until a stop flag is raised on the device:
 *   done        dlogz / maxiter / maxcall / plateau reached (sampler.py:1095-1120)
 *   need_bound  1 = update interval reached (sampler.py:648-651), 2 = a start point is outside
 *               the bound (forced update, :485-489), 3 = dead-point buffer full, 4 = the FIRST bound is
 *               due (unit-cube phase: enough calls and low efficiency, sampler.py:640-647)
 * The caller then updates the bound from b2n_ns_get_live (b2n_multi_decompose / b2n_bound_set as
 * usual), calls b2n_ns_bound_updated and runs on.  Random streams: chain c of round r is the
 * B2N chain (seed, chain0 + r*batch + c); the round driver (start rows, ellipsoid picks) is the
 * chain (seed, 2^62 + r), tick 0 / 1 = one uniform vector event each (oracle/nsloop.py).      */
typedef struct {
    int32_t nlive, ndim, ncdim, batch;
    int32_t sampler;          /* 0 rwalk, 1 rslice, 2 slice, 3 unif (steps ignored)             */
    int32_t steps;            /* walks / slices                                                  */
    int32_t model_id;
    int32_t strict_contains;  /* 1: MultiEllipsoid.contains (d2 < 1), 0: Ellipsoid.contains (<= 1) */
    double  facc;             /* rwalk target acceptance (internal_samplers.py:449-451)          */
    double  dlogz;
    int64_t maxiter, maxcall; /* in device-buffer iterations / total calls                       */
    int64_t update_interval;  /* bound update every this many calls (dynesty.py:213-240)         */
    uint64_t seed, chain0;
    const uint8_t* dimflags;  /* HOST, ndim B2N_DIM_* flags or NULL (copied)                      */
    /* -- the phase before the first bound (sampler.py:407-409, 625-674; _initialize_live_points + UnitCubeSampler,
     *    sampler.py:56-262, internal_samplers.py:343-441): with unit_cube_phase = 1 the run STARTS with rounds whose
     *    chains draw from the prior (b2n_unitcube_batch) and raises need_bound = 4 once ncall >= first_min_ncall and
     *    the efficiency 100 (it0 + it) / ncall has fallen below first_min_eff; b2n_ns_bound_updated ends the phase. */
    int32_t unit_cube_phase;
    int32_t use_logl_max;     /* 1: stop (done) once the lowest live logl exceeds logl_max (the end of a
                                 dynamic-sampler batch, dynamicsampler.py:1338-1345)                */
    int64_t first_min_ncall;
    double  first_min_eff;
    double  logl_max;
    int64_t it0;              /* iterations of the run before this device phase (enters the efficiency) */
} b2n_ns_config;

typedef struct {
    int64_t it, ncall, rounds;       /* dead points in the device buffer, total calls, rounds done */
    double logz, logvol, loglstar, lmax, delta_logz, scale;
    int32_t done, need_bound, doubling, error;
    int64_t ncall_last_update;       /* calls at the last bound update (restorable state)            */
} b2n_ns_status;

int b2n_ns_create(b2n_ctx* ctx, const b2n_ns_config* cfg, int64_t dead_capacity);
int b2n_ns_destroy(b2n_ctx* ctx);
/* host arrays: the live set (nlive x ndim, nlive) and the scalars of the run so far */
int b2n_ns_set_state(b2n_ctx* ctx, const double* live_u, const double* live_v, const double* live_logl,
                     double logvol, double logz, double loglstar, int64_t it, int64_t ncall, double scale);
/* enqueue up to max_rounds rounds, reading the stop flags every check_every rounds (<= 0: once at
 * the end); synchronises; returns the status (and the sampler error status, e.g.
 * B2N_ERR_SLICE_FAIL, if a chain failed). */
int b2n_ns_run(b2n_ctx* ctx, int32_t max_rounds, int32_t check_every, b2n_ns_status* status);
/* Rounds whose chains are STEPPED (b2n_rwalk_step's walk, likelihood outside the library).  b2n_ns_create takes
 * model_id = -1 ("no in-kernel model") for such a run: sampler 0 (rwalk), unit_cube_phase 0, ndim from the config;
 * b2n_ns_run refuses it with B2N_ERR_UNSUPPORTED.  The caller enqueues, with no synchronisation in between,
 *   b2n_ns_step(3) | b2n_ns_rwalk_step(0) .. b2n_ns_rwalk_step(steps)   per round, then b2n_ns_step(1),
 * with its likelihood between the stepped launches as for b2n_rwalk_step (start rows: st->u_start, which step 0
 * must be given here), and reads the flags with b2n_ns_status_get.
 * b2n_ns_step: one launch of the round kernel; mode 3 = commit the pending round and propose the next, 1 = the
 * closing commit.  b2n_ns_rwalk_step: one stepped launch bound to the current round -- threshold, scale, chain ids,
 * worklist and skip from the round's device state, start rows and outputs the round's own buffers; the order / cta /
 * ncta fields of st are not used.  A round skipped on the device (a stop flag) makes its launches return at once. */
int b2n_ns_step(b2n_ctx* ctx, int32_t mode);
int b2n_ns_rwalk_step(b2n_ctx* ctx, int32_t step, b2n_rwalk_state* st);
int b2n_ns_status_get(b2n_ctx* ctx, b2n_ns_status* status);
/* restore the counters a snapshot of a run carries besides b2n_ns_set_state's arguments (utils.py:2321-2355
 * save / restore of the reference pickles the whole sampler; here: live set + scalars + these): the round
 * index (chain ids and the round driver's stream depend on it), the calls at the last bound update, the
 * slice-doubling switch.  A run restored this way continues bit-identically. */
int b2n_ns_set_counters(b2n_ctx* ctx, int64_t rounds, int64_t ncall_last_update, int32_t doubling);
/* after the caller replaced the resident bound: clears need_bound, restarts the update interval, ends the
 * unit-cube phase */
int b2n_ns_bound_updated(b2n_ctx* ctx);
/* Sampler.update_bound (sampler.py:493-510) WITHOUT leaving the device: fits the bound to the run's live points
 * where they lie in HBM (multi = 1: MultiEllipsoid.update, bounding.py:632-686 -- b2n_multi_decompose; 0:
 * Ellipsoid.update, :345-414 -- b2n_bounding_ellipsoid; first ncdim coordinates), enlarges it
 * (scale_to_logvol(logvol + ln enlarge), sampler.py:506-508) and makes it the resident bound of the ctx -- no
 * live-set download, no bound upload.  Bootstrap expansion is not part of this entry (callers that need it take
 * the host route: b2n_ns_get_live + b2n_bootstrap_expand + b2n_bound_set).  nells / logvol (ln of the summed
 * volumes) / warn: host outputs, may be NULL.  Follow with b2n_ns_bound_updated.  Synchronises. */
int b2n_ns_update_bound(b2n_ctx* ctx, int32_t multi, double enlarge, int32_t* nells, double* logvol, uint32_t* warn);
/* the bound b2n_ns_update_bound built last (host outputs sized for max_ells >= nells; each may be NULL) */
int b2n_ns_get_bound(b2n_ctx* ctx, int32_t max_ells, double* ctrs, double* covs, double* ams, double* axes,
                     double* axlens, double* logvols);
/* grow the dead-point buffer to `capacity` rows (keeps the rows written so far); clears need_bound == 3 */
int b2n_ns_reserve_dead(b2n_ctx* ctx, int64_t capacity);
/* host outputs (each may be NULL) */
int b2n_ns_get_live(b2n_ctx* ctx, double* live_u, double* live_v, double* live_logl);
int b2n_ns_get_dead(b2n_ctx* ctx, int64_t first, int64_t count, double* u, double* v, double* logl,
                    double* logvol, int32_t* ncall);
/* Strands (the reference's samples_id / samples_it, sampler.py:1107, 1182).  Every round records, for its j-th removal,
 * the live slot it occupied (slot[it0 + j] = its row in the live set) and the number of dead rows recorded before it
 * entered the live set (it[it0 + j]); the slot's new occupant then gets it0 + K, the dead rows after the round, so its
 * birth threshold is the logl of dead row it0 + K - 1, the round threshold.  Unit-cube rounds record the same.  Counts
 * are in the numbering of this device buffer (row 0 = the first row after b2n_ns_set_state); b2n_ns_set_state sets
 * every slot's count to 0, b2n_ns_set_live_it replaces them (a hand-over from a host loop or a checkpoint, in the
 * same numbering: negative for points that entered before row 0).  Host outputs (each may be NULL), N = nlive. */
int b2n_ns_get_strands(b2n_ctx* ctx, int64_t first, int64_t count, int32_t* slot, int64_t* it);
int b2n_ns_set_live_it(b2n_ctx* ctx, const int64_t* live_it);
int b2n_ns_get_live_it(b2n_ctx* ctx, int64_t* live_it);

#ifdef __cplusplus
}
#endif
#endif /* B200NEST_H_ */

/*
 * mbar_b200.h — C ABI of libmbar_b200.so: the MBAR solve hot path on NVIDIA H100 (sm_90a).
 *
 * Drop-in boundary.  pymbar has no native FFI; its "operator API" for this path is the set of
 * module-level functions in pymbar/mbar_solvers.py that pymbar.MBAR reaches by attribute lookup
 * (mbar.py:413, :437, :455, :910).  Each entry point below names the reference function it stands
 * in for (paths relative to the pymbar package directory).  INTEGRATION.md shows the ctypes stub a
 * pymbar maintainer would add beside the numpy/JAX switch at mbar_solvers.py:25-87.
 *
 * Conventions
 *   - plain C types only; every pointer is caller-owned HOST memory unless the name says "_dev";
 *   - all functions return 0 (MBAR_B200_OK) or a negative mbar_b200_status; no exceptions, no
 *     callbacks; mbar_b200_last_error() gives the message of the last failure on this thread;
 *   - one context = one GPU = one contiguous slice [n0, n0+N_local) of the samples.  K-sized
 *     state (N_k, f_k) is global and replicated.  With a communicator attached
 *     (mbar_b200_comm_init) every reduction over samples is followed by one sum all-reduce of the
 *     packed partials, so every rank returns identical K-vectors;
 *   - u_kn is float64 [K, N] row-major on the host exactly as pymbar.MBAR holds it (mbar.py:243).
 *     In HBM it is re-tiled to [N/32][K][32] and shifted per sample (see DESIGN.md "HBM layout");
 *   - states with N_k == 0 are "unsampled": they never enter a denominator and only
 *     mbar_b200_self_consistent_update / mbar_b200_log_W_nk produce values for them, exactly as in
 *     the reference (mbar_solvers.py:1002-1012);
 *   - stored range: every sample is shifted by x_n (its lowest sampled-state energy) and stored as
 *     min(u_kn - x_n, 1e6).  +inf is legal anywhere and has weight exactly 0 (an unsampled state whose
 *     energies are all +inf gets f = +inf, log W = -inf).  An unsampled or appended state whose energies
 *     all lie 1e6 - 800 or more above x_n, at least one of them finite, is outside the stored range: the
 *     entry points that read unsampled rows (self_consistent_update, weight_moments, log_W_nk, bin_moments
 *     with C / D) return MBAR_B200_ERR_RANGE; the sampled-state entry points are unaffected.  -inf in any
 *     row is rejected at upload / append with MBAR_B200_ERR_NAN (in a sampled row the sample has "no finite
 *     energy"; in an unsampled row the reference's f would be -inf).
 */
#ifndef MBAR_B200_H
#define MBAR_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MBAR_B200_ABI_VERSION 1

/* Largest number of states a context takes: mbar_b200_create's K and create_augmented's K + n_extra. */
#define MBAR_B200_MAX_STATES 8192

/* Largest number of rows R_p = K_p + M_p of a batch problem with appended rows (mbar_b200_batch_set_unsampled):
 * 3 * 64, so the 3K rows of compute_entropy_and_enthalpy fit every problem a batch holds. */
#define MBAR_B200_BATCH_MAX_ROWS 192

#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

typedef struct mbar_b200_ctx mbar_b200_ctx;

typedef enum mbar_b200_status {
    MBAR_B200_OK = 0,
    MBAR_B200_ERR_INVALID = -1,      /* bad argument (shape, NULL, K<1, ...)  -> ParameterError/ValueError */
    MBAR_B200_ERR_CUDA = -2,         /* CUDA runtime failure                                             */
    MBAR_B200_ERR_NO_DEVICE = -3,    /* no usable sm_90 GPU: there is NO CPU fallback                     */
    MBAR_B200_ERR_NOT_READY = -4,    /* u_kn not uploaded / synthesised yet                               */
    MBAR_B200_ERR_NAN = -5,          /* NaN found in u_kn at upload                                       */
    MBAR_B200_ERR_RANGE = -6,        /* f_k + log N_k outside the supported +-1e6 range                   */
    MBAR_B200_ERR_COMM = -7,         /* NCCL failure or libnccl not loadable                              */
    MBAR_B200_ERR_SINGULAR = -8,     /* Newton system not positive definite (disconnected states)         */
    MBAR_B200_ERR_NOMEM = -9
} mbar_b200_status;

/* Which kernel family a pass uses (mbar_b200_set_pass_kernel). AUTO = fused when it applies. */
typedef enum mbar_b200_kernel {
    MBAR_B200_KERNEL_AUTO = 0,
    MBAR_B200_KERNEL_FUSED = 1,      /* TMA-pipelined persistent kernel (clusters of CTAs above K = 256), K <= 2048 */
    MBAR_B200_KERNEL_GENERIC = 2     /* any K, log-domain for unsampled states                            */
} mbar_b200_kernel;

/* Result of a native solve (reference: the `results` dict of adaptive(), mbar_solvers.py:662-665). */
typedef struct mbar_b200_solve_result {
    int32_t success;          /* results["success"]                                                   */
    int32_t iterations;       /* loop iterations executed                                             */
    int32_t nr_iterations;    /* Newton-Raphson steps taken (nr_iter, mbar_solvers.py:620)            */
    int32_t sci_iterations;   /* self-consistent steps taken (sci_iter, mbar_solvers.py:610)          */
    int32_t passes;           /* full streaming passes over u_kn                                      */
    int32_t hessian_passes;   /* of which with the K x K Hessian                                      */
    double max_delta;         /* last relative change (mbar_solvers.py:631)                           */
    double gnorm;             /* ||gradient||_2 at the returned f_k (mbar_solvers.py:938-940)          */
    double device_ms;         /* CUDA-event time of the whole solve on this rank                      */
} mbar_b200_solve_result;

/* Synthetic-input family of SURVEY.md 8(d): harmonic oscillators, samples in block order. */
typedef struct mbar_b200_synth {
    uint64_t seed;            /* Philox-4x32-10 key; counter = GLOBAL sample index                     */
    int64_t n_offset;         /* global index of this context's first sample                           */
    int64_t N_global;         /* total samples over all ranks (defines the state of origin of n)       */
    const double* O_k;        /* [K] oscillator centres                                                */
    const double* k_k;        /* [K] spring constants (beta = 1)                                       */
} mbar_b200_synth;

/* ---- library ------------------------------------------------------------------------------- */
int mbar_b200_abi_version(void);
const char* mbar_b200_last_error(void);
int mbar_b200_device_count(int* count);
/* Pinned host memory for zero-staging uploads/downloads (cudaHostAlloc / cudaFreeHost). */
int mbar_b200_host_alloc(void** ptr, uint64_t bytes);
int mbar_b200_host_free(void* ptr);
/* NUMA node the GPU hangs off (sysfs), -1 when the host exposes none.  Pinned staging buffers are allocated with
 * that node preferred so uploads / downloads do not cross the inter-socket link. */
int mbar_b200_gpu_numa_node(int device, int* node);

/* 64-bit content hash of a host matrix of `rows` rows of `row_bytes` bytes, row stride `stride_bytes` (threaded,
 * memory-bandwidth bound, independent of the thread count).  A binding that keeps u_kn resident between the
 * reference's pure-function calls keys its cache on this, never on a sample of the contents. */
int mbar_b200_host_hash(const void* base, int64_t rows, int64_t row_bytes, int64_t stride_bytes, uint64_t* hash_out);

/* Release the buffers parked by destroyed contexts (at most one u_kn-sized device buffer and one staging set
 * per device are kept for the next context; MBAR_B200_NO_POOL=1 in the environment disables the parking). */
int mbar_b200_trim(void);

/* ---- context ------------------------------------------------------------------------------- */
/* N_k: [K] global sample counts as float64 (validate_inputs casts to float, mbar_solvers.py:198). */
int mbar_b200_create(mbar_b200_ctx** ctx, int device, int32_t K, int64_t N_local, const double* N_k);
int mbar_b200_destroy(mbar_b200_ctx* ctx);
int mbar_b200_get_shape(const mbar_b200_ctx* ctx, int32_t* K, int64_t* N_local);
int mbar_b200_set_pass_kernel(mbar_b200_ctx* ctx, int kernel /* mbar_b200_kernel */);
/* Counters since creation: kernel launches, streaming passes, bytes moved H2D / D2H. */
int mbar_b200_get_counters(const mbar_b200_ctx* ctx, int64_t* launches, int64_t* passes,
                           int64_t* h2d_bytes, int64_t* d2h_bytes);
/* CUDA-event duration (ms) of the most recent pass kernel on the context's stream. */
int mbar_b200_last_pass_ms(mbar_b200_ctx* ctx, double* ms);

/* ---- data in / out -------------------------------------------------------------------------- */
/* Replaces the host copies at mbar.py:243 and mbar_solvers.py:1003: u_host is [K, N_local]
 * row-major with row stride `ld` (elements).  Pinned memory is DMA'd directly; pageable memory is
 * staged through internal pinned buffers.  NaN anywhere -> MBAR_B200_ERR_NAN.  Once a communicator is
 * attached (mbar_b200_comm_init) the uploads and mbar_b200_synthesize are collective: every rank calls them, since
 * the ranks agree on each state's lowest shifted energy, which decides the kernel of all-state passes. */
int mbar_b200_upload_u_kn(mbar_b200_ctx* ctx, const double* u_host, int64_t ld);
/* Same, from a row-major DEVICE buffer on ctx's device (e.g. a torch tensor's data_ptr).  Ordered after all work
 * already submitted to the device, on any stream (it synchronises the device first): a tensor filled
 * asynchronously just before the call is read complete.  The caller may reuse u_dev once the call returns. */
int mbar_b200_upload_u_kn_dev(mbar_b200_ctx* ctx, const double* u_dev, int64_t ld);
/* A new context holding the samples of `base` plus n_extra UNSAMPLED states whose energies are u_extra_host
 * [n_extra, N_local] (row stride ld).  The resident tiles are copied device-to-device; only the new rows cross
 * PCIe.  This is how expectations / perturbed free energies (the columns mbar.py:886-940 appends to Log_W_nk)
 * reuse the resident u_kn.  `base` stays valid and independent. */
int mbar_b200_create_augmented(mbar_b200_ctx* base, int32_t n_extra, const double* u_extra_host, int64_t ld,
                               mbar_b200_ctx** ctx_out);
/* Fill the context on device from the synthetic family (no host traffic). */
int mbar_b200_synthesize(mbar_b200_ctx* ctx, const mbar_b200_synth* spec);
/* Per-sample multiplicities w_n >= 0 ([N_local] host doubles; NULL restores w_n = 1).  Every sum over
 * samples becomes a weighted sum (S_k = sum_n w_n W_nk, sum_n w_n L_n, W^T diag(w) W) while the denominators
 * L_n are untouched: a bootstrap replicate of mbar.py:417-449 (`u_kn[:, rints]`, an 8*K*N gather per
 * replicate) is the same data with w_n = number of times sample n was drawn — no copy, same kernels. */
int mbar_b200_set_sample_weights(mbar_b200_ctx* ctx, const double* w_host);
/* Read back columns [n0, n0+n) of the ORIGINAL (unshifted) u_kn as [K, n] row-major, stride ld. */
int mbar_b200_download_u_kn(mbar_b200_ctx* ctx, int64_t n0, int64_t n, double* u_host, int64_t ld);

/* ---- the streaming pass and the reference primitives built on it ---------------------------- */
/* One read of u_kn at f_k.  Outputs (any may be NULL):
 *   S[K]    S_k = sum_n W_nk  (0 for unsampled states)
 *   sumL    sum_n L_n,  L_n = log sum_k N_k exp(f_k - u_kn)   (mbar_solvers.py:238)
 *   G[K*K]  G = W^T W row-major (0 rows/cols for unsampled states); costs the Hessian pass.
 * With a communicator the outputs are the all-reduced global sums. */
int mbar_b200_pass(mbar_b200_ctx* ctx, const double* f_k, double* S, double* sumL, double* G);

/* The same pass at M (1 or 2) candidate vectors f[m][K] in one call, one host synchronisation: what adaptive()
 * needs to compare its self-consistent and Newton-Raphson candidates (mbar_solvers.py:590-607 evaluates
 * mbar_gradient at both).  S is [M][K], sumL is [M]; either may be NULL. */
int mbar_b200_pass_multi(mbar_b200_ctx* ctx, int32_t M, const double* f, double* S, double* sumL);

/* self_consistent_update(u_kn, N_k, f_k)  — mbar_solvers.py:206-257, Eq. C3, ALL states. */
int mbar_b200_self_consistent_update(mbar_b200_ctx* ctx, const double* f_k, double* f_out);
/* mbar_gradient — mbar_solvers.py:260-292, Eq. C6.  Unsampled states get 0 (-N_k * ...). */
int mbar_b200_gradient(mbar_b200_ctx* ctx, const double* f_k, double* g_out);
/* mbar_objective_and_gradient — mbar_solvers.py:341-392 (g_out may be NULL = mbar_objective). */
int mbar_b200_objective_and_gradient(mbar_b200_ctx* ctx, const double* f_k, double* obj_out,
                                     double* g_out);
/* mbar_hessian — mbar_solvers.py:395-436, Eq. C9, [K, K] row-major. */
int mbar_b200_hessian(mbar_b200_ctx* ctx, const double* f_k, double* H_out);
/* mbar_log_W_nk — mbar_solvers.py:439-473: [N_local, K] row-major (note: transposed w.r.t. u_kn),
 * row stride ld_out elements; exponentiate != 0 gives mbar_W_nk (mbar_solvers.py:476-507). */
int mbar_b200_log_W_nk(mbar_b200_ctx* ctx, const double* f_k, double* logW_host, int64_t ld_out,
                       int exponentiate);
/* Rows [n0, n0 + n) of the same matrix (n0 a multiple of 32): lets a caller page through Log_W_nk, or fetch the
 * part an estimator needs, instead of materialising N x K doubles on the host (mbar.py:455 keeps all of it). */
int mbar_b200_log_W_nk_rows(mbar_b200_ctx* ctx, const double* f_k, int64_t n0, int64_t n, double* logW_host,
                            int64_t ld_out, int exponentiate);
/* Sums and second moments of the weights of ALL K states (sampled or not) at f_k:
 *   S[K] = sum_n W_nk,  G[K*K] = W^T W.
 * Everything MBAR's asymptotic covariance (mbar.py:1837-1858, "svd-ew"), compute_overlap (mbar.py:605-606) and
 * compute_effective_sample_number (mbar.py:546-549) need, without materialising the N x K weight matrix. */
int mbar_b200_weight_moments(mbar_b200_ctx* ctx, const double* f_k, double* S_out, double* G_out);
/* Per-sample log denominators L_n [N_local] (the logsumexp at mbar_solvers.py:238). */
int mbar_b200_log_denominator(mbar_b200_ctx* ctx, const double* f_k, double* L_host);
/* Histogram FES of one target state (pymbar fes.py:388-600 and :1382-1415).  u_n [N_local] is the target
 * state's reduced potential for every sample (+inf allowed = weight 0, NaN -> MBAR_B200_ERR_NAN); bin_n
 * [N_local] is a dense bin index in [0, nbins) (anything else -> MBAR_B200_ERR_INVALID).  With
 * multiplicities c_n (mbar_b200_set_sample_weights, default 1):
 *   f_bin[nbins]  f_i  = -log sum_{n in i} c_n exp(-u_n - L_n)                          (required)
 *   C[K*nbins]    C_ki = sum_{n in i} c_n W_nk w^_n,  w^_n = exp(-u_n - L_n + f_i)      (row-major, may be NULL)
 *   D[nbins]      D_i  = sum_{n in i} c_n w^_n^2                                         (may be NULL)
 * W_nk covers ALL K states, sampled or not, as Log_W_nk does.  Together with mbar_b200_weight_moments this is
 * W_aug^T W_aug of the augmented matrix W_aug = [W | B], B_ni = w^_n [bin(n) = i], without materialising it.
 * Range: at the converged f_k every W_nk <= 1 and w^_n <= 1 / c_n.  An exponent of W_nk or w^_n above 700 (f_k
 * far from the solution), or a bin with no sample of finite weight (empty, all u_n = +inf or all c_n = 0),
 * returns MBAR_B200_ERR_RANGE.  Two calls on the same inputs return bit-identical results.  Sharded contexts
 * (communicator attached) are not supported: MBAR_B200_ERR_INVALID. */
int mbar_b200_bin_moments(mbar_b200_ctx* ctx, const double* f_k, const double* u_n, const int32_t* bin_n,
                          int32_t nbins, double* f_bin, double* C, double* D);
/* Unsampled-state updates of B bootstrap replicates of the resident samples in one call.  Replicate b draws sample n
 * counts[b, n] times ([B, N_local] row-major) and has free energies F[b] ([B, K] row-major; only sampled entries are
 * read).  For every replicate and every unsampled state j (N_k = 0, in index order; n_u of them):
 *   out[b, j] = -log sum_n counts[b,n] exp(-u_jn - L_bn),   L_bn = log sum_{k: N_k > 0} N_k exp(F[b,k] - u_kn),
 * i.e. what mbar_b200_set_sample_weights(counts[b]) + mbar_b200_self_consistent_update(F[b]) return for row j.
 * +inf where no term is nonzero (a row of +inf energies).  Range errors are those of self_consistent_update for
 * every replicate (check_range on each F[b]; check_unsampled_clamp).  A replicate whose counts sum to 0, B < 1, or a
 * context with a communicator -> MBAR_B200_ERR_INVALID.  Multiplicities set by mbar_b200_set_sample_weights are
 * neither used nor changed.  Row b is summed in an order fixed by N and K alone: it does not depend on B or on the
 * other replicates, repeat calls are bit-identical, and there are no floating-point atomics.  A failed call leaves
 * the context usable.  The counts go to the device one batch of 8 replicates at a time, one batch ahead of the
 * kernels (2 * 8 * 2 * N_local bytes of device memory whatever B is). */
int mbar_b200_replicate_unsampled(mbar_b200_ctx* ctx, int64_t B, const uint16_t* counts, const double* F,
                                  double* out);
/* CUDA-event time of the kernels of the last call, its replicate batches, and the exps it evaluated. */
int mbar_b200_last_replicate_stats(mbar_b200_ctx* ctx, double* ms, int32_t* batches, int64_t* exps);

/* ---- kernel-density sums (pymbar FES with fes_type="kde", independent of any u_kn context) ------ */
/* For the resident samples x_n in R^D with weights w_n >= 0 and query points y_q:
 *   out[q] = log sum_n w_n k(d_qn / h),   d_qn = sqrt(sum_{j<D} (y_qj - x_nj)^2),
 * the unnormalised log kernel sum behind sklearn's KernelDensity.score_samples (fes.py:1566): the caller adds the
 * kernel's normalisation and subtracts log sum_n w_n.  The log-kernels are sklearn's: gaussian -d^2/(2h^2),
 * exponential -d/h; tophat 0, epanechnikov log(1 - d^2/h^2), linear log(1 - d/h), cosine log cos(pi d / (2h)), each
 * for d < h only, with d the correctly rounded square root of the rounded squares summed in dimension order, as
 * sklearn computes it.  out[q] is finite whenever some w_n k > 0, however far below the fp64 range the linear sum
 * lies, and -inf when none is.  A query's result depends only on it and the samples (not on Q or the other queries),
 * and repeat calls are bit-identical. */
typedef enum mbar_b200_kde_kernel {
    MBAR_B200_KDE_GAUSSIAN = 0,
    MBAR_B200_KDE_TOPHAT = 1,
    MBAR_B200_KDE_EPANECHNIKOV = 2,
    MBAR_B200_KDE_EXPONENTIAL = 3,
    MBAR_B200_KDE_LINEAR = 4,
    MBAR_B200_KDE_COSINE = 5
} mbar_b200_kde_kernel;
typedef struct mbar_b200_kde mbar_b200_kde;
/* Upload N samples x_host [N, D] row-major and their weights w_host [N] once.  D outside 1..4, a negative, NaN or
 * infinite weight, or weights that sum to 0 -> MBAR_B200_ERR_INVALID; a NaN or infinite coordinate ->
 * MBAR_B200_ERR_NAN. */
int mbar_b200_kde_create(int device, int64_t N, int32_t D, const double* x_host, const double* w_host,
                         mbar_b200_kde** out);
int mbar_b200_kde_destroy(mbar_b200_kde* kde);
/* out [Q] for the queries y_host [Q, D] row-major.  An unknown kernel (mbar_b200_kde_kernel), or h <= 0 or not finite
 * -> MBAR_B200_ERR_INVALID; a NaN or infinite query coordinate -> MBAR_B200_ERR_NAN.  A failed call leaves the object
 * usable. */
int mbar_b200_kde_log_sum(mbar_b200_kde* kde, int32_t kernel, double h, int64_t Q, const double* y_host, double* out);
/* Bootstrap replicates of the resident samples (pymbar FES with fes_type="kde" and n_bootstraps > 0, fes.py:388-430,
 * :690-699, :1590-1601): replicate b puts weight V_host[b, n] >= 0 on sample n (row-major [B, N]).  The reference fits
 * replicate b to x_n[idx_b] with the weights of b = 0 by position, so V_bn is the sum of w_m over the positions m with
 * idx_b[m] = n.  The weights stay on the device until the next call replaces them: 8 nPad (9 ceil(B/8) + 1) bytes,
 * nPad = N rounded up to 256.  The host side is built one batch of 8 replicates at a time (8 * 9 nPad bytes).
 * B < 1, or a negative, NaN or infinite weight -> MBAR_B200_ERR_INVALID (the object then holds no replicates). */
int mbar_b200_kde_set_replicates(mbar_b200_kde* kde, int64_t B, const double* V_host);
/* out [B, Q] row-major: out[b, q] = log sum_n V_bn k(d_qn / h), the log sum of mbar_b200_kde_log_sum with replicate
 * b's weights, behind score_samples of the reference's B replicate KernelDensity objects (fes.py:1598-1601).  Every
 * batch of 8 replicates is one pass over the samples: the distance, the kernel and one exp per (query, sample) pair
 * serve the whole batch, under one running scale per query (the largest log V_bn + log k_qn of the batch).  Where
 * that shared scale may have cut a replicate short (its log sum more than 549 - log N below the batch's scale at
 * the query, -inf included: far queries), the entry is recomputed with the single-replicate pass, so every out[b, q]
 * agrees with mbar_b200_kde_log_sum on weights V_b to 1e-12 relative and is -inf exactly when no V_bn k is nonzero.
 * Results do not depend on Q, on the other queries or on replicates of other batches, and repeat calls are
 * bit-identical.
 * Errors as mbar_b200_kde_log_sum; no replicates uploaded -> MBAR_B200_ERR_NOT_READY. */
int mbar_b200_kde_log_sum_replicates(mbar_b200_kde* kde, int32_t kernel, double h, int64_t Q, const double* y_host,
                                     double* out);
/* CUDA-event time of the kernels of the last mbar_b200_kde_log_sum or mbar_b200_kde_log_sum_replicates, and the number
 * of sample chunks they split N into. */
int mbar_b200_last_kde_stats(mbar_b200_kde* kde, double* ms, int32_t* chunks);
/* Many sample sets in one object (DESIGN.md 3.5h''): KDE surfaces of many small problems, and every bootstrap
 * replicate of each, scored in one call.  Only the coordinates are resident; the weights travel with each request.
 * Set s holds N[s] >= 1 samples in D[s] dimensions (1..4); x concatenates the sets' row-major [N_s, D_s].  D outside
 * 1..4 or N < 1 -> MBAR_B200_ERR_INVALID; a NaN or infinite coordinate -> MBAR_B200_ERR_NAN. */
typedef struct mbar_b200_kde_many mbar_b200_kde_many;
int mbar_b200_kde_many_create(int device, int32_t n_sets, const int32_t* D, const int64_t* N, const double* x,
                              mbar_b200_kde_many** out);
int mbar_b200_kde_many_destroy(mbar_b200_kde_many* kde);
/* Request r names set[r], a kernel[r] (mbar_b200_kde_kernel), a bandwidth h[r], weights w [N_set] and Q[r] >= 0 query
 * points y [Q_r, D_set] row-major; w, y and out concatenate the requests'.  out[q] = log sum_n w_n k(d_qn / h): the
 * same bits mbar_b200_kde_log_sum returns on an mbar_b200_kde created from (x of set[r], that w) for the same kernel, h
 * and query.  A request gives the same bits alone, among any others, in any order and on repeat calls.  One partial
 * launch per distinct (D, kernel) and one combine launch for all requests, and one synchronisation; the requests are
 * cut into sub-batches (more launches, the same results) when their chunk partials would pass 64 MiB.  Before any
 * device work, leaving the object usable: a bad set or kernel, an h <= 0 or not finite, a negative, NaN or infinite
 * weight, or weights that sum to 0 -> MBAR_B200_ERR_INVALID; a NaN or infinite query -> MBAR_B200_ERR_NAN.  A call
 * whose buffers do not fit in device memory -> MBAR_B200_ERR_NOMEM with the byte count in the message. */
int mbar_b200_kde_many_log_sum(mbar_b200_kde_many* kde, int32_t n_requests, const int32_t* set, const int32_t* kernel,
                               const double* h, const double* w, const int64_t* Q, const double* y, double* out);
/* CUDA-event time of the kernels of the last mbar_b200_kde_many_log_sum, its kernel launches and its (query, sample)
 * pairs. */
int mbar_b200_last_kde_many_stats(mbar_b200_kde_many* kde, double* ms, int32_t* launches, int64_t* pairs);

/* ---- B-spline basis sums (pymbar FES with fes_type="spline", independent of any u_kn context) --- */
/* For the resident samples x_n with weights w_n and state labels s_n, and the nb = n_knots - degree - 1 basis
 * functions B_i of the knot vector t:
 *   S_ki = sum_{n: s_n = k} B_i(x_n),   A_i = sum_n w_n B_i(x_n),
 * the sums that the sample terms of the spline fit's objective, gradient and MC likelihood are linear in
 * (fes.py:2102-2306, :1954-2010).  B_i(x) is scipy.interpolate.BSpline(t, e_i, degree)(x) with extrapolate=True, bit
 * for bit: the interval scipy picks (x on a knot, repeated knots, x outside [t_k, t_nb] on the end polynomials) and
 * its Cox-de Boor arithmetic.  Repeat calls are bit-identical, S and A do not depend on whether the other is asked for
 * or on earlier knot vectors, and there are no floating-point atomics. */
typedef struct mbar_b200_bspline mbar_b200_bspline;
/* Upload N samples x [N], weights w [N] (NULL: no A) and labels s [N] in [0, K) (NULL: no S) once.  A negative, NaN
 * or infinite weight, or a label outside [0, K) -> MBAR_B200_ERR_INVALID; a NaN or infinite x -> MBAR_B200_ERR_NAN. */
int mbar_b200_bspline_create(int device, int64_t N, const double* x, const double* w, const int32_t* s, int32_t K,
                             mbar_b200_bspline** out);
int mbar_b200_bspline_destroy(mbar_b200_bspline* bspline);
/* S [K * nb] row-major and A [nb]; either may be NULL.  degree outside 0..7, a non-finite or decreasing knot,
 * n_knots < 2 (degree + 1), t[degree] = t[nb], nb + n_knots above 13824 (one shared-memory accumulator), or S / A
 * asked of an object created without labels / weights -> MBAR_B200_ERR_INVALID.  A failed call leaves the object
 * usable.  When K * nb does not fit one accumulator, further state chunks cover the rest (tiles without a sample of
 * a chunk's states are skipped). */
int mbar_b200_bspline_moments(mbar_b200_bspline* bspline, int32_t degree, int64_t n_knots, const double* t, double* S,
                              double* A);
/* Upload the weights V [B, N] row-major (V_bn >= 0) of B bootstrap replicates of the resident samples, replacing any
 * uploaded before; they stay on the device (8 B nPad bytes, nPad = N rounded up to 32) until the next call or destroy.
 * B < 1, or a negative, NaN or infinite weight -> MBAR_B200_ERR_INVALID, and the object then holds no replicates.
 * The weights w and labels s of create are not touched. */
int mbar_b200_bspline_set_replicates(mbar_b200_bspline* bspline, int64_t B, const double* V_host);
/* out [B, nb] row-major: out[b, i] = sum_n V_bn B_i(x_n), the A of mbar_b200_bspline_moments with replicate b's
 * weights, for every uploaded replicate in one call.  Each pass over the samples evaluates the basis once per sample
 * for a batch of replicates.  Row b is summed in an order fixed by N and nb alone: it does not depend on B or on the
 * other rows, and repeat calls are bit-identical; there are no floating-point atomics.  Degree and knot errors are
 * those of mbar_b200_bspline_moments; no replicates uploaded -> MBAR_B200_ERR_NOT_READY.  A failed call leaves the
 * object usable. */
int mbar_b200_bspline_replicate_sums(mbar_b200_bspline* bspline, int32_t degree, int64_t n_knots, const double* t,
                                     double* out);
/* CUDA-event time of the kernels of the last mbar_b200_bspline_moments or mbar_b200_bspline_replicate_sums and the
 * number of row chunks (moments) or replicate batches (replicate_sums) they took. */
int mbar_b200_last_bspline_stats(mbar_b200_bspline* bspline, double* ms, int32_t* chunks);

/* ---- lag sums of timeseries (pymbar.timeseries, independent of any u_kn context) --------------- */
/* For a start s of the resident series A (and B; NULL: B = A) of length T, m = T - s, the means mu_A, mu_B of A[s:],
 * B[s:], dA = A - mu_A, dB = B - mu_B, and
 *   sigma^2 = sum_{n >= s} dA[n] dB[n] / m,
 *   C(t) = sum_{n = s}^{T-1-t} (dA[n] dB[n+t] + dB[n] dA[n+t]) / (2.0 (m - t) sigma^2),
 * with every term and quotient rounded as numpy rounds the reference's (timeseries.py:156-196, :474-497); only the
 * sums run in another order (sequential within chunks whose bounds depend on T alone, the chunks in order).  A
 * start's results do not depend on the other starts of a call or on how its lags were batched, and repeat calls are
 * bit-identical; there are no floating-point atomics. */
typedef struct mbar_b200_acf mbar_b200_acf;
/* Upload A [T] and B [T] (or NULL) once.  n_segments > 0: A is K concatenated series with offsets [K + 1] (0 = offsets[0]
 * < offsets[1] < ... < offsets[K] = T), and no lag pair crosses a series (statistical_inefficiency_multiple).  NaN or
 * infinite values -> MBAR_B200_ERR_NAN; T < 1 or bad offsets -> MBAR_B200_ERR_INVALID. */
int mbar_b200_acf_create(int device, int64_t T, const double* a, const double* b, int32_t n_segments,
                         const int64_t* offsets, mbar_b200_acf** out);
int mbar_b200_acf_destroy(mbar_b200_acf* acf);
/* The reference's statistical-inefficiency loop for every start: t = 1, 2, ... (fast: increments 1, 2, 3, ...) while
 * t < m - 1, stopping after the first C(t) <= 0 with t > mintime, g += 2.0 * C * (1.0 - t / m) * increment.
 * rule 1 (a segmented autocorrelation object, the single start 0) is statistical_inefficiency_multiple's loop instead:
 * C(t) = (sum of single products over the series / sum_k max(N_k - t, 0)) / sigma^2, t < max N_k - 1, stop at
 * C <= 0 with t > 10, g += 2.0 * C * (1.0 - t / navg) * increment.  Per start: mean_a, mean_b, sigma2 (may be NULL),
 * g before the g >= 1 clamp, last_lag (the last t whose C was computed, 0 if none) and status (1: sigma^2 == 0, the
 * reference's ParameterError; g = 1 and no lag evaluated).  trace [n_starts][trace_cap] (trace_cap may be 0) gets
 * C at the first trace_cap lag indices evaluated, NaN after the last.  Lags are evaluated in rounds of 8, 8, 16, 32,
 * ... lag indices for all active starts, with one host poll per round.
 * rule 2 (an unsegmented autocorrelation object, fast = 0, any starts) is statistical_inefficiency_fft's loop over
 * statsmodels' acf(adjusted=True): C(t) = (S(t) / (m - t)) / sigma^2 with S(t) the single-product sum
 * sum_{n = s}^{T-1-t} dA[n] dA[n+t], evaluated by direct lag sums (not an FFT), t = 1 .. m - 1 inclusive, stop at the
 * first C <= 0 with t > mintime (that lag excluded), g += 2.0 * C * (1.0 - t / m).  A start outside [0, T) or a rule
 * the object cannot take -> MBAR_B200_ERR_INVALID.  A failed call leaves the object usable. */
int mbar_b200_acf_inefficiency(mbar_b200_acf* acf, int64_t n_starts, const int64_t* starts, int32_t fast,
                               int32_t mintime, int32_t rule, double navg, int64_t trace_cap, double* mean_a,
                               double* mean_b, double* sigma2, double* g, int64_t* last_lag, int32_t* status,
                               double* trace);
/* Rule 0 of mbar_b200_acf_inefficiency for n requests on a segmented object (autocorrelation or cross): request r is
 * series series[r] taken alone, from starts[r] counted from that series' first sample.  Every output of request r is
 * bit for bit what mbar_b200_acf_inefficiency returns for that start on an unsegmented object holding series[r] alone:
 * each series is cut into its own chunks of max(512, ceil(N_k / 1024)) samples, the lag launch covers only the
 * (request, chunk) pairs a request reads, and the rounds (8, 8, 16, 32, ... lag indices, one host poll each) are shared
 * by all active requests, each retired at its own limit.  n < 1 or n >= 2^31, a series index outside [0, K), a start
 * outside [0, N_k) or an unsegmented object -> MBAR_B200_ERR_INVALID before anything runs.  mean_a, mean_b and sigma2
 * may be NULL.  mbar_b200_last_acf_stats reports the call's rounds and terms. */
int mbar_b200_acf_inefficiency_series(mbar_b200_acf* acf, int64_t n, const int32_t* series, const int64_t* starts,
                                      int32_t fast, int32_t mintime, double* mean_a, double* mean_b, double* sigma2,
                                      double* g, int64_t* last_lag, int32_t* status);
/* C(t) for t = 0 .. n_max of one start (normalized_fluctuation_correlation_function), with its means and sigma^2.
 * n_max outside [0, T - start - 1], a segmented object or sigma^2 == 0 -> MBAR_B200_ERR_INVALID. */
int mbar_b200_acf_correlation(mbar_b200_acf* acf, int64_t start, int64_t n_max, double* C, double* mean_a,
                              double* mean_b, double* sigma2);
/* normalized_fluctuation_correlation_function_multiple of a segmented object (K series, A and optionally B): pooled
 * means mu_A, mu_B over all N = T samples, S_k(t) = sum_{n < N_k - t} dA_k[n] dB_k[n + t] (one product, over the
 * series with N_k > t), C(t) = ((0.0 + sum_k S_k(t)) / sum_k (N_k - t)) / sigma^2 with sigma^2 = sum_k S_k(0) / N
 * (so C(0) == 1.0), for t = 0 .. n_max into C [n_max + 1].  Each series is cut into its own chunks of
 * max(512, ceil(N_k / 1024)) samples; a (series, lag) sum adds its chunk partials in order and the numerator the
 * series in list order, so results are bit-identical across calls and launch splits, with no floating-point atomics.
 * n_out gets the length the reference returns: n_max, or with truncate the first t at which a running numerator
 * (after each series, in list order) is negative; truncate evaluates lags in rounds of 8, 8, 16, 32, ... and leaves
 * NaN in C past the last round.  mean_a, mean_b, sigma2 may be NULL.  An unsegmented object, n_max outside
 * [0, max N_k - 1] or sigma^2 == 0 -> MBAR_B200_ERR_INVALID. */
int mbar_b200_acf_correlation_multiple(mbar_b200_acf* acf, int64_t n_max, int32_t truncate, double* C, int64_t* n_out,
                                       double* mean_a, double* mean_b, double* sigma2);
/* CUDA-event time of the last call, its lag rounds (host polls), and the (start, lag, n) terms of lags >= 1 it
 * evaluated and of those up to each start's last lag; terms / useful_terms is the speculative batches' waste.  After
 * mbar_b200_acf_correlation_multiple: its truncate rounds (0 without truncate) and the (series, lag, n) terms of
 * lags >= 0 evaluated and of those through the reference's last lag. */
int mbar_b200_last_acf_stats(mbar_b200_acf* acf, double* ms, int32_t* rounds, int64_t* terms, int64_t* useful_terms);

/* ---- sums over work vectors (pymbar.other_estimators: BAR, EXP, Gaussian EXP; no u_kn context) -- */
/* A request (vector v, kind, c1, c2) over the resident vector w = w_v of n values returns out [3], every term in the
 * reference's fp64 formula with its own max shifts (other_estimators.py:120-145, :489-504, :617-636, :694-696), and
 * logsumexp(t) = log(sum exp(t - M)) + M with M = max t, replaced by 0 when it is not finite (utils.py:315-320):
 *   FERMI:          a = (w + c1) + c2, m = max(a, 0), t = -m - log(exp(-m) + exp(a - m)):  logsumexp(t), 0, 0
 *   FERMI_MOMENTS:  a = w + c1, A = max(a), t = -log(exp(-A) + exp(a - A)):  logsumexp(t), logsumexp(2 t), A
 *   EXP:            x = exp(-w - max(-w)):  log(sum x) + max(-w), sum x, sum (x - sum x / n)^2
 *   GAUSS:          sum w, sum (w - sum w / n)^2, 0
 * Each sum runs over chunks whose bounds depend on n alone (sequential per thread, a fixed tree per chunk, the chunks
 * in order): a request's out is the same bits whichever requests share the call, repeat calls are bit-identical, and
 * there are no floating-point atomics. */
#define MBAR_B200_WORK_FERMI 0
#define MBAR_B200_WORK_FERMI_MOMENTS 1
#define MBAR_B200_WORK_EXP 2
#define MBAR_B200_WORK_GAUSS 3
typedef struct mbar_b200_work mbar_b200_work;
/* Upload V concatenated vectors w [n_total] with offsets [V + 1] once; each vector's min and max are kept.  NaN or
 * infinite values -> MBAR_B200_ERR_NAN; an empty vector or bad offsets -> MBAR_B200_ERR_INVALID. */
int mbar_b200_work_create(int device, int64_t n_total, const double* w, int32_t n_vectors, const int64_t* offsets,
                          mbar_b200_work** out);
int mbar_b200_work_destroy(mbar_b200_work* work);
/* out [n_requests][3] for the requests (vector[r], kind[r], c1[r], c2[r]): two passes over each requested vector,
 * four launches and one host synchronisation per call.  A vector outside [0, V) or an unknown kind ->
 * MBAR_B200_ERR_INVALID.  A failed call leaves the object usable. */
int mbar_b200_work_evaluate(mbar_b200_work* work, int32_t n_requests, const int32_t* vector, const int32_t* kind,
                            const double* c1, const double* c2, double* out);
/* CUDA-event time of the kernels of the last mbar_b200_work_evaluate, its launches and the work values it read. */
int mbar_b200_last_work_stats(mbar_b200_work* work, double* ms, int32_t* launches, int64_t* values_read);

/* ---- many small MBAR problems in lockstep (pymbar_b200.mbar_many; DESIGN.md 3.5g) ------------------------------ */
/* P problems, problem p with K_p (1 to 64) states and N_p >= 1 samples: u concatenates each problem's row-major
 * u_kn [K_p][N_p], N_k concatenates each problem's N_k [K_p] (at least one positive entry each).  One H2D copy, then
 * every problem is shifted per sample and tiled on the device.  NaN or -inf energies -> MBAR_B200_ERR_NAN; a bad
 * shape or N_k -> MBAR_B200_ERR_INVALID; a batch that does not fit in device memory -> MBAR_B200_ERR_NOMEM (the
 * message gives the allocation in bytes). */
typedef struct mbar_b200_batch mbar_b200_batch;
int mbar_b200_batch_create(int device, int32_t n_problems, const int32_t* K, const int64_t* N, const double* N_k,
                           const double* u, mbar_b200_batch** out);
int mbar_b200_batch_destroy(mbar_b200_batch* batch);
/* For each request r (problem[r], f: the concatenation of the requests' f [K_p]): S_k = sum_n e^{f_k - u_kn - L_n},
 * log S_k, sum_n L_n with L_n = log sum_{j sampled} N_j e^{f_j - u_jn}, a flag and, when G is not NULL, the Gram
 * Ghat_ij = sum_n w_in w_jn with w_kn = N_k W_nk on sampled rows and W_nk on unsampled rows if all_rows (0
 * otherwise).  S and log S cover the sampled rows, and all rows if all_rows.  flag[r] = 1: a NaN reached the sums,
 * a sampled S_k lies outside (1e-280, 1e300), or (all_rows) an unsampled S_k is NaN or overflows.  Outputs are
 * concatenated by request (G: K_p x K_p each, row-major).  Two kernel launches and one synchronisation; a request's
 * results are the same bits whichever requests share the call. */
int mbar_b200_batch_moments(mbar_b200_batch* batch, int32_t n_requests, const int32_t* problem, const double* f,
                            int32_t all_rows, double* S, double* log_S, double* sum_L, int32_t* flag, double* G);
/* The adaptive solver of mbar_b200_solve_adaptive's host-stepped loop (same step, Newton retries, step choice and
 * convergence rule) for every problem at once, one moments call (both candidates of every unfinished problem) per
 * iteration.  f [sum K_p] in/out: the sampled states of each problem, gauge f[first sampled] = 0; unsampled states
 * are left untouched.  status[p]: 0 converged (or nothing to solve), 1 maxiter reached, 2 the batched sums could
 * not represent an iterate (flag set or a non-finite candidate; f is then the last good iterate).  iterations[p]:
 * the iterations problem p took.  A sampled |f_k| >= 5e5 -> MBAR_B200_ERR_RANGE. */
int mbar_b200_batch_solve(mbar_b200_batch* batch, double* f_inout, double tol, int32_t maxiter, int32_t min_sc_iter,
                          double gamma, int32_t* status, int32_t* iterations);
/* Replicate slots (DESIGN.md 3.5g'): replaces the resident slots with n_slots bootstrap replicates, slot s of problem
 * problem[s] with the uint16 multiplicities counts [N_p] (counts concatenates the slots), and computes each slot's
 * sum_n c_n x_n once.  A slot naming a bad problem or whose counts do not sum to N_p -> MBAR_B200_ERR_INVALID;
 * slots that do not fit in device memory -> MBAR_B200_ERR_NOMEM (the message gives the allocation in bytes).  A
 * failed call leaves no slot.  n_slots = 0 drops every slot. */
int mbar_b200_batch_set_replicates(mbar_b200_batch* batch, int32_t n_slots, const int32_t* problem,
                                   const uint16_t* counts);
/* mbar_b200_batch_moments with every request naming a slot (slot[r]) instead of a problem: the sums of its problem
 * with sample n counted c_n times, S_k = sum_n c_n e^{f_k - u_kn - L_n}, Ghat_ij = sum_n c_n w_in w_jn and
 * sum_n c_n L_n, where L_n keeps N_k.  These are the values DeviceProblem.set_sample_weights(c) and the matching
 * single-problem call give; the flag follows the same rules.  All-ones counts give the bits of the unweighted
 * request, and a request's results are the same bits whichever requests share the call. */
int mbar_b200_batch_replicate_moments(mbar_b200_batch* batch, int32_t n_requests, const int32_t* slot,
                                      const double* f, int32_t all_rows, double* S, double* log_S, double* sum_L,
                                      int32_t* flag, double* G);
/* mbar_b200_batch_solve over the slots: the same loop with units that are slots rather than problems.  f_inout
 * [sum over slots of K_p], status and iterations [n_slots]; the same status codes. */
int mbar_b200_batch_solve_replicates(mbar_b200_batch* batch, double* f_inout, double tol, int32_t maxiter,
                                     int32_t min_sc_iter, double gamma, int32_t* status, int32_t* iterations);
/* Appended rows (DESIGN.md 3.5g''): replaces the resident appended rows with those of n problems, problem problem[i]
 * getting M[i] unsampled rows [M_i][N_p] (rows concatenates them, row-major).  They are stored as tiles of u - x_n,
 * shifted by the problem's resident x_n and padded with +inf past N_p.  NaN or -inf -> MBAR_B200_ERR_NAN; a bad or
 * repeated problem index, M_i < 1 or K_p + M_i > MBAR_B200_BATCH_MAX_ROWS -> MBAR_B200_ERR_INVALID; rows that do not
 * fit in device memory -> MBAR_B200_ERR_NOMEM (the message gives the allocation in bytes).  A failed call leaves no
 * appended rows.  n = 0 drops them all. */
int mbar_b200_batch_set_unsampled(mbar_b200_batch* batch, int32_t n, const int32_t* problem, const int32_t* M,
                                  const double* rows);
/* The moments of the augmented problems: request r names problem[r], which must hold appended rows, and f its
 * R_p = K_p + M_p free energies (f concatenates the requests').  L_n is taken over the sampled rows only, as in
 * mbar_b200_batch_moments.  S and log S [R_p] cover every row (sampled rows as batch_moments with all_rows = 1
 * gives them; unsampled and appended rows as running (max, sum) pairs), then sum_n L_n, the flag of batch_moments
 * applied to every row and, when G is not NULL, the N-scaled Gram Ghat [R_p][R_p] of all rows (sampled rows scaled by
 * N_k, the others by 1).  Appended weights are not shifted: ask for the Gram at a normalised f, where they are at
 * most 1; a Ghat entry that is not finite sets the flag.  Three kernel launches with the Gram (two without) and one
 * synchronisation; a request's results are the same bits whichever requests share the call. */
int mbar_b200_batch_augmented_moments(mbar_b200_batch* batch, int32_t n_requests, const int32_t* problem,
                                      const double* f, double* S, double* log_S, double* sum_L, int32_t* flag,
                                      double* G);
/* mbar_b200_batch_augmented_moments with every request naming a replicate slot (slot[r]) whose problem holds
 * appended rows, and f its R_p = K_p + M_p values: the sums of the augmented problem with sample n counted c_n times,
 * S_k = sum_n c_n e^{f_k - u_kn - L_n}, log S_k and sum_n c_n L_n, where L_n keeps N_k, and the flag of
 * batch_augmented_moments.  These are the values DeviceProblem.replicate_unsampled gives for the appended rows.  No
 * Gram.  A slot out of range or whose problem holds no appended rows -> MBAR_B200_ERR_INVALID.  Two kernel launches
 * and one synchronisation; all-ones counts give the bits of the unweighted request, a zero-count sample enters no sum
 * and a request's results are the same bits whichever requests share the call. */
int mbar_b200_batch_replicate_augmented_moments(mbar_b200_batch* batch, int32_t n_requests, const int32_t* slot,
                                                const double* f, double* S, double* log_S, double* sum_L,
                                                int32_t* flag);
/* Histogram FES of many problems (DESIGN.md 3.5h): mbar_b200_bin_moments for every request in one call.  Request r
 * names problem[r] and gives its converged f [K_p], a target state's reduced potentials u_n [N_p] and dense bin
 * indices bin_n [N_p] in [0, nbins[r]); f, u_n and bin_n concatenate the requests'.  With L_n = log sum_{k sampled}
 * N_k exp(f_k - u_kn):
 *   f_bin [nbins_r]         f_i  = -log sum_{n in i} exp(-u_n - L_n)                          (required)
 *   C     [K_p * nbins_r]   C_ki = sum_{n in i} W_nk w^_n,  w^_n = exp(-u_n - L_n + f_i)      (row-major, may be NULL)
 *   D     [nbins_r]         D_i  = sum_{n in i} w^_n^2                                         (may be NULL)
 * each concatenated by request, W_nk over all K_p rows, sampled or not.  Only u_n and bin_n are uploaded: the
 * problem's resident tiles, x_n and log N_k serve the rest.  Before any device work: a bad problem index, nbins < 1
 * or a bin index outside [0, nbins) -> MBAR_B200_ERR_INVALID, a NaN u_n -> MBAR_B200_ERR_NAN.  +inf in u_n is weight
 * 0.  flag[r] = 1 where an exponent of W_nk or w^_n exceeds 700, a bin has no sample of finite weight, or a sample's
 * L_n is not a number; the call still succeeds.  Five kernel launches (seven with C or D) and one synchronisation.  No
 * floating-point atomics: a request's results are the same bits whichever requests share the call, and repeat calls
 * are bit-identical. */
int mbar_b200_batch_bin_moments(mbar_b200_batch* batch, int32_t n_requests, const int32_t* problem, const double* f,
                                const double* u_n, const int32_t* bin_n, const int32_t* nbins, double* f_bin,
                                double* C, double* D, int32_t* flag);
/* Histogram FES of bootstrap replicates (DESIGN.md 3.5h'): the f_bin of mbar_b200_batch_bin_moments with sample n
 * counted c_n times, for replicate slots of many problems in one call.  Target t names target_problem[t] and gives
 * that problem's target-state u_n [N_p] and dense bin indices bin_n [N_p] in [0, nbins[t]) (u_n and bin_n
 * concatenate the targets'); each target is uploaded once, however many requests read it.  Request r names a
 * resident replicate slot slot[r], a target target[r] of the slot's problem and the replicate's converged f [K_p]
 * (f concatenates the requests').  With L_n = log sum_{k sampled} N_k exp(f_k - u_kn), which keeps N_k:
 *   f_bin [nbins of target[r]]   f_i = -log sum_{n in i} c_n exp(-u_n - L_n)
 * concatenated by request: what DeviceProblem.set_sample_weights(c) and mbar_b200_bin_moments(want_C = 0) give.  No
 * C and no D.  A sample with c_n = 0 enters no sum and no maximum, and its NaN L_n does not flag; all-ones counts give
 * the bits of batch_bin_moments' f_bin.  flag[r] follows batch_bin_moments' rules over the drawn samples.  Before any
 * device work: a slot or target out of range, a slot whose problem is not its target's, nbins < 1 or a bin index
 * outside [0, nbins) -> MBAR_B200_ERR_INVALID, a NaN u_n -> MBAR_B200_ERR_NAN; the batch stays usable.  Five kernel
 * launches and one synchronisation for all requests; the work split of a request depends on (N_p, K_p, nbins) alone
 * and there are no floating-point atomics, so its results are the same bits whichever requests share the call. */
int mbar_b200_batch_replicate_bin_moments(mbar_b200_batch* batch, int32_t n_targets, const int32_t* target_problem,
                                          const double* u_n, const int32_t* bin_n, const int32_t* nbins,
                                          int32_t n_requests, const int32_t* slot, const int32_t* target,
                                          const double* f, double* f_bin, int32_t* flag);
/* Target-state log weights of many problems (DESIGN.md 3.5h''): for request r, problem[r] with its converged f [K_p]
 * and a target state's reduced potentials u_n [N_p] (f and u_n concatenate the requests'),
 *   log_w [N_p] = -u_n - L_n,   L_n = log sum_{k sampled} N_k exp(f_k - u_kn),
 * concatenated by request, from the resident tiles: L_n is batch_bin_moments' per-sample denominator.  u_n = +inf
 * gives -inf.  A NaN log w_n sets flag[r]; the call still succeeds.  Before any device work, leaving the batch usable:
 * a bad problem index -> MBAR_B200_ERR_INVALID, a NaN u_n -> MBAR_B200_ERR_NAN.  One kernel launch and one
 * synchronisation. */
int mbar_b200_batch_log_weights(mbar_b200_batch* batch, int32_t n_requests, const int32_t* problem, const double* f,
                                const double* u_n, double* log_w, int32_t* flag);
/* CUDA-event time of the kernels of the last batch_moments, batch_solve, batch_replicate_moments,
 * batch_solve_replicates, batch_augmented_moments, batch_replicate_augmented_moments, batch_bin_moments,
 * batch_replicate_bin_moments or batch_log_weights call, its
 * kernel launches, its iterations (solves) and the bytes of u_kn tiles (appended tiles, counts) its passes read. */
int mbar_b200_last_batch_stats(mbar_b200_batch* batch, double* kernel_ms, int32_t* launches, int32_t* iterations,
                               int64_t* bytes_read);

/* ---- native solver loops (no Python between iterations) ------------------------------------- */
/* Plain self-consistent iteration f <- f - log S(f), gauge f[first sampled] = 0 each step, until
 * max |delta f / f| < tol (the convergence rule of mbar_solvers.py:627-640) or maxiter. */
int mbar_b200_solve_sci(mbar_b200_ctx* ctx, double* f_inout, double tol, int32_t maxiter,
                        mbar_b200_solve_result* result);
/* adaptive() — mbar_solvers.py:510-667: Newton vs self-consistent step by gradient norm.
 * f_inout covers all K states; unsampled states are carried through untouched. */
int mbar_b200_solve_adaptive(mbar_b200_ctx* ctx, double* f_inout, double tol, int32_t maxiter,
                             int32_t min_sc_iter, double gamma, mbar_b200_solve_result* result);
/* How the two solvers above iterate.  mode 0 (default): device resident — every quantity of an iteration
 * (gradient, candidates, K x K Cholesky of the Newton system, step choice mbar_solvers.py:607, convergence test
 * :627-640) stays on the GPU, `batch` iterations are enqueued between two polls of a small state struct and
 * kernels of iterations past convergence exit immediately; jax_core_adaptive (mbar_solvers.py:670-694) is the
 * reference's counterpart of that single fused step.  mode 1: host-stepped (one round trip per pass), which is
 * also what mode 0 falls back to when the fast kernels cannot represent an iterate.  batch < 1 keeps the
 * current batch size. */
int mbar_b200_set_loop_mode(mbar_b200_ctx* ctx, int32_t mode, int32_t batch);
/* Host synchronisations spent polling the device-resident loops since creation, current mode and batch. */
int mbar_b200_get_loop_stats(const mbar_b200_ctx* ctx, int64_t* polls, int32_t* mode, int32_t* batch);
/* The adaptive iteration is captured into a CUDA graph after the first batch a context runs and relaunched once
 * per iteration: how often it was captured / launched (MBAR_B200_NO_GRAPH=1 disables the capture). */
int mbar_b200_get_graph_stats(const mbar_b200_ctx* ctx, int64_t* captures, int64_t* launches);
/* How the last mbar_b200_solve_adaptive on this context ran.  The Newton counters cover the device-resident loop
 * only (the host-stepped loop retries its own factorisations, up to four times with a growing additive ridge). */
typedef struct mbar_b200_adaptive_stats {
    int32_t device_iterations;  /* iterations the device-resident loop completed and kept                       */
    int32_t fell_back;          /* 1: the host-stepped loop finished the solve from the last polled f           */
    int32_t ridge_retries;      /* factorisations of H[1:,1:] retried with the 1e-10 relative ridge             */
    int32_t newton_failed;      /* iterations without a Newton candidate: the retry was not positive definite  */
    int32_t newton_rejected;    /* Newton candidates rejected as non-finite or outside 0.5 C_RANGE              */
    int32_t newton_threads;     /* CTA size of the Newton kernel, 0 when it never ran                            */
    int32_t newton_smem;        /* 1: the matrix sat in shared memory, 0: the L2-resident variant ran           */
    int32_t reserved;
} mbar_b200_adaptive_stats;
int mbar_b200_get_adaptive_stats(const mbar_b200_ctx* ctx, mbar_b200_adaptive_stats* stats);
/* Run exactly `iters` self-consistent passes back to back with no host round trip (bench). */
int mbar_b200_sci_iterate(mbar_b200_ctx* ctx, double* f_inout, int32_t iters);

/* CUDA-event timing of the last mbar_b200_sci_iterate on the context's stream: whole loop (pass +
 * all-reduce + K-vector epilogue per iteration) and the sum of the pass-kernel launch durations. */
int mbar_b200_last_loop_ms(mbar_b200_ctx* ctx, double* total_ms, double* kernel_ms_sum, int32_t* iters);

/* ---- introspection for the benchmark ---------------------------------------------------------- */
/* Human-readable description of the pass-kernel / Hessian-kernel variants launched last (buffers of `len`). */
int mbar_b200_last_kernels(const mbar_b200_ctx* ctx, char* pass_kernel, char* hessian_kernel, int32_t len);
/* CUDA-event durations of the last Hessian evaluation: weight materialisation and DMMA kernel + reduction. */
int mbar_b200_last_hessian_ms(mbar_b200_ctx* ctx, double* weights_ms, double* hessian_ms);
/* CUDA-event duration of the kernels of the last mbar_b200_bin_moments after its pass (bin sums, C and D), and
 * the number of bin chunks (reads of u_kn) its C / D step took (0 when C and D were not requested). */
int mbar_b200_last_bin_stats(mbar_b200_ctx* ctx, double* ms, int32_t* chunks);
/* fp64 ceilings of this GPU measured in place (register-only DMMA.8x8x4 and DFMA loops), in TFLOP/s: the
 * roofline denominator of mbar_b200_hessian (MEASURED_PEAKS.json has no fp64 figure). */
int mbar_b200_measure_fp64_peak(int device, double* dmma_tflops, double* dfma_tflops);
/* Development probe of the device exp: out[i] = exp(a[i]) for n host arguments, evaluated by
 * which = 0: exp_fast (generic pass, Hessian weights); 1: the fused pass's exp with the state constant in the
 * exponent (MODE=1); 2: its multiplicative form e0 = exp(-u') (MODE=3).  Arguments below about -707.7 return
 * a value in [0, 2^-1020]; arguments above 709.7 are outside the contract (the host never passes them). */
int mbar_b200_probe_exp(int device, int which, int64_t n, const double* a_host, double* out_host);

/* ---- one-shot, host-buffer entry (what a binding without residency would call) --------------- */
/* self_consistent_update on host buffers: upload u_kn, one pass, f_out — copies inside the call. */
int mbar_b200_self_consistent_update_host(int device, int32_t K, int64_t N, const double* u_host,
                                          int64_t ld, const double* N_k, const double* f_k,
                                          double* f_out);

/* ---- multi-GPU: samples sharded over ranks, one all-reduce per pass -------------------------- */
#define MBAR_B200_UNIQUE_ID_BYTES 128
int mbar_b200_comm_unique_id(void* id_out /* [128] */);
/* Collective over all ranks; call it after this rank's u_kn is uploaded / synthesised. */
int mbar_b200_comm_init(mbar_b200_ctx* ctx, int32_t nranks, int32_t rank, const void* unique_id);
int mbar_b200_comm_destroy(mbar_b200_ctx* ctx);

/* Peer-memory exchange for the device-resident iteration: every rank exports a 64-byte cudaIpc handle
 * of its inbox, the caller distributes them (any transport), every rank attaches all of them.  After
 * that mbar_b200_sci_iterate runs ONE kernel per iteration: the pass kernel's last CTA stores its
 * K+2 partial sums into every peer's inbox over NVLink, waits for the peers' flags, sums in rank order
 * and applies the K-vector update — no NCCL call and no second launch on the iteration's critical path. */
#define MBAR_B200_IPC_HANDLE_BYTES 64
int mbar_b200_peer_export(mbar_b200_ctx* ctx, void* handle_out /* [64] */);
/* (needs mbar_b200_comm_init first: every host-stepped path and the K x K Hessian reduce through the communicator;
 * at most 16 ranks) */
int mbar_b200_peer_attach(mbar_b200_ctx* ctx, int32_t nranks, int32_t rank, const void* handles /* [nranks][64] */);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif

#ifdef __cplusplus
}
#endif
#endif /* MBAR_B200_H */

// mbar_b200_batch_*: many small MBAR problems (1 <= K_p <= 64 states each) resident on one GPU, their sums evaluated
// in one launch for every problem and the adaptive solver stepped for all of them in lockstep (DESIGN.md 3.5g).
//
// Layout.  Problem p keeps its own tiles [nT_p][K_p][32] of shifted energies u'_kn = u_kn - x_n with
// x_n = min over the sampled states of u_kn (0 when every such entry is +inf), as the single-problem upload stores
// them (DESIGN.md 2).  Samples past N_p in the last tile hold +inf.  Per problem the device also keeps N_k, log N_k
// and sum_n x_n.
//
// Moments.  A request names a problem and a vector f [K_p].  With c_k = f_k + log N_k over the sampled states,
//   L'_n = log sum_{k sampled} e^{c_k - u'_kn}      (per-sample max shift, exact exp)
//   a_kn = f_k - u'_kn - L'_n,   log S_k = logsumexp_n a_kn,   sum L = sum_n L'_n - sum_n x_n
// and, on request, the Gram Ghat_ij = sum_n w_in w_jn with w_kn = N_k e^{a_kn} (sampled rows) and e^{a_kn} (unsampled
// rows, only when all rows are asked for) — the row scaling of launch_hessian.  A sampled row has e^{a_kn} <= 1 / N_k
// and is summed linearly, as the single-problem pass sums it: its S_k carries a relative error of a few ulp, which the
// adaptive loop's relative-change test at tol = 1e-12 needs when f_k is near 0.  An unsampled row is kept as a running
// (max, sum) pair, so it neither under- nor overflows inside the pass.  The finalize kernel sets the request's flag
// where a sum is not a usable number (see batch_finalize_kernel).
//
// Replicate slots.  A slot is a bootstrap replicate of one problem: uint16 multiplicities c_n over its N_p samples,
// padded with 0 to the problem's tiles, and sum_n c_n x_n, computed once when the slots are set (x_n stays resident
// for that).  A weighted request names a slot and gets exactly what DeviceProblem.set_sample_weights(c) and the
// matching single-problem call give: S_k = sum_n c_n e^{a_kn}, Ghat_ij = sum_n c_n w_in w_jn and
// sum L = sum_n c_n L'_n - sum_n c_n x_n, with L'_n itself unweighted (the denominators keep N_k).  It is the same
// kernel instantiated with W = true.  Multiplying by c_n = 1 is exact and the order of operations is the same in both
// instantiations, so all-ones counts give the bits of the unweighted request.  A zero-count sample enters no sum: its
// L'_n is not added to sum L and its a_kn is -inf before the NaN test and the warp max of an unsampled row, as
// log c_n = -inf is in the single-problem pass, so an undrawn sample whose sampled energies are all +inf does not flag
// its replicate.
//
// Determinism.  Work items are (request, chunk) pairs; a chunk is CT_p tiles with CT_p a function of (N_p, K_p) alone.
// Warp w of a CTA takes the chunk's tiles w, w + 4, ... in order and folds each tile into its own (max, sum) pairs;
// the four warps' pairs, the 128 thread sums of L' and the per-thread Gram sums are combined in a fixed order, and
// the finalize kernel adds a request's chunk partials in chunk order.  There are no atomics: a request's sums are the
// same bits whichever requests share the launch, and repeat calls are bit-identical.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

#include "internal.cuh"

namespace mbar {

constexpr int BATCH_MAX_K = 64;
constexpr int BATCH_THREADS = 128;                  // four warps, one tile each per round
constexpr int BATCH_WARPS = BATCH_THREADS / 32;
constexpr int BATCH_ROUND = BATCH_THREADS;          // samples per round
constexpr int BATCH_SW_LD = BATCH_ROUND + 1;        // leading dimension of the staged weights (bank spread)
constexpr int BATCH_GSLOTS = (BATCH_MAX_K * (BATCH_MAX_K + 1) / 2 + BATCH_THREADS - 1) / BATCH_THREADS;
constexpr int BATCH_FINALIZE_THREADS = 256;         // one CTA per request: up to 18528 Gram entries at R = 192
constexpr int64_t BATCH_MAX_CHUNKS = 4096;

// tiles per chunk: about 64k entries of u' per chunk, at most BATCH_MAX_CHUNKS chunks per problem
__host__ __device__ __forceinline__ int64_t batch_chunk_tiles(int64_t nT, int K) {
    const int64_t base = 2048 / K > 4 ? 2048 / K : 4;
    const int64_t need = (nT + BATCH_MAX_CHUNKS - 1) / BATCH_MAX_CHUNKS;
    return base > need ? base : need;
}

// One request: a problem's K rows, a replicate slot's, or a problem's (or a replicate slot's) K resident rows followed
// by the problem's M appended rows; R = K + M rows in all.
struct BatchReq {
    int64_t uoff;     // first double of the problem's tiles
    int64_t N, nT;    // samples and tiles of the problem
    int64_t ct;       // tiles per chunk
    int64_t item0;    // first (request, chunk) item
    int64_t poff;     // first double of the request's chunk partials
    int64_t ooff;     // first double of the request's packed output
    int64_t voff;     // first entry of the problem's K-vectors (N_k, log N_k)
    int64_t foff;     // first entry of the request's f
    int32_t K;
    int32_t prob;     // the problem, or for a weighted request its replicate slot: indexes sum x (sum c x)
    int32_t allRows, wantG;
    // appended rows (M = 0 for every other request); the Gram of such a request is batch_aug_gram_kernel's
    int32_t M;
    int64_t aoff;     // first double of the problem's appended tiles
    int64_t gct;      // tiles per Gram chunk
    int64_t gitem0;   // first (request, block pair, Gram chunk) item
    int64_t gpoff;    // first double of the request's Gram partials
    int64_t loff;     // first entry of the request's L'_n scratch
};

// per-request packed output: [0, R) S, [R, 2R) log S, [2R] sum L, [2R + 1] flag, then R x R Ghat when asked for
__host__ __device__ __forceinline__ int64_t batch_out_size(int R, bool G) {
    return 2 * R + 2 + (G ? (int64_t)R * R : 0);
}
// per-chunk partial: R (max, sum) pairs, sum L', bad flag, then, with the in-pass Gram, its R (R + 1) / 2
// lower-triangle entries
__host__ __device__ __forceinline__ int64_t batch_part_size(int R, bool G) {
    return 2 * R + 2 + (G ? (int64_t)R * (R + 1) / 2 : 0);
}

// one problem's layout for the upload kernels: raw offset, tile offset, first tile, samples, K-vector offset, states
struct BatchProbDev {
    int64_t roff, uoff, tile0, N, voff;
    int32_t K;
};

// ---- appended rows and the augmented moments (DESIGN.md 3.5g'') ----
constexpr int AUG_MAX_R = MBAR_B200_BATCH_MAX_ROWS;
constexpr int AUG_BLOCK = 32;                       // Gram rows per block: a work item is one pair of row blocks
constexpr int AUG_SW_LD = BATCH_ROUND + 1;          // leading dimension of a staged weight block
constexpr int64_t AUG_GRAM_MIN_TILES = 512;         // a Gram chunk holds at least 16384 samples ...
constexpr int64_t AUG_GRAM_MAX_CHUNKS = 64;         // ... and a problem at most 64 Gram chunks
constexpr size_t AUG_GRAM_SMEM = 2 * AUG_BLOCK * AUG_SW_LD * sizeof(double);

__host__ __device__ __forceinline__ int64_t aug_gram_tiles(int64_t nT) {
    const int64_t need = (nT + AUG_GRAM_MAX_CHUNKS - 1) / AUG_GRAM_MAX_CHUNKS;
    return need > AUG_GRAM_MIN_TILES ? need : AUG_GRAM_MIN_TILES;
}
__host__ __device__ __forceinline__ int aug_blocks(int R) { return (R + AUG_BLOCK - 1) / AUG_BLOCK; }

// one problem's appended rows for the upload kernel: raw offset, appended tile offset, first tile of the problem
// (indexes x_n), first tile among the appended problems, samples, rows
struct AugProbDev {
    int64_t roff, aoff, tile0, atile0, N;
    int32_t M;
};

}  // namespace mbar

struct mbar_b200_batch : mbar::Resident {
    int P = 0;
    std::vector<int> K;
    std::vector<int64_t> N, nT, uoff, voff;
    std::vector<double> Nk;                     // concatenated N_k
    int64_t uTotal = 0;
    mbar::DevArray<double> d_u, d_Nk, d_logNk, d_sumx;
    mbar::DevArray<double> d_x;                 // x_n [tiles * 32], kept for the slots' sum_n c_n x_n
    mbar::DevArray<mbar::BatchProbDev> d_prob;  // per-problem layout, as the upload kernels read it
    // replicate slots (mbar_b200_batch_set_replicates)
    int nSlots = 0;
    std::vector<int> slotProb;
    std::vector<int64_t> slotCoff;              // first count of each slot in d_counts
    mbar::DevArray<uint16_t> d_counts;          // each slot's c_n, padded with 0 to its problem's tiles
    mbar::DevArray<int64_t> d_slotCoff;
    mbar::DevArray<int32_t> d_slotProb;
    mbar::DevArray<double> d_sumxw;             // sum_n c_n x_n of each slot
    // appended rows (mbar_b200_batch_set_unsampled)
    std::vector<int> M;                         // appended rows of each problem (0: none)
    std::vector<int64_t> aoff;                  // first double of each problem's appended tiles
    mbar::DevArray<double> d_ua;                // appended tiles [nT_p][M_p][32] of u - x_n
    mbar::DevArray<double> d_L, d_gpart;        // L'_n of each Gram request, Gram chunk partials
    // per-call buffers, grown on demand
    mbar::DevArray<mbar::BatchReq> d_req;
    mbar::DevArray<double> d_f, d_part, d_out;
    mbar::HostPinned<double> h_f;               // pinned staging of f and of the packed output
    mbar::HostPinned<double> h_out;
    mbar::HostPinned<int32_t> h_bin;            // pinned staging of the bin indices (mbar_b200_batch_bin_moments)
    // the last moments / solve call
    int32_t lastLaunches = 0, lastIterations = 0;
    int64_t lastBytes = 0;
};

namespace mbar {

// entry e = i (i + 1) / 2 + j of a lower triangle -> (row i, column j), i >= j
__device__ __forceinline__ int2 tri_decode(int e) {
    int i = (int)((sqrt(8.0 * e + 1.0) - 1.0) * 0.5);
    while ((i + 1) * (i + 2) / 2 <= e) ++i;
    while (i * (i + 1) / 2 > e) --i;
    return make_int2(i, e - i * (i + 1) / 2);
}

// ---- upload: raw row-major problems -> shifted tiles, x_n, sum x_n -------------------------------------------------

// one warp per tile, one lane per sample; bad[0] counts NaN or -inf energies
__global__ void __launch_bounds__(256) batch_retile_kernel(const double* __restrict__ raw,
                                                           const BatchProbDev* __restrict__ pr, int P,
                                                           int64_t nTiles, const double* __restrict__ Nk,
                                                           double* __restrict__ u, double* __restrict__ x,
                                                           unsigned int* bad) {
    const int64_t tile = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (tile >= nTiles) return;
    const int lane = threadIdx.x & 31;
    const int p = find_segment(P, tile, [&](int s) { return pr[s].tile0; });
    const BatchProbDev q = pr[p];
    const int64_t t = tile - q.tile0;
    const int64_t n = t * 32 + lane;
    const bool valid = n < q.N;
    double xn = INFINITY;
    bool nan = false;
    if (valid)
        for (int k = 0; k < q.K; ++k) {
            const double v = raw[q.roff + (int64_t)k * q.N + n];
            if (v != v || v == -INFINITY) nan = true;
            if (Nk[q.voff + k] > 0.0) xn = fmin(xn, v);
        }
    if (!(xn < INFINITY)) xn = 0.0;
    double* dst = u + q.uoff + t * q.K * 32 + lane;
    for (int k = 0; k < q.K; ++k) dst[k * 32] = valid ? raw[q.roff + (int64_t)k * q.N + n] - xn : INFINITY;
    x[tile * 32 + lane] = valid ? xn : 0.0;
    if (nan) atomicAdd(bad, 1u);        // an error count, not a result
}

// sum_n x_n of each problem (W = false, one CTA per problem) or sum_n c_n x_n of each replicate slot (W = true, one
// CTA per slot), in a fixed order that is the same for both: all-ones counts give the problem's bits
template <bool W>
__global__ void __launch_bounds__(256) batch_sumx_kernel(const double* __restrict__ x,
                                                         const BatchProbDev* __restrict__ pr,
                                                         const int32_t* __restrict__ slotProb,
                                                         const int64_t* __restrict__ slotCoff,
                                                         const uint16_t* __restrict__ counts,
                                                         double* __restrict__ sumx) {
    __shared__ double sh[256];
    const BatchProbDev q = pr[W ? slotProb[blockIdx.x] : blockIdx.x];
    double s = 0.0;
    for (int64_t n = threadIdx.x; n < q.N; n += 256) {
        if constexpr (W) s += (double)counts[slotCoff[blockIdx.x] + n] * x[q.tile0 * 32 + n];
        else s += x[q.tile0 * 32 + n];
    }
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) sumx[blockIdx.x] = sh[0];
}

// appended rows -> shifted tiles: one warp per appended tile, one lane per sample
__global__ void __launch_bounds__(256) batch_aug_retile_kernel(const double* __restrict__ raw,
                                                               const AugProbDev* __restrict__ pr, int n,
                                                               int64_t nTiles, const double* __restrict__ x,
                                                               double* __restrict__ ua) {
    const int64_t tile = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (tile >= nTiles) return;
    const int lane = threadIdx.x & 31;
    const AugProbDev q = pr[find_segment(n, tile, [&](int p) { return pr[p].atile0; })];
    const int64_t t = tile - q.atile0;
    const int64_t s = t * 32 + lane;
    const bool valid = s < q.N;
    const double xn = x[(q.tile0 + t) * 32 + lane];
    double* dst = ua + q.aoff + t * q.M * 32 + lane;
    for (int m = 0; m < q.M; ++m) dst[m * 32] = valid ? raw[q.roff + (int64_t)m * q.N + s] - xn : INFINITY;
}

// ---- the pass ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_max(double x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x = fmax(x, __shfl_xor_sync(0xffffffffu, x, o));
    return x;
}

// fold the pair (m2, s2) into (m, s): the running log-sum-exp m + log s
__device__ __forceinline__ void pair_merge(double& m, double& s, double m2, double s2) {
    if (!(s2 > 0.0)) return;
    if (m2 > m) {
        s = s * exp(m - m2) + s2;
        m = m2;
    } else {
        s += s2 * exp(m2 - m);
    }
}

// row k of a request at tile t: the problem's own tiles for k < K, its appended tiles after
__device__ __forceinline__ const double* batch_row(const double* __restrict__ u, const double* __restrict__ ua,
                                                   const BatchReq& q, int64_t t, int k, int lane) {
    return k < q.K ? u + q.uoff + (t * q.K + k) * 32 + lane : ua + q.aoff + (t * q.M + (k - q.K)) * 32 + lane;
}

// One CTA per (request, chunk) item; every request of a launch is of one kind:
//   W: weighted requests (q.prob names a replicate slot; its counts start at slotCoff[q.prob]);
//   APPENDED: requests with appended rows, every row asked for; with the Gram, L'_n goes to Lbuf for
//     batch_aug_gram_kernel instead of an in-pass Gram;
//   both: a replicate slot with its problem's appended rows, never with the Gram (DESIGN.md 3.5g''').
template <bool W, bool APPENDED>
__global__ void __launch_bounds__(BATCH_THREADS) batch_pass_kernel(
    const double* __restrict__ u, const BatchReq* __restrict__ req, int nReq, const double* __restrict__ fAll,
    const double* __restrict__ NkAll, const double* __restrict__ logNkAll, double* __restrict__ part,
    const int64_t* __restrict__ slotCoff, const uint16_t* __restrict__ counts, const double* __restrict__ ua,
    double* __restrict__ Lbuf) {
    constexpr int MAX_R = APPENDED ? AUG_MAX_R : BATCH_MAX_K;
    extern __shared__ __align__(16) double sW[];                  // [K][BATCH_SW_LD] staged Gram weights
    __shared__ double sM[BATCH_WARPS][MAX_R], sS[BATCH_WARPS][MAX_R];
    __shared__ double sF[MAX_R], sC[BATCH_MAX_K], sLs[BATCH_MAX_K];
    __shared__ int sRow[MAX_R];                                   // 1 sampled, 2 unsampled and asked for, 0 neither
    __shared__ double sRed[BATCH_THREADS];
    __shared__ int sBad;
    const int64_t item = blockIdx.x;
    const BatchReq q = req[find_segment(nReq, item, [&](int r) { return req[r].item0; })];
    const int64_t chunk = item - q.item0;
    const int K = q.K, R = APPENDED ? K + q.M : K;
    const bool G = !APPENDED && q.wantG;                          // the in-pass Gram
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int k0 = 0; k0 < MAX_R; k0 += BATCH_THREADS) {            // thread tid takes rows tid, tid + 128, ...
        const int k = k0 + tid;
        if (k >= R) break;
        const bool sampled = k < K && NkAll[q.voff + k] > 0.0;
        sF[k] = fAll[q.foff + k];
        if (k < K) {
            sC[k] = sampled ? sF[k] + logNkAll[q.voff + k] : -INFINITY;
            if (!APPENDED) sLs[k] = sampled ? logNkAll[q.voff + k] : 0.0;
        }
        sRow[k] = sampled ? 1 : (q.allRows ? 2 : 0);
    }
    for (int k = tid; k < BATCH_WARPS * MAX_R; k += BATCH_THREADS) {
        (&sM[0][0])[k] = -INFINITY;
        (&sS[0][0])[k] = 0.0;
    }
    if (tid == 0) sBad = 0;
    // lower-triangle Gram entries of this thread: e = tid + BATCH_THREADS * slot, row i >= column j
    const int E = G ? K * (K + 1) / 2 : 0;
    int gi[BATCH_GSLOTS], gj[BATCH_GSLOTS];
    double gacc[BATCH_GSLOTS];
#pragma unroll
    for (int sl = 0; sl < BATCH_GSLOTS; ++sl) {
        const int2 ij = tri_decode(tid + BATCH_THREADS * sl);
        gi[sl] = ij.x;
        gj[sl] = ij.y;
        gacc[sl] = 0.0;
    }
    __syncthreads();
    double* sCn = nullptr;                                        // the round's counts, for the Gram
    const uint16_t* cq = nullptr;
    if constexpr (W) {
        __shared__ double sCnBuf[BATCH_ROUND];
        sCn = sCnBuf;
        cq = counts + slotCoff[q.prob];
    }
    const int64_t t0 = chunk * q.ct, t1 = min(q.nT, t0 + q.ct);
    const int rounds = (int)((q.ct + BATCH_WARPS - 1) / BATCH_WARPS);
    double sumL = 0.0;
    bool bad = false;
    for (int r = 0; r < rounds; ++r) {
        const int64_t t = t0 + (int64_t)r * BATCH_WARPS + warp;
        const bool tileOn = t < t1;                                  // warp-uniform
        const int64_t n = t * 32 + lane;
        const bool valid = tileOn && n < q.N;
        const double* ut = u + q.uoff + t * (int64_t)K * 32 + lane;
        double cn = 1.0;
        if constexpr (W) {
            cn = valid ? (double)__ldg(cq + n) : 0.0;
            if (G) sCn[tid] = cn;
        }
        double Lp = 0.0;
        if (valid) {
            double m = -INFINITY;
            for (int k = 0; k < K; ++k)
                if (sRow[k] == 1) m = fmax(m, sC[k] - __ldg(ut + k * 32));
            double D = 0.0;
            for (int k = 0; k < K; ++k)
                if (sRow[k] == 1) D += exp(sC[k] - __ldg(ut + k * 32) - m);
            Lp = m + log(D);
            if constexpr (W) {
                if (cn != 0.0) sumL += cn * Lp;
            } else {
                sumL += Lp;
            }
        }
        if (tileOn) {
            if (APPENDED && !W && q.wantG) Lbuf[q.loff + n] = Lp;      // weighted requests have no Gram
            for (int k = 0; k < R; ++k) {
                if (sRow[k] == 0) {
                    if (G) sW[k * BATCH_SW_LD + tid] = 0.0;
                    continue;
                }
                double a = valid ? sF[k] - __ldg(APPENDED ? batch_row(u, ua, q, t, k, lane) : ut + k * 32) - Lp
                                 : -INFINITY;
                if constexpr (W)
                    if (cn == 0.0) a = -INFINITY;      // before the NaN test: an undrawn sample enters no sum
                if (a != a) {
                    bad = true;
                    a = -INFINITY;
                }
                // sampled rows: e^a <= 1 / N_k, summed linearly (the pair keeps max 0) as the single-problem pass
                // sums them; every other row: shifted by the warp's max
                const double wm = sRow[k] == 1 ? 0.0 : warp_max(a);
                double e = wm > -INFINITY ? exp(a - wm) : 0.0;
                if constexpr (W) e *= cn;
                const double ws = warp_sum(e);
                if (lane == 0) pair_merge(sM[warp][k], sS[warp][k], wm, ws);
                if (G) sW[k * BATCH_SW_LD + tid] = exp(a + sLs[k]);
            }
        } else if (G)
            for (int k = 0; k < K; ++k) sW[k * BATCH_SW_LD + tid] = 0.0;
        if (G) {
            __syncthreads();
#pragma unroll
            for (int sl = 0; sl < BATCH_GSLOTS; ++sl) {
                if (tid + BATCH_THREADS * sl < E) {
                    const double* wi = sW + gi[sl] * BATCH_SW_LD;
                    const double* wj = sW + gj[sl] * BATCH_SW_LD;
                    double acc = gacc[sl];
                    if constexpr (W)
                        for (int s = 0; s < BATCH_ROUND; ++s) acc = fma(wi[s] * sCn[s], wj[s], acc);
                    else
                        for (int s = 0; s < BATCH_ROUND; ++s) acc = fma(wi[s], wj[s], acc);
                    gacc[sl] = acc;
                }
            }
            __syncthreads();
        }
    }
    if (bad) sBad = 1;
    sRed[tid] = sumL;
    __syncthreads();
    for (int o = BATCH_THREADS / 2; o > 0; o >>= 1) {
        if (tid < o) sRed[tid] += sRed[tid + o];
        __syncthreads();
    }
    const int64_t stride = batch_part_size(R, G);
    double* pc = part + q.poff + chunk * stride;
#pragma unroll
    for (int k0 = 0; k0 < MAX_R; k0 += BATCH_THREADS) {
        const int k = k0 + tid;
        if (k >= R) break;
        double m = sM[0][k], s = sS[0][k];
        for (int w = 1; w < BATCH_WARPS; ++w) pair_merge(m, s, sM[w][k], sS[w][k]);
        pc[2 * k] = m;
        pc[2 * k + 1] = s;
    }
    if (tid == 0) {
        pc[2 * R] = sRed[0];
        pc[2 * R + 1] = sBad ? 1.0 : 0.0;
    }
#pragma unroll
    for (int sl = 0; sl < BATCH_GSLOTS; ++sl) {
        const int e = tid + BATCH_THREADS * sl;
        if (e < E) pc[2 * R + 2 + e] = gacc[sl];
    }
}

// The Gram of appended-row requests, over (request, pair of 32-row blocks bi >= bj, Gram chunk) items: it rebuilds the
// two blocks' weights of 128 samples at a time from the tiles and the pass's L'_n, stages them in shared memory and
// accumulates a 2 x 4 patch of the 32 x 32 block per thread with DFMA, samples in order: thread
// (ti, tj) = (tid / 8, tid % 8) owns rows 2 ti, 2 ti + 1 of block bi and columns tj + 8 c (c < 4) of block bj.  No
// atomics, and the Gram chunking is a function of N_p alone.
__global__ void __launch_bounds__(BATCH_THREADS) batch_aug_gram_kernel(
    const double* __restrict__ u, const double* __restrict__ ua, const BatchReq* __restrict__ req, int nReq,
    const double* __restrict__ fAll, const double* __restrict__ NkAll, const double* __restrict__ logNkAll,
    const double* __restrict__ Lbuf, double* __restrict__ gpart) {
    extern __shared__ __align__(16) double sAug[];               // [2][AUG_BLOCK][AUG_SW_LD] staged weights
    __shared__ double sF[2][AUG_BLOCK], sLs[2][AUG_BLOCK];
    const int64_t item = blockIdx.x;
    const BatchReq q = req[find_segment(nReq, item, [&](int r) { return req[r].gitem0; })];
    const int R = q.K + q.M;
    const int64_t ngc = (q.nT + q.gct - 1) / q.gct;
    const int64_t local = item - q.gitem0;
    const int pair = (int)(local / ngc);
    const int64_t gc = local - (int64_t)pair * ngc;
    const int2 b2 = tri_decode(pair);
    const int bi = b2.x, bj = b2.y;
    const int nh = bi == bj ? 1 : 2;                             // a diagonal block stages one row block
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 2 * AUG_BLOCK) {
        const int h = tid / AUG_BLOCK, i = tid % AUG_BLOCK;
        const int k = (h ? bj : bi) * AUG_BLOCK + i;
        const bool s = k < q.K && NkAll[q.voff + k] > 0.0;
        sF[h][i] = k < R ? fAll[q.foff + k] : 0.0;
        sLs[h][i] = s ? logNkAll[q.voff + k] : 0.0;
    }
    double* sWi = sAug;
    double* sWj = nh == 2 ? sAug + AUG_BLOCK * AUG_SW_LD : sAug;
    const int ti = tid >> 3, tj = tid & 7;
    double acc[2][4];
#pragma unroll
    for (int e = 0; e < 2; ++e)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[e][c] = 0.0;
    __syncthreads();
    const int64_t t0 = gc * q.gct, t1 = min(q.nT, t0 + q.gct);
    const int64_t rounds = (t1 - t0 + BATCH_WARPS - 1) / BATCH_WARPS;
    for (int64_t r = 0; r < rounds; ++r) {
        const int64_t t = t0 + r * BATCH_WARPS + warp;
        const int64_t n = t * 32 + lane;
        const bool valid = t < t1 && n < q.N;
        const double Lp = valid ? Lbuf[q.loff + n] : 0.0;
        for (int h = 0; h < nh; ++h) {
            const int b = h ? bj : bi;
            double* w = h ? sWj : sWi;
            for (int i = 0; i < AUG_BLOCK; ++i) {
                const int k = b * AUG_BLOCK + i;
                double x = 0.0;
                if (valid && k < R) x = exp(sF[h][i] - __ldg(batch_row(u, ua, q, t, k, lane)) - Lp + sLs[h][i]);
                w[i * AUG_SW_LD + tid] = x;
            }
        }
        __syncthreads();
        const double* wa = sWi + (2 * ti) * AUG_SW_LD;
        const double* wb = sWj + tj * AUG_SW_LD;
#pragma unroll 4
        for (int s = 0; s < BATCH_ROUND; ++s) {
            const double a0 = wa[s], a1 = wa[AUG_SW_LD + s];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const double bc = wb[c * 8 * AUG_SW_LD + s];
                acc[0][c] = fma(a0, bc, acc[0][c]);
                acc[1][c] = fma(a1, bc, acc[1][c]);
            }
        }
        __syncthreads();
    }
    double* pg = gpart + q.gpoff + local * (AUG_BLOCK * AUG_BLOCK);
#pragma unroll
    for (int e = 0; e < 2; ++e)
#pragma unroll
        for (int c = 0; c < 4; ++c) pg[(2 * ti + e) * AUG_BLOCK + tj + 8 * c] = acc[e][c];
}

// A request's partials in chunk order -> its packed output.  The flag is set when a NaN reached a sum, when a
// sampled row's S_k is outside (1e-280, 1e300) (the range the fused pass and the adaptive loop accept), when any
// other row asked for has a NaN or overflowing S_k, or, with the Gram, when an entry of Ghat is not finite: an
// unsampled row's Gram weight e^{a_kn} is not shifted, so a weight above about e^355 overflows Ghat_kk while S_k is
// still finite.  An unsampled row whose every weight is zero (all its energies +inf) reports S_k = 0,
// log S_k = -inf, as the single-problem path does.  The Gram partials are the pass's per-chunk lower triangles or,
// for appended rows, those of batch_aug_gram_kernel: block pair (bi, bj) and Gram chunk c at
// gpoff + (pair * nGc + c) * 1024.
__global__ void __launch_bounds__(BATCH_FINALIZE_THREADS) batch_finalize_kernel(const BatchReq* __restrict__ req,
                                                                                const double* __restrict__ part,
                                                                                const double* __restrict__ gpart,
                                                                                const double* __restrict__ NkAll,
                                                                                const double* __restrict__ sumx,
                                                                                double* __restrict__ out) {
    __shared__ int sFlag;
    const BatchReq q = req[blockIdx.x];
    const int K = q.K, R = q.K + q.M, tid = threadIdx.x;
    const int64_t stride = batch_part_size(R, q.wantG && q.M == 0);
    const int64_t nc = (q.nT + q.ct - 1) / q.ct;
    const double* p0 = part + q.poff;
    double* o = out + q.ooff;
    if (tid == 0) sFlag = 0;
    __syncthreads();
    for (int k = tid; k < R; k += BATCH_FINALIZE_THREADS) {
        double m = -INFINITY, s = 0.0;
        for (int64_t c = 0; c < nc; ++c) pair_merge(m, s, p0[c * stride + 2 * k], p0[c * stride + 2 * k + 1]);
        const double logS = s > 0.0 ? m + log(s) : -INFINITY;
        const double S = m == 0.0 ? s : exp(logS);      // sampled rows: the linear sum itself
        o[k] = S;
        o[R + k] = logS;
        const bool sampled = k < K && NkAll[q.voff + k] > 0.0;
        if (sampled && !(S > 1e-280 && S < 1e300)) sFlag = 1;
        if (!sampled && q.allRows && (logS != logS || !(S < INFINITY))) sFlag = 1;
    }
    if (tid == 0) {
        double sl = 0.0, bad = 0.0;
        for (int64_t c = 0; c < nc; ++c) {
            sl += p0[c * stride + 2 * R];
            bad = fmax(bad, p0[c * stride + 2 * R + 1]);
        }
        o[2 * R] = sl - sumx[q.prob];
        if (bad > 0.0 || sl != sl) sFlag = 1;
    }
    if (q.wantG) {
        const int E = R * (R + 1) / 2;
        for (int e = tid; e < E; e += BATCH_FINALIZE_THREADS) {
            const int2 ij = tri_decode(e);
            const int i = ij.x, j = ij.y;
            const double* pg = p0 + 2 * R + 2 + e;        // entry e of chunk c at pg[c * gs], c < ngc
            int64_t gs = stride, ngc = nc;
            if (q.M > 0) {
                const int bi = i / AUG_BLOCK, bj = j / AUG_BLOCK;
                gs = AUG_BLOCK * AUG_BLOCK;
                ngc = (q.nT + q.gct - 1) / q.gct;
                pg = gpart + q.gpoff + (int64_t)(bi * (bi + 1) / 2 + bj) * ngc * gs + (i % AUG_BLOCK) * AUG_BLOCK +
                     j % AUG_BLOCK;
            }
            double g = 0.0;
            for (int64_t c = 0; c < ngc; ++c) g += pg[c * gs];
            if (!isfinite(g)) sFlag = 1;
            o[2 * R + 2 + (int64_t)i * R + j] = g;
            o[2 * R + 2 + (int64_t)j * R + i] = g;
        }
    }
    __syncthreads();
    if (tid == 0) o[2 * R + 1] = sFlag ? 1.0 : 0.0;
}

// What the ids of a call name: problems, replicate slots (weighted requests), problems with their appended rows, or
// replicate slots with their problem's appended rows (weighted requests with appended rows).
enum class Units { problems, slots, appended, slot_appended };

static inline bool units_weighted(Units kind) { return kind == Units::slots || kind == Units::slot_appended; }
static inline bool units_appended(Units kind) { return kind == Units::appended || kind == Units::slot_appended; }

// One request of a call: f (R_p values) at unit `id`.
struct Ask {
    int id;
    const double* f;
    bool G;
};

// the problem of unit `id`
static inline int unit_problem(const mbar_b200_batch* b, Units kind, int id) {
    return units_weighted(kind) ? b->slotProb[id] : id;
}

// the rows of unit `id`: K_p, or K_p + M_p with the appended rows
static inline int unit_rows(const mbar_b200_batch* b, Units kind, int id) {
    const int p = unit_problem(b, kind, id);
    return b->K[p] + (units_appended(kind) ? b->M[p] : 0);
}

// Sets a kernel's dynamic shared memory limit once per device.
template <auto Kernel, size_t Bytes>
static int smem_limit(int device) {
    static bool done[16] = {false};
    if (!done[device & 15]) {
        MBAR_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Bytes));
        done[device & 15] = true;
    }
    return MBAR_B200_OK;
}

constexpr size_t BATCH_GRAM_SMEM = BATCH_MAX_K * BATCH_SW_LD * sizeof(double);

// Evaluate the requests, all naming units of one kind, in one launch of each kernel (pass, the appended rows' Gram
// when asked for, finalize) and one synchronisation; returns the packed outputs in b->h_out, request r's at
// offsets[r] (batch_out_size(R_p, G) doubles each).
static int batch_run(mbar_b200_batch* b, Units kind, const std::vector<Ask>& asks, bool allRows,
                     std::vector<int64_t>& offsets, double* msAcc) {
    const bool weighted = units_weighted(kind), appended = units_appended(kind);
    const int nReq = (int)asks.size();
    std::vector<BatchReq> req((size_t)nReq);
    int64_t items = 0, gitems = 0, parts = 0, gparts = 0, outs = 0, fs = 0, Ls = 0, bytes = 0;
    int maxKG = 0;
    offsets.resize(nReq);
    for (int r = 0; r < nReq; ++r) {
        const int p = unit_problem(b, kind, asks[r].id);
        BatchReq& q = req[r];
        q.K = b->K[p];
        q.M = appended ? b->M[p] : 0;
        q.prob = asks[r].id;
        q.allRows = allRows || appended ? 1 : 0;
        q.wantG = asks[r].G ? 1 : 0;
        const int R = q.K + q.M;
        q.N = b->N[p];
        q.nT = b->nT[p];
        q.ct = batch_chunk_tiles(q.nT, R);
        q.uoff = b->uoff[p];
        q.voff = b->voff[p];
        q.item0 = items;
        q.poff = parts;
        q.ooff = outs;
        q.foff = fs;
        const int64_t nc = (q.nT + q.ct - 1) / q.ct;
        items += nc;
        parts += nc * batch_part_size(R, q.wantG && !appended);
        bytes += q.nT * 32 * R * 8 + (weighted ? q.nT * 32 * 2 : 0);
        if (appended) {
            q.aoff = b->aoff[p];
            q.gct = aug_gram_tiles(q.nT);
            q.gitem0 = gitems;
            q.gpoff = gparts;
            q.loff = Ls;
        }
        if (appended && q.wantG) {
            const int nb = aug_blocks(R);
            const int64_t ngc = (q.nT + q.gct - 1) / q.gct;
            gitems += (int64_t)nb * (nb + 1) / 2 * ngc;
            gparts += (int64_t)nb * (nb + 1) / 2 * ngc * AUG_BLOCK * AUG_BLOCK;
            Ls += q.nT * 32;
            bytes += q.nT * 32 * 8 * (int64_t)nb * R;             // every row is staged by nb block pairs
        } else if (q.wantG) {
            maxKG = std::max(maxKG, q.K);
        }
        offsets[r] = outs;
        outs += batch_out_size(R, q.wantG);
        fs += R;
    }
    MBAR_REQUIRE(items < INT32_MAX && gitems < INT32_MAX, MBAR_B200_ERR_INVALID, "batch: %lld chunks in one call",
                 (long long)(items + gitems));
    MBAR_TRY(b->d_req.grow(nReq, "batch"));
    MBAR_TRY(b->d_f.grow(fs, "batch"));
    MBAR_TRY(b->d_part.grow(parts, "batch"));
    MBAR_TRY(b->d_out.grow(outs, "batch"));
    if (gitems > 0) {
        MBAR_TRY(b->d_gpart.grow(gparts, "batch"));
        MBAR_TRY(b->d_L.grow(Ls, "batch"));
        MBAR_TRY((smem_limit<batch_aug_gram_kernel, AUG_GRAM_SMEM>(b->device)));
    }
    MBAR_TRY(b->h_f.grow((size_t)fs + (size_t)nReq * sizeof(BatchReq) / 8 + 1, "batch"));
    MBAR_TRY(b->h_out.grow((size_t)outs, "batch"));
    for (int r = 0; r < nReq; ++r) std::memcpy(b->h_f + req[r].foff, asks[r].f,
                                             (size_t)(req[r].K + req[r].M) * sizeof(double));
    BatchReq* hreq = reinterpret_cast<BatchReq*>(b->h_f + fs);
    std::memcpy(hreq, req.data(), req.size() * sizeof(BatchReq));
    MBAR_CUDA(cudaMemcpyAsync(b->d_f, b->h_f, (size_t)fs * sizeof(double), cudaMemcpyHostToDevice, b->stream));
    MBAR_CUDA(cudaMemcpyAsync(b->d_req, hreq, req.size() * sizeof(BatchReq), cudaMemcpyHostToDevice, b->stream));
    const size_t shBytes = (size_t)maxKG * BATCH_SW_LD * sizeof(double);
    if (shBytes > 0)
        MBAR_TRY((weighted ? smem_limit<batch_pass_kernel<true, false>, BATCH_GRAM_SMEM>(b->device)
                           : smem_limit<batch_pass_kernel<false, false>, BATCH_GRAM_SMEM>(b->device)));
    const auto pass = weighted ? (appended ? batch_pass_kernel<true, true> : batch_pass_kernel<true, false>)
                               : appended ? batch_pass_kernel<false, true> : batch_pass_kernel<false, false>;
    MBAR_CUDA(cudaEventRecord(b->ev0, b->stream));
    pass<<<(unsigned)items, BATCH_THREADS, shBytes, b->stream>>>(b->d_u, b->d_req, nReq, b->d_f, b->d_Nk, b->d_logNk,
                                                                 b->d_part, b->d_slotCoff, b->d_counts, b->d_ua,
                                                                 b->d_L);
    if (gitems > 0)
        batch_aug_gram_kernel<<<(unsigned)gitems, BATCH_THREADS, AUG_GRAM_SMEM, b->stream>>>(
            b->d_u, b->d_ua, b->d_req, nReq, b->d_f, b->d_Nk, b->d_logNk, b->d_L, b->d_gpart);
    batch_finalize_kernel<<<(unsigned)nReq, BATCH_FINALIZE_THREADS, 0, b->stream>>>(
        b->d_req, b->d_part, b->d_gpart, b->d_Nk, weighted ? b->d_sumxw : b->d_sumx, b->d_out);
    MBAR_CUDA(cudaGetLastError());
    MBAR_CUDA(cudaEventRecord(b->ev1, b->stream));
    MBAR_CUDA(cudaMemcpyAsync(b->h_out, b->d_out, (size_t)outs * sizeof(double), cudaMemcpyDeviceToHost, b->stream));
    MBAR_CUDA(cudaStreamSynchronize(b->stream));
    float e = 0.f;
    if (event_ms(b->ev0, b->ev1, &e)) *msAcc += e;
    b->lastLaunches += gitems > 0 ? 3 : 2;
    b->lastBytes += bytes;
    return MBAR_B200_OK;
}

// Per-unit state of the batched adaptive loop.
struct BatchSolver {
    std::vector<int> active;
    StepRows rows;
    std::vector<double> cur, f_sci, f_nr, g, S, logS, G, A, rhs;
    mbar_b200_solve_result r{};
    bool haveNr = false;
};

// The adaptive loop of mbar_b200_batch_solve over U units: the problems (weighted = false, U = P) or the replicate
// slots (weighted = true, U = nSlots), each unit with its problem's K_p entries of f in unit order.  Every iteration
// evaluates both candidates of every unfinished unit in one batch_run.
static int batch_solve_units(mbar_b200_batch* b, bool weighted, double* f, double tol, int32_t maxiter,
                             int32_t min_sc_iter, double gamma, int32_t* status, int32_t* iterations, const char* who) {
    MBAR_REQUIRE(maxiter >= 0, MBAR_B200_ERR_INVALID, "%s: maxiter=%d", who, (int)maxiter);
    MBAR_CUDA(cudaSetDevice(b->device));
    b->lastLaunches = 0;
    b->lastBytes = 0;
    b->lastIterations = 0;
    double ms = 0.0;
    const Units kind = weighted ? Units::slots : Units::problems;
    const int U = weighted ? b->nSlots : b->P;
    std::vector<BatchSolver> sv((size_t)U);
    std::vector<int64_t> foff((size_t)U + 1, 0);
    std::vector<int> work;                    // units still iterating, in index order
    for (int u = 0; u < U; ++u) {
        BatchSolver& s = sv[u];
        const int p = unit_problem(b, kind, u);
        const int K = b->K[p];
        foff[u + 1] = foff[u] + K;
        const double* Nk = b->Nk.data() + b->voff[p];
        for (int k = 0; k < K; ++k)
            if (Nk[k] > 0.0) s.active.push_back(k);
        s.rows = StepRows{K, s.active.data(), (int)s.active.size(), Nk};
        double* fp = f + foff[u];
        s.cur.assign(fp, fp + K);
        for (int k : s.active) s.cur[k] -= fp[s.active[0]];
        for (int k : s.active)
            MBAR_REQUIRE(std::isfinite(s.cur[k]) && std::fabs(s.cur[k]) < 0.5 * C_RANGE, MBAR_B200_ERR_RANGE,
                         "%s: %s %d has f[%d]=%g", who, weighted ? "slot" : "problem", u, k, fp[k]);
        s.g.assign(K, 0.0);
        status[u] = 1;
        iterations[u] = 0;
        if (s.active.size() < 2 || maxiter < 1) status[u] = 0;     // nothing to solve: the gauge fixes f
        else work.push_back(u);
    }
    std::vector<Ask> asks;
    std::vector<int64_t> off;
    auto take = [&](BatchSolver& s, const double* o) {
        const int K = s.rows.K;
        s.S.assign(o, o + K);
        s.logS.assign(o + K, o + 2 * K);
        s.G.assign(o + 2 * K + 2, o + 2 * K + 2 + (size_t)K * K);
    };
    // the sums at the starting points
    for (int u : work) asks.push_back(Ask{u, sv[u].cur.data(), true});
    if (!work.empty()) MBAR_TRY(batch_run(b, kind, asks, false, off, &ms));
    {
        std::vector<int> next;
        for (size_t i = 0; i < work.size(); ++i) {
            const int u = work[i];
            const double* o = b->h_out + off[i];
            if (o[2 * sv[u].rows.K + 1] != 0.0) {
                status[u] = 2;
                continue;
            }
            take(sv[u], o);
            next.push_back(u);
        }
        work.swap(next);
    }
    // one launch per iteration: both candidates of every unit, with their second moments, so that the chosen one's
    // sums are the next iteration's sums at f
    while (!work.empty()) {
        asks.clear();
        std::vector<int> first(work.size());
        for (size_t i = 0; i < work.size(); ++i) {
            BatchSolver& s = sv[work[i]];
            step_gradient(s.rows, s.S.data(), s.g);
            step_sci(s.rows, s.cur, s.logS.data(), s.f_sci);
            s.haveNr = step_newton(s.rows, s.S.data(), s.G.data(), s.g, s.cur, gamma, s.A, s.rhs, s.f_nr);
            first[i] = (int)asks.size();
            asks.push_back(Ask{work[i], s.f_sci.data(), true});
            if (s.haveNr) asks.push_back(Ask{work[i], s.f_nr.data(), true});
        }
        MBAR_TRY(batch_run(b, kind, asks, false, off, &ms));
        b->lastIterations++;
        std::vector<int> next;
        for (size_t i = 0; i < work.size(); ++i) {
            const int u = work[i];
            BatchSolver& s = sv[u];
            const int K = s.rows.K;
            const double* oS = b->h_out + off[first[i]];
            const double* oN = s.haveNr ? b->h_out + off[first[i] + 1] : nullptr;
            bool finite = true;
            for (int k : s.active) finite = finite && std::isfinite(s.f_sci[k]);
            if (oS[2 * K + 1] != 0.0 || !finite) {
                status[u] = 2;              // the self-consistent candidate left the range this loop serves
                iterations[u] = s.r.iterations;
                continue;
            }
            std::vector<double> gtmp(K);
            const double gn_sci = step_gradient(s.rows, oS, gtmp);
            const bool nrOk = s.haveNr && oN[2 * K + 1] == 0.0;
            const double gn_nr = nrOk ? step_gradient(s.rows, oN, gtmp) : INFINITY;
            const int nrBefore = s.r.nr_iterations;
            const bool done = step_choose(s.rows, s.f_sci, s.f_nr, nrOk, gn_sci, gn_nr, tol, min_sc_iter, s.cur, s.r);
            take(s, s.r.nr_iterations > nrBefore ? oN : oS);
            iterations[u] = s.r.iterations;
            if (done) status[u] = 0;
            else if (s.r.iterations < maxiter) next.push_back(u);
        }
        work.swap(next);
    }
    for (int u = 0; u < U; ++u) {
        double* fp = f + foff[u];
        for (int k : sv[u].active) fp[k] = sv[u].cur[k];
    }
    b->lastMs = ms;
    return MBAR_B200_OK;
}

// The moments of mbar_b200_batch_moments (ids name problems), mbar_b200_batch_replicate_moments (ids name slots),
// mbar_b200_batch_augmented_moments (ids name problems with appended rows) or
// mbar_b200_batch_replicate_augmented_moments (ids name slots whose problems hold appended rows), unpacked into the
// caller's arrays.
static int batch_moments_call(mbar_b200_batch* b, Units kind, int32_t n, const int32_t* ids, const double* f,
                              int32_t all_rows, double* S, double* logS, double* sumL, int32_t* flag, double* G,
                              const char* who) {
    MBAR_REQUIRE(b, MBAR_B200_ERR_INVALID, "%s: NULL object", who);
    MBAR_REQUIRE(n >= 1 && ids && f, MBAR_B200_ERR_INVALID, "%s: %d requests", who, (int)n);
    const int U = units_weighted(kind) ? b->nSlots : b->P;
    std::vector<Ask> asks((size_t)n);
    int64_t fo = 0;
    for (int r = 0; r < n; ++r) {
        const int id = ids[r];
        MBAR_REQUIRE(id >= 0 && id < U, MBAR_B200_ERR_INVALID, "%s: request %d names %s %d of %d", who, r,
                     units_weighted(kind) ? "slot" : "problem", id, U);
        const int p = unit_problem(b, kind, id);
        MBAR_REQUIRE(!units_appended(kind) || (p < (int)b->M.size() && b->M[p] > 0), MBAR_B200_ERR_INVALID,
                     "%s: request %d names %s %d of problem %d, which holds no appended rows", who, r,
                     units_weighted(kind) ? "slot" : "problem", id, p);
        asks[r] = Ask{id, f + fo, G != nullptr};
        fo += unit_rows(b, kind, id);
    }
    MBAR_CUDA(cudaSetDevice(b->device));
    b->lastLaunches = 0;
    b->lastBytes = 0;
    b->lastIterations = 0;
    double ms = 0.0;
    std::vector<int64_t> off;
    MBAR_TRY(batch_run(b, kind, asks, all_rows != 0, off, &ms));
    b->lastMs = ms;
    int64_t ko = 0, go = 0;
    for (int r = 0; r < n; ++r) {
        const int R = unit_rows(b, kind, asks[r].id);
        const double* o = b->h_out + off[r];
        if (S) std::memcpy(S + ko, o, R * sizeof(double));
        if (logS) std::memcpy(logS + ko, o + R, R * sizeof(double));
        if (sumL) sumL[r] = o[2 * R];
        if (flag) flag[r] = o[2 * R + 1] != 0.0;
        if (G) std::memcpy(G + go, o + 2 * R + 2, (size_t)R * R * sizeof(double));
        ko += R;
        go += (int64_t)R * R;
    }
    return MBAR_B200_OK;
}

// ---- histogram bin moments (DESIGN.md 3.5h) -------------------------------------------------------------------------
// A request names a problem p, its converged f [K_p], a target state's u_n [N_p] and dense bin indices bin_n [N_p] in
// [0, nbins).  With the shifted tiles u'_kn = u_kn - x_n,
//   L'_n = log sum_{k sampled} N_k e^{f_k - u'_kn},   log w_n = -(u_n - x_n) - L'_n   (= -u_n - L_n)
//   f_i  = -log sum_{n in i} w_n,   C_ki = sum_{n in i} W_nk w^_n,   D_i = sum_{n in i} w^_n^2,
//   W_nk = e^{f_k - u'_kn - L'_n} (every row),   w^_n = e^{log w_n + f_i}
// as mbar_b200_bin_moments gives them on one context.  Five kernels (seven with C and D), all requests in each:
//   1. batch_bin_prep_kernel: L'_n and log w_n per sample, each bin's maximum m_i by an atomic max on the
//      order-preserving key (a maximum does not depend on order);
//   2. batch_bin_max_kernel: m_i from the keys;
//   3. batch_bin_accum_kernel<false> + batch_bin_reduce_kernel<false>: s_i = sum_{n in i} e^{log w_n - m_i};
//   4. batch_bin_f_kernel: f_i = -(m_i + log s_i);
//   5. batch_bin_accum_kernel<true> + batch_bin_reduce_kernel<true>: the K_p rows of C and the row of D.
// The accumulation is that of bins.cu (warp_groups): work items are (request, bin chunk, sample chunk); a CTA keeps a
// [rows x bin chunk] accumulator in shared memory, warps own disjoint rows, and the last lane of each group of equal
// bins adds the group's sum to its own cell.  Each sample chunk writes its block of partials, and the reduce kernel
// adds them in chunk order.  The chunking is a function of (N_p, K_p, nbins) alone, there are no floating-point
// atomics, so a request's results are the same bits whichever requests share the call.
constexpr int BB_THREADS = 256;
constexpr int BB_WARPS = BB_THREADS / 32;
constexpr int BB_MAX_RW = (BATCH_MAX_K + 1 + BB_WARPS - 1) / BB_WARPS;   // rows per warp at K_p + 1 = 65 rows
constexpr int BB_ACC_DOUBLES = (108 * 1024) / 8;    // shared accumulator per CTA: two CTAs per SM, as bins.cu
constexpr int64_t BB_MIN_TILES = 64;                // a sample chunk holds at least 2048 samples ...
constexpr int64_t BB_MAX_CHUNKS = 64;               // ... a request at most 64 sample chunks ...
constexpr int64_t BB_PARTIAL_BYTES = 4 << 20;       // ... and at most 4 MB of partials (one chunk at least)
constexpr double BB_MAX_ARG = 700.0;                // range contract of the W_nk and w^_n exponents

// one pass's work items of a request: bin chunks of BC bins, sample chunks of ct tiles
struct BinGeo {
    int64_t item0;    // first (request, bin chunk, sample chunk) item
    int64_t poff;     // first double of the request's partials [nsc][rows][nbins]
    int64_t ct;       // tiles per sample chunk
    int32_t BC, nbc, nsc;
};

static BinGeo bin_geometry(int64_t nT, int rows, int nbins) {
    BinGeo g{};
    g.BC = std::min(nbins, BB_ACC_DOUBLES / rows);
    g.nbc = (nbins + g.BC - 1) / g.BC;
    const int64_t cap = std::max<int64_t>(1, BB_PARTIAL_BYTES / ((int64_t)rows * nbins * 8));
    const int64_t nsc = std::min(std::min((nT + BB_MIN_TILES - 1) / BB_MIN_TILES, BB_MAX_CHUNKS), cap);
    g.ct = (nT + nsc - 1) / nsc;
    g.nsc = (int32_t)((nT + g.ct - 1) / g.ct);
    return g;
}

struct BinReq {
    int64_t uoff;     // first double of the problem's tiles
    int64_t xoff;     // first x_n of the problem
    int64_t soff;     // first sample slot of the request (u_n -> log w_n, L'_n, bin index; nT_p * 32 slots)
    int64_t N, nT;
    int64_t boff;     // first bin of the request (keys, m, o, s, f_bin)
    int64_t ooff;     // first entry of the request's [K_p + 1][nbins] C and D
    int64_t foff;     // first entry of the request's f
    int64_t voff;     // first entry of the problem's K-vectors (N_k, log N_k)
    int32_t K, nbins;
    BinGeo geo[2];    // 0: the bin sums (one row), 1: C and D (K_p + 1 rows)
};

// L'_n = log sum_{k sampled} e^{f_k + log N_k - u'_kn} of sample n < N_p of request q (per-sample max shift)
__device__ __forceinline__ double bin_log_denominator(const double* __restrict__ u, const BinReq& q, int64_t n,
                                                      const double* __restrict__ fAll,
                                                      const double* __restrict__ NkAll,
                                                      const double* __restrict__ logNkAll) {
    const double* ut = u + q.uoff + (n >> 5) * (int64_t)q.K * 32 + (n & 31);
    const double* f = fAll + q.foff;
    const double* Nk = NkAll + q.voff;
    const double* logNk = logNkAll + q.voff;
    double m = -INFINITY;
    for (int k = 0; k < q.K; ++k)
        if (Nk[k] > 0.0) m = fmax(m, f[k] + logNk[k] - __ldg(ut + k * 32));
    double D = 0.0;
    for (int k = 0; k < q.K; ++k)
        if (Nk[k] > 0.0) D += exp(f[k] + logNk[k] - __ldg(ut + k * 32) - m);
    return m + log(D);
}

// lw [slots]: u_n on entry (+inf past N_p), log w_n on exit (-inf past N_p and where u_n = +inf); Lp [slots]: L'_n.
// A NaN log w_n (a sample whose sampled energies are all +inf) flags its request.
__global__ void __launch_bounds__(256) batch_bin_prep_kernel(const double* __restrict__ u,
                                                             const BinReq* __restrict__ req, int nReq, int64_t slots,
                                                             const double* __restrict__ fAll,
                                                             const double* __restrict__ NkAll,
                                                             const double* __restrict__ logNkAll,
                                                             const double* __restrict__ x, const int* __restrict__ bin,
                                                             double* __restrict__ lw, double* __restrict__ Lp,
                                                             unsigned long long* __restrict__ keys,
                                                             int* __restrict__ rflag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= slots) return;
    const int r = find_segment(nReq, i, [&](int s) { return req[s].soff; });
    const BinReq& q = req[r];
    const int64_t n = i - q.soff;
    if (n >= q.N) {
        lw[i] = -INFINITY;
        Lp[i] = 0.0;
        return;
    }
    const double L = bin_log_denominator(u, q, n, fAll, NkAll, logNkAll);
    const double un = lw[i];
    // u_n = +inf: weight exactly 0, as np.exp(-inf) in the reference
    const double v = un < INFINITY ? -(un - x[q.xoff + n]) - L : -INFINITY;
    Lp[i] = L;
    lw[i] = v;
    if (v != v) atomicOr(&rflag[r], 1);
    const unsigned long long key = ordered_key(v);
    unsigned long long* kb = keys + q.boff + bin[i];
    if (v > -INFINITY && key > *((volatile unsigned long long*)kb)) atomicMax(kb, key);
}

// Target-state log weights (mbar_b200_batch_log_weights, DESIGN.md 3.5h''): batch_bin_prep_kernel's log w_n, without
// bins.  lw [slots]: u_n on entry (+inf past N_p), log w_n on exit (samples past N_p are left as they are).  A NaN
// log w_n flags its request.
__global__ void __launch_bounds__(256) batch_log_weights_kernel(const double* __restrict__ u,
                                                                const BinReq* __restrict__ req, int nReq, int64_t slots,
                                                                const double* __restrict__ fAll,
                                                                const double* __restrict__ NkAll,
                                                                const double* __restrict__ logNkAll,
                                                                const double* __restrict__ x, double* __restrict__ lw,
                                                                int* __restrict__ rflag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= slots) return;
    const int r = find_segment(nReq, i, [&](int s) { return req[s].soff; });
    const BinReq& q = req[r];
    const int64_t n = i - q.soff;
    if (n >= q.N) return;
    const double L = bin_log_denominator(u, q, n, fAll, NkAll, logNkAll);
    const double un = lw[i];
    const double v = un < INFINITY ? -(un - x[q.xoff + n]) - L : -INFINITY;
    lw[i] = v;
    if (v != v) atomicOr(&rflag[r], 1);
}

// The replicate part of a weighted request (mbar_b200_batch_replicate_bin_moments): its target's first sample in the
// per-target u_n and bin index arrays, and its slot's first count.
struct RepBinReq {
    int64_t toff;
    int64_t coff;
};

// batch_bin_prep_kernel for replicate slots.  u_n and the bin index come from the request's target (uploaded once per
// target); lw, Lp and bin [slots] are the request's own.  A drawn sample (c_n > 0) gets
// log w_n + log c_n (c_n = 1 adds nothing, so all-ones counts give the unweighted bits) and its bin index; an undrawn
// one, like the padding, gets lw = -inf and bin -1, so that it enters no maximum and no sum and its L'_n is neither
// computed nor able to flag the request.
__global__ void __launch_bounds__(256) batch_rep_bin_prep_kernel(const double* __restrict__ u,
                                                                 const BinReq* __restrict__ req,
                                                                 const RepBinReq* __restrict__ rreq, int nReq,
                                                                 int64_t slots, const double* __restrict__ fAll,
                                                                 const double* __restrict__ NkAll,
                                                                 const double* __restrict__ logNkAll,
                                                                 const double* __restrict__ x,
                                                                 const uint16_t* __restrict__ counts,
                                                                 const double* __restrict__ ut,
                                                                 const int* __restrict__ bt, double* __restrict__ lw,
                                                                 double* __restrict__ Lp, int* __restrict__ bin,
                                                                 unsigned long long* __restrict__ keys,
                                                                 int* __restrict__ rflag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= slots) return;
    const int r = find_segment(nReq, i, [&](int s) { return req[s].soff; });
    const BinReq& q = req[r];
    const RepBinReq& w = rreq[r];
    const int64_t n = i - q.soff;
    const int c = counts[w.coff + n];                   // 0 past N_p: the slot's counts are padded to the tiles
    if (c == 0) {
        lw[i] = -INFINITY;
        Lp[i] = 0.0;
        bin[i] = -1;
        return;
    }
    const double L = bin_log_denominator(u, q, n, fAll, NkAll, logNkAll);
    const double un = ut[w.toff + n];
    double v = un < INFINITY ? -(un - x[q.xoff + n]) - L : -INFINITY;
    if (c != 1) v += log((double)c);
    const int b = bt[w.toff + n];
    Lp[i] = L;
    lw[i] = v;
    bin[i] = b;
    if (v != v) atomicOr(&rflag[r], 1);
    const unsigned long long key = ordered_key(v);
    unsigned long long* kb = keys + q.boff + b;
    if (v > -INFINITY && key > *((volatile unsigned long long*)kb)) atomicMax(kb, key);
}

// m_i from the keys, o = -m_i (the offset of the bin-sum pass).  A bin without a finite maximum (no sample, every
// u_n = +inf, or a u_n = -inf) flags its request.
__global__ void batch_bin_max_kernel(const BinReq* __restrict__ req, int nReq, int64_t bins,
                                     const unsigned long long* __restrict__ keys, double* __restrict__ m,
                                     double* __restrict__ o, int* __restrict__ rflag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= bins) return;
    const double v = ordered_value(keys[i]);
    if (!isfinite(v)) atomicOr(&rflag[find_segment(nReq, i, [&](int s) { return req[s].boff; })], 1);
    m[i] = v;
    o[i] = -v;
}

// f_i = -(m_i + log s_i), o = f_i (the offset of the moments pass)
__global__ void batch_bin_f_kernel(const BinReq* __restrict__ req, int nReq, int64_t bins,
                                   const double* __restrict__ m, const double* __restrict__ s,
                                   double* __restrict__ fbin, double* __restrict__ o, int* __restrict__ rflag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= bins) return;
    const double fb = -(m[i] + log(s[i]));
    if (!isfinite(fb)) atomicOr(&rflag[find_segment(nReq, i, [&](int r) { return req[r].boff; })], 1);
    fbin[i] = fb;
    o[i] = fb;
}

// One CTA per (request, bin chunk, sample chunk) item.  MOM = false: one row of ones against e^{log w_n - m_i} (the bin
// sums); MOM = true: the K_p rows of W_nk and one row of w^_n against w^_n (C and D).
template <bool MOM>
__global__ void __launch_bounds__(BB_THREADS, 2) batch_bin_accum_kernel(
    const double* __restrict__ u, const BinReq* __restrict__ req, int nReq, const double* __restrict__ fAll,
    const double* __restrict__ lw, const double* __restrict__ Lp, const int* __restrict__ bin,
    const double* __restrict__ o, double* __restrict__ part, int* __restrict__ rflag) {
    extern __shared__ double acc[];                     // [rows][BC]
    __shared__ int perm[BB_WARPS][32];
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int r = find_segment(nReq, blockIdx.x, [&](int s) { return req[s].geo[MOM].item0; });
    const BinReq& q = req[r];
    const BinGeo g = q.geo[MOM];
    const int64_t local = blockIdx.x - g.item0;
    const int sc = (int)(local % g.nsc), bc = (int)(local / g.nsc);
    const int K = q.K, nbins = q.nbins;
    const int Kw = MOM ? K : 0, rows = Kw + 1;
    const int b0 = bc * g.BC, bw = min(g.BC, nbins - b0);
    for (int i = threadIdx.x; i < rows * g.BC; i += BB_THREADS) acc[i] = 0.0;
    __syncthreads();
    const int myRows = (warp < rows) ? (rows - 1 - warp) / BB_WARPS + 1 : 0;   // rows warp, warp + 8, ...
    const int64_t t0 = (int64_t)sc * g.ct, t1 = min(q.nT, t0 + g.ct);
    const double* f = fAll + q.foff;
    const double* ob = o + q.boff;
    bool range = false;
    for (int64_t t = t0; t < t1 && myRows > 0; ++t) {
        const int64_t i = q.soff + t * 32 + lane;
        const int b = bin[i];
        if (!__any_sync(FULL, b >= b0 && b < b0 + bw)) continue;
        // this tile's energies first, so that the loads of all rows are in flight together
        const double* tp = u + q.uoff + t * (int64_t)K * 32 + lane;
        double uu[BB_MAX_RW];
#pragma unroll
        for (int j = 0; j < BB_MAX_RW; ++j) {
            const int rl = warp + BB_WARPS * j;
            uu[j] = (j < myRows && rl < Kw) ? __ldg(tp + rl * 32) : 0.0;
        }
        const double L = Lp[i];
        const double eo = (b >= 0) ? lw[i] + ob[b] : -INFINITY;
        if (eo > BB_MAX_ARG) range = true;
        const double e0 = exp(eo);                      // w^_n (moments) | e^{log w_n - m_i} (bin sums)
        const double aux = MOM ? e0 : 1.0;
        const WarpGroups grp = warp_groups(b, perm[warp]);
        const int col = (grp.tail && grp.key >= b0 && grp.key < b0 + bw) ? grp.key - b0 : -1;
#pragma unroll
        for (int j = 0; j < BB_MAX_RW; ++j) {
            const int rl = warp + BB_WARPS * j;
            if (j >= myRows) continue;                  // warp-uniform
            double a = aux;
            if (rl < Kw) {
                // +inf energies (and the padding past N_p) have weight exactly 0
                const double e = f[rl] - uu[j] - L;
                if (b >= 0 && e > BB_MAX_ARG) range = true;
                a = exp(e);
            }
            if (b < 0) a = 0.0;
            const double v = warp_group_sum(grp, a * e0);
            if (col >= 0) acc[rl * g.BC + col] += v;
        }
        __syncwarp();
    }
    if (range) atomicOr(&rflag[r], 1);
    __syncthreads();
    double* dst = part + g.poff + (int64_t)sc * rows * nbins + b0;
    for (int i = threadIdx.x; i < rows * bw; i += BB_THREADS) {
        const int rl = i / bw, c = i - rl * bw;
        dst[(int64_t)rl * nbins + c] = acc[rl * g.BC + c];
    }
}

// out[i] over every request's [rows][nbins] entries (MOM = false: the bin sums at boff; true: C and D at ooff): the
// sum over the request's sample chunks, in chunk order
template <bool MOM>
__global__ void batch_bin_reduce_kernel(const BinReq* __restrict__ req, int nReq, int64_t total,
                                        const double* __restrict__ part, double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const BinReq& q = req[find_segment(nReq, i, [&](int s) { return MOM ? req[s].ooff : req[s].boff; })];
    const BinGeo& g = q.geo[MOM];
    const int rows = MOM ? q.K + 1 : 1;
    const int64_t e = i - (MOM ? q.ooff : q.boff);    // row * nbins + bin
    double s = 0.0;
    for (int c = 0; c < g.nsc; ++c) s += part[g.poff + (int64_t)c * rows * q.nbins + e];
    out[i] = s;
}

}  // namespace mbar

using namespace mbar;

int mbar_b200_batch_create(int device, int32_t n_problems, const int32_t* K, const int64_t* N, const double* N_k,
                           const double* u, mbar_b200_batch** out) {
    MBAR_REQUIRE(out && K && N && N_k && u, MBAR_B200_ERR_INVALID, "batch_create: NULL argument");
    *out = nullptr;
    MBAR_REQUIRE(n_problems >= 1, MBAR_B200_ERR_INVALID, "batch_create: %d problems", (int)n_problems);
    std::unique_ptr<mbar_b200_batch> o(new mbar_b200_batch());
    o->P = n_problems;
    int64_t rawTotal = 0, vTotal = 0, tiles = 0;
    std::vector<BatchProbDev> pr((size_t)n_problems);
    for (int p = 0; p < n_problems; ++p) {
        MBAR_REQUIRE(K[p] >= 1 && K[p] <= BATCH_MAX_K, MBAR_B200_ERR_INVALID,
                     "batch_create: problem %d has K=%d states (1 to %d)", p, (int)K[p], BATCH_MAX_K);
        MBAR_REQUIRE(N[p] >= 1 && N[p] < (int64_t(1) << 36), MBAR_B200_ERR_INVALID,
                     "batch_create: problem %d has N=%lld samples", p, (long long)N[p]);
        bool any = false;
        for (int k = 0; k < K[p]; ++k) {
            const double n = N_k[vTotal + k];
            MBAR_REQUIRE(n >= 0.0 && n < INFINITY, MBAR_B200_ERR_INVALID, "batch_create: problem %d has N_k[%d]=%g", p,
                         k, n);
            any = any || n > 0.0;
        }
        MBAR_REQUIRE(any, MBAR_B200_ERR_INVALID, "batch_create: problem %d has no sampled state", p);
        const int64_t nT = (N[p] + 31) / 32;
        o->K.push_back(K[p]);
        o->N.push_back(N[p]);
        o->nT.push_back(nT);
        o->uoff.push_back(o->uTotal);
        o->voff.push_back(vTotal);
        pr[p] = BatchProbDev{rawTotal, o->uTotal, tiles, N[p], vTotal, K[p]};
        rawTotal += (int64_t)K[p] * N[p];
        o->uTotal += nT * 32 * K[p];
        vTotal += K[p];
        tiles += nT;
    }
    o->Nk.assign(N_k, N_k + vTotal);
    std::vector<double> logNk((size_t)vTotal);
    for (int64_t i = 0; i < vTotal; ++i) logNk[i] = o->Nk[i] > 0.0 ? std::log(o->Nk[i]) : -INFINITY;
    MBAR_TRY(open_device(device, nullptr));
    MBAR_TRY(o->open(device, "batch_create"));
    NvtxRange nvtx_("mbar_b200::batch_create");
    MBAR_TRY(o->upload(o->d_Nk, o->Nk.data(), (size_t)vTotal, "batch_create"));
    MBAR_TRY(o->upload(o->d_logNk, logNk.data(), (size_t)vTotal, "batch_create"));
    MBAR_TRY(o->d_u.reserve((size_t)o->uTotal, "batch_create (tiles)"));
    MBAR_TRY(o->d_sumx.reserve((size_t)n_problems, "batch_create"));
    MBAR_TRY(o->d_x.reserve((size_t)tiles * 32, "batch_create (x_n)"));
    MBAR_TRY(o->upload(o->d_prob, pr.data(), pr.size(), "batch_create"));
    {
        CallBuffers cb("batch_create (staging)");
        double* raw = nullptr;
        unsigned int* bad = nullptr;
        MBAR_TRY(cb.alloc(&raw, (size_t)rawTotal));
        MBAR_TRY(cb.alloc(&bad, 1));
        MBAR_CUDA(cudaMemcpyAsync(raw, u, (size_t)rawTotal * sizeof(double), cudaMemcpyHostToDevice, o->stream));
        MBAR_CUDA(cudaMemsetAsync(bad, 0, sizeof(unsigned int), o->stream));
        batch_retile_kernel<<<(unsigned)((tiles + 7) / 8), 256, 0, o->stream>>>(raw, o->d_prob, n_problems, tiles,
                                                                               o->d_Nk, o->d_u, o->d_x, bad);
        batch_sumx_kernel<false><<<(unsigned)n_problems, 256, 0, o->stream>>>(o->d_x, o->d_prob, nullptr, nullptr,
                                                                               nullptr, o->d_sumx);
        MBAR_CUDA(cudaGetLastError());
        unsigned int hbad = 0;
        MBAR_CUDA(cudaMemcpyAsync(&hbad, bad, sizeof(hbad), cudaMemcpyDeviceToHost, o->stream));
        MBAR_CUDA(cudaStreamSynchronize(o->stream));
        MBAR_REQUIRE(hbad == 0, MBAR_B200_ERR_NAN, "batch_create: %u samples hold NaN or -inf energies", hbad);
    }
    *out = o.release();
    return MBAR_B200_OK;
}

int mbar_b200_batch_destroy(mbar_b200_batch* b) { return destroy_resident(b); }

int mbar_b200_batch_moments(mbar_b200_batch* b, int32_t n_requests, const int32_t* problem, const double* f,
                            int32_t all_rows, double* S, double* logS, double* sumL, int32_t* flag, double* G) {
    NvtxRange nvtx_("mbar_b200::batch_moments");
    return batch_moments_call(b, Units::problems, n_requests, problem, f, all_rows, S, logS, sumL, flag, G,
                              "batch_moments");
}

int mbar_b200_batch_solve(mbar_b200_batch* b, double* f, double tol, int32_t maxiter, int32_t min_sc_iter,
                          double gamma, int32_t* status, int32_t* iterations) {
    MBAR_REQUIRE(b && f && status && iterations, MBAR_B200_ERR_INVALID, "batch_solve: NULL argument");
    NvtxRange nvtx_("mbar_b200::batch_solve");
    return batch_solve_units(b, false, f, tol, maxiter, min_sc_iter, gamma, status, iterations, "batch_solve");
}

int mbar_b200_batch_set_replicates(mbar_b200_batch* b, int32_t n_slots, const int32_t* problem,
                                   const uint16_t* counts) {
    MBAR_REQUIRE(b, MBAR_B200_ERR_INVALID, "batch_set_replicates: NULL object");
    b->nSlots = 0;                            // a failed call leaves no slot
    MBAR_REQUIRE(n_slots >= 0 && (n_slots == 0 || (problem && counts)), MBAR_B200_ERR_INVALID,
                 "batch_set_replicates: %d slots", (int)n_slots);
    std::vector<int64_t> coff((size_t)n_slots);
    int64_t padded = 0, src = 0;
    for (int s = 0; s < n_slots; ++s) {
        const int p = problem[s];
        MBAR_REQUIRE(p >= 0 && p < b->P, MBAR_B200_ERR_INVALID, "batch_set_replicates: slot %d names problem %d of %d",
                     s, p, b->P);
        int64_t sum = 0;
        for (int64_t n = 0; n < b->N[p]; ++n) sum += counts[src + n];
        MBAR_REQUIRE(sum == b->N[p], MBAR_B200_ERR_INVALID,
                     "batch_set_replicates: slot %d counts sum to %lld, problem %d has %lld samples", s,
                     (long long)sum, p, (long long)b->N[p]);
        coff[s] = padded;
        padded += b->nT[p] * 32;
        src += b->N[p];
    }
    MBAR_CUDA(cudaSetDevice(b->device));
    NvtxRange nvtx_("mbar_b200::batch_set_replicates");
    b->slotProb.assign(problem, problem + n_slots);
    b->slotCoff = coff;
    if (n_slots == 0) return MBAR_B200_OK;
    std::vector<uint16_t> hc((size_t)padded, 0);
    src = 0;
    for (int s = 0; s < n_slots; ++s) {
        const int64_t N = b->N[problem[s]];
        std::memcpy(hc.data() + coff[s], counts + src, (size_t)N * sizeof(uint16_t));
        src += N;
    }
    MBAR_TRY(b->upload(b->d_counts, hc.data(), hc.size(), "batch_set_replicates (counts)"));
    MBAR_TRY(b->upload(b->d_slotCoff, coff.data(), coff.size(), "batch_set_replicates"));
    MBAR_TRY(b->upload(b->d_slotProb, problem, (size_t)n_slots, "batch_set_replicates"));
    MBAR_TRY(b->d_sumxw.reserve((size_t)n_slots, "batch_set_replicates"));
    batch_sumx_kernel<true><<<(unsigned)n_slots, 256, 0, b->stream>>>(b->d_x, b->d_prob, b->d_slotProb, b->d_slotCoff,
                                                                       b->d_counts, b->d_sumxw);
    MBAR_CUDA(cudaGetLastError());
    MBAR_CUDA(cudaStreamSynchronize(b->stream));
    b->nSlots = n_slots;
    return MBAR_B200_OK;
}

int mbar_b200_batch_replicate_moments(mbar_b200_batch* b, int32_t n_requests, const int32_t* slot, const double* f,
                                      int32_t all_rows, double* S, double* logS, double* sumL, int32_t* flag,
                                      double* G) {
    NvtxRange nvtx_("mbar_b200::batch_replicate_moments");
    return batch_moments_call(b, Units::slots, n_requests, slot, f, all_rows, S, logS, sumL, flag, G,
                              "batch_replicate_moments");
}

int mbar_b200_batch_solve_replicates(mbar_b200_batch* b, double* f, double tol, int32_t maxiter,
                                     int32_t min_sc_iter, double gamma, int32_t* status, int32_t* iterations) {
    MBAR_REQUIRE(b && f && status && iterations, MBAR_B200_ERR_INVALID, "batch_solve_replicates: NULL argument");
    NvtxRange nvtx_("mbar_b200::batch_solve_replicates");
    return batch_solve_units(b, true, f, tol, maxiter, min_sc_iter, gamma, status, iterations,
                             "batch_solve_replicates");
}

int mbar_b200_batch_set_unsampled(mbar_b200_batch* b, int32_t n, const int32_t* problem, const int32_t* M,
                                  const double* rows) {
    MBAR_REQUIRE(b, MBAR_B200_ERR_INVALID, "batch_set_unsampled: NULL object");
    b->M.assign((size_t)b->P, 0);             // a failed call leaves no appended rows
    b->aoff.assign((size_t)b->P, 0);
    MBAR_REQUIRE(n >= 0 && (n == 0 || (problem && M && rows)), MBAR_B200_ERR_INVALID,
                 "batch_set_unsampled: %d problems", (int)n);
    std::vector<AugProbDev> pr((size_t)n);
    std::vector<char> seen((size_t)b->P, 0);
    std::vector<int64_t> tile0((size_t)b->P, 0);  // first tile of each problem: indexes x_n
    for (int p = 1; p < b->P; ++p) tile0[p] = tile0[p - 1] + b->nT[p - 1];
    int64_t raw = 0, total = 0, tiles = 0;
    for (int i = 0; i < n; ++i) {
        const int p = problem[i];
        MBAR_REQUIRE(p >= 0 && p < b->P && !seen[p], MBAR_B200_ERR_INVALID,
                     "batch_set_unsampled: entry %d names problem %d of %d%s", i, p, b->P,
                     p >= 0 && p < b->P ? " twice" : "");
        seen[p] = 1;
        MBAR_REQUIRE(M[i] >= 1 && b->K[p] + M[i] <= AUG_MAX_R, MBAR_B200_ERR_INVALID,
                     "batch_set_unsampled: problem %d has K=%d states and M=%d appended rows (K + M: at most %d)", p,
                     b->K[p], (int)M[i], AUG_MAX_R);
        pr[i] = AugProbDev{raw, total, tile0[p], tiles, b->N[p], M[i]};
        raw += (int64_t)M[i] * b->N[p];
        total += b->nT[p] * 32 * M[i];
        tiles += b->nT[p];
    }
    int64_t bad = 0;
    for (int64_t j = 0; j < raw; ++j) bad += rows[j] != rows[j] || rows[j] == -INFINITY;
    MBAR_REQUIRE(bad == 0, MBAR_B200_ERR_NAN, "batch_set_unsampled: %lld appended energies are NaN or -inf",
                 (long long)bad);
    if (n == 0) return MBAR_B200_OK;
    MBAR_CUDA(cudaSetDevice(b->device));
    NvtxRange nvtx_("mbar_b200::batch_set_unsampled");
    MBAR_TRY(b->d_ua.reserve((size_t)total, "batch_set_unsampled (appended tiles)"));
    {
        CallBuffers cb("batch_set_unsampled (staging)");
        double* draw = nullptr;
        AugProbDev* dpr = nullptr;
        MBAR_TRY(cb.alloc(&draw, (size_t)raw));
        MBAR_TRY(cb.alloc(&dpr, pr.size()));
        MBAR_CUDA(cudaMemcpyAsync(draw, rows, (size_t)raw * sizeof(double), cudaMemcpyHostToDevice, b->stream));
        MBAR_CUDA(cudaMemcpyAsync(dpr, pr.data(), pr.size() * sizeof(AugProbDev), cudaMemcpyHostToDevice, b->stream));
        batch_aug_retile_kernel<<<(unsigned)((tiles + 7) / 8), 256, 0, b->stream>>>(draw, dpr, n, tiles, b->d_x,
                                                                                    b->d_ua);
        MBAR_CUDA(cudaGetLastError());
        MBAR_CUDA(cudaStreamSynchronize(b->stream));
    }
    for (int i = 0; i < n; ++i) {
        b->M[problem[i]] = M[i];
        b->aoff[problem[i]] = pr[i].aoff;
    }
    return MBAR_B200_OK;
}

int mbar_b200_batch_augmented_moments(mbar_b200_batch* b, int32_t n_requests, const int32_t* problem,
                                      const double* f, double* S, double* logS, double* sumL, int32_t* flag,
                                      double* G) {
    NvtxRange nvtx_("mbar_b200::batch_augmented_moments");
    return batch_moments_call(b, Units::appended, n_requests, problem, f, 1, S, logS, sumL, flag, G,
                              "batch_augmented_moments");
}

int mbar_b200_batch_replicate_augmented_moments(mbar_b200_batch* b, int32_t n_requests, const int32_t* slot,
                                                const double* f, double* S, double* logS, double* sumL,
                                                int32_t* flag) {
    NvtxRange nvtx_("mbar_b200::batch_replicate_augmented_moments");
    return batch_moments_call(b, Units::slot_appended, n_requests, slot, f, 1, S, logS, sumL, flag, nullptr,
                              "batch_replicate_augmented_moments");
}

int mbar_b200_batch_bin_moments(mbar_b200_batch* b, int32_t n, const int32_t* problem, const double* f,
                                const double* u_n, const int32_t* bin_n, const int32_t* nbins, double* f_bin,
                                double* C, double* D, int32_t* flag) {
    MBAR_REQUIRE(b, MBAR_B200_ERR_INVALID, "batch_bin_moments: NULL object");
    MBAR_REQUIRE(n >= 1 && problem && f && u_n && bin_n && nbins && f_bin && flag, MBAR_B200_ERR_INVALID,
                 "batch_bin_moments: %d requests or a NULL argument", (int)n);
    const bool wantC = C || D;
    std::vector<BinReq> req((size_t)n);
    std::vector<int64_t> tile0((size_t)b->P, 0);  // first tile of each problem: indexes x_n
    for (int p = 1; p < b->P; ++p) tile0[p] = tile0[p - 1] + b->nT[p - 1];
    int64_t slots = 0, bins = 0, outs = 0, fs = 0, items0 = 0, items1 = 0, parts0 = 0, parts1 = 0, bytes = 0, src = 0;
    size_t smem1 = 0;
    for (int r = 0; r < n; ++r) {
        const int p = problem[r];
        MBAR_REQUIRE(p >= 0 && p < b->P, MBAR_B200_ERR_INVALID, "batch_bin_moments: request %d names problem %d of %d",
                     r, p, b->P);
        MBAR_REQUIRE(nbins[r] >= 1, MBAR_B200_ERR_INVALID, "batch_bin_moments: request %d has nbins = %d", r,
                     (int)nbins[r]);
        BinReq& q = req[r];
        q.K = b->K[p];
        q.nbins = nbins[r];
        q.N = b->N[p];
        q.nT = b->nT[p];
        q.uoff = b->uoff[p];
        q.voff = b->voff[p];
        q.xoff = tile0[p] * 32;
        q.soff = slots;
        q.boff = bins;
        q.ooff = outs;
        q.foff = fs;
        for (int64_t i = 0; i < q.N; ++i)
            MBAR_REQUIRE(bin_n[src + i] >= 0 && bin_n[src + i] < q.nbins, MBAR_B200_ERR_INVALID,
                         "batch_bin_moments: request %d: bin index %d of sample %lld lies outside [0, %d)", r,
                         (int)bin_n[src + i], (long long)i, (int)q.nbins);
        src += q.N;
        for (int pass = 0; pass < 2; ++pass) {
            BinGeo& g = q.geo[pass];
            g = bin_geometry(q.nT, pass ? q.K + 1 : 1, q.nbins);
            int64_t& items = pass ? items1 : items0;
            int64_t& parts = pass ? parts1 : parts0;
            g.item0 = items;
            g.poff = parts;
            items += (int64_t)g.nbc * g.nsc;
            parts += (int64_t)g.nsc * (pass ? q.K + 1 : 1) * q.nbins;
        }
        smem1 = std::max(smem1, (size_t)(q.K + 1) * q.geo[1].BC * sizeof(double));
        bytes += q.nT * 32 * q.K * 8 * (1 + (wantC ? q.geo[1].nbc : 0));   // the prep pass, then C's bin chunks
        slots += q.nT * 32;
        bins += q.nbins;
        outs += (int64_t)(q.K + 1) * q.nbins;
        fs += q.K;
    }
    for (int64_t i = 0; i < src; ++i)
        MBAR_REQUIRE(u_n[i] == u_n[i], MBAR_B200_ERR_NAN, "batch_bin_moments: NaN in u_n (entry %lld)", (long long)i);
    MBAR_REQUIRE(items0 < INT32_MAX && items1 < INT32_MAX, MBAR_B200_ERR_INVALID,
                 "batch_bin_moments: %lld work items in one call", (long long)std::max(items0, items1));
    MBAR_CUDA(cudaSetDevice(b->device));
    NvtxRange nvtx_("mbar_b200::batch_bin_moments");
    b->lastLaunches = 0;
    b->lastBytes = 0;
    b->lastIterations = 0;
    // pinned staging: f, u_n padded with +inf to the tiles and the requests; the bin indices, padded with -1 (no bin)
    const size_t reqDoubles = ((size_t)n * sizeof(BinReq) + 7) / 8;
    MBAR_TRY(b->h_f.grow((size_t)fs + (size_t)slots + reqDoubles, "batch_bin_moments"));
    MBAR_TRY(b->h_bin.grow((size_t)slots, "batch_bin_moments"));
    double* hu = b->h_f + fs;
    src = 0;
    int64_t fo = 0;
    for (int r = 0; r < n; ++r) {
        const BinReq& q = req[r];
        std::memcpy(b->h_f + q.foff, f + fo, (size_t)q.K * sizeof(double));
        std::memcpy(hu + q.soff, u_n + src, (size_t)q.N * sizeof(double));
        std::memcpy(b->h_bin + q.soff, bin_n + src, (size_t)q.N * sizeof(int32_t));
        for (int64_t i = q.N; i < q.nT * 32; ++i) {
            hu[q.soff + i] = INFINITY;
            b->h_bin[q.soff + i] = -1;
        }
        src += q.N;
        fo += q.K;
    }
    BinReq* hreq = reinterpret_cast<BinReq*>(b->h_f + fs + slots);
    std::memcpy(hreq, req.data(), req.size() * sizeof(BinReq));
    CallBuffers buf("batch_bin_moments");
    BinReq* d_req;
    int *d_bin, *d_rflag;
    double *d_f, *d_lw, *d_Lp, *d_m, *d_o, *d_s, *d_fbin, *d_part, *d_out = nullptr;
    unsigned long long* d_keys;
    MBAR_TRY(buf.alloc(&d_req, (size_t)n));
    MBAR_TRY(buf.alloc(&d_f, (size_t)fs));
    MBAR_TRY(buf.alloc(&d_lw, (size_t)slots));
    MBAR_TRY(buf.alloc(&d_Lp, (size_t)slots));
    MBAR_TRY(buf.alloc(&d_bin, (size_t)slots));
    MBAR_TRY(buf.alloc(&d_keys, (size_t)bins));
    MBAR_TRY(buf.alloc(&d_m, (size_t)bins));
    MBAR_TRY(buf.alloc(&d_o, (size_t)bins));
    MBAR_TRY(buf.alloc(&d_s, (size_t)bins));
    MBAR_TRY(buf.alloc(&d_fbin, (size_t)bins));
    MBAR_TRY(buf.alloc(&d_part, (size_t)std::max(parts0, wantC ? parts1 : 0)));
    MBAR_TRY(buf.alloc(&d_rflag, (size_t)n));
    if (wantC) MBAR_TRY(buf.alloc(&d_out, (size_t)outs));
    cudaStream_t s = b->stream;
    MBAR_CUDA(cudaMemcpyAsync(d_f, b->h_f, (size_t)fs * sizeof(double), cudaMemcpyHostToDevice, s));
    MBAR_CUDA(cudaMemcpyAsync(d_lw, hu, (size_t)slots * sizeof(double), cudaMemcpyHostToDevice, s));
    MBAR_CUDA(cudaMemcpyAsync(d_bin, b->h_bin, (size_t)slots * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    MBAR_CUDA(cudaMemcpyAsync(d_req, hreq, req.size() * sizeof(BinReq), cudaMemcpyHostToDevice, s));
    MBAR_CUDA(cudaMemsetAsync(d_keys, 0, (size_t)bins * sizeof(unsigned long long), s));
    MBAR_CUDA(cudaMemsetAsync(d_rflag, 0, (size_t)n * sizeof(int), s));
    const size_t smem0 = (size_t)BB_ACC_DOUBLES * sizeof(double);
    MBAR_CUDA(cudaFuncSetAttribute(batch_bin_accum_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)smem0));
    MBAR_CUDA(cudaFuncSetAttribute(batch_bin_accum_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)smem0));
    // the largest shared-memory carveout, so that two CTAs with the largest accumulator share an SM
    MBAR_CUDA(cudaFuncSetAttribute(batch_bin_accum_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    MBAR_CUDA(cudaFuncSetAttribute(batch_bin_accum_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    size_t smemS = 0;
    for (const BinReq& q : req) smemS = std::max(smemS, (size_t)q.geo[0].BC * sizeof(double));
    MBAR_CUDA(cudaEventRecord(b->ev0, s));
    batch_bin_prep_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, s>>>(
        b->d_u, d_req, n, slots, d_f, b->d_Nk, b->d_logNk, b->d_x, d_bin, d_lw, d_Lp, d_keys, d_rflag);
    batch_bin_max_kernel<<<(unsigned)((bins + 255) / 256), 256, 0, s>>>(d_req, n, bins, d_keys, d_m, d_o, d_rflag);
    batch_bin_accum_kernel<false><<<(unsigned)items0, BB_THREADS, smemS, s>>>(b->d_u, d_req, n, d_f, d_lw, d_Lp, d_bin,
                                                                              d_o, d_part, d_rflag);
    batch_bin_reduce_kernel<false><<<(unsigned)((bins + 255) / 256), 256, 0, s>>>(d_req, n, bins, d_part, d_s);
    batch_bin_f_kernel<<<(unsigned)((bins + 255) / 256), 256, 0, s>>>(d_req, n, bins, d_m, d_s, d_fbin, d_o, d_rflag);
    b->lastLaunches = 5;
    if (wantC) {
        batch_bin_accum_kernel<true><<<(unsigned)items1, BB_THREADS, smem1, s>>>(b->d_u, d_req, n, d_f, d_lw, d_Lp,
                                                                                 d_bin, d_o, d_part, d_rflag);
        batch_bin_reduce_kernel<true><<<(unsigned)((outs + 255) / 256), 256, 0, s>>>(d_req, n, outs, d_part, d_out);
        b->lastLaunches += 2;
    }
    MBAR_CUDA(cudaGetLastError());
    MBAR_CUDA(cudaEventRecord(b->ev1, s));
    MBAR_TRY(b->h_out.grow((size_t)bins + (wantC ? (size_t)outs : 0), "batch_bin_moments"));
    std::vector<int> hflag((size_t)n);
    MBAR_CUDA(cudaMemcpyAsync(b->h_out, d_fbin, (size_t)bins * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (wantC)
        MBAR_CUDA(cudaMemcpyAsync(b->h_out + bins, d_out, (size_t)outs * sizeof(double), cudaMemcpyDeviceToHost, s));
    MBAR_CUDA(cudaMemcpyAsync(hflag.data(), d_rflag, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, s));
    MBAR_CUDA(cudaStreamSynchronize(s));
    float ms = 0.f;
    b->lastMs = event_ms(b->ev0, b->ev1, &ms) ? ms : 0.0;
    b->lastBytes = bytes;
    int64_t co = 0;
    for (int r = 0; r < n; ++r) {
        const BinReq& q = req[r];
        flag[r] = hflag[r] != 0;
        std::memcpy(f_bin + q.boff, b->h_out + q.boff, (size_t)q.nbins * sizeof(double));
        const double* o = b->h_out + bins + q.ooff;
        if (C) std::memcpy(C + co, o, (size_t)q.K * q.nbins * sizeof(double));
        if (D) std::memcpy(D + q.boff, o + (size_t)q.K * q.nbins, (size_t)q.nbins * sizeof(double));
        co += (int64_t)q.K * q.nbins;
    }
    return MBAR_B200_OK;
}

int mbar_b200_batch_replicate_bin_moments(mbar_b200_batch* b, int32_t n_targets, const int32_t* target_problem,
                                          const double* u_n, const int32_t* bin_n, const int32_t* nbins,
                                          int32_t n, const int32_t* slot, const int32_t* target, const double* f,
                                          double* f_bin, int32_t* flag) {
    MBAR_REQUIRE(b, MBAR_B200_ERR_INVALID, "batch_replicate_bin_moments: NULL object");
    MBAR_REQUIRE(n_targets >= 1 && target_problem && u_n && bin_n && nbins, MBAR_B200_ERR_INVALID,
                 "batch_replicate_bin_moments: %d targets or a NULL argument", (int)n_targets);
    MBAR_REQUIRE(n >= 1 && slot && target && f && f_bin && flag, MBAR_B200_ERR_INVALID,
                 "batch_replicate_bin_moments: %d requests or a NULL argument", (int)n);
    // targets: u_n and bin indices, each padded to its problem's tiles
    std::vector<int64_t> toff((size_t)n_targets);
    int64_t tslots = 0, src = 0;
    for (int t = 0; t < n_targets; ++t) {
        const int p = target_problem[t];
        MBAR_REQUIRE(p >= 0 && p < b->P, MBAR_B200_ERR_INVALID,
                     "batch_replicate_bin_moments: target %d names problem %d of %d", t, p, b->P);
        MBAR_REQUIRE(nbins[t] >= 1, MBAR_B200_ERR_INVALID, "batch_replicate_bin_moments: target %d has nbins = %d",
                     t, (int)nbins[t]);
        for (int64_t i = 0; i < b->N[p]; ++i)
            MBAR_REQUIRE(bin_n[src + i] >= 0 && bin_n[src + i] < nbins[t], MBAR_B200_ERR_INVALID,
                         "batch_replicate_bin_moments: target %d: bin index %d of sample %lld lies outside [0, %d)",
                         t, (int)bin_n[src + i], (long long)i, (int)nbins[t]);
        toff[t] = tslots;
        tslots += b->nT[p] * 32;
        src += b->N[p];
    }
    for (int64_t i = 0; i < src; ++i)
        MBAR_REQUIRE(u_n[i] == u_n[i], MBAR_B200_ERR_NAN, "batch_replicate_bin_moments: NaN in u_n (entry %lld)",
                     (long long)i);
    std::vector<BinReq> req((size_t)n);
    std::vector<RepBinReq> rreq((size_t)n);
    std::vector<int64_t> tile0((size_t)b->P, 0);  // first tile of each problem: indexes x_n
    for (int p = 1; p < b->P; ++p) tile0[p] = tile0[p - 1] + b->nT[p - 1];
    int64_t slots = 0, bins = 0, fs = 0, items = 0, parts = 0, bytes = 0;
    for (int r = 0; r < n; ++r) {
        const int s = slot[r], t = target[r];
        MBAR_REQUIRE(s >= 0 && s < b->nSlots, MBAR_B200_ERR_INVALID,
                     "batch_replicate_bin_moments: request %d names slot %d of %d", r, s, b->nSlots);
        MBAR_REQUIRE(t >= 0 && t < n_targets, MBAR_B200_ERR_INVALID,
                     "batch_replicate_bin_moments: request %d names target %d of %d", r, t, (int)n_targets);
        const int p = b->slotProb[s];
        MBAR_REQUIRE(target_problem[t] == p, MBAR_B200_ERR_INVALID,
                     "batch_replicate_bin_moments: request %d: slot %d is of problem %d, target %d of problem %d", r,
                     s, p, t, (int)target_problem[t]);
        BinReq& q = req[r];
        q = BinReq{};
        q.K = b->K[p];
        q.nbins = nbins[t];
        q.N = b->N[p];
        q.nT = b->nT[p];
        q.uoff = b->uoff[p];
        q.voff = b->voff[p];
        q.xoff = tile0[p] * 32;
        q.soff = slots;
        q.boff = bins;
        q.foff = fs;
        BinGeo& g = q.geo[0];
        g = bin_geometry(q.nT, 1, q.nbins);
        g.item0 = items;
        g.poff = parts;
        items += (int64_t)g.nbc * g.nsc;
        parts += (int64_t)g.nsc * q.nbins;
        rreq[r] = RepBinReq{toff[t], b->slotCoff[s]};
        bytes += q.nT * 32 * ((int64_t)q.K * 8 + 2);     // the prep pass: tiles and counts
        slots += q.nT * 32;
        bins += q.nbins;
        fs += q.K;
    }
    MBAR_REQUIRE(items < INT32_MAX, MBAR_B200_ERR_INVALID, "batch_replicate_bin_moments: %lld work items in one call",
                 (long long)items);
    MBAR_CUDA(cudaSetDevice(b->device));
    NvtxRange nvtx_("mbar_b200::batch_replicate_bin_moments");
    b->lastLaunches = 0;
    b->lastBytes = 0;
    b->lastIterations = 0;
    // pinned staging: f, the targets' u_n padded with +inf and the requests; the targets' bin indices padded with -1
    const size_t reqDoubles = ((size_t)n * sizeof(BinReq) + 7) / 8;
    const size_t rreqDoubles = ((size_t)n * sizeof(RepBinReq) + 7) / 8;
    MBAR_TRY(b->h_f.grow((size_t)fs + (size_t)tslots + reqDoubles + rreqDoubles, "batch_replicate_bin_moments"));
    MBAR_TRY(b->h_bin.grow((size_t)tslots, "batch_replicate_bin_moments"));
    std::memcpy(b->h_f, f, (size_t)fs * sizeof(double));
    double* hu = b->h_f + fs;
    src = 0;
    for (int t = 0; t < n_targets; ++t) {
        const int p = target_problem[t];
        std::memcpy(hu + toff[t], u_n + src, (size_t)b->N[p] * sizeof(double));
        std::memcpy(b->h_bin + toff[t], bin_n + src, (size_t)b->N[p] * sizeof(int32_t));
        for (int64_t i = b->N[p]; i < b->nT[p] * 32; ++i) {
            hu[toff[t] + i] = INFINITY;
            b->h_bin[toff[t] + i] = -1;
        }
        src += b->N[p];
    }
    BinReq* hreq = reinterpret_cast<BinReq*>(b->h_f + fs + tslots);
    std::memcpy(hreq, req.data(), req.size() * sizeof(BinReq));
    RepBinReq* hrreq = reinterpret_cast<RepBinReq*>(b->h_f + fs + tslots + reqDoubles);
    std::memcpy(hrreq, rreq.data(), rreq.size() * sizeof(RepBinReq));
    CallBuffers buf("batch_replicate_bin_moments");
    BinReq* d_req;
    RepBinReq* d_rreq;
    int *d_bt, *d_bin, *d_rflag;
    double *d_f, *d_ut, *d_lw, *d_Lp, *d_m, *d_o, *d_s, *d_fbin, *d_part;
    unsigned long long* d_keys;
    MBAR_TRY(buf.alloc(&d_req, (size_t)n));
    MBAR_TRY(buf.alloc(&d_rreq, (size_t)n));
    MBAR_TRY(buf.alloc(&d_f, (size_t)fs));
    MBAR_TRY(buf.alloc(&d_ut, (size_t)tslots));
    MBAR_TRY(buf.alloc(&d_bt, (size_t)tslots));
    MBAR_TRY(buf.alloc(&d_lw, (size_t)slots));
    MBAR_TRY(buf.alloc(&d_Lp, (size_t)slots));
    MBAR_TRY(buf.alloc(&d_bin, (size_t)slots));
    MBAR_TRY(buf.alloc(&d_keys, (size_t)bins));
    MBAR_TRY(buf.alloc(&d_m, (size_t)bins));
    MBAR_TRY(buf.alloc(&d_o, (size_t)bins));
    MBAR_TRY(buf.alloc(&d_s, (size_t)bins));
    MBAR_TRY(buf.alloc(&d_fbin, (size_t)bins));
    MBAR_TRY(buf.alloc(&d_part, (size_t)parts));
    MBAR_TRY(buf.alloc(&d_rflag, (size_t)n));
    cudaStream_t st = b->stream;
    MBAR_CUDA(cudaMemcpyAsync(d_f, b->h_f, (size_t)fs * sizeof(double), cudaMemcpyHostToDevice, st));
    MBAR_CUDA(cudaMemcpyAsync(d_ut, hu, (size_t)tslots * sizeof(double), cudaMemcpyHostToDevice, st));
    MBAR_CUDA(cudaMemcpyAsync(d_bt, b->h_bin, (size_t)tslots * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    MBAR_CUDA(cudaMemcpyAsync(d_req, hreq, req.size() * sizeof(BinReq), cudaMemcpyHostToDevice, st));
    MBAR_CUDA(cudaMemcpyAsync(d_rreq, hrreq, rreq.size() * sizeof(RepBinReq), cudaMemcpyHostToDevice, st));
    MBAR_CUDA(cudaMemsetAsync(d_keys, 0, (size_t)bins * sizeof(unsigned long long), st));
    MBAR_CUDA(cudaMemsetAsync(d_rflag, 0, (size_t)n * sizeof(int), st));
    const size_t smem0 = (size_t)BB_ACC_DOUBLES * sizeof(double);
    MBAR_CUDA(cudaFuncSetAttribute(batch_bin_accum_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)smem0));
    MBAR_CUDA(cudaFuncSetAttribute(batch_bin_accum_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    size_t smemS = 0;
    for (const BinReq& q : req) smemS = std::max(smemS, (size_t)q.geo[0].BC * sizeof(double));
    MBAR_CUDA(cudaEventRecord(b->ev0, st));
    batch_rep_bin_prep_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, st>>>(
        b->d_u, d_req, d_rreq, n, slots, d_f, b->d_Nk, b->d_logNk, b->d_x, b->d_counts, d_ut, d_bt, d_lw, d_Lp, d_bin,
        d_keys, d_rflag);
    batch_bin_max_kernel<<<(unsigned)((bins + 255) / 256), 256, 0, st>>>(d_req, n, bins, d_keys, d_m, d_o, d_rflag);
    batch_bin_accum_kernel<false><<<(unsigned)items, BB_THREADS, smemS, st>>>(b->d_u, d_req, n, d_f, d_lw, d_Lp, d_bin,
                                                                              d_o, d_part, d_rflag);
    batch_bin_reduce_kernel<false><<<(unsigned)((bins + 255) / 256), 256, 0, st>>>(d_req, n, bins, d_part, d_s);
    batch_bin_f_kernel<<<(unsigned)((bins + 255) / 256), 256, 0, st>>>(d_req, n, bins, d_m, d_s, d_fbin, d_o, d_rflag);
    MBAR_CUDA(cudaGetLastError());
    MBAR_CUDA(cudaEventRecord(b->ev1, st));
    MBAR_TRY(b->h_out.grow((size_t)bins, "batch_replicate_bin_moments"));
    std::vector<int> hflag((size_t)n);
    MBAR_CUDA(cudaMemcpyAsync(b->h_out, d_fbin, (size_t)bins * sizeof(double), cudaMemcpyDeviceToHost, st));
    MBAR_CUDA(cudaMemcpyAsync(hflag.data(), d_rflag, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
    MBAR_CUDA(cudaStreamSynchronize(st));
    float ms = 0.f;
    b->lastMs = event_ms(b->ev0, b->ev1, &ms) ? ms : 0.0;
    b->lastLaunches = 5;
    b->lastBytes = bytes;
    std::memcpy(f_bin, b->h_out, (size_t)bins * sizeof(double));
    for (int r = 0; r < n; ++r) flag[r] = hflag[r] != 0;
    return MBAR_B200_OK;
}

int mbar_b200_batch_log_weights(mbar_b200_batch* b, int32_t n, const int32_t* problem, const double* f,
                                const double* u_n, double* log_w, int32_t* flag) {
    MBAR_REQUIRE(b, MBAR_B200_ERR_INVALID, "batch_log_weights: NULL object");
    MBAR_REQUIRE(n >= 1 && problem && f && u_n && log_w && flag, MBAR_B200_ERR_INVALID,
                 "batch_log_weights: %d requests or a NULL argument", (int)n);
    std::vector<BinReq> req((size_t)n);
    std::vector<int64_t> tile0((size_t)b->P, 0);  // first tile of each problem: indexes x_n
    for (int p = 1; p < b->P; ++p) tile0[p] = tile0[p - 1] + b->nT[p - 1];
    int64_t slots = 0, fs = 0, src = 0, bytes = 0;
    for (int r = 0; r < n; ++r) {
        const int p = problem[r];
        MBAR_REQUIRE(p >= 0 && p < b->P, MBAR_B200_ERR_INVALID, "batch_log_weights: request %d names problem %d of %d",
                     r, p, b->P);
        BinReq& q = req[r];
        q = BinReq{};
        q.K = b->K[p];
        q.N = b->N[p];
        q.nT = b->nT[p];
        q.uoff = b->uoff[p];
        q.voff = b->voff[p];
        q.xoff = tile0[p] * 32;
        q.soff = slots;
        q.foff = fs;
        bytes += q.nT * 32 * q.K * 8;
        slots += q.nT * 32;
        fs += q.K;
        src += q.N;
    }
    for (int64_t i = 0; i < src; ++i)
        MBAR_REQUIRE(u_n[i] == u_n[i], MBAR_B200_ERR_NAN, "batch_log_weights: NaN in u_n (entry %lld)", (long long)i);
    MBAR_CUDA(cudaSetDevice(b->device));
    NvtxRange nvtx_("mbar_b200::batch_log_weights");
    b->lastLaunches = 0;
    b->lastBytes = 0;
    b->lastIterations = 0;
    // pinned staging: f, u_n padded with +inf to the tiles, the requests; log w_n comes back through the u_n slots
    const size_t reqDoubles = ((size_t)n * sizeof(BinReq) + 7) / 8;
    MBAR_TRY(b->h_f.grow((size_t)fs + (size_t)slots + reqDoubles, "batch_log_weights"));
    std::memcpy(b->h_f, f, (size_t)fs * sizeof(double));
    double* hu = b->h_f + fs;
    src = 0;
    for (int r = 0; r < n; ++r) {
        const BinReq& q = req[r];
        std::memcpy(hu + q.soff, u_n + src, (size_t)q.N * sizeof(double));
        for (int64_t i = q.N; i < q.nT * 32; ++i) hu[q.soff + i] = INFINITY;
        src += q.N;
    }
    BinReq* hreq = reinterpret_cast<BinReq*>(b->h_f + fs + slots);
    std::memcpy(hreq, req.data(), req.size() * sizeof(BinReq));
    CallBuffers buf("batch_log_weights");
    BinReq* d_req;
    int* d_rflag;
    double *d_f, *d_lw;
    MBAR_TRY(buf.alloc(&d_req, (size_t)n));
    MBAR_TRY(buf.alloc(&d_f, (size_t)fs));
    MBAR_TRY(buf.alloc(&d_lw, (size_t)slots));
    MBAR_TRY(buf.alloc(&d_rflag, (size_t)n));
    cudaStream_t s = b->stream;
    MBAR_CUDA(cudaMemcpyAsync(d_f, b->h_f, (size_t)fs * sizeof(double), cudaMemcpyHostToDevice, s));
    MBAR_CUDA(cudaMemcpyAsync(d_lw, hu, (size_t)slots * sizeof(double), cudaMemcpyHostToDevice, s));
    MBAR_CUDA(cudaMemcpyAsync(d_req, hreq, req.size() * sizeof(BinReq), cudaMemcpyHostToDevice, s));
    MBAR_CUDA(cudaMemsetAsync(d_rflag, 0, (size_t)n * sizeof(int), s));
    MBAR_CUDA(cudaEventRecord(b->ev0, s));
    batch_log_weights_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, s>>>(b->d_u, d_req, n, slots, d_f, b->d_Nk,
                                                                            b->d_logNk, b->d_x, d_lw, d_rflag);
    MBAR_CUDA(cudaGetLastError());
    MBAR_CUDA(cudaEventRecord(b->ev1, s));
    MBAR_TRY(b->h_out.grow((size_t)slots, "batch_log_weights"));
    std::vector<int> hflag((size_t)n);
    MBAR_CUDA(cudaMemcpyAsync(b->h_out, d_lw, (size_t)slots * sizeof(double), cudaMemcpyDeviceToHost, s));
    MBAR_CUDA(cudaMemcpyAsync(hflag.data(), d_rflag, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, s));
    MBAR_CUDA(cudaStreamSynchronize(s));
    float ms = 0.f;
    b->lastMs = event_ms(b->ev0, b->ev1, &ms) ? ms : 0.0;
    b->lastLaunches = 1;
    b->lastBytes = bytes;
    src = 0;
    for (int r = 0; r < n; ++r) {
        const BinReq& q = req[r];
        std::memcpy(log_w + src, b->h_out + q.soff, (size_t)q.N * sizeof(double));
        flag[r] = hflag[r] != 0;
        src += q.N;
    }
    return MBAR_B200_OK;
}

int mbar_b200_last_batch_stats(mbar_b200_batch* b, double* ms, int32_t* launches, int32_t* iterations,
                               int64_t* bytes_read) {
    MBAR_REQUIRE(b, MBAR_B200_ERR_INVALID, "NULL batch object");
    if (ms) *ms = b->lastMs;
    if (launches) *launches = b->lastLaunches;
    if (iterations) *iterations = b->lastIterations;
    if (bytes_read) *bytes_read = b->lastBytes;
    return MBAR_B200_OK;
}

// mbar_b200_bin_moments: the histogram free-energy surface of one target state (pymbar fes.py:388-600) and the
// blocks its analytical uncertainty needs (fes.py:1382-1415), without the N x (K + nbins) augmented weight matrix.
//
//   log w_n = -(u_n - x_n) - L'_n            (shifted frame: the per-sample shift x_n cancels, as in logw.cu)
//   f_i     = -(m_i + log sum_{n in i} c_n exp(log w_n - m_i)),   m_i = max_{n in i, c_n > 0} log w_n
//   C_ki    = sum_{n in i} c_n W_nk w^_n,   D_i = sum_{n in i} c_n w^_n^2,   w^_n = exp(log w_n + f_i)
//
// Four steps on the context's stream, each deterministic:
//   1. bin_prep_kernel: log w_n into a per-sample buffer, the bin index checked, each bin's maximum m_i by an
//      atomic max on the order-preserving integer form of the double (order-independent, hence deterministic);
//   2. bin_accum_kernel with one "row" of ones against c_n exp(log w_n - m_i) -> the bin sums, then f_i;
//   3. bin_accum_kernel with the K rows of W_nk plus one row of w^_n against c_n w^_n -> C and D;
//   4. bin_reduce_kernel: the per-CTA partial blocks summed in CTA order.
//
// bin_accum_kernel: a CTA owns a block of rows (warps own disjoint rows) and a contiguous range of tiles, and keeps a
// [rows x bin chunk] fp64 accumulator in shared memory.  Per tile a warp groups its lanes (= samples) by bin once
// (__match_any_sync), sorts them so that each group is contiguous, and reuses that order for all of its rows: one
// shuffle into sorted order, a segmented scan of ceil(log2(largest group)) steps, and the last lane of each group adds
// the group's sum to its own cell.  No two threads ever write the same cell, so there are no atomics and the order
// of every sum is fixed by the inputs.  Bins that do not fit in one chunk are covered by further chunks, each one more
// read of u_kn; tiles with no sample in the current chunk are skipped without being read.
#include <algorithm>
#include <cmath>
#include <vector>

#include "internal.cuh"

namespace mbar {

constexpr int BIN_THREADS = 256;
constexpr int BIN_WARPS = BIN_THREADS / 32;
constexpr int BIN_MAX_RW = 8;                          // rows per warp
constexpr int BIN_ACC_DOUBLES = (108 * 1024) / 8;      // shared accumulator per CTA: two CTAs per SM
constexpr size_t BIN_PARTIAL_BYTES = 256ull << 20;     // cap of the per-CTA partial blocks
constexpr double BIN_MAX_ARG = 700.0;                  // range contract of W_nk and w^_n exponents
enum { BINF_INVALID = 1, BINF_NAN = 2, BINF_RANGE = 4 };

// lw [nPad]: u_n on entry (first N), log w_n on exit (-inf for padding and for samples of multiplicity 0);
// bin [nPad]: the caller's bin index on entry, -1 for padding on exit.
__global__ void bin_prep_kernel(int64_t N, int64_t nPad, int nbins, int* __restrict__ bin, double* __restrict__ lw,
                                const double* __restrict__ Lp, const double* __restrict__ xshift,
                                const double* __restrict__ wgt, unsigned long long* __restrict__ keys,
                                int* __restrict__ flag) {
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= nPad) return;
    if (n >= N) {
        bin[n] = -1;
        lw[n] = -INFINITY;
        return;
    }
    int b = bin[n];
    const double u = lw[n];
    if (b < 0 || b >= nbins) {
        atomicOr(flag, BINF_INVALID);
        b = -1;
    }
    if (isnan(u)) atomicOr(flag, BINF_NAN);
    const double c = wgt ? wgt[n] : 1.0;
    // u_n = +inf: weight exactly 0, as np.exp(-inf) in the reference
    const double v = (c > 0.0 && u < INFINITY) ? -(u - xshift[n]) - Lp[n] : -INFINITY;
    bin[n] = b;
    lw[n] = v;
    // skip the atomic when the (possibly stale) maximum already beats this sample: few bins, many samples
    const unsigned long long key = ordered_key(v);
    if (b >= 0 && v > -INFINITY && key > *((volatile unsigned long long*)&keys[b])) atomicMax(&keys[b], key);
}

// m_i from the keys; o = -m (offset of the bin-sum pass).  A bin without a finite maximum (no sample, every u_n = +inf
// or every multiplicity 0, or a u_n = -inf) has no finite free energy.
__global__ void bin_max_kernel(int nbins, const unsigned long long* __restrict__ keys, double* __restrict__ m,
                               double* __restrict__ o, int* __restrict__ flag) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nbins) return;
    const double v = ordered_value(keys[b]);
    if (!isfinite(v)) atomicOr(flag, BINF_RANGE);
    m[b] = v;
    o[b] = -v;
}

// f_i = -(m_i + log s_i); o = f (offset of the moments pass)
__global__ void bin_f_kernel(int nbins, const double* __restrict__ m, const double* __restrict__ s,
                             double* __restrict__ f, double* __restrict__ o, int* __restrict__ flag) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nbins) return;
    const double fb = -(m[b] + log(s[b]));
    if (!isfinite(fb)) atomicOr(flag, BINF_RANGE);
    f[b] = fb;
    o[b] = fb;
}

struct BinParams {
    const double* u;        // [nTiles][K][32] shifted energies
    const double* Lp;       // [nPad] shifted-frame L'_n
    const double* f;        // [K] f_k
    const double* lw;       // [nPad] log w_n
    const int* bin;         // [nPad] bin index, -1 = none
    const double* o;        // [nbins] per-bin offset of the exponent of the right-hand factor
    const double* wgt;      // [nPad] multiplicities or NULL
    double* partial;        // [nGroups][nrows][BC]
    int* flag;
    int64_t nTiles;
    int K;                  // states in the tiles (row stride)
    int Kw;                 // rows of W_nk (K, or 0 for the bin-sum pass)
    int nrows;              // Kw + 1: the last row is w^_n (moments) or 1 (bin sums)
    int R, RW, nRowBlocks, nGroups;
    int b0, bw, BC;         // bins [b0, b0 + bw) in this chunk, accumulator row stride BC
};

__global__ void __launch_bounds__(BIN_THREADS, 2) bin_accum_kernel(BinParams p) {
    extern __shared__ double acc[];                     // [R][BC]
    __shared__ int perm[BIN_WARPS][32];
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int rb = blockIdx.x % p.nRowBlocks, g = blockIdx.x / p.nRowBlocks;
    const int row0 = rb * p.R;
    for (int i = threadIdx.x; i < p.R * p.BC; i += BIN_THREADS) acc[i] = 0.0;
    __syncthreads();
    const int64_t t0 = (int64_t)g * p.nTiles / p.nGroups, t1 = (int64_t)(g + 1) * p.nTiles / p.nGroups;
    const int myRows = (warp < p.R) ? (p.R - 1 - warp) / BIN_WARPS + 1 : 0;   // rows warp, warp + 8, ... below R
    bool range = false;
    for (int64_t t = t0; t < t1 && myRows > 0 && row0 + warp < p.nrows; ++t) {
        const int64_t n = t * TILE_N + lane;
        const int b = p.bin[n];
        if (!__any_sync(FULL, b >= p.b0 && b < p.b0 + p.bw)) continue;
        // this tile's energies first, so that the loads of all rows are in flight together
        const double* tp = p.u + t * (int64_t)p.K * TILE_N + lane;
        double uu[BIN_MAX_RW];
#pragma unroll
        for (int j = 0; j < BIN_MAX_RW; ++j) {
            const int r = row0 + warp + BIN_WARPS * j;
            uu[j] = (j < myRows && r < p.Kw) ? tp[(int64_t)r * TILE_N] : 0.0;
        }
        const double L = p.Lp[n];
        const double lwn = p.lw[n];
        const double eo = (b >= 0) ? lwn + p.o[b] : -INFINITY;
        if (eo > BIN_MAX_ARG) range = true;
        const double e0 = exp(eo);                      // w^_n (moments) | exp(log w_n - m_i) (bin sums)
        const double right = (p.wgt ? p.wgt[n] : 1.0) * e0;
        const double aux = (p.Kw == 0) ? 1.0 : e0;
        // group the lanes by bin and make every group contiguous, groups in the order of their lowest lane
        const WarpGroups grp = warp_groups(b, perm[warp]);
        const int col = (grp.tail && grp.key >= p.b0 && grp.key < p.b0 + p.bw) ? grp.key - p.b0 : -1;
        // predicated rather than an early exit, so that the rows' exps and shuffles can interleave
#pragma unroll
        for (int j = 0; j < BIN_MAX_RW; ++j) {
            const int rl = warp + BIN_WARPS * j;
            const int r = row0 + rl;
            if (j >= myRows || r >= p.nrows) continue;     // warp-uniform
            double a = aux;
            if (r < p.Kw) {
                const double e = p.f[r] - uu[j] - L;
                if (b >= 0 && e > BIN_MAX_ARG) range = true;
                // energies clamped at upload (+inf in the caller's array) have weight exactly 0
                a = (uu[j] >= U_CLAMP) ? 0.0 : exp(e);
            }
            if (b < 0) a = 0.0;
            const double v = warp_group_sum(grp, a * right);
            if (col >= 0) acc[rl * p.BC + col] += v;
        }
        __syncwarp();
    }
    if (range) atomicOr(p.flag, BINF_RANGE);
    __syncthreads();
    double* dst = p.partial + (int64_t)g * p.nrows * p.BC;
    for (int i = threadIdx.x; i < p.R * p.BC; i += BIN_THREADS) {
        const int r = row0 + i / p.BC;
        if (r < p.nrows) dst[(int64_t)r * p.BC + i % p.BC] = acc[i];
    }
}

// out[r][b0 + b] = sum over groups g, in order, of partial[g][r][b]
__global__ void bin_reduce_kernel(const double* __restrict__ partial, int nGroups, int nrows, int BC, int bw, int b0,
                                  int nbins, double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)nrows * bw) return;
    const int r = (int)(i / bw), b = (int)(i % bw);
    double s = 0.0;
    for (int g = 0; g < nGroups; ++g) s += partial[((int64_t)g * nrows + r) * BC + b];
    out[(int64_t)r * nbins + b0 + b] = s;
}

struct BinPlan {
    int RW, R, BC, chunks, nRowBlocks, nGroups;
};

// Rows per warp and bin-chunk width: fewest reads of u_kn, weighed against the loads a warp has in flight per tile.
static BinPlan plan_bins(int nrows, int nbins, int64_t nTiles, int smCount) {
    BinPlan best{};
    double bestCost = 0.0;
    for (int RW = 1; RW <= BIN_MAX_RW; RW *= 2) {
        const int R = std::min(BIN_WARPS * RW, nrows);
        const int BC = std::min(nbins, BIN_ACC_DOUBLES / R);
        const int chunks = (nbins + BC - 1) / BC;
        const double cost = (double)chunks * 4.0 / std::min(RW, 4);
        if (RW == 1 || cost < bestCost) {
            bestCost = cost;
            best = BinPlan{RW, R, BC, chunks, 0, 0};
        }
        if (R == nrows) break;
    }
    // spread the rows evenly over the row blocks
    best.nRowBlocks = (nrows + best.R - 1) / best.R;
    const int per = (nrows + best.nRowBlocks - 1) / best.nRowBlocks;
    best.RW = (per + BIN_WARPS - 1) / BIN_WARPS;
    best.R = std::min(BIN_WARPS * best.RW, nrows);
    best.BC = std::min(nbins, BIN_ACC_DOUBLES / best.R);
    best.chunks = (nbins + best.BC - 1) / best.BC;
    best.nRowBlocks = (nrows + best.R - 1) / best.R;
    // one wave of two CTAs per SM, each group a contiguous range of tiles
    int64_t groups = std::max<int64_t>(1, (2 * (int64_t)smCount) / best.nRowBlocks);
    groups = std::min<int64_t>(groups, nTiles);
    const int64_t cap = (int64_t)(BIN_PARTIAL_BYTES / ((size_t)nrows * best.BC * sizeof(double)));
    groups = std::max<int64_t>(1, std::min(groups, cap));
    best.nGroups = (int)groups;
    return best;
}

// nrows x nbins sums of a * right over the bins: rows [0, Kw) are W_nk, row Kw the auxiliary row.
static int run_accum(mbar_b200_ctx* c, BinParams p, int nbins, double* d_out, double* d_partial, const BinPlan& pl) {
    p.partial = d_partial;
    p.R = pl.R;
    p.RW = pl.RW;
    p.nRowBlocks = pl.nRowBlocks;
    p.nGroups = pl.nGroups;
    p.BC = pl.BC;
    const size_t smem = (size_t)pl.R * pl.BC * sizeof(double);
    MBAR_CUDA(cudaFuncSetAttribute(bin_accum_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // the largest shared-memory carveout, so that two CTAs with the largest accumulator share an SM
    MBAR_CUDA(cudaFuncSetAttribute(bin_accum_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    for (int b0 = 0; b0 < nbins; b0 += pl.BC) {
        p.b0 = b0;
        p.bw = std::min(pl.BC, nbins - b0);
        bin_accum_kernel<<<pl.nRowBlocks * pl.nGroups, BIN_THREADS, smem, c->stream>>>(p);
        const int64_t cells = (int64_t)p.nrows * p.bw;
        bin_reduce_kernel<<<(unsigned)((cells + 255) / 256), 256, 0, c->stream>>>(d_partial, pl.nGroups, p.nrows,
                                                                                  pl.BC, p.bw, b0, nbins, d_out);
        c->launches += 2;
        MBAR_CUDA(cudaGetLastError());
    }
    return MBAR_B200_OK;
}

}  // namespace mbar

using namespace mbar;

int mbar_b200_bin_moments(mbar_b200_ctx* c, const double* f_k, const double* u_n, const int32_t* bin_n,
                          int32_t nbins, double* f_bin, double* C, double* D) {
    MBAR_REQUIRE(c && f_k && u_n && bin_n && f_bin, MBAR_B200_ERR_INVALID, "bin_moments: NULL argument");
    MBAR_REQUIRE(nbins >= 1, MBAR_B200_ERR_INVALID, "bin_moments: nbins = %d must be at least 1", (int)nbins);
    MBAR_REQUIRE(!c->comm && c->nranks == 1, MBAR_B200_ERR_INVALID,
                 "bin_moments: sharded contexts are not supported (a communicator is attached)");
    PassWant w;
    w.L = true;
    MBAR_TRY(run_pass(c, f_k, w));
    if (C || D) MBAR_TRY(check_unsampled_clamp(c));   // C covers every state
    NvtxRange nvtx_("mbar_b200::bin_moments");
    const int K = c->K;
    const int64_t N = c->N, nPad = c->nTiles * TILE_N;
    const bool wantC = C || D;
    const BinPlan sumPlan = plan_bins(1, nbins, c->nTiles, c->smCount);
    const BinPlan momPlan = plan_bins(K + 1, nbins, c->nTiles, c->smCount);
    CallBuffers buf("bin_moments");
    int* d_bin;
    int* d_flag;
    double *d_lw, *d_f, *d_m, *d_o, *d_s, *d_fbin, *d_partial, *d_out = nullptr;
    unsigned long long* d_keys;
    size_t partialDoubles = (size_t)sumPlan.nGroups * sumPlan.BC;
    if (wantC) partialDoubles = std::max(partialDoubles, (size_t)momPlan.nGroups * (K + 1) * momPlan.BC);
    MBAR_TRY(buf.alloc(&d_bin, (size_t)nPad));
    MBAR_TRY(buf.alloc(&d_lw, (size_t)nPad));
    MBAR_TRY(buf.alloc(&d_flag, 1));
    MBAR_TRY(buf.alloc(&d_f, (size_t)K));
    MBAR_TRY(buf.alloc(&d_keys, (size_t)nbins));
    MBAR_TRY(buf.alloc(&d_m, (size_t)nbins));
    MBAR_TRY(buf.alloc(&d_o, (size_t)nbins));
    MBAR_TRY(buf.alloc(&d_s, (size_t)nbins));
    MBAR_TRY(buf.alloc(&d_fbin, (size_t)nbins));
    MBAR_TRY(buf.alloc(&d_partial, partialDoubles));
    if (wantC) MBAR_TRY(buf.alloc(&d_out, (size_t)(K + 1) * nbins));
    cudaStream_t s = c->stream;
    MBAR_CUDA(cudaMemcpyAsync(d_bin, bin_n, (size_t)N * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    MBAR_CUDA(cudaMemcpyAsync(d_lw, u_n, (size_t)N * sizeof(double), cudaMemcpyHostToDevice, s));
    MBAR_CUDA(cudaMemcpyAsync(d_f, f_k, (size_t)K * sizeof(double), cudaMemcpyHostToDevice, s));
    MBAR_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), s));
    MBAR_CUDA(cudaMemsetAsync(d_keys, 0, (size_t)nbins * sizeof(unsigned long long), s));
    c->h2dBytes += N * 12 + K * 8;
    Events ev;
    MBAR_TRY(ev.create(2));
    MBAR_CUDA(cudaEventRecord(ev[0], s));
    bin_prep_kernel<<<(unsigned)((nPad + 255) / 256), 256, 0, s>>>(N, nPad, nbins, d_bin, d_lw, c->d_L, c->d_xshift,
                                                                   c->d_wgt, d_keys, d_flag);
    bin_max_kernel<<<(nbins + 255) / 256, 256, 0, s>>>(nbins, d_keys, d_m, d_o, d_flag);
    c->launches += 2;
    MBAR_CUDA(cudaGetLastError());
    BinParams p{};
    p.u = c->d_u;
    p.Lp = c->d_L;
    p.f = d_f;
    p.lw = d_lw;
    p.bin = d_bin;
    p.o = d_o;
    p.wgt = c->d_wgt;
    p.flag = d_flag;
    p.nTiles = c->nTiles;
    p.K = K;
    // 2. bin sums s_i = sum c_n exp(log w_n - m_i) -> f_i
    p.Kw = 0;
    p.nrows = 1;
    MBAR_TRY(run_accum(c, p, nbins, d_s, d_partial, sumPlan));
    bin_f_kernel<<<(nbins + 255) / 256, 256, 0, s>>>(nbins, d_m, d_s, d_fbin, d_o, d_flag);
    c->launches++;
    // 3. C and D
    if (wantC) {
        p.Kw = K;
        p.nrows = K + 1;
        MBAR_TRY(run_accum(c, p, nbins, d_out, d_partial, momPlan));
    }
    MBAR_CUDA(cudaEventRecord(ev[1], s));
    int flag = 0;
    MBAR_CUDA(cudaMemcpyAsync(&flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
    MBAR_CUDA(cudaStreamSynchronize(s));
    float ms = 0.f;
    if (event_ms(ev[0], ev[1], &ms)) c->lastBinMs = ms;
    c->lastBinChunks = wantC ? momPlan.chunks : 0;
    MBAR_REQUIRE(!(flag & BINF_INVALID), MBAR_B200_ERR_INVALID, "bin_moments: a bin index lies outside [0, %d)",
                 (int)nbins);
    MBAR_REQUIRE(!(flag & BINF_NAN), MBAR_B200_ERR_NAN, "bin_moments: NaN in u_n");
    MBAR_REQUIRE(!(flag & BINF_RANGE), MBAR_B200_ERR_RANGE,
                 "bin_moments: a bin has no sample of finite weight, or a weight exponent exceeds 700 (f_k far from "
                 "the solution)");
    MBAR_CUDA(cudaMemcpy(f_bin, d_fbin, (size_t)nbins * sizeof(double), cudaMemcpyDeviceToHost));
    if (C) MBAR_CUDA(cudaMemcpy(C, d_out, (size_t)K * nbins * sizeof(double), cudaMemcpyDeviceToHost));
    if (D) MBAR_CUDA(cudaMemcpy(D, d_out + (size_t)K * nbins, (size_t)nbins * sizeof(double), cudaMemcpyDeviceToHost));
    c->d2hBytes += (int64_t)nbins * 8 * ((C ? K : 0) + (D ? 1 : 0) + 1);
    return MBAR_B200_OK;
}

int mbar_b200_last_bin_stats(mbar_b200_ctx* c, double* ms, int32_t* chunks) {
    MBAR_REQUIRE(c, MBAR_B200_ERR_INVALID, "NULL context");
    if (ms) *ms = c->lastBinMs;
    if (chunks) *chunks = c->lastBinChunks;
    return MBAR_B200_OK;
}

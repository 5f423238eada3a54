// mbar_b200_replicate_unsampled: the unsampled-state updates of B bootstrap replicates of the resident samples in one
// call, what set_sample_weights(c_b) + self_consistent_update(F_b) return for the unsampled rows, replicate by
// replicate (DESIGN.md 3.5f).  The bootstrap expectations of pymbar (mbar.py:890-971) need exactly these numbers: the
// appended rows of an augmented problem under each replicate's multiplicities and free energies.
//
// Shifted frame, as the passes (u' = u - x_n, L' = L - x_n; the shift cancels in -u'_jn - L'_bn):
//   L'_bn    = log sum_{k sampled} exp(c_bk - u'_kn),   c_bk = F[b, k] + log N_k
//   out[b,j] = -log sum_n c_bn exp(-u'_jn - L'_bn)       (unsampled j)
//
// rep_partial_kernel: a CTA owns a contiguous range of tiles (fixed by N and K alone) and a chunk of up to
// REP_THREADS * RPT unsampled rows; one launch serves a batch of up to REP_BATCH replicates.  Per tile:
//   1. the (replicate, sample) pairs of the batch with c_bn > 0 are listed in shared memory, grouped by replicate and in
//      sample order (one ballot per warp: warp b reads replicate b's counts); pairs with c_bn = 0 cost nothing after
//      this step;
//   2. thread i evaluates pair i's denominator with an exact per-pair max, the generic pass's two sweeps over the
//      sampled rows (read through L1 / L2: every pair of the tile reads the same rows), and keeps log c_bn - L'_bn;
//   3. the tile's rows of the chunk, staged in shared memory once per tile for the whole batch, are folded in: thread r
//      owns row r of the chunk and, replicate by replicate, updates a running (max, sum) in registers with one exp per
//      pair.
// Row b's pairs are visited in sample order whatever the other replicates draw, so its sums depend only on N, K and
// its own counts.  rep_combine_kernel merges the per-CTA (max, sum) pairs in CTA order.  No floating-point atomics.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "internal.cuh"

namespace mbar {

constexpr int REP_THREADS = 256;
constexpr int REP_WARPS = REP_THREADS / 32;
constexpr int REP_BATCH = 8;           // replicates per launch: one warp each lists a replicate's pairs of a tile
static_assert(REP_BATCH <= REP_WARPS && REP_BATCH * TILE_N <= REP_THREADS, "one pair per thread in step 2");

struct RepParams {
    const double* u;            // [nTiles][K][32] shifted, clamped energies
    const uint16_t* counts;     // [RB][nPad] this batch's multiplicities (0 past N)
    const double* c;            // [RB][Ks] c_bk of the sampled states, in the order of act
    const int* act;             // [Ks] sampled rows
    const int* uns;             // [nu] unsampled rows
    double2* partial;           // [nGroups * chunks][REP_BATCH][JC] (max, sum) per CTA
    int64_t nTiles, nPad;
    int K, Ks, nu, RB, nGroups, chunks, JC;
};

template <int RPT>
__global__ void __launch_bounds__(REP_THREADS) rep_partial_kernel(RepParams p) {
    extern __shared__ __align__(16) double rep_smem[];
    double* tab = rep_smem;                           // [32] exp table
    double* ut = tab + 32;                            // [JC][33] the chunk's rows of the current tile
    double* lv = ut + (size_t)p.JC * 33;              // [REP_THREADS] log c_bn - L'_bn of pair i
    __shared__ int s_n[REP_THREADS];                  // sample (lane) of pair i
    __shared__ int s_cnt[REP_WARPS];                  // pairs of replicate b in this tile
    const unsigned FULL = 0xffffffffu;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 32) tab[tid] = MBAR_EXP_TABLE[tid];
    const int g = blockIdx.x, y = blockIdx.y;
    const int j0 = y * p.JC;
    const int rows = min(p.JC, p.nu - j0);
    double M[RPT][REP_BATCH], S[RPT][REP_BATCH];
#pragma unroll
    for (int r = 0; r < RPT; ++r)
#pragma unroll
        for (int b = 0; b < REP_BATCH; ++b) {
            M[r][b] = -INFINITY;
            S[r][b] = 0.0;
        }
    const int64_t t0 = (int64_t)g * p.nTiles / p.nGroups, t1 = (int64_t)(g + 1) * p.nTiles / p.nGroups;
    for (int64_t t = t0; t < t1; ++t) {
        // 1. the pairs of the batch with c_bn > 0, grouped by replicate, in sample order
        const int cb = (warp < p.RB) ? (int)p.counts[(int64_t)warp * p.nPad + t * TILE_N + lane] : 0;
        const unsigned bal = __ballot_sync(FULL, cb > 0);
        if (lane == 0) s_cnt[warp] = __popc(bal);
        if (!__syncthreads_or(bal != 0u)) continue;       // no pair in this tile: nothing is read
        const double* tp = p.u + t * (int64_t)p.K * TILE_N;
        for (int i = tid; i < rows * TILE_N; i += REP_THREADS) {
            const int r = i >> 5, l = i & 31;
            ut[r * 33 + l] = tp[(int64_t)__ldg(p.uns + j0 + r) * TILE_N + l];
        }
        int seg[REP_BATCH + 1];
        seg[0] = 0;
#pragma unroll
        for (int b = 0; b < REP_BATCH; ++b) seg[b + 1] = seg[b] + s_cnt[b];
        const int total = seg[REP_BATCH];
        if (cb > 0) {
            int base = 0;
#pragma unroll
            for (int b = 0; b < REP_BATCH; ++b)
                if (b < warp) base += s_cnt[b];
            const int pos = base + __popc(bal & ((1u << lane) - 1u));
            s_n[pos] = lane;
            lv[pos] = log((double)cb);
        }
        __syncthreads();
        // 2. one pair per thread: L'_bn with an exact per-pair max
        if (tid < total) {
            int b = 0;
#pragma unroll
            for (int q = 1; q < REP_BATCH; ++q)
                if (tid >= seg[q]) b = q;
            const double* cr = p.c + (size_t)b * p.Ks;
            const double* un = tp + s_n[tid];
            double m = -INFINITY;
            int k = 0;
            for (; k + 4 <= p.Ks; k += 4) {
                double v[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) v[i] = un[(int64_t)__ldg(p.act + k + i) * TILE_N];
#pragma unroll
                for (int i = 0; i < 4; ++i) m = fmax(m, __ldg(cr + k + i) - v[i]);
            }
            for (; k < p.Ks; ++k) m = fmax(m, __ldg(cr + k) - un[(int64_t)__ldg(p.act + k) * TILE_N]);
            double D = 0.0;
            k = 0;
            for (; k + 4 <= p.Ks; k += 4) {
                double v[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) v[i] = un[(int64_t)__ldg(p.act + k + i) * TILE_N];
#pragma unroll
                for (int i = 0; i < 4; ++i) D += exp_fast(fmax(__ldg(cr + k + i) - v[i] - m, -800.0), tab);
            }
            for (; k < p.Ks; ++k)
                D += exp_fast(fmax(__ldg(cr + k) - un[(int64_t)__ldg(p.act + k) * TILE_N] - m, -800.0), tab);
            lv[tid] -= m + log(D);
        }
        __syncthreads();
        // 3. the chunk's rows: a running (max, sum) per (row, replicate), one exp per pair
#pragma unroll
        for (int rr = 0; rr < RPT; ++rr) {
            const int r = tid + rr * REP_THREADS;
            if (r < rows) {
                const double* ur = ut + r * 33;
#pragma unroll
                for (int b = 0; b < REP_BATCH; ++b) {
                    double m = M[rr][b], s = S[rr][b];
                    for (int i = seg[b]; i < seg[b + 1]; ++i) {
                        const double v = lv[i] - ur[s_n[i]];
                        const double d = v - m;
                        const double e = exp_fast(fmax(-fabs(d), -800.0), tab);
                        s = (d > 0.0) ? fma(s, e, 1.0) : s + e;
                        m = fmax(m, v);
                    }
                    M[rr][b] = m;
                    S[rr][b] = s;
                }
            }
        }
        __syncthreads();
    }
    double2* P = p.partial + ((size_t)g * p.chunks + y) * REP_BATCH * p.JC;
#pragma unroll
    for (int rr = 0; rr < RPT; ++rr) {
        const int r = tid + rr * REP_THREADS;
        if (r < rows)
#pragma unroll
            for (int b = 0; b < REP_BATCH; ++b) P[(size_t)b * p.JC + r] = make_double2(M[rr][b], S[rr][b]);
    }
}

// out[b, j] = -(M + log sum_g s_g exp(M_g - M)), M = max_g M_g, the CTAs g of row j's chunk in index order
__global__ void rep_combine_kernel(const double2* __restrict__ partial, int nGroups, int chunks, int JC, int nu, int RB,
                                   double* __restrict__ out) {
    __shared__ double tab[32];
    if (threadIdx.x < 32) tab[threadIdx.x] = MBAR_EXP_TABLE[threadIdx.x];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)RB * nu) return;
    const int b = (int)(i / nu), j = (int)(i % nu);
    const int y = j / JC, r = j % JC;
    const size_t stride = (size_t)chunks * REP_BATCH * JC;
    const double2* q = partial + ((size_t)y * REP_BATCH + b) * JC + r;
    double M = -INFINITY;
    for (int g = 0; g < nGroups; ++g) M = fmax(M, q[g * stride].x);
    if (M == -INFINITY) {
        out[i] = INFINITY;
        return;
    }
    double s = 0.0;
    for (int g = 0; g < nGroups; ++g) {
        const double2 v = q[g * stride];
        if (v.x > -INFINITY) s += v.y * exp_fast(fmax(v.x - M, -800.0), tab);
    }
    out[i] = -(M + log(s));
}

}  // namespace mbar

using namespace mbar;

int mbar_b200_replicate_unsampled(mbar_b200_ctx* c, int64_t B, const uint16_t* counts, const double* F, double* out) {
    MBAR_REQUIRE(c && counts && F && out, MBAR_B200_ERR_INVALID, "replicate_unsampled: NULL argument");
    MBAR_REQUIRE(B >= 1, MBAR_B200_ERR_INVALID, "replicate_unsampled: B = %lld must be at least 1", (long long)B);
    MBAR_REQUIRE(!c->comm && c->nranks == 1, MBAR_B200_ERR_INVALID,
                 "replicate_unsampled: sharded contexts are not supported (a communicator is attached)");
    MBAR_REQUIRE(c->ready, MBAR_B200_ERR_NOT_READY, "u_kn has not been uploaded");
    MBAR_CUDA(cudaSetDevice(c->device));
    const int K = c->K;
    for (int64_t b = 0; b < B; ++b) MBAR_TRY(check_range(c, F + (size_t)b * K));
    MBAR_TRY(check_unsampled_clamp(c));
    const int64_t N = c->N, nPad = c->nTiles * TILE_N;
    int64_t pairs = 0;
    for (int64_t b = 0; b < B; ++b) {
        const uint16_t* cb = counts + (size_t)b * N;
        int64_t sum = 0, nz = 0;
        for (int64_t n = 0; n < N; ++n) {
            sum += cb[n];
            nz += cb[n] > 0;
        }
        MBAR_REQUIRE(sum > 0, MBAR_B200_ERR_INVALID, "replicate_unsampled: the counts of replicate %lld sum to 0",
                     (long long)b);
        pairs += nz;
    }
    std::vector<int> uns;
    for (int k = 0; k < K; ++k)
        if (!(c->h_Nk[k] > 0)) uns.push_back(k);
    const int nu = (int)uns.size(), Ks = (int)c->active.size();
    c->lastRepMs = 0.0;
    c->lastRepBatches = 0;
    c->lastRepExps = 0;
    if (nu == 0) return MBAR_B200_OK;
    NvtxRange nvtx_("mbar_b200::replicate_unsampled");

    // rows per thread and CTAs: fixed by N and K alone, so that no row's sums depend on B
    const int RPT = nu > REP_THREADS ? 2 : 1;
    const int JC = REP_THREADS * RPT;
    const int chunks = (nu + JC - 1) / JC;
    const size_t smem = (32 + (size_t)JC * 33 + REP_THREADS) * sizeof(double);
    const int perSm = RPT == 1 ? 3 : 1;
    const int64_t groups =
        std::max<int64_t>(1, std::min<int64_t>(c->nTiles, ((int64_t)perSm * c->smCount + chunks - 1) / chunks));
    const int64_t nBatches = (B + REP_BATCH - 1) / REP_BATCH;

    // c_bk of the sampled states for every replicate, in the order of `active`
    std::vector<double> h_c((size_t)B * Ks);
    for (int64_t b = 0; b < B; ++b)
        for (int q = 0; q < Ks; ++q) {
            const int k = c->active[q];
            h_c[(size_t)b * Ks + q] = F[(size_t)b * K + k] + c->h_logNk[k];
        }
    CallBuffers buf("replicate_unsampled");
    uint16_t* d_counts;
    double *d_c, *d_out;
    int *d_act, *d_uns;
    double2* d_partial;
    MBAR_TRY(buf.alloc(&d_counts, 2 * (size_t)REP_BATCH * nPad));
    MBAR_TRY(buf.alloc(&d_c, (size_t)B * Ks));
    MBAR_TRY(buf.alloc(&d_out, (size_t)B * nu));
    MBAR_TRY(buf.alloc(&d_act, (size_t)Ks));
    MBAR_TRY(buf.alloc(&d_uns, (size_t)nu));
    MBAR_TRY(buf.alloc(&d_partial, (size_t)groups * chunks * REP_BATCH * JC));
    // pinned staging of the counts (two batches) and the call's events: copied[2], used[2], start, end
    const size_t slotElems = (size_t)REP_BATCH * nPad;
    HostPinned<uint16_t> pinned;
    Events ev;
    StreamDrain guard{c};
    MBAR_TRY(pinned.reserve(2 * slotElems, "replicate_unsampled"));
    MBAR_TRY(ev.create(6));
    const cudaEvent_t* copied = ev.ev.data();
    const cudaEvent_t* used = copied + 2;
    cudaStream_t s = c->stream;
    MBAR_CUDA(cudaMemcpyAsync(d_c, h_c.data(), h_c.size() * sizeof(double), cudaMemcpyHostToDevice, s));
    MBAR_CUDA(cudaMemcpyAsync(d_act, c->active.data(), (size_t)Ks * sizeof(int), cudaMemcpyHostToDevice, s));
    MBAR_CUDA(cudaMemcpyAsync(d_uns, uns.data(), (size_t)nu * sizeof(int), cudaMemcpyHostToDevice, s));
    MBAR_CUDA(cudaStreamSynchronize(s));      // the host vectors go out of scope with this call
    c->h2dBytes += (int64_t)h_c.size() * 8 + (int64_t)(Ks + nu) * 4;
    auto kern = RPT == 1 ? rep_partial_kernel<1> : rep_partial_kernel<2>;
    MBAR_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));

    RepParams p{};
    p.u = c->d_u;
    p.act = d_act;
    p.uns = d_uns;
    p.partial = d_partial;
    p.nTiles = c->nTiles;
    p.nPad = nPad;
    p.K = K;
    p.Ks = Ks;
    p.nu = nu;
    p.nGroups = (int)groups;
    p.chunks = chunks;
    p.JC = JC;
    // counts go up one batch ahead on the copy stream, through two pinned slots (zero past N once for all)
    for (int slot = 0; slot < 2; ++slot)
        for (int b = 0; b < REP_BATCH; ++b)
            std::memset(pinned + slot * slotElems + (size_t)b * nPad + N, 0, (size_t)(nPad - N) * sizeof(uint16_t));
    for (int64_t i = 0; i < nBatches; ++i) {
        const int slot = (int)(i & 1);
        const int64_t b0 = i * REP_BATCH;
        const int RB = (int)std::min<int64_t>(REP_BATCH, B - b0);
        if (i >= 2) MBAR_CUDA(cudaEventSynchronize(used[slot]));     // batch i - 2 no longer reads this slot
        uint16_t* hp = pinned + slot * slotElems;
        for (int b = 0; b < RB; ++b)
            std::memcpy(hp + (size_t)b * nPad, counts + (size_t)(b0 + b) * N, (size_t)N * sizeof(uint16_t));
        uint16_t* dp = d_counts + slot * slotElems;
        MBAR_CUDA(cudaMemcpyAsync(dp, hp, (size_t)RB * nPad * sizeof(uint16_t), cudaMemcpyHostToDevice,
                                  c->copyStream));
        MBAR_CUDA(cudaEventRecord(copied[slot], c->copyStream));
        c->h2dBytes += (int64_t)RB * nPad * 2;
        MBAR_CUDA(cudaStreamWaitEvent(s, copied[slot], 0));
        if (i == 0) MBAR_CUDA(cudaEventRecord(ev[4], s));
        p.counts = dp;
        p.c = d_c + (size_t)b0 * Ks;
        p.RB = RB;
        kern<<<dim3((unsigned)groups, (unsigned)chunks), REP_THREADS, smem, s>>>(p);
        const int64_t cells = (int64_t)RB * nu;
        rep_combine_kernel<<<(unsigned)((cells + 255) / 256), 256, 0, s>>>(d_partial, (int)groups, chunks, JC, nu, RB,
                                                                          d_out + (size_t)b0 * nu);
        c->launches += 2;
        MBAR_CUDA(cudaGetLastError());
        MBAR_CUDA(cudaEventRecord(used[slot], s));
    }
    MBAR_CUDA(cudaEventRecord(ev[5], s));
    MBAR_CUDA(cudaMemcpyAsync(out, d_out, (size_t)B * nu * sizeof(double), cudaMemcpyDeviceToHost, s));
    MBAR_CUDA(cudaStreamSynchronize(s));
    c->d2hBytes += (int64_t)B * nu * 8;
    // an unsampled row of +inf only was stored clamped; the reference's answer is +inf (as run_pass gives it)
    for (int q = 0; q < nu; ++q) {
        const int k = uns[q];
        if (c->h_ufar[k] != 0.0 && c->h_uclamp[k] == 0.0)
            for (int64_t b = 0; b < B; ++b) out[(size_t)b * nu + q] = INFINITY;
    }
    float ms = 0.f;
    if (event_ms(ev[4], ev[5], &ms)) c->lastRepMs = ms;
    c->lastRepBatches = (int)nBatches;
    c->lastRepExps = pairs * ((int64_t)Ks * chunks + nu);
    return MBAR_B200_OK;
}

int mbar_b200_last_replicate_stats(mbar_b200_ctx* c, double* ms, int32_t* batches, int64_t* exps) {
    MBAR_REQUIRE(c, MBAR_B200_ERR_INVALID, "NULL context");
    if (ms) *ms = c->lastRepMs;
    if (batches) *batches = c->lastRepBatches;
    if (exps) *exps = c->lastRepExps;
    return MBAR_B200_OK;
}

// Fused streaming pass, K <= 512: ONE read of u_kn per solver iteration.
//
// Reference being replaced: the two logsumexp sweeps of self_consistent_update / mbar_gradient /
// mbar_objective (mbar_solvers.py:231-242, :284-292, :327-355).  One launch yields S_k = sum_n W_nk and
// sum_n L_n, from which  f_sci = f - log S,  g = N (S - 1),  obj = sum L - N.f  all follow; in the
// device-resident iteration the launch also exchanges the sums with the other GPUs and applies the update.
//
// Structure (persistent, one CTA of 8 warps per SM; clusters of two CTAs when 256 < K <= 512):
//   * thread 0 streams whole stages (contiguous extents of the tile-major layout) into a 3..8-deep
//     shared-memory ring with cp.async.bulk (TMA engine, SASS UBLKCP) completing on mbarriers.  There is
//     no producer warp: a 9th warp would cap every thread at 168 registers instead of 255;
//   * lane = sample, warp = contiguous chunk of <= R states.  Each thread pulls its R energies out of
//     shared memory ONCE, does one fp64 exp per entry (table entry from a lane-replicated 8 KB table,
//     binary exponent on the integer pipe) and keeps R per-state accumulators in registers for the whole
//     kernel: no shuffles, no atomics, no re-reads in the steady state;
//   * the per-sample denominator is exchanged between the Wk warps of a sample group through 4 KB of
//     shared memory + one named barrier per tile (none when K <= 32); between the two CTAs of a cluster
//     through distributed shared memory + one cluster barrier per tile;
//   * per-CTA partials -> global; the last CTA (ticket) reduces them in CTA order (deterministic),
//     optionally gathers the other GPUs' sums through peer memory and applies the K-vector update.
//
// No per-sample max is needed: samples are pre-shifted so that min over sampled k of u'_kn = 0, hence
// max_k (c_k - u'_kn) lies in [min c, max c]; with c centred on `mid` and max c - min c < 1200 every
// exponent stays inside the fp64 range.  The kernel still verifies D_n per sample and raises a flag
// (host falls back to the generic kernel) if that assumption is ever violated.
//
// fp64-pipe budget per (k, n) entry: 9 (exp) + 1 (D) + 1 (accumulate) = 11 when the state constant is
// applied multiplicatively (spread(c) <= 600), 12 otherwise.  See DESIGN.md 3.1 for measurements.
#include <cmath>
#include <cstdlib>

#include "internal.cuh"

namespace mbar {


// denominator-exchange slots per parity: 16 inside one CTA, CL * 8 across a cluster of CL CTAs
__host__ __device__ constexpr int fused_slots(int CL) { return CL > 1 ? CL * 8 : 16; }
constexpr uint32_t FUSED_COPY_CHUNK = 32768;

__host__ __device__ inline size_t fused_smem_header(int K, int CL, int M = 1) {
    // tab[32] | c_s[M][K + 32] | xD[2][M][slots][32] | sred[M][256] | sumL[M][16] | bad[M][32] | full[8] | empty[8]
    // (c_s carries 32 spare entries.  A masked CTA zeroes c_s[Kl, max(Kl + 32, (Wk - 1) Rw + R)): it reads the
    //  constants of all R register rows of every warp.  Wk Rw < Kh + 2 Wk and R < Rw + 8 keep the highest read
    //  below Kh + 24, which is K + 24 for CL = 1 and at most K / 2 + 26 for CL > 1: K + 32 entries hold it.
    //  M = 2: a second candidate f-vector is evaluated on the same staged tiles)
    size_t b = 256 + (size_t)M * (((size_t)K + 32) * 8 + 2 * (size_t)fused_slots(CL) * 32 * 8 + 256 * 8 + 128 + 128) +
               64 + 64;
    return (b + 127) & ~(size_t)127;
}

__device__ __forceinline__ double lds_f64(const double* p) {
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(smem_u32(p)));
    return v;
}

// exp of `B` independent arguments a[i] = c[i] - u[i], stage by stage, so the fp64 pipe always has
// B independent chains in flight.  Shared-memory latency is hidden explicitly: the table lookups
// are issued right after the rounding step (5 polynomial stages ahead of their use) and the
// energies of the NEXT batch are fetched before this batch's polynomial (volatile loads keep their
// program position; two consumer warps per scheduler cannot hide ~30-cycle LDS otherwise).
// How the 2^(j/32) table is gathered and how the state constant enters:
//   MODE bit 0: 0 = table entry `lane` in two registers, gathered with two index shuffles;
//               1 = lane-replicated table in shared memory (tab[j][lane], 8 KB): one conflict-free
//                   LDS.64 whose address is (n << 8 & 0x1f00) | laneBase — cheaper to issue than two SHFL;
//   MODE bit 1: 0 = e = exp(c_k - u'), D += e                       (12 fp64 ops per entry)
//               1 = e0 = exp(-u'), D += E_k * e0 with E_k = exp(c_k) (11 fp64 ops; needs spread(c) <= 600)
struct TabRef {
    int hi, lo;          // shuffle mode
    uint32_t laneBase;   // LDS mode: shared address of tab[0][lane]
};

template <int R, int B, int R0, bool PREFETCH, int MODE, bool MASKED>
__device__ __forceinline__ void exp_batch(const double (&cu)[B], const double (&uu)[B], const TabRef tr,
                                          double (&e)[R], double& Dp, const double* nextC,
                                          const double* nextU, double (&cn)[B], double (&un)[B],
                                          uint32_t actbits) {
    constexpr bool LDSTAB = MODE & 1, ETRICK = MODE & 2;
    double t[B], r[B], pl[B], T[B];
#pragma unroll
    for (int i = 0; i < B; ++i) {
        if (ETRICK) {
            r[i] = uu[i];                                        // r holds +u' here (argument is -u')
            t[i] = fma(uu[i], -MBAR_EXP_SCALE, EXP_MAGIC);
        } else {
            r[i] = cu[i] - uu[i];
            t[i] = fma(r[i], MBAR_EXP_SCALE, EXP_MAGIC);
        }
    }
#pragma unroll
    for (int i = 0; i < B; ++i) {
        const int n = __double2loint(t[i]);
        if (LDSTAB) {
            const uint32_t addr = (((uint32_t)n << 8) & 0x1f00u) | tr.laneBase;
            asm volatile("ld.shared.f64 %0, [%1];" : "=d"(T[i]) : "r"(addr));
        } else {
            T[i] = __hiloint2double(__shfl_sync(0xffffffffu, tr.hi, n), __shfl_sync(0xffffffffu, tr.lo, n));
        }
    }
    if (PREFETCH) {
#pragma unroll
        for (int i = 0; i < B; ++i) un[i] = lds_f64(nextU + i * TILE_N);
#pragma unroll
        for (int i = 0; i < B; i += 2) {
            double2 c2;
            asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(c2.x), "=d"(c2.y) : "r"(smem_u32(nextC + i)));
            cn[i] = c2.x;
            cn[i + 1] = c2.y;
        }
    }
    if (ETRICK) {
        // rp = u' + n*ln2/32 = -(reduced argument); odd coefficients carry the sign
#pragma unroll
        for (int i = 0; i < B; ++i) r[i] = fma(t[i] - EXP_MAGIC, MBAR_EXP_LN2N, r[i]);
#pragma unroll
        for (int i = 0; i < B; ++i) pl[i] = fma(-MBAR_EXP_C5, r[i], MBAR_EXP_C4);
#pragma unroll
        for (int i = 0; i < B; ++i) pl[i] = fma(pl[i], r[i], -MBAR_EXP_C3);
#pragma unroll
        for (int i = 0; i < B; ++i) pl[i] = fma(pl[i], r[i], MBAR_EXP_C2);
#pragma unroll
        for (int i = 0; i < B; ++i) pl[i] = fma(pl[i], r[i], -MBAR_EXP_C1);
    } else {
#pragma unroll
        for (int i = 0; i < B; ++i) r[i] = fma(t[i] - EXP_MAGIC, -MBAR_EXP_LN2N, r[i]);   // (see exp_split)
#pragma unroll
        for (int i = 0; i < B; ++i) pl[i] = fma(MBAR_EXP_C5, r[i], MBAR_EXP_C4);
#pragma unroll
        for (int i = 0; i < B; ++i) pl[i] = fma(pl[i], r[i], MBAR_EXP_C3);
#pragma unroll
        for (int i = 0; i < B; ++i) pl[i] = fma(pl[i], r[i], MBAR_EXP_C2);
#pragma unroll
        for (int i = 0; i < B; ++i) pl[i] = fma(pl[i], r[i], MBAR_EXP_C1);
    }
#pragma unroll
    for (int i = 0; i < B; ++i) pl[i] = pl[i] * r[i];
#pragma unroll
    for (int i = 0; i < B; ++i) {
        e[R0 + i] = scale2(fma(T[i], pl[i], T[i]), __double2loint(t[i]) >> 5);
        // rows this warp does not own (K not a multiple of the warp tiling, unsampled states) were
        // computed on whatever bytes sit there; a select (not a multiply) discards them, NaN included
        if (MASKED && !((actbits >> (R0 + i)) & 1u)) e[R0 + i] = 0.0;
        if (ETRICK)
            Dp = fma(cu[i], e[R0 + i], Dp);
        else
            Dp += e[R0 + i];
    }
}

// All R rows of a thread in batches of B with two alternating input register sets (no copies).
template <int R, int B, int R0, int MODE, bool MASKED>
__device__ __forceinline__ void exp_rows(double (&cA)[B], double (&uA)[B], double (&cB)[B], double (&uB)[B],
                                         const TabRef tr, double (&e)[R], double& Dp,
                                         const double* cbase, const double* ubase, uint32_t actbits) {
    if constexpr (R0 + B < R) {
        exp_batch<R, B, R0, true, MODE, MASKED>(cA, uA, tr, e, Dp, cbase + R0 + B,
                                                ubase + (R0 + B) * TILE_N, cB, uB, actbits);
        exp_rows<R, B, R0 + B, MODE, MASKED>(cB, uB, cA, uA, tr, e, Dp, cbase, ubase, actbits);
    } else {
        exp_batch<R, B, R0, false, MODE, MASKED>(cA, uA, tr, e, Dp, nullptr, nullptr, cB, uB, actbits);
    }
}

// sum_n log D_n without a log per sample: D = m * 2^x with m in [1, 2); the exponents are summed as
// integers and the mantissas multiplied (renormalised by the caller before they can overflow).
__device__ __forceinline__ void logprod_push(double D, double& mprod, int& esum) {
    const int hi = __double2hiint(D);
    esum += (hi >> 20) - 1023;
    mprod *= __hiloint2double((hi & 0x000fffff) | 0x3ff00000, __double2loint(D));
}
__device__ __forceinline__ void logprod_renorm(double& mprod, int& esum) {
    const int hi = __double2hiint(mprod);
    esum += (hi >> 20) - 1023;
    mprod = __hiloint2double((hi & 0x000fffff) | 0x3ff00000, __double2loint(mprod));
}

// ---- thread-block-cluster helpers (CL = 2: two CTAs on two SMs share one tile, half the states each)
__device__ __forceinline__ unsigned cluster_ctarank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void st_cluster_f64(double* localPtr, unsigned rank, double v) {
    uint32_t ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(smem_u32(localPtr)), "r"(rank));
    asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(ra), "d"(v) : "memory");
}
__device__ __forceinline__ void cluster_barrier() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// CL = 1: one CTA per tile group, K <= 256.  CL = 2, 4, 8 (K <= 512, 1024, 2048): a cluster of CL CTAs (CL
// SMs) works on the same tile; CTA `half` (its rank in the cluster) owns states [half*Kh, ...), pulls only
// those rows from HBM (no redundant traffic) and the per-sample denominators are completed by exchanging
// the warps' partial sums through distributed shared memory + one cluster barrier per tile.
// WST: the launch also materialises the weights N_k W_nk = e_kn / D_n for the Hessian kernels (tile-major like
// u_kn, every 256-byte row XOR-swizzled for the DMMA fragment loads): the values sit in registers at that
// point, so the Newton half of an iteration costs one extra HBM write instead of a separate read+exp+write sweep.
// M = 2 (candidate-batched pass, SURVEY.md 8b `mbar_pass(ctx, M, f[M][K], ...)`): a second candidate vector is
// evaluated on the SAME staged tile.  With the multiplicative state constant the expensive part, e0 = exp(-u'),
// does not depend on f at all: the second candidate costs one more FMA per entry for its denominator
// (D2 += E2_k e0) and one for its accumulator — 13 instead of 2 x 11 fp64 operations per entry, and one read of
// u_kn instead of two.  It needs a second accumulator set, so it runs with <= 16 states per thread.
template <int R, bool FULL, int CW, int BATCH, int MODE, int CL, bool WST = false, int M = 1>
__global__ void __launch_bounds__(CW * 32, 1) pass_fused_kernel(const FusedParams p) {
    static_assert(M == 1 || ((MODE & 2) && R <= 16 && !WST), "M = 2 needs the multiplicative constant and R <= 16");
    extern __shared__ __align__(128) unsigned char smem_raw[];
    // device-resident loops: a converged (or failed) solver turns the rest of the enqueued batch into no-ops.
    // `done` is only written by the last CTA of a launch, after every CTA has taken its ticket, so all CTAs
    // (and all ranks: the state is bit-identical everywhere) take the same branch.
    if (p.loop && *reinterpret_cast<volatile int*>(&p.loop->done)) return;
    const int K = p.K;
    const int half = (CL > 1) ? (int)cluster_ctarank() : 0;             // rank of this CTA in its cluster
    const int kbase = (CL > 1) ? half * p.Kh : 0;                        // first state of this CTA
    const int Kl = (CL > 1) ? max(0, min(p.Kh, K - kbase)) : K;         // states of this CTA
    const unsigned nGroups = gridDim.x / CL, grp = blockIdx.x / CL;      // CTA (pair) index
    double* tab = reinterpret_cast<double*>(smem_raw);
    double* c_s = tab + 32;
    double* c_s2 = c_s + (K + 32);               // constants of the second candidate (M == 2)
    double* xD = c_s + M * (K + 32);             // [2][M][slots][32]
    constexpr int SLOTS = fused_slots(CL);
    double* sred = xD + 2 * M * SLOTS * 32;      // [M][Wn][K]  (Wn * K <= 256)
    double* s_sumL = sred + M * 256;             // [M][16]
    int* s_bad = reinterpret_cast<int*>(s_sumL + M * 16);     // [M][32]
    uint64_t* bar_full = reinterpret_cast<uint64_t*>(s_sumL + M * 32);
    uint64_t* bar_empty = bar_full + 8;
    unsigned char* stages = smem_raw + fused_smem_header(K, CL, M);
    __shared__ bool s_last;

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < 32) tab[threadIdx.x] = MBAR_EXP_TABLE[threadIdx.x];
    // state constants: c_k, or E_k = exp(c_k) when the constant is applied multiplicatively
    for (int k = threadIdx.x; k < Kl; k += blockDim.x)
        c_s[k] = (MODE & 2) ? exp(p.c[kbase + k]) : p.c[kbase + k];
    // keep the constants past this CTA's rows finite (a stale inf or NaN would turn D += E_k * 0 into NaN): the
    // masked variants read all R register rows of every warp, owned or not, up to c_s[(Wk - 1) * Rw + R - 1], which
    // for the last CTA of a cluster (Kl < Kh) can lie past Kl + 31.  The FULL variants read their own rows only.
    for (int i = threadIdx.x; i < 32; i += blockDim.x) c_s[Kl + i] = 0.0;
    if constexpr (!FULL)
        for (int i = Kl + 32 + threadIdx.x; i < (p.Wk - 1) * p.Rw + R; i += blockDim.x) c_s[i] = 0.0;
    if constexpr (M == 2) {
        for (int k = threadIdx.x; k < Kl; k += blockDim.x) c_s2[k] = exp(p.c2[kbase + k]);
        for (int i = threadIdx.x; i < 32; i += blockDim.x) c_s2[Kl + i] = 0.0;
        if constexpr (!FULL)
            for (int i = Kl + 32 + threadIdx.x; i < (p.Wk - 1) * p.Rw + R; i += blockDim.x) c_s2[i] = 0.0;
    }
    for (int i = threadIdx.x; i < 2 * M * SLOTS * 32; i += blockDim.x) xD[i] = 0.0;
    // lane-replicated exp table, 8 KB aligned so that its address bits never overlap the index bits
    const uint32_t tabRep = (smem_u32(stages + (size_t)p.NS * p.stageBytes) + 8191u) & ~8191u;
    if (MODE & 1)
        for (int i = threadIdx.x; i < 32 * 32; i += blockDim.x)
            asm volatile("st.shared.f64 [%0], %1;" ::"r"(tabRep + i * 8), "d"(MBAR_EXP_TABLE[i >> 5]));
    if (threadIdx.x == 0) {
        for (int i = 0; i < p.NS; ++i) {
            mbar_init(smem_u32(&bar_full[i]), 1);
            mbar_init(smem_u32(&bar_empty[i]), CW);
        }
        mbar_fence_init();
    }
    __syncthreads();
    // distributed shared memory may only be touched once every CTA of the cluster is running, and a
    // partner's first remote store must not land before this CTA has finished initialising xD
    if (CL > 1) cluster_barrier();

    const int tilesPerStage = p.Wn * p.TPW;
    double acc[R];
    double acc2[M == 2 ? R : 1];
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = 0.0;
#pragma unroll
    for (int r = 0; r < (M == 2 ? R : 1); ++r) acc2[r] = 0.0;
    double sumL = 0.0, sumL2 = 0.0;
    int bad = 0, bad2 = 0;
    const int g = warp / p.Wk, w = warp % p.Wk;   // sample group, state chunk (consumers)
    const int k0 = w * p.Rw;

    // Producer duty rides on thread 0 (a dedicated producer warp would put a third warp on one
    // scheduler and cut the register budget of EVERY thread from 255 to 168).  `issue(it)` streams the
    // it-th stage of this CTA into ring slot it % NS.
    // (slot, wrap) are carried incrementally by the callers: no integer division in the loop
    auto issue = [&](int it2, int slot2, int wrap2) {
        const int64_t s2 = (int64_t)grp + (int64_t)it2 * nGroups;
        if (s2 >= p.nStages) return;
        if (wrap2 > 0) mbar_wait(smem_u32(&bar_empty[slot2]), (wrap2 - 1) & 1);
        const int64_t tile0 = s2 * tilesPerStage;
        const int64_t ntl = min((int64_t)tilesPerStage, p.nTiles - tile0);
        const uint32_t fb = smem_u32(&bar_full[slot2]);
        const uint32_t dst = smem_u32(stages + (size_t)slot2 * p.stageBytes);
        if (Kl <= 0) {
            mbar_arrive_expect_tx(fb, 0);                           // (a trailing CTA without states)
        } else if (CL == 1) {
            const uint32_t bytes = (uint32_t)ntl * p.tileBytes;     // whole tiles are contiguous
            mbar_arrive_expect_tx(fb, bytes);
            const unsigned char* src =
                reinterpret_cast<const unsigned char*>(p.u) + (size_t)tile0 * p.tileBytes;
            for (uint32_t off = 0; off < bytes; off += FUSED_COPY_CHUNK)
                bulk_g2s(dst + off, src + off, min(FUSED_COPY_CHUNK, bytes - off), fb);
        } else {
            const uint32_t tb = (uint32_t)Kl * TILE_N * 8;          // this CTA's rows of each tile
            mbar_arrive_expect_tx(fb, (uint32_t)ntl * tb);
            for (int64_t t = 0; t < ntl; ++t)
                bulk_g2s(dst + (uint32_t)t * tb,
                         reinterpret_cast<const unsigned char*>(p.u) + (size_t)(tile0 + t) * p.tileBytes +
                             (size_t)kbase * TILE_N * 8,
                         tb, fb);
        }
    };
    if (threadIdx.x == 0)
        for (int i = 0; i < p.NS - 1; ++i) issue(i, i, 0);
    {
        // ------------------------------ consumers -----------------------------
        uint32_t actbits = 0;
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int k = kbase + k0 + r;
            if (r < p.Rw && k0 + r < Kl && ((p.rowmask[k >> 6] >> (k & 63)) & 1ull)) actbits |= 1u << r;
        }
        int par = 0;
        int it = 0;
        double mprod = 1.0;   // running product of the mantissas of D_n (see logprod_push)
        int esum = 0, npush = 0;
        double mprod2 = 1.0;
        int esum2 = 0;
        TabRef tr;
        tr.hi = __double2hiint(MBAR_EXP_TABLE[lane]);
        tr.lo = __double2loint(MBAR_EXP_TABLE[lane]);
        tr.laneBase = tabRep + lane * 8;
        int slot = 0, wrap = 0;              // it = wrap * NS + slot
        int pslot = p.NS - 1, pwrap = 0;     // ring position of stage it + NS - 1
        for (int64_t s = grp; s < p.nStages; s += nGroups, ++it) {
            // keep NS-1 stages in flight: stage it+NS-1 goes into the slot consumed at iteration it-1,
            // which every warp released before it could pass that iteration's denominator barrier
            if (threadIdx.x == 0) issue(it + p.NS - 1, pslot, pwrap);
            if (++pslot == p.NS) { pslot = 0; ++pwrap; }
            mbar_wait(smem_u32(&bar_full[slot]), wrap & 1);
            const double* sb = reinterpret_cast<const double*>(stages + (size_t)slot * p.stageBytes);
            for (int j = 0; j < p.TPW; ++j) {
                if (p.debugSkip) break;   // development probe: memory pipeline only
                const int tis = j * p.Wn + g;
                const int64_t tile = s * tilesPerStage + tis;
                if (tile >= p.nTiles) break;   // uniform over the sample group
                const double* tp = sb + ((size_t)tis * Kl + k0) * TILE_N + lane;
                // bootstrap multiplicity of this lane's sample (issued early; used after the exps)
                // (only the masked kernel family carries the weighted path: the FULL family stays lean)
                const double wn = (!FULL && p.wgt) ? __ldg(p.wgt + tile * TILE_N + lane) : 1.0;
                double e[R];
                double Dp = 0.0;
                {
                    // branch-free, 8 rows at a time; FULL: every warp owns exactly R sampled rows,
                    // otherwise the same code runs on all R register rows and masks the foreign ones
                    constexpr int B = R < BATCH ? R : BATCH;
                    double cA[B], uA[B], cB[B], uB[B];
#pragma unroll
                    for (int i = 0; i < B; ++i) {
                        uA[i] = lds_f64(tp + i * TILE_N);
                        cA[i] = lds_f64(c_s + k0 + i);
                    }
                    exp_rows<R, B, 0, MODE, !FULL>(cA, uA, cB, uB, tr, e, Dp, c_s + k0, tp, actbits);
                }
                double D = Dp, D2 = 0.0, Dp2 = 0.0;
                if constexpr (M == 2) {
                    // second candidate's partial denominator from the same e0 (state constants: broadcast loads)
#pragma unroll
                    for (int r = 0; r < R; ++r) Dp2 = fma(lds_f64(c_s2 + k0 + r), e[r], Dp2);
                    D2 = Dp2;
                }
                if (CL >= 4) {
                    // Two-level exchange (K > 512): the 8 warps of this CTA first combine their partial sums
                    // locally (slots CL .. CL+7 of this parity, one named barrier), then ONE warp publishes the
                    // CTA's sum to every partner through distributed shared memory and all CTAs add the CL
                    // sums in rank order — 8x fewer remote stores and CL instead of 8 CL additions per thread
                    // than the flat scheme used for pairs of CTAs.
                    double* xb = xD + par * M * SLOTS * 32 + lane;
                    xb[(CL + w) * 32] = Dp;
                    if constexpr (M == 2) xb[(SLOTS + CL + w) * 32] = Dp2;
                    named_bar_sync(1, CW * 32);
                    if (w == 0) {
                        double s1 = 0.0, s2 = 0.0;
#pragma unroll
                        for (int ww = 0; ww < 8; ++ww) s1 += xb[(CL + ww) * 32];
                        if constexpr (M == 2) {
#pragma unroll
                            for (int ww = 0; ww < 8; ++ww) s2 += xb[(SLOTS + CL + ww) * 32];
                        }
                        double* x = xb + half * 32;
                        *x = s1;
                        if constexpr (M == 2) x[SLOTS * 32] = s2;
#pragma unroll
                        for (int q = 1; q < CL; ++q) {
                            st_cluster_f64(x, (unsigned)((half + q) % CL), s1);
                            if constexpr (M == 2) st_cluster_f64(x + SLOTS * 32, (unsigned)((half + q) % CL), s2);
                        }
                    }
                    cluster_barrier();
                    D = 0.0;
#pragma unroll
                    for (int q = 0; q < CL; ++q) D += xb[q * 32];
                    if constexpr (M == 2) {
                        D2 = 0.0;
#pragma unroll
                        for (int q = 0; q < CL; ++q) D2 += xb[(SLOTS + q) * 32];
                    }
                    par ^= 1;
                } else if (CL > 1) {
                    // CL*8 partial sums per sample: slot = owner rank * 8 + warp, written locally and into
                    // every partner CTA's shared memory; all CTAs then add them in the same order
                    double* x = xD + (par * M * SLOTS + half * 8 + w) * 32 + lane;
                    *x = Dp;
                    if constexpr (M == 2) x[SLOTS * 32] = Dp2;
#pragma unroll
                    for (int q = 1; q < CL; ++q) {
                        st_cluster_f64(x, (unsigned)((half + q) % CL), Dp);
                        if constexpr (M == 2) st_cluster_f64(x + SLOTS * 32, (unsigned)((half + q) % CL), Dp2);
                    }
                    cluster_barrier();
                    const double* xs = xD + par * M * SLOTS * 32 + lane;
                    D = 0.0;
#pragma unroll
                    for (int ww = 0; ww < CL * 8; ++ww) D += xs[ww * 32];
                    if constexpr (M == 2) {
                        D2 = 0.0;
#pragma unroll
                        for (int ww = 0; ww < CL * 8; ++ww) D2 += xs[(SLOTS + ww) * 32];
                    }
                    par ^= 1;
                } else if (p.Wk > 1) {
                    double* x = xD + (par * M * SLOTS + g * p.Wk) * 32 + lane;
                    x[w * 32] = Dp;
                    if constexpr (M == 2) x[(SLOTS + w) * 32] = Dp2;
                    named_bar_sync(1 + g, p.Wk * 32);
                    D = 0.0;
                    for (int ww = 0; ww < p.Wk; ++ww) D += x[ww * 32];
                    if constexpr (M == 2) {
                        D2 = 0.0;
                        for (int ww = 0; ww < p.Wk; ++ww) D2 += x[(SLOTS + ww) * 32];
                    }
                    par ^= 1;
                }
                const bool valid = tile * TILE_N + lane < p.N;
                if (valid && !(D > 1e-250 && D < 1e250)) bad = 1;
                const double rD = 1.0 / D;
                const double invD = valid ? (FULL ? rD : rD * wn) : 0.0;
#pragma unroll
                for (int r = 0; r < R; ++r) acc[r] = fma(e[r], invD, acc[r]);
                if constexpr (M == 2) {
                    if (valid && !(D2 > 1e-250 && D2 < 1e250)) bad2 = 1;
                    const double rD2 = 1.0 / D2;
                    const double invD2 = valid ? (FULL ? rD2 : rD2 * wn) : 0.0;
#pragma unroll
                    for (int r = 0; r < R; ++r) acc2[r] = fma(e[r], invD2, acc2[r]);
                }
                if (WST) {
                    // weights of this lane's sample, rows of this warp (bootstrap multiplicities enter the
                    // second moments as sqrt(w_n) on both factors)
                    const double inv0 = valid ? ((!FULL && p.wgt) ? rD * sqrt(wn) : rD) : 0.0;
                    double* wp = p.Wout + ((size_t)tile * K + kbase + k0) * TILE_N;
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        if (FULL || (r < p.Rw && k0 + r < Kl)) {
                            double wv = e[r] * inv0;
                            if (MODE & 2) wv *= lds_f64(c_s + k0 + r);
                            const int k = kbase + k0 + r;
                            wp[r * TILE_N + (lane ^ ((k & 7) << 2))] = wv;
                        }
                    }
                }
                if (w == 0 && half == 0) {
                    if (valid) {
                        if (!FULL && p.wgt) {
                            sumL += wn * log(D);          // general multiplicities: one log per sample
                            if constexpr (M == 2) sumL2 += wn * log(D2);
                        } else {
                            logprod_push(D, mprod, esum);
                            if constexpr (M == 2) logprod_push(D2, mprod2, esum2);
                            if ((++npush & 255) == 0) {
                                logprod_renorm(mprod, esum);
                                if constexpr (M == 2) logprod_renorm(mprod2, esum2);
                            }
                        }
                    }
                    if (p.Lout) p.Lout[tile * TILE_N + lane] = log(D) + p.mid;
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(smem_u32(&bar_empty[slot]));
            if (++slot == p.NS) { slot = 0; ++wrap; }
        }
        // per-warp lane reduction of the R accumulators (once per kernel)
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const double t = warp_sum(acc[r]);
            if (lane == 0 && r < p.Rw && k0 + r < Kl) sred[g * Kl + k0 + r] = t;
        }
        sumL += (double)esum * 0.693147180559945309417232 + log(mprod);
        sumL = warp_sum(sumL);
        bad = __any_sync(0xffffffffu, bad);
        if (lane == 0) {
            s_sumL[warp] = (w == 0 && half == 0) ? sumL : 0.0;
            s_bad[warp] = bad;
        }
        if constexpr (M == 2) {
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const double t = warp_sum(acc2[r]);
                if (lane == 0 && r < p.Rw && k0 + r < Kl) sred[256 + g * Kl + k0 + r] = t;
            }
            sumL2 += (double)esum2 * 0.693147180559945309417232 + log(mprod2);
            sumL2 = warp_sum(sumL2);
            bad2 = __any_sync(0xffffffffu, bad2);
            if (lane == 0) {
                s_sumL[16 + warp] = (w == 0 && half == 0) ? sumL2 : 0.0;
                s_bad[32 + warp] = bad2;
            }
        }
    }
    if (CL > 1) cluster_barrier();    // a partner may not exit while it can still be written to
    __syncthreads();

    constexpr int PW = M;                               // partial blocks of K + 2 doubles per CTA group
    double* P = p.partial + (size_t)grp * (PW * (K + 2));
    for (int k = threadIdx.x; k < Kl; k += blockDim.x) {
        double t = 0.0;
        for (int gg = 0; gg < p.Wn; ++gg) t += sred[gg * Kl + k];
        P[kbase + k] = t;
        if constexpr (M == 2) {
            double t2 = 0.0;
            for (int gg = 0; gg < p.Wn; ++gg) t2 += sred[256 + gg * Kl + k];
            P[K + 2 + kbase + k] = t2;
        }
    }
    if (threadIdx.x == 0 && half == 0) {
        double t = 0.0;
        int b = 0;
        for (int i = 0; i < CW; ++i) {
            t += s_sumL[i];
            b |= s_bad[i];
        }
        P[K] = t;
        P[K + 1] = (double)b;
        if constexpr (M == 2) {
            double t2 = 0.0;
            int b2 = 0;
            for (int i = 0; i < CW; ++i) {
                t2 += s_sumL[16 + i];
                b2 |= s_bad[32 + i];
            }
            P[K + 2 + K] = t2;
            P[K + 2 + K + 1] = (double)b2;
        }
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicInc(p.ticket, gridDim.x - 1);
        s_last = (prev == gridDim.x - 1);
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    const PassLayout lay{K};
    // ---- last CTA: deterministic reduction over CTAs, optional exchange with the other GPUs, optional
    // ---- self-consistent epilogue (f <- f - log S, gauge, c for the next launch): one kernel per iteration
    double* tot = reinterpret_cast<double*>(stages);     // [M][K + 2] (the ring is idle now)
    constexpr int TW = M;
    const int totN = TW * (K + 2);
    // Entries whose exp argument lay below the normal range were floored at up to 2^-1020 (scale2), and
    // D_n >= exp(c_min - mid) amplifies each by at most exp(mid - c_min), c_min over the sampled states (each
    // sample has a sampled state with u' = 0; unsampled rows only add to D_n): a raw sum sum_n e_kn / D_n below
    // 2^53 * N times that bound could be made of floored entries.  Such an S_k is poisoned (NaN) and every
    // consumer treats it as underflowed (log-domain redo).  (In S_k = E_k * sum / N_k the bound carries the
    // same factor E_k / N_k as S_k itself, so one threshold, floorSum, serves all states.)
    __shared__ double s_cmin[2][32];
    {
        double m1 = INFINITY, m2 = INFINITY;
        for (int k = threadIdx.x; k < K; k += blockDim.x)
            if ((p.sampledmask[k >> 6] >> (k & 63)) & 1ull) {
                m1 = fmin(m1, p.c[k]);
                if constexpr (M == 2) m2 = fmin(m2, p.c2[k]);
            }
        for (int o = 16; o > 0; o >>= 1) {
            m1 = fmin(m1, __shfl_xor_sync(0xffffffffu, m1, o));
            m2 = fmin(m2, __shfl_xor_sync(0xffffffffu, m2, o));
        }
        if (lane == 0) {
            s_cmin[0][warp] = m1;
            s_cmin[1][warp] = m2;
        }
    }
    for (int k = threadIdx.x; k < totN; k += blockDim.x) {
        double t = 0.0;
        for (unsigned b = 0; b < nGroups; ++b) t += p.partial[(size_t)b * totN + k];
        if (k == K) t += p.sumW * p.mid;
        if (M == 2 && k == K + 2 + K) t += p.sumW * p.mid2;
        tot[k] = t;
    }
    __syncthreads();
    double floorSum[2] = {INFINITY, INFINITY};
    for (int w2 = 0; w2 < (int)(blockDim.x >> 5); ++w2) {
        floorSum[0] = fmin(floorSum[0], s_cmin[0][w2]);
        floorSum[1] = fmin(floorSum[1], s_cmin[1][w2]);
    }
    floorSum[0] = exp(p.logFloorN - floorSum[0]);
    if (M == 2) floorSum[1] = exp(p.logFloorN - floorSum[1]);
    if (p.peer.nranks > 1) {
        // One-shot all-gather of the K+2 partial sums through peer memory (NVLink stores into every
        // rank's inbox, then a release flag), followed by a sum in RANK ORDER so that every GPU
        // computes bit-identical totals.  Replaces ncclAllReduce + a separate epilogue launch.
        __shared__ unsigned long long s_seq;
        if (threadIdx.x == 0) s_seq = ++(*p.peer.seq);   // only this CTA of this launch touches the counter
        __syncthreads();
        const unsigned long long seq = s_seq;
        const int par = (int)(seq & 1ull);
        const int P = p.peer.nranks, me = p.peer.rank;
        for (int q = 0; q < P; ++q) {
            double* dst = p.peer.inbox[q] + ((size_t)par * P + me) * totN;
            for (int k = threadIdx.x; k < totN; k += blockDim.x) dst[k] = tot[k];
        }
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x < P) {
            unsigned long long* flag = p.peer.flags[threadIdx.x] + (size_t)par * P + me;
            asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(flag), "l"(seq) : "memory");
        }
        __shared__ int s_timeout;
        if (threadIdx.x == 0) s_timeout = 0;
        __syncthreads();
        if (threadIdx.x < P) {
            const unsigned long long* flag = p.peer.flags[me] + (size_t)par * P + threadIdx.x;
            const long long t0 = clock64();
            unsigned long long v;
            for (;;) {
                asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(flag) : "memory");
                if (v == seq) break;
                // ~20 s: a peer died; fail instead of hanging the GPU.  (The host lines the ranks up with a
                // stream-ordered all-reduce before the first exchange of every loop, so live ranks arrive
                // within microseconds of each other.)
                if (clock64() - t0 > 40000000000ll) {
                    s_timeout = 1;
                    break;
                }
                __nanosleep(100);
            }
        }
        __syncthreads();
        const double* in = p.peer.inbox[me] + (size_t)par * P * totN;
        for (int k = threadIdx.x; k < totN; k += blockDim.x) {
            double t = 0.0;
            for (int q = 0; q < P; ++q) t += __ldcv(in + (size_t)q * totN + k);
            tot[k] = t;
        }
        __syncthreads();
        if (threadIdx.x == 0 && s_timeout) {
            tot[K + 1] += 1.0e6;   // flag > 0 -> host reports the failure
            if (M == 2) tot[K + 2 + K + 1] += 1.0e6;
        }
        __syncthreads();
    }
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        const bool act = (p.rowmask[k >> 6] >> (k & 63)) & 1ull;
        double t = tot[k];
        // (floor-aware underflow test on the raw sum, see floorSum)
        const bool under = !(t > floorSum[0]);
        if ((MODE & 2) && act) t *= exp(p.c[k]);      // S_k = E_k * sum_n e0_kn / D_n / N_k
        t = act ? (under ? NAN : t / p.Nk[k]) : 0.0;
        p.out[lay.S() + k] = t;
        p.out[lay.logS() + k] = 0.0;
        tot[k] = t;
    }
    if (threadIdx.x == 0) {
        p.out[lay.sumL()] = tot[K];
        p.out[lay.flag()] = tot[K + 1];
    }
    if constexpr (M == 2) {
        for (int k = threadIdx.x; k < K; k += blockDim.x) {
            const bool act = (p.rowmask[k >> 6] >> (k & 63)) & 1ull;
            double t = tot[K + 2 + k];
            const bool under = !(t > floorSum[1]);
            if (act) t *= exp(p.c2[k]);
            p.out2[lay.S() + k] = act ? (under ? NAN : t / p.Nk[k]) : 0.0;
            p.out2[lay.logS() + k] = 0.0;
        }
        if (threadIdx.x == 0) {
            p.out2[lay.sumL()] = tot[K + 2 + K];
            p.out2[lay.flag()] = tot[K + 2 + K + 1];
        }
    }
    if (p.epi) {
        __syncthreads();
        __shared__ double s_f0;
        __shared__ double s_md[32];
        __shared__ int s_nan[32];
        if (threadIdx.x == 0) s_f0 = p.f[p.first] - log(tot[p.first]);
        __syncthreads();
        // relative change of this step (mbar_solvers.py:627-631): entries with |f| below min(1e-8, tol) are
        // compared absolutely, the gauge state is skipped
        const double thr = p.loop ? fmin(1.0e-8, p.loop->tol) : 1.0e-8;
        double md = 0.0;
        int sawNan = 0;
        for (int k = threadIdx.x; k < K; k += blockDim.x) {
            if (p.Nk[k] > 0.0 && ((p.rowmask[k >> 6] >> (k & 63)) & 1ull)) {
                // an underflowed S_k poisons the result so the host redoes the step in the log domain
                const double fo = p.f[k];
                const double fn = (tot[k] > 1e-280) ? fo - log(tot[k]) - s_f0 : NAN;
                p.f[k] = fn;
                p.cnext[k] = fn + log(p.Nk[k]) - p.mid;
                if (fn != fn) sawNan = 1;
                if (k != p.first) {
                    double div = fabs(fn);
                    if (div < thr) div = 1.0;
                    md = fmax(md, fabs(fn - fo) / div);
                }
            }
        }
        if (p.loop) {
            for (int o = 16; o > 0; o >>= 1) md = fmax(md, __shfl_xor_sync(0xffffffffu, md, o));
            sawNan = __any_sync(0xffffffffu, sawNan);
            if (lane == 0) {
                s_md[warp] = md;
                s_nan[warp] = sawNan;
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                double m = 0.0;
                int nn = 0;
                for (int w2 = 0; w2 < (int)(blockDim.x >> 5); ++w2) {
                    m = fmax(m, s_md[w2]);
                    nn |= s_nan[w2];
                }
                LoopState* L = p.loop;
                const int it = L->iterations + 1;
                L->iterations = it;
                L->sci_iterations = it;
                L->max_delta = m;
                if (nn || tot[K + 1] != 0.0) {
                    L->status = tot[K + 1] >= 1.0e6 ? 2 : 1;   // comm time-out | range problem: robust redo
                    L->done = 1;
                } else if (m < L->tol) {
                    L->success = 1;
                    L->done = 1;
                } else if (it >= L->maxiter) {
                    L->done = 1;
                }
            }
        }
    }
}

// kernel mode (see TabRef): bit 0 = LDS-replicated exp table, bit 1 = multiplicative state constant.
// MBAR_B200_FUSED_MODE overrides the default for experiments.
static int fused_mode(double spread) {
    int mode = 3;
    if (const char* v = std::getenv("MBAR_B200_FUSED_MODE")) mode = std::atoi(v) & 3;
    mode |= 1;   // the shuffle-gathered table (bit 0 clear) was measured 10 % slower and is retired
    if (spread > 600.0) mode &= 1;   // exp(c_k) * exp(-u') needs the spread inside the exponent range
    return mode;
}

bool fused_applicable(const mbar_b200_ctx* ctx, const double* h_f, bool allStates, double* midOut,
                      double* spreadOut) {
    if (ctx->K > 2048) return false;
    double lo = INFINITY, hi = -INFINITY;
    for (int k = 0; k < ctx->K; ++k) {
        if (!allStates && !(ctx->h_Nk[k] > 0)) continue;
        const double c = h_f[k] + ctx->h_logNkEff[k];
        if (!std::isfinite(c)) return false;
        lo = std::fmin(lo, c);
        hi = std::fmax(hi, c);
    }
    if (hi - lo >= FUSED_SPREAD) return false;
    if (std::fabs(hi) > C_RANGE || std::fabs(lo) > C_RANGE) return false;
    if (allStates) {
        // Sampled rows have u' >= 0, unsampled rows may lie far below the sampled minimum.  An exp argument above
        // ~709.78 would overflow the binary exponent that scale2 adds to the high word and wrap it into the sign
        // bit (NaN, negative, or a small positive number that no later check can tell from a right answer): such
        // all-state passes take the log-domain kernel.
        const bool mult = fused_mode(hi - lo) & 2;
        const double mid = 0.5 * (hi + lo);
        for (int k = 0; k < ctx->K; ++k) {
            if (ctx->h_Nk[k] > 0) continue;
            const double arg = (mult ? 0.0 : h_f[k] + ctx->h_logNkEff[k] - mid) - ctx->h_urowmin[k];
            if (arg > FUSED_MAX_ARG) return false;
        }
    }
    if (midOut) *midOut = 0.5 * (hi + lo);
    if (spreadOut) *spreadOut = hi - lo;
    return true;
}

// Configure the fused kernel for f (host) and stage c = f + log N - mid on the device.
int fused_prepare(mbar_b200_ctx* ctx, const double* h_f, bool wantL, bool allStates, FusedParams* out,
                  bool* ok, double* d_cdst, double* h_stage, bool wantW, int M, double midQuantum) {
    if (!d_cdst) d_cdst = ctx->dc(ROW_C);
    if (!h_stage) h_stage = ctx->hf(ROW_C);
    *ok = false;
    double mid = 0.0, spread = 0.0;
    if (!fused_applicable(ctx, h_f, allStates, &mid, &spread)) return MBAR_B200_OK;
    // (any centring within a few units of the midpoint is as good; a quantised one lets consecutive batches and
    //  solves of the device-resident loops launch with identical parameters, i.e. reuse one captured graph)
    if (midQuantum > 0.0) mid = midQuantum * std::nearbyint(mid / midQuantum);
    const int K = ctx->K;
    FusedParams p{};
    p.K = K;
    const int mode = fused_mode(spread);
    p.logFloorN = LOG_FLOOR_S + std::log(ctx->N_total_states);
    p.allStates = allStates ? 1 : 0;
    p.M = M;
    // two candidates per launch: second accumulator set -> at most 16 states per thread, hence K <= 1024, and the
    // e0 = exp(-u') sharing needs the multiplicative constant; the caller falls back to two launches otherwise
    if (M == 2 && (!(mode & 2) || K > 1024 || K < 2 || allStates || wantW)) return MBAR_B200_OK;
    // Above 128 states the second accumulator set forces clusters of CTAs with 16 states per thread, and the
    // per-tile cluster barrier then outweighs the shared exp (measured at K = 256: 8.0 ms vs 2 x 3.5 ms for two
    // plain launches): the batched kernel is the default only where one CTA holds all states.
    if (M == 2 && K > 128 && !std::getenv("MBAR_B200_M2_CLUSTERS")) return MBAR_B200_OK;
    const int cw = 8;
    const int rmax = (M == 2) ? 16 : 32;
    const int perCta = cw * rmax;                          // states one CTA can hold
    p.CL = K > 4 * perCta ? 8 : K > 2 * perCta ? 4 : K > perCta ? 2 : 1;   // clusters of CL CTAs, K/CL states each
    p.Kh = (K + p.CL - 1) / p.CL;
    if (p.CL > 1) p.Kh = (p.Kh + 1) & ~1;   // even split point: 16-byte aligned pairs of state constants
    int wk = 1;
    while (wk * rmax < p.Kh) wk *= 2;
    p.Wk = wk;
    p.CW = cw;
    p.batch = 8;
    p.mode = mode;
    p.debugSkip = std::getenv("MBAR_B200_FUSED_SKIP") ? 1 : 0;
    p.Wn = cw / p.Wk;
    p.Rw = (p.Kh + p.Wk - 1) / p.Wk;
    p.Rw = (p.Rw + 1) & ~1;   // even: the state constants are fetched as 16-byte pairs
    p.tileBytes = (uint32_t)K * TILE_N * 8;                        // stride between tiles in HBM
    const uint32_t ctaTileBytes = (uint32_t)p.Kh * TILE_N * 8;    // what one CTA pulls per tile
    int tpw = (int)(65536u / (p.Wn * ctaTileBytes));
    p.TPW = tpw < 1 ? 1 : (tpw > 8 ? 8 : tpw);
    p.stageBytes = (uint32_t)p.Wn * p.TPW * ctaTileBytes;
    {
        // the masked variants read (and discard) up to R rows per warp regardless of how many it owns:
        // pad every ring slot so that those reads never touch a slot the TMA engine may be filling
        const int rt = p.Rw <= 8 ? 8 : p.Rw <= 16 ? 16 : p.Rw <= 24 ? 24 : 32;
        const int over = (p.Wk - 1) * p.Rw + rt - p.Kh;          // rows past the CTA's last state
        if (over > 0) p.stageBytes += (uint32_t)over * TILE_N * 8;
        p.stageBytes = (p.stageBytes + 127u) & ~127u;
    }
    const size_t header = fused_smem_header(K, p.CL, M);
    int ns = (int)((225 * 1024 - header - 16384) / p.stageBytes);   // (CL >= 4 -> 2 stages of 64 KB)
    while (ns < 2 && p.TPW > 1) {
        // (M = 2 with 8-CTA clusters: two sets of 64 exchange slots leave room for single-tile stages only)
        const uint32_t pad = p.stageBytes - (uint32_t)p.Wn * p.TPW * ctaTileBytes;
        p.TPW /= 2;
        p.stageBytes = (((uint32_t)p.Wn * p.TPW * ctaTileBytes + pad) + 127u) & ~127u;
        ns = (int)((225 * 1024 - header - 16384) / p.stageBytes);
    }
    p.NS = ns > 8 ? 8 : ns;
    if (p.NS < 2) return MBAR_B200_OK;
    const int tilesPerStage = p.Wn * p.TPW;
    p.nStages = (ctx->nTiles + tilesPerStage - 1) / tilesPerStage;
    p.N = ctx->N;
    p.nTiles = ctx->nTiles;
    p.mid = mid;
    p.u = ctx->d_u;
    p.c = d_cdst;
    // allStates: unsampled rows take part with weight e^-80 (see LOG_EPS_UNSAMPLED)
    p.rowmask = allStates ? ctx->d_onesmask : ctx->d_rowmask;
    p.sampledmask = ctx->d_rowmask;
    p.Nk = allStates ? ctx->d_NkEff : ctx->d_Nk;
    p.partial = ctx->d_partial;
    p.out = ctx->d_out;
    p.ticket = ctx->d_ticket;
    if (wantL) MBAR_TRY(ensure_L(ctx));
    p.Lout = wantL ? ctx->d_L.ptr : nullptr;
    // weights for the K > 64 Hessian path ride along when the caller is about to evaluate the Hessian at this f
    p.Wout = (wantW && !allStates && M == 1 && ensure_weight_buffer(ctx)) ? ctx->d_Wt.ptr : nullptr;
    p.wgt = ctx->d_wgt;
    p.sumW = ctx->d_wgt ? ctx->sumW : (double)ctx->N;
    for (int k = 0; k < K; ++k)
        h_stage[k] = (!allStates && std::isinf(ctx->h_logNk[k])) ? 0.0 : h_f[k] + ctx->h_logNkEff[k] - mid;
    MBAR_CUDA(cudaMemcpyAsync(d_cdst, h_stage, (size_t)K * sizeof(double), cudaMemcpyHostToDevice,
                              ctx->stream));
    ctx->h2dBytes += K * 8;
    *out = p;
    *ok = true;
    return MBAR_B200_OK;
}

// Launch with whatever c currently sits in ctx->d_c (device-resident iteration).
int fused_enqueue(mbar_b200_ctx* ctx, const FusedParams& p) {
    const size_t smem = fused_smem_header(p.K, p.CL, p.M) + (size_t)p.NS * p.stageBytes + 16384;
    int64_t grid = p.nStages < ctx->smCount / p.CL ? p.nStages : ctx->smCount / p.CL;
    grid *= p.CL;
    // register rows per thread: 8 / 16 / 24 / 32 (24 keeps K = 96, 192, 384, 768, 1536 and their neighbours on
    // the unmasked family: 8 warps x 24 states instead of 32 register rows of which a quarter is discarded)
    const int Rt = p.Rw <= 8 ? 8 : p.Rw <= 16 ? 16 : (p.Rw <= 24 && p.M == 1) ? 24 : 32;
    const bool full = (p.Rw == Rt) && (p.K == p.CL * p.Wk * p.Rw) &&
                      ((int)ctx->active.size() == p.K || p.allStates) && !p.wgt;
    void (*kern)(const FusedParams) = nullptr;
    int which = 0;
#define PICK(R_, CL_, ID_)                                                                           \
    if (Rt == R_ && p.CL == CL_) {                                                                   \
        if (!full && !(p.mode & 2)) { kern = pass_fused_kernel<R_, false, 8, 8, 1, CL_>; which = ID_; } \
        else if (!full) { kern = pass_fused_kernel<R_, false, 8, 8, 3, CL_>; which = ID_ + 1; }        \
        else if (!(p.mode & 2)) { kern = pass_fused_kernel<R_, true, 8, 8, 1, CL_>; which = ID_ + 2; } \
        else { kern = pass_fused_kernel<R_, true, 8, 8, 3, CL_>; which = ID_ + 3; }                    \
    }
#define PICKW(R_, CL_, ID_)                                                                          \
    if (Rt == R_ && p.CL == CL_ && p.Wout) {                                                         \
        if (!full && !(p.mode & 2)) { kern = pass_fused_kernel<R_, false, 8, 8, 1, CL_, true>; which = ID_; } \
        else if (!full) { kern = pass_fused_kernel<R_, false, 8, 8, 3, CL_, true>; which = ID_ + 1; }        \
        else if (!(p.mode & 2)) { kern = pass_fused_kernel<R_, true, 8, 8, 1, CL_, true>; which = ID_ + 2; } \
        else { kern = pass_fused_kernel<R_, true, 8, 8, 3, CL_, true>; which = ID_ + 3; }                    \
    }
#define PICKM(R_, CL_, ID_)                                                                          \
    if (Rt == R_ && p.CL == CL_) {                                                                   \
        if (!full) { kern = pass_fused_kernel<R_, false, 8, 8, 3, CL_, false, 2>; which = ID_; }     \
        else { kern = pass_fused_kernel<R_, true, 8, 8, 3, CL_, false, 2>; which = ID_ + 1; }        \
    }
    if (p.M == 2) {
        MBAR_REQUIRE((p.mode & 2) && !p.Wout && p.c2 && p.out2, MBAR_B200_ERR_INVALID, "bad M = 2 launch");
        PICKM(8, 1, 40) PICKM(16, 1, 42) PICKM(16, 2, 44) PICKM(16, 4, 46) PICKM(16, 8, 48)
    } else {
        PICK(8, 1, 0) PICK(16, 1, 4) PICK(32, 1, 8) PICK(32, 2, 12) PICK(32, 4, 16) PICK(32, 8, 20)
        PICK(24, 1, 60) PICK(24, 2, 64) PICK(24, 4, 68) PICK(24, 8, 72)
        PICKW(32, 1, 24) PICKW(32, 2, 28) PICKW(32, 4, 32) PICKW(32, 8, 36) PICKW(16, 1, 52) PICKW(8, 1, 56)
        PICKW(24, 1, 76) PICKW(24, 2, 80) PICKW(24, 4, 84) PICKW(24, 8, 88)
    }
#undef PICKM
#undef PICKW
#undef PICK
    MBAR_REQUIRE(kern, MBAR_B200_ERR_INVALID, "no fused kernel variant for K=%d", p.K);
    const bool isW = (which >= 24 && which < 40) || (which >= 52 && which < 60) || which >= 76;
    MBAR_REQUIRE(!p.Wout || isW, MBAR_B200_ERR_INVALID, "no weight-storing fused variant for K=%d", p.K);
    snprintf(ctx->lastKernel, sizeof(ctx->lastKernel),
             "pass_fused_kernel<R=%d, %s, CW=8, BATCH=8, MODE=%d (%s), CL=%d%s> grid=%lld NS=%d TPW=%d", Rt,
             full ? "FULL" : "MASKED", (p.mode & 2) ? 3 : 1,
             (p.mode & 2) ? "LDS table + multiplicative state constant" : "LDS table", p.CL,
             (which >= 40 && which < 52) ? ", M=2 (two candidates per launch)"
                           : isW ? ", WST (weights stored for the Hessian)" : "",
             (long long)grid, p.NS, p.TPW);
    static size_t attrSetAll[16][96] = {{0}};          // per device: the attribute belongs to the context
    size_t* attrSet = attrSetAll[ctx->device & 15];
    if (attrSet[which] < smem) {
        MBAR_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attrSet[which] = smem;
    }
    if (!ctx->capturing) MBAR_CUDA(cudaEventRecord(ctx->ev0, ctx->stream));
    if (p.CL == 1) {
        kern<<<(unsigned)grid, p.CW * 32, smem, ctx->stream>>>(p);
    } else {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)grid);
        cfg.blockDim = dim3(p.CW * 32);
        cfg.dynamicSmemBytes = smem;
        cfg.stream = ctx->stream;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = (unsigned)p.CL;
        at[0].val.clusterDim.y = 1;
        at[0].val.clusterDim.z = 1;
        cfg.attrs = at;
        cfg.numAttrs = 1;
        MBAR_CUDA(cudaLaunchKernelEx(&cfg, kern, p));
    }
    if (!ctx->capturing) MBAR_CUDA(cudaEventRecord(ctx->ev1, ctx->stream));
    ctx->launches++;
    ctx->passes++;
    MBAR_CUDA(cudaGetLastError());
    return MBAR_B200_OK;
}

int launch_pass_fused(mbar_b200_ctx* ctx, const double* h_f, bool wantL, bool allStates, bool* usedOut,
                      bool wantW, bool* wroteW) {
    FusedParams p;
    if (wroteW) *wroteW = false;
    MBAR_TRY(fused_prepare(ctx, h_f, wantL, allStates, &p, usedOut, nullptr, nullptr, wantW));
    if (!*usedOut) return MBAR_B200_OK;
    if (wroteW) *wroteW = p.Wout != nullptr;
    return fused_enqueue(ctx, p);
}

// Development probe (mbar_b200_probe_exp): exp(a[i]) through exactly the device code the passes run.
// which = 0: exp_fast; 1: the fused exp_batch body with the constant in the exponent (MODE=1, c = a, u' = 0);
// 2: its multiplicative form (MODE=3, e0 = exp(-u') with u' = -a).  One warp per 256 arguments, 8 per lane.
__global__ void __launch_bounds__(32) probe_exp_kernel(int which, int64_t n, const double* __restrict__ a,
                                                       double* __restrict__ out) {
    __shared__ double tab[MBAR_EXP_NT];
    __shared__ double rep[2 * 32 * 32];    // holds the lane-replicated table 8 KB aligned, as in the pass
    const int lane = threadIdx.x;
    tab[lane] = MBAR_EXP_TABLE[lane];
    const uint32_t tabRep = (smem_u32(rep) + 8191u) & ~8191u;
    for (int i = lane; i < 32 * 32; i += 32)
        asm volatile("st.shared.f64 [%0], %1;" ::"r"(tabRep + i * 8), "d"(MBAR_EXP_TABLE[i >> 5]));
    __syncwarp();
    TabRef tr;
    tr.hi = __double2hiint(MBAR_EXP_TABLE[lane]);
    tr.lo = __double2loint(MBAR_EXP_TABLE[lane]);
    tr.laneBase = tabRep + lane * 8;
    const int64_t base = (int64_t)blockIdx.x * 256;
    double cu[8], uu[8], e[8], cn[8], un[8], Dp = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int64_t j = base + i * 32 + lane;
        const double x = j < n ? a[j] : 0.0;
        cu[i] = which == 1 ? x : 0.0;
        uu[i] = which == 1 ? 0.0 : -x;
        e[i] = which == 0 ? exp_fast(x, tab) : 0.0;
    }
    if (which == 1) exp_batch<8, 8, 0, false, 1, false>(cu, uu, tr, e, Dp, nullptr, nullptr, cn, un, 0u);
    if (which == 2) exp_batch<8, 8, 0, false, 3, false>(cu, uu, tr, e, Dp, nullptr, nullptr, cn, un, 0u);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int64_t j = base + i * 32 + lane;
        if (j < n) out[j] = e[i];
    }
}

int probe_exp_launch(int which, int64_t n, const double* d_a, double* d_out) {
    probe_exp_kernel<<<(unsigned)((n + 255) / 256), 32>>>(which, n, d_a, d_out);
    MBAR_CUDA(cudaGetLastError());
    return MBAR_B200_OK;
}

}  // namespace mbar

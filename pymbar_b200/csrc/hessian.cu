// K x K second-moment matrix of the weights, Ghat = (N W)^T (N W), on the fp64 tensor pipe.
//
// Reference being replaced: mbar_hessian (mbar_solvers.py:395-411): W = exp(f - u^T - L) [N,K];
// H = -( (W^T W) * N N^T - diag(N_k sum_n W_nk) ).  With  w_kn = N_k W_nk = exp(c_k - u'_kn - L'_n):
//   H_ij = delta_ij N_i S_i - Ghat_ij,   Ghat_ij = sum_n w_in w_jn.
// This is the only compute-bound piece of the path (2 K^2 N flop vs 8 K N bytes).  wgmma has no fp64 kind,
// so it uses the warp-level DMMA (mma.sync.m8n8k4.f64, SASS DMMA.8x8x4).  On sm_90a the larger PTX shapes are
// native too (m16n8k4 -> DMMA.16x8x4, m16n8k16 -> DMMA.16x8x16, checked with cuobjdump); these kernels do not
// use them yet.  The DMMA shares the fp64 datapath with DFMA, so every exp evaluated inside this kernel costs
// MMA time.
//
// Round-2 structure (three kernels, chosen by K):
//   K <= 64   hessian_small_kernel<KT>: one warp owns one 32-sample tile and the whole lower triangle of
//             Ghat in registers (KT(KT+1)/2 8x8 DMMA tiles).  The A and B fragments of a symmetric product are
//             the same registers, so every weight is needed by exactly one lane: energies go TMA -> shared
//             (rows padded to 36 doubles: conflict-free fragment loads) -> registers, the exp is evaluated
//             in the fragment, nothing is written back and there is no block-level synchronisation.
//   K > 64    weights_kernel materialises w_kn ONCE per Hessian (tile-major like u_kn, rows XOR-swizzled) —
//             the round-1 kernel re-evaluated every panel's exps in each of the block pairs that used it (4x
//             for K = 256) and needed a __syncthreads per tile between conversion and multiplication;
//             hessian_big_kernel then is pure TMA -> DMMA: 128 x 128 block pairs of the lower block
//             triangle, 16 warps with 32 x 32 register tiles, mbarrier ring, no __syncthreads in the loop.
//             Diagonal pairs run their 6 full + 4 triangular 32 x 32 sub-blocks on 10 warps placed so that
//             the four schedulers carry 32/32/36/36 DMMA per k-step (off-diagonal pairs: 64).
//   fallback  hessian_inplace_kernel (round 1: in-place conversion) when the 8*K*N weight buffer cannot be
//             allocated (on an 80 GB part: once u_kn and the weights, 16*K*N bytes, no longer fit, e.g. K = 512,
//             N = 1.25e7), for every K.
// Per-CTA partial blocks are reduced by a second kernel in CTA order (deterministic).
#include <cmath>
#include <cstdlib>
#include <vector>

#include "internal.cuh"

namespace mbar {

constexpr int HB = 128;                    // block edge
constexpr int HNS = 3;                     // ring depth
constexpr uint32_t HPANEL = HB * TILE_N * 8;   // 32 KB

__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

// Converts row `row` of a 128 x 32 energy panel into weights in place (swizzled store).
__device__ __forceinline__ void convert_row(double* P, int row, int lane, double ck, bool act, bool valid,
                                            double L, const double* tab, double sw) {
    const double v = P[row * TILE_N + lane];
    __syncwarp();   // every lane has read the row before any lane overwrites a permuted slot of it
    double wv = 0.0;
    if (valid && act) wv = sw * exp_fast(fmin(fmax(ck - v - L, -800.0), 700.0), tab);
    P[row * TILE_N + (lane ^ ((row & 7) << 2))] = wv;
}

// Work split: CTAs [pairStart[p], pairStart[p+1]) own block pair p and share its tiles evenly.  Diagonal
// pairs only multiply the 10 lower-triangular 32 x 32 sub-blocks (3 instead of 4 per scheduler), so
// they get 3/4 of the CTAs an off-diagonal pair gets.
struct HessSplit {
    int nPairs;        // pairs handled by THIS launch
    int pairBase;      // global index of its first pair (K > 2048 needs several launches)
    int pairStart[140];
};

__global__ void __launch_bounds__(512, 1)
hessian_inplace_kernel(const double* __restrict__ u, const double* __restrict__ Lp,
               const double* __restrict__ c, const unsigned long long* __restrict__ rowmask, int K,
               int64_t N, int64_t nTiles, const HessSplit split, double* __restrict__ Gpart,
               const double* __restrict__ sqrtw, const LoopState* loop) {
    if (loop && *reinterpret_cast<const volatile int*>(&loop->done)) return;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    double* tab = reinterpret_cast<double*>(smem_raw);                      // [32]
    uint64_t* bar_full = reinterpret_cast<uint64_t*>(tab + 32);             // [HNS]
    uint64_t* bar_empty = bar_full + 4;                                     // [HNS]
    unsigned char* ring = smem_raw + 512;                                   // [HNS][2][HPANEL]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;             // 16 warps

    int pair = 0;
    while (pair + 1 < split.nPairs && (int)blockIdx.x >= split.pairStart[pair + 1]) ++pair;
    const int chunk = blockIdx.x - split.pairStart[pair];
    const int nChunks = split.pairStart[pair + 1] - split.pairStart[pair];
    int bi = 0, rem = pair + split.pairBase;      // pairs enumerated (0,0),(1,0),(1,1),(2,0),...
    while (rem > bi) { rem -= bi + 1; ++bi; }
    const int bj = rem;
    const bool diag = (bi == bj);
    const int64_t t0 = nTiles * chunk / nChunks, t1 = nTiles * (chunk + 1) / nChunks;
    const int rowsI = min(HB, K - bi * HB), rowsJ = min(HB, K - bj * HB);

    if (threadIdx.x < 32) tab[threadIdx.x] = MBAR_EXP_TABLE[threadIdx.x];
    if (threadIdx.x == 0) {
        for (int i = 0; i < HNS; ++i) {
            mbar_init(smem_u32(&bar_full[i]), 1);
            mbar_init(smem_u32(&bar_empty[i]), 16);
        }
        mbar_fence_init();
    }
    __syncthreads();

    auto issue = [&](int it) {
        const int64_t tile = t0 + it;
        if (tile >= t1) return;
        const int slot = it % HNS;
        if (it >= HNS) mbar_wait(smem_u32(&bar_empty[slot]), ((it / HNS) - 1) & 1);
        const uint32_t fb = smem_u32(&bar_full[slot]);
        const uint32_t bytesI = (uint32_t)rowsI * TILE_N * 8, bytesJ = (uint32_t)rowsJ * TILE_N * 8;
        mbar_arrive_expect_tx(fb, bytesI + (diag ? 0u : bytesJ));
        const double* base = u + tile * (int64_t)K * TILE_N;
        const uint32_t dst = smem_u32(ring + (size_t)slot * 2 * HPANEL);
        bulk_g2s(dst, base + (int64_t)bi * HB * TILE_N, bytesI, fb);
        if (!diag) bulk_g2s(dst + HPANEL, base + (int64_t)bj * HB * TILE_N, bytesJ, fb);
    };
    if (threadIdx.x == 0) {
        issue(0);
        issue(1);
    }

    // conversion (vector fp64 pipe): warp owns rows warp*8 .. +7 of each panel, lane = sample.
    // MMA (tensor pipe): warp tile 32 (i) x 32 (j).  Off-diagonal pair: wm = warp / 4, wn = warp % 4.
    // Diagonal pair: only the 10 sub-blocks with wm >= wn are needed (Ghat is symmetric); warps 0..9 take
    // them, which loads the four schedulers 3/3/2/2 instead of 4/4/4/4, warps 10..15 only convert.
    int wm = warp >> 2, wn = warp & 3;
    bool mmaWarp = true;
    if (diag) {
        mmaWarp = warp < 10;
        int t = warp < 10 ? warp : 0;
        wm = 0;
        while (t > wm) { t -= wm + 1; ++wm; }     // triangular enumeration (0,0),(1,0),(1,1),(2,0),...
        wn = t;
    }
    double acc[4][4][2];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b][0] = acc[a][b][1] = 0.0;

    double cI[8], cJ[8];
    uint32_t actI = 0, actJ = 0;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const int ki = bi * HB + warp * 8 + r, kj = bj * HB + warp * 8 + r;
        const bool ai = ki < K && ((rowmask[ki >> 6] >> (ki & 63)) & 1ull);
        const bool aj = kj < K && ((rowmask[kj >> 6] >> (kj & 63)) & 1ull);
        cI[r] = ai ? c[ki] : 0.0;
        cJ[r] = aj ? c[kj] : 0.0;
        actI |= (uint32_t)ai << r;
        actJ |= (uint32_t)aj << r;
    }
    const int fragCol = lane & 3, fragRow = lane >> 2;   // DMMA fragment coordinates of this lane
    const int nIter = (int)(t1 - t0);

    // prologue: weights of the first tile
    if (nIter > 0) {
        const double L = Lp[t0 * TILE_N + lane];
        const double sw0 = sqrtw ? sqrtw[t0 * TILE_N + lane] : 1.0;   // sqrt of the bootstrap multiplicity
        const bool valid = t0 * TILE_N + lane < N;
        mbar_wait(smem_u32(&bar_full[0]), 0);
        double* Pi = reinterpret_cast<double*>(ring);
        double* Pj = Pi + HB * TILE_N;
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            convert_row(Pi, warp * 8 + r, lane, cI[r], (actI >> r) & 1u, valid, L, tab, sw0);
            if (!diag) convert_row(Pj, warp * 8 + r, lane, cJ[r], (actJ >> r) & 1u, valid, L, tab, sw0);
        }
    }
    __syncthreads();

    for (int it = 0; it < nIter; ++it) {
        const int slot = it % HNS;
        const int64_t tile = t0 + it;
        if (threadIdx.x == 0) issue(it + 2);          // slot (it+2)%3 was released at the end of it-1
        // the NEXT tile's energies are converted while this tile is multiplied (separate pipes)
        const bool haveNext = it + 1 < nIter;
        const int nslot = (it + 1) % HNS;
        double Ln = 0.0, swn = 1.0;
        bool validN = false;
        if (haveNext) {
            Ln = Lp[(tile + 1) * TILE_N + lane];
            if (sqrtw) swn = sqrtw[(tile + 1) * TILE_N + lane];
            validN = (tile + 1) * TILE_N + lane < N;
            mbar_wait(smem_u32(&bar_full[nslot]), ((it + 1) / HNS) & 1);
        }
        double* Ni = reinterpret_cast<double*>(ring + (size_t)nslot * 2 * HPANEL);
        double* Nj = Ni + HB * TILE_N;
        const double* Pi = reinterpret_cast<const double*>(ring + (size_t)slot * 2 * HPANEL);
        const double* Pj = diag ? Pi : Pi + HB * TILE_N;
        const double* Ai = Pi + (wm * 32 + fragRow) * TILE_N;
        const double* Bj = Pj + (wn * 32 + fragRow) * TILE_N;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
            if (haveNext) {
                convert_row(Ni, warp * 8 + ks, lane, cI[ks], (actI >> ks) & 1u, validN, Ln, tab, swn);
                if (!diag) convert_row(Nj, warp * 8 + ks, lane, cJ[ks], (actJ >> ks) & 1u, validN, Ln, tab, swn);
            }
            if (!mmaWarp) continue;
            const int col = ((ks ^ fragRow) << 2) + fragCol;      // (4 ks + fragCol) ^ (fragRow << 2)
            double a[4], b[4];
#pragma unroll
            for (int mt = 0; mt < 4; ++mt) a[mt] = Ai[mt * 8 * TILE_N + col];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) b[nt] = Bj[nt * 8 * TILE_N + col];
#pragma unroll
            for (int mt = 0; mt < 4; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) dmma884(acc[mt][nt][0], acc[mt][nt][1], a[mt], b[nt]);
        }
        fence_proxy_async_smem();   // slot `slot` was written in place; its next writer is the TMA engine
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&bar_empty[slot]));
        __syncthreads();            // next tile's weights are complete for every warp
    }
    // write this CTA's 128 x 128 partial block: Gpart[chunk][pair][128][128]
    double* out = Gpart + (size_t)blockIdx.x * HB * HB;
    if (mmaWarp)
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const int row = wm * 32 + mt * 8 + (lane >> 2);
            const int col = wn * 32 + nt * 8 + (lane & 3) * 2;
            out[row * HB + col] = acc[mt][nt][0];
            out[row * HB + col + 1] = acc[mt][nt][1];
        }
}

// Sum the partial blocks of each pair over its CTAs (in order: deterministic) and scatter to the full
// symmetric K x K matrix.  Diagonal pairs only hold sub-blocks with row-block >= column-block.
__global__ void __launch_bounds__(256)
hessian_reduce_kernel(const double* __restrict__ Gpart, int K, const HessSplit split, double* __restrict__ G,
                      const LoopState* loop) {
    if (loop && *reinterpret_cast<const volatile int*>(&loop->done)) return;
    const int pair = blockIdx.x;
    int bi = 0, rem = pair + split.pairBase;
    while (rem > bi) { rem -= bi + 1; ++bi; }
    const int bj = rem;
    const int c0 = split.pairStart[pair], c1 = split.pairStart[pair + 1];
    for (int e = blockIdx.y * blockDim.x + threadIdx.x; e < HB * HB; e += gridDim.y * blockDim.x) {
        const int r = e / HB, cidx = e % HB;
        const int i = bi * HB + r, j = bj * HB + cidx;
        if (i >= K || j >= K) continue;
        if (bi == bj && (r >> 5) < (cidx >> 5)) continue;      // filled by its mirror image below
        double s = 0.0;
        for (int ch = c0; ch < c1; ++ch) s += Gpart[(size_t)ch * HB * HB + e];
        G[(size_t)i * K + j] = s;
        if (bi != bj || (r >> 5) > (cidx >> 5)) G[(size_t)j * K + i] = s;
    }
}

// ------------------------------------------------------------------------------------------------
// Round 2, K > 64: weights materialised once, then a pure TMA -> DMMA kernel.
// ------------------------------------------------------------------------------------------------
// w_kn = sqrt(mult_n) * exp(c_k - u'_kn - L'_n), written tile-major like u_kn with the XOR swizzle the DMMA
// fragment loads want (element (k, s) at column s ^ ((k & 7) << 2): a permutation inside one 256-byte row, so
// both the read and the write stay fully coalesced).  HBM-bound: reads and writes 8*K*N bytes each.
__global__ void __launch_bounds__(256)
weights_kernel(const double* __restrict__ u, const double* __restrict__ Lp, const double* __restrict__ c,
               const unsigned long long* __restrict__ rowmask, int K, int64_t N, int64_t nTiles,
               const double* __restrict__ sqrtw, double* __restrict__ Wt, const LoopState* loop) {
    if (loop && *reinterpret_cast<const volatile int*>(&loop->done)) return;
    __shared__ double tab[32];
    if (threadIdx.x < 32) tab[threadIdx.x] = MBAR_EXP_TABLE[threadIdx.x];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t tile = blockIdx.x; tile < nTiles; tile += gridDim.x) {
        const double L = Lp[tile * TILE_N + lane];
        const double sw = sqrtw ? sqrtw[tile * TILE_N + lane] : 1.0;
        const bool valid = tile * TILE_N + lane < N;
        const double* src = u + tile * (int64_t)K * TILE_N;
        double* dst = Wt + tile * (int64_t)K * TILE_N;
        // 8 rows per thread in flight: the sweep is bound by bytes in flight per SM, not by the exps
        for (int k0 = warp; k0 < K; k0 += 64) {
            double v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = (k0 + 8 * i < K) ? src[(k0 + 8 * i) * TILE_N + lane] : 0.0;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int k = k0 + 8 * i;
                if (k < K) {
                    const bool act = (rowmask[k >> 6] >> (k & 63)) & 1ull;
                    double wv = 0.0;
                    if (valid && act) wv = sw * exp_fast(fmin(fmax(__ldg(c + k) - v[i] - L, -800.0), 700.0), tab);
                    dst[k * TILE_N + (lane ^ ((k & 7) << 2))] = wv;
                }
            }
        }
    }
}

// Diagonal block pairs: 6 full + 4 triangular 32 x 32 sub-blocks on 10 of the 16 warps, placed so that the four
// schedulers (warp % 4) carry 32 / 32 / 36 / 36 DMMA per k-step.  -1: the warp idles in a diagonal pair.
__constant__ signed char HD_M[16] = {1, 2, 3, 3, 2, 3, 0, 2, -1, -1, 1, 3, -1, -1, -1, -1};
__constant__ signed char HD_N[16] = {0, 1, 1, 2, 0, 0, 0, 2, -1, -1, 1, 3, -1, -1, -1, -1};

__global__ void __launch_bounds__(512, 1)
hessian_big_kernel(const double* __restrict__ Wt, int K, int64_t nTiles, const HessSplit split,
                   double* __restrict__ Gpart, const LoopState* loop) {
    if (loop && *reinterpret_cast<const volatile int*>(&loop->done)) return;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem_raw);             // [HNS]
    uint64_t* bar_empty = bar_full + 4;                                     // [HNS]
    unsigned char* ring = smem_raw + 512;                                   // [HNS][2][HPANEL]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;             // 16 warps

    int pair = 0;
    while (pair + 1 < split.nPairs && (int)blockIdx.x >= split.pairStart[pair + 1]) ++pair;
    const int chunk = blockIdx.x - split.pairStart[pair];
    const int nChunks = split.pairStart[pair + 1] - split.pairStart[pair];
    int bi = 0, rem = pair + split.pairBase;      // pairs enumerated (0,0),(1,0),(1,1),(2,0),...
    while (rem > bi) { rem -= bi + 1; ++bi; }
    const int bj = rem;
    const bool diag = (bi == bj);
    const int64_t t0 = nTiles * chunk / nChunks, t1 = nTiles * (chunk + 1) / nChunks;
    const int rowsI = min(HB, K - bi * HB), rowsJ = min(HB, K - bj * HB);

    // role of this warp: 32 x 32 sub-block (wm, wn) of the 128 x 128 block; tri = only its lower 8 x 8 tiles
    int wm = diag ? (int)HD_M[warp] : (warp >> 2), wn = diag ? (int)HD_N[warp] : (warp & 3);
    const bool tri = diag && wm == wn;
    const bool active = wm >= 0 && wm * 32 < rowsI && wn * 32 < rowsJ;
    int nAct = 0, prodWarp = -1;
    for (int w2 = 0; w2 < 16; ++w2) {
        const int m2 = diag ? (int)HD_M[w2] : (w2 >> 2), n2 = diag ? (int)HD_N[w2] : (w2 & 3);
        if (m2 >= 0 && m2 * 32 < rowsI && n2 * 32 < rowsJ) {
            if (prodWarp < 0) prodWarp = w2;
            ++nAct;
        }
    }
    if (threadIdx.x == 0) {
        for (int i = 0; i < HNS; ++i) {
            mbar_init(smem_u32(&bar_full[i]), 1);
            mbar_init(smem_u32(&bar_empty[i]), nAct);
        }
        mbar_fence_init();
    }
    __syncthreads();
    if (!active) return;
    const bool producer = (warp == prodWarp) && lane == 0;
    const int nIter = (int)(t1 - t0);

    auto issue = [&](int it) {
        if (it >= nIter) return;
        const int64_t tile = t0 + it;
        const int slot = it % HNS;
        if (it >= HNS) mbar_wait(smem_u32(&bar_empty[slot]), ((it / HNS) - 1) & 1);
        const uint32_t fb = smem_u32(&bar_full[slot]);
        const uint32_t bytesI = (uint32_t)rowsI * TILE_N * 8, bytesJ = (uint32_t)rowsJ * TILE_N * 8;
        mbar_arrive_expect_tx(fb, bytesI + (diag ? 0u : bytesJ));
        const double* base = Wt + tile * (int64_t)K * TILE_N;
        const uint32_t dst = smem_u32(ring + (size_t)slot * 2 * HPANEL);
        bulk_g2s(dst, base + (int64_t)bi * HB * TILE_N, bytesI, fb);
        if (!diag) bulk_g2s(dst + HPANEL, base + (int64_t)bj * HB * TILE_N, bytesJ, fb);
    };
    if (producer) {
        issue(0);
        issue(1);
    }

    double acc[4][4][2];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b][0] = acc[a][b][1] = 0.0;
    const int fragCol = lane & 3, fragRow = lane >> 2;   // DMMA fragment coordinates of this lane

    for (int it = 0; it < nIter; ++it) {
        const int slot = it % HNS;
        mbar_wait(smem_u32(&bar_full[slot]), (it / HNS) & 1);
        const double* Pi = reinterpret_cast<const double*>(ring + (size_t)slot * 2 * HPANEL);
        const double* Pj = diag ? Pi : Pi + HB * TILE_N;
        const double* Ai = Pi + (wm * 32 + fragRow) * TILE_N;
        const double* Bj = Pj + (wn * 32 + fragRow) * TILE_N;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
            const int col = ((ks ^ fragRow) << 2) + fragCol;      // (4 ks + fragCol) ^ (fragRow << 2)
            double a[4], b[4];
#pragma unroll
            for (int mt = 0; mt < 4; ++mt) a[mt] = Ai[mt * 8 * TILE_N + col];
            if (tri) {
                // symmetric sub-block: the B fragments are the A fragments; only tiles with mt >= nt
#pragma unroll
                for (int mt = 0; mt < 4; ++mt)
#pragma unroll
                    for (int nt = 0; nt <= mt; ++nt) dmma884(acc[mt][nt][0], acc[mt][nt][1], a[mt], a[nt]);
            } else {
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) b[nt] = Bj[nt * 8 * TILE_N + col];
#pragma unroll
                for (int mt = 0; mt < 4; ++mt)
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) dmma884(acc[mt][nt][0], acc[mt][nt][1], a[mt], b[nt]);
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&bar_empty[slot]));
        // refill the slot consumed one iteration ago (every warp has very likely released it by now, so the
        // producer lane does not stall its own warp), keeping two tiles in flight
        if (producer) issue(it + 2);
    }
    // write this CTA's 128 x 128 partial block: Gpart[cta][128][128] (only the tiles this warp computed)
    double* out = Gpart + (size_t)blockIdx.x * HB * HB;
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            if (tri && nt > mt) continue;
            const int row = wm * 32 + mt * 8 + (lane >> 2);
            const int col = wn * 32 + nt * 8 + (lane & 3) * 2;
            out[row * HB + col] = acc[mt][nt][0];
            out[row * HB + col + 1] = acc[mt][nt][1];
        }
}

// Sum the partial blocks of each pair over its CTAs (in order: deterministic) and scatter to the full symmetric
// K x K matrix.  Diagonal pairs hold only the 8 x 8 tiles on or below the diagonal.
__global__ void __launch_bounds__(256)
hessian_big_reduce_kernel(const double* __restrict__ Gpart, int K, const HessSplit split, double* __restrict__ G,
                          const LoopState* loop) {
    if (loop && *reinterpret_cast<const volatile int*>(&loop->done)) return;
    const int pair = blockIdx.x;
    int bi = 0, rem = pair + split.pairBase;
    while (rem > bi) { rem -= bi + 1; ++bi; }
    const int bj = rem;
    const int c0 = split.pairStart[pair], c1 = split.pairStart[pair + 1];
    for (int e = blockIdx.y * blockDim.x + threadIdx.x; e < HB * HB; e += gridDim.y * blockDim.x) {
        const int r = e / HB, cidx = e % HB;
        const int i = bi * HB + r, j = bj * HB + cidx;
        if (i >= K || j >= K) continue;
        if (bi == bj && (r >> 3) < (cidx >> 3)) continue;      // filled by its mirror image below
        double s = 0.0;
        for (int ch = c0; ch < c1; ++ch) s += Gpart[(size_t)ch * HB * HB + e];
        G[(size_t)i * K + j] = s;
        if (bi != bj || (r >> 3) > (cidx >> 3)) G[(size_t)j * K + i] = s;
    }
}

// ------------------------------------------------------------------------------------------------
// Round 2, K <= 64: a pair of warps owns one 32-sample tile (16 samples each) and the whole lower triangle.
// ------------------------------------------------------------------------------------------------
// Ring of NSLOT one-tile slots (K*256 bytes, one bulk copy each).  Pair q of the CTA takes local tiles q, q+4,
// q+8, ...; NSLOT is a multiple of 4, so a pair always reuses its own slots and the even warp of the pair can
// refill a slot as soon as both warps have released it: no CTA-wide barrier in the loop.
// WIN: the tiles come from the weight buffer the fused pass filled (FusedParams::Wout: N_k W_nk, rows
// XOR-swizzled) — no exp, conflict-free fragment loads, the DMMA pipe has the fp64 datapath to itself; otherwise
// they are energies and every lane converts the entries of its own fragment.
template <int KT, bool WIN>
__global__ void __launch_bounds__(256, 1)
hessian_small_kernel(const double* __restrict__ u, const double* __restrict__ Lp, const double* __restrict__ c,
                     const unsigned long long* __restrict__ rowmask, int K, int64_t N, int64_t nTiles, int NSLOT,
                     double* __restrict__ Gpart, const double* __restrict__ sqrtw, const LoopState* loop) {
    if (loop && *reinterpret_cast<const volatile int*>(&loop->done)) return;
    constexpr int KP = KT * 8;                    // padded number of states
    constexpr int NT = KT * (KT + 1) / 2;         // 8 x 8 tiles of the lower triangle
    extern __shared__ __align__(128) unsigned char smem_raw[];
    double* tab = reinterpret_cast<double*>(smem_raw);                      // [32]
    uint64_t* bar_full = reinterpret_cast<uint64_t*>(tab + 32);             // [32]
    uint64_t* bar_empty = bar_full + 32;                                    // [32]
    unsigned char* ring = smem_raw + 1024;                                  // [NSLOT][KP*256]
    const uint32_t slotBytes = KP * TILE_N * 8;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int q = warp >> 1, h = warp & 1;

    const int64_t t0 = nTiles * blockIdx.x / gridDim.x, t1 = nTiles * (blockIdx.x + 1) / gridDim.x;
    const int n = (int)(t1 - t0);
    if (threadIdx.x < 32) tab[threadIdx.x] = MBAR_EXP_TABLE[threadIdx.x];
    if (threadIdx.x == 0) {
        for (int i = 0; i < NSLOT; ++i) {
            mbar_init(smem_u32(&bar_full[i]), 1);
            mbar_init(smem_u32(&bar_empty[i]), 2);
        }
        mbar_fence_init();
    }
    __syncthreads();

    const uint32_t tileBytes = (uint32_t)K * TILE_N * 8;
    auto issue = [&](int j) {          // local tile j -> slot j % NSLOT (caller guarantees the slot is free)
        const int slot = j % NSLOT;
        const uint32_t fb = smem_u32(&bar_full[slot]);
        mbar_arrive_expect_tx(fb, tileBytes);
        bulk_g2s(smem_u32(ring + (size_t)slot * slotBytes), u + (t0 + j) * (int64_t)K * TILE_N, tileBytes, fb);
    };
    if (h == 0 && lane == 0)
        for (int j = q; j < n && j < NSLOT; j += 4) issue(j);

    const int fragCol = lane & 3, fragRow = lane >> 2;
    double cr[KT];
    uint32_t act = 0;
#pragma unroll
    for (int mt = 0; mt < KT; ++mt) {
        const int k = mt * 8 + fragRow;
        const bool a = k < K && (WIN || ((rowmask[k >> 6] >> (k & 63)) & 1ull));
        cr[mt] = (a && !WIN) ? c[k] : 0.0;
        act |= (uint32_t)a << mt;
    }
    double acc[NT][2];
#pragma unroll
    for (int i = 0; i < NT; ++i) acc[i][0] = acc[i][1] = 0.0;

    for (int j = q; j < n; j += 4) {
        const int slot = j % NSLOT;
        const uint32_t par = (uint32_t)(j / NSLOT) & 1u;
        const int64_t tile = t0 + j;
        double Lt = 0.0, swt = 1.0;
        if (!WIN) {
            Lt = Lp[tile * TILE_N + lane];
            if (sqrtw) swt = sqrtw[tile * TILE_N + lane];
        }
        mbar_wait(smem_u32(&bar_full[slot]), par);
        const double* P = reinterpret_cast<const double*>(ring + (size_t)slot * slotBytes);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const int ks = 4 * h + kk;
            const int s = ks * 4 + fragCol;                    // sample of this lane's fragment column
            double a[KT];
            if (WIN) {
                const int col = ((ks ^ fragRow) << 2) + fragCol;   // (4 ks + fragCol) ^ (fragRow << 2)
#pragma unroll
                for (int mt = 0; mt < KT; ++mt) {
                    const double v = P[(mt * 8 + fragRow) * TILE_N + col];
                    a[mt] = ((act >> mt) & 1u) ? v : 0.0;      // rows >= K of the slot were never loaded
                }
            } else {
                const double L = __shfl_sync(0xffffffffu, Lt, s);
                const double sw = __shfl_sync(0xffffffffu, swt, s);
                const bool valid = tile * TILE_N + s < N;
#pragma unroll
                for (int mt = 0; mt < KT; ++mt) {
                    const double v = P[(mt * 8 + fragRow) * TILE_N + s];
                    const double e = sw * exp_fast(fmin(fmax(cr[mt] - v - L, -800.0), 700.0), tab);
                    a[mt] = (valid && ((act >> mt) & 1u)) ? e : 0.0;     // select: garbage rows (k >= K) never count
                }
            }
#pragma unroll
            for (int mt = 0; mt < KT; ++mt)
#pragma unroll
                for (int nt = 0; nt <= mt; ++nt)
                    dmma884(acc[mt * (mt + 1) / 2 + nt][0], acc[mt * (mt + 1) / 2 + nt][1], a[mt], a[nt]);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&bar_empty[slot]));
        if (h == 0 && lane == 0 && j + NSLOT < n) {
            mbar_wait(smem_u32(&bar_empty[slot]), par);      // both warps of the pair are done with this use
            issue(j + NSLOT);
        }
    }
    // deterministic in-CTA reduction over the 8 warps (warp order), then one partial block per CTA
    __syncthreads();
    double* red = reinterpret_cast<double*>(ring);              // [KP][KP]
    for (int w2 = 0; w2 < 8; ++w2) {
        if (warp == w2) {
#pragma unroll
            for (int mt = 0; mt < KT; ++mt)
#pragma unroll
                for (int nt = 0; nt <= mt; ++nt) {
                    const int row = mt * 8 + (lane >> 2), col = nt * 8 + (lane & 3) * 2;
                    const int idx = mt * (mt + 1) / 2 + nt;
                    if (w2 == 0) {
                        red[row * KP + col] = acc[idx][0];
                        red[row * KP + col + 1] = acc[idx][1];
                    } else {
                        red[row * KP + col] += acc[idx][0];
                        red[row * KP + col + 1] += acc[idx][1];
                    }
                }
        }
        __syncthreads();
    }
    double* out = Gpart + (size_t)blockIdx.x * KP * KP;
    for (int e = threadIdx.x; e < KP * KP; e += blockDim.x)
        if (((e / KP) >> 3) >= ((e % KP) >> 3)) out[e] = red[e];
}

__global__ void __launch_bounds__(256)
hessian_small_reduce_kernel(const double* __restrict__ Gpart, int K, int KP, int nCtas, double* __restrict__ G,
                            const LoopState* loop) {
    if (loop && *reinterpret_cast<const volatile int*>(&loop->done)) return;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < KP * KP; e += gridDim.x * blockDim.x) {
        const int i = e / KP, j = e % KP;
        if (i >= K || j >= K || (i >> 3) < (j >> 3)) continue;
        double s = 0.0;
        for (int b = 0; b < nCtas; ++b) s += Gpart[(size_t)b * KP * KP + e];
        G[(size_t)i * K + j] = s;
        if ((i >> 3) > (j >> 3)) G[(size_t)j * K + i] = s;
    }
}

bool ensure_weight_buffer(mbar_b200_ctx* ctx) {
    static const bool forceOld = std::getenv("MBAR_B200_HESSIAN_INPLACE") != nullptr;
    if (forceOld) return false;
    if (ctx->d_Wt) return true;
    if (ctx->wtAllocFailed) return false;
    if (ctx->d_Wt.reserve((size_t)ctx->nTiles * ctx->K * TILE_N, "hessian") != MBAR_B200_OK) {
        ctx->wtAllocFailed = true;
        return false;
    }
    return true;
}

// Requires ctx->d_L (shifted-frame L'_n) from the preceding pass at the same f; d_ch = c_k = f_k + log N_k on
// the device (unsampled rows: f_k when allRows, else ignored).
int launch_hessian_dev(mbar_b200_ctx* ctx, const double* d_ch, bool allRows, LoopState* loop, bool weightsReady) {
    const int K = ctx->K;
    MBAR_REQUIRE(ctx->d_L, MBAR_B200_ERR_NOT_READY, "hessian: per-sample L not available");
    const PassLayout lay{K};
    const unsigned long long* mask = allRows ? ctx->d_onesmask : ctx->d_rowmask;
    static const bool forceOld = std::getenv("MBAR_B200_HESSIAN_INPLACE") != nullptr;
    if (!ctx->capturing) MBAR_CUDA(cudaEventRecord(ctx->evH[0], ctx->stream));
    if (K <= 64 && !forceOld) {
        const int KT = K <= 16 ? 2 : K <= 32 ? 4 : 8;
        const int KP = KT * 8;
        const size_t slotBytes = (size_t)KP * TILE_N * 8;
        int nslot = (int)((200 * 1024) / slotBytes) & ~3;
        if (nslot > 32) nslot = 32;
        int64_t grid = ctx->smCount;
        if (grid > (ctx->nTiles + 3) / 4) grid = (ctx->nTiles + 3) / 4;
        if (grid < 1) grid = 1;
        MBAR_TRY(ctx->d_W.reserve((size_t)grid * KP * KP, "hessian"));
        const size_t smem = 1024 + (size_t)nslot * slotBytes;
        const bool win = weightsReady && !allRows && ctx->d_Wt;
        void (*kern)(const double*, const double*, const double*, const unsigned long long*, int, int64_t, int64_t,
                     int, double*, const double*, const LoopState*) =
            win ? (KT == 2 ? hessian_small_kernel<2, true> : KT == 4 ? hessian_small_kernel<4, true>
                                                                     : hessian_small_kernel<8, true>)
                : (KT == 2 ? hessian_small_kernel<2, false> : KT == 4 ? hessian_small_kernel<4, false>
                                                                      : hessian_small_kernel<8, false>);
        static size_t attr[16][6] = {{0}};
        size_t& a = attr[ctx->device & 15][(KT == 2 ? 0 : KT == 4 ? 1 : 2) + (win ? 3 : 0)];
        if (a < smem) {
            MBAR_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            a = smem;
        }
        if (!ctx->capturing) MBAR_CUDA(cudaEventRecord(ctx->evH[1], ctx->stream));
        kern<<<(unsigned)grid, 256, smem, ctx->stream>>>(win ? ctx->d_Wt : ctx->d_u, ctx->d_L, d_ch, mask, K, ctx->N,
                                                        ctx->nTiles, nslot, ctx->d_W, ctx->d_sqrtw, loop);
        MBAR_CUDA(cudaGetLastError());
        hessian_small_reduce_kernel<<<(KP * KP + 255) / 256, 256, 0, ctx->stream>>>(ctx->d_W, K, KP, (int)grid,
                                                                                    ctx->d_out + lay.G(), loop);
        MBAR_CUDA(cudaGetLastError());
        if (!ctx->capturing) MBAR_CUDA(cudaEventRecord(ctx->evH[2], ctx->stream));
        snprintf(ctx->lastHessKernel, sizeof(ctx->lastHessKernel), "hessian_small_kernel<KT=%d, %s> grid=%lld NSLOT=%d",
                 KT, win ? "weights stored by the fused pass (WST)" : "in-register conversion", (long long)grid, nslot);
        ctx->launches += 2;
        ctx->passes++;
        return MBAR_B200_OK;
    }

    const int nB = (K + HB - 1) / HB;
    const int nPairsAll = nB * (nB + 1) / 2;
    // weight buffer (8*K*N bytes, kept for the life of the context); without it: round-1 in-place kernel
    const bool materialise = !forceOld && ensure_weight_buffer(ctx);
    // CTAs per pair proportional to its cost per tile: off-diagonal 64 DMMA per k-step on the busiest scheduler,
    // diagonal 36 (materialised) | 4 vs 3 (in-place kernel)
    const double wOff = materialise ? 64.0 : 4.0, wDiag = materialise ? 36.0 : 3.0;
    static bool attr[16][2] = {{false}};
    const size_t smem = 512 + (size_t)HNS * 2 * HPANEL;
    if (materialise && !(weightsReady && !allRows)) {
        // (the fused pass at this f normally wrote the weights already: FusedParams::Wout)
        int64_t wgrid = (int64_t)ctx->smCount * 8;
        if (wgrid > ctx->nTiles) wgrid = ctx->nTiles;
        weights_kernel<<<(unsigned)wgrid, 256, 0, ctx->stream>>>(ctx->d_u, ctx->d_L, d_ch, mask, K, ctx->N,
                                                                ctx->nTiles, ctx->d_sqrtw, ctx->d_Wt, loop);
        MBAR_CUDA(cudaGetLastError());
        ctx->launches++;
    }
    if (!ctx->capturing) MBAR_CUDA(cudaEventRecord(ctx->evH[1], ctx->stream));
    // pairs in launches of at most 128 (K <= 2048: one launch; the split table is a kernel parameter)
    int totalCtas = 0;
    for (int base = 0; base < nPairsAll; base += 128) {
        const int nPairs = std::min(128, nPairsAll - base);
        HessSplit split{};
        split.nPairs = nPairs;
        split.pairBase = base;
        std::vector<char> isDiag(nPairs);
        {
            int bi = 0, rem = base;
            while (rem > bi) { rem -= bi + 1; ++bi; }
            int bj = rem;
            for (int p = 0; p < nPairs; ++p) {
                isDiag[p] = (bi == bj);
                if (++bj > bi) { ++bi; bj = 0; }
            }
        }
        double wsum = 0.0;
        for (int p = 0; p < nPairs; ++p) wsum += isDiag[p] ? wDiag : wOff;
        const int total = ctx->smCount > nPairs ? ctx->smCount : nPairs;
        // largest-remainder apportionment of `total` CTAs (every SM gets exactly one CTA when it fits)
        int used = 0;
        std::vector<int> cnt(nPairs);
        std::vector<double> frac(nPairs);
        for (int p = 0; p < nPairs; ++p) {
            const double x = total * (isDiag[p] ? wDiag : wOff) / wsum;
            cnt[p] = (int)x;
            if (cnt[p] < 1) cnt[p] = 1;
            frac[p] = x - (int)x;
            used += cnt[p];
        }
        while (used < total) {
            int best = 0;
            for (int p = 1; p < nPairs; ++p)
                if (frac[p] > frac[best]) best = p;
            cnt[best]++;
            frac[best] = -1.0;
            used++;
        }
        used = 0;
        for (int p = 0; p < nPairs; ++p) {
            if ((int64_t)cnt[p] > ctx->nTiles) cnt[p] = (int)ctx->nTiles;
            split.pairStart[p] = used;
            used += cnt[p];
        }
        split.pairStart[nPairs] = used;
        const int nCtas = used;
        totalCtas += nCtas;
        MBAR_TRY(ctx->d_W.reserve((size_t)nCtas * HB * HB, "hessian"));
        if (materialise) {
            if (!attr[ctx->device & 15][0]) {
                MBAR_CUDA(cudaFuncSetAttribute(hessian_big_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                attr[ctx->device & 15][0] = true;
            }
            hessian_big_kernel<<<nCtas, 512, smem, ctx->stream>>>(ctx->d_Wt, K, ctx->nTiles, split, ctx->d_W, loop);
            MBAR_CUDA(cudaGetLastError());
            hessian_big_reduce_kernel<<<dim3(nPairs, 16), 256, 0, ctx->stream>>>(ctx->d_W, K, split,
                                                                                ctx->d_out + lay.G(), loop);
            MBAR_CUDA(cudaGetLastError());
        } else {
            if (!attr[ctx->device & 15][1]) {
                MBAR_CUDA(cudaFuncSetAttribute(hessian_inplace_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                attr[ctx->device & 15][1] = true;
            }
            hessian_inplace_kernel<<<nCtas, 512, smem, ctx->stream>>>(ctx->d_u, ctx->d_L, d_ch, mask, K, ctx->N,
                                                                     ctx->nTiles, split, ctx->d_W, ctx->d_sqrtw, loop);
            MBAR_CUDA(cudaGetLastError());
            hessian_reduce_kernel<<<dim3(nPairs, 16), 256, 0, ctx->stream>>>(ctx->d_W, K, split, ctx->d_out + lay.G(),
                                                                            loop);
            MBAR_CUDA(cudaGetLastError());
        }
        ctx->launches += 2;
    }
    if (materialise)
        snprintf(ctx->lastHessKernel, sizeof(ctx->lastHessKernel),
                 "%s + hessian_big_kernel (128x128 block pairs: %d, CTAs %d)",
                 (weightsReady && !allRows) ? "weights stored by the fused pass (WST)" : "weights_kernel", nPairsAll,
                 totalCtas);
    else
        snprintf(ctx->lastHessKernel, sizeof(ctx->lastHessKernel), "hessian_inplace_kernel (round 1), CTAs %d", totalCtas);
    if (!ctx->capturing) MBAR_CUDA(cudaEventRecord(ctx->evH[2], ctx->stream));
    ctx->passes++;
    return MBAR_B200_OK;
}

int launch_hessian(mbar_b200_ctx* ctx, const double* h_f, bool allRows, bool weightsReady) {
    const int K = ctx->K;
    // sampled rows carry N_k W_nk (c = f + log N); with allRows the unsampled rows carry W_nk (c = f)
    double* c = ctx->hf(ROW_HESS_C);
    for (int k = 0; k < K; ++k)
        c[k] = std::isinf(ctx->h_logNk[k]) ? (allRows ? h_f[k] : 0.0) : h_f[k] + ctx->h_logNk[k];
    MBAR_CUDA(cudaMemcpyAsync(ctx->dc(ROW_HESS_C), c, (size_t)K * sizeof(double), cudaMemcpyHostToDevice,
                              ctx->stream));
    return launch_hessian_dev(ctx, ctx->dc(ROW_HESS_C), allRows, nullptr, weightsReady);
}

}  // namespace mbar

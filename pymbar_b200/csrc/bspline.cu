// mbar_b200_bspline_*: per-state and weighted sums of B-spline basis functions over resident samples, the only part
// of pymbar's spline free-energy fit that grows with N (fes.py:2102-2306, :1954-2010).  The fit's sample terms are
// linear in the coefficients c: sum_n w_n F(x_n) = sum_i c_i A_i and sum_{n in k} F(x_n) = sum_i c_i S_ki, with
//
//   S_ki = sum_{n: s_n = k} B_i(x_n),   A_i = sum_n w_n B_i(x_n).
//
// B_i are scipy's (BSpline(t, e_i, k), extrapolate=True): the interval l is the last one in [k, nb - 1] whose left
// knot is <= x (clamped to the first and last interval outside [t_k, t_nb]), and the k + 1 nonzero values come from
// scipy's Cox-de Boor triangle in the same fp64 operations, without contraction, so that every basis value is
// scipy's bit for bit (degree 0 included, where the interval alone decides the value).
//
// Decomposition.  Per call, the rows (the A row, then the states) are cut into chunks whose [rows x nb] fp64
// accumulator fits one CTA's shared memory.  Per chunk, CTA g owns a contiguous range of 32-sample tiles (a
// function of N alone) and steps through it, one tile per warp per step.  A warp groups its lanes by (state, first
// basis index) with __match_any_sync, makes each group contiguous, and runs k + 1 rounds: in round r each group adds
// its segmented sum of B_{first + r} to cell (state, first + r), so no two lanes of a round write the same cell.  The
// warps of a CTA write one after the other, so a cell receives its terms in tile order.  The A row is grouped by
// first index alone.  The per-CTA blocks are then summed in CTA order.  There are no atomics: the order of every
// sum is fixed by N and the inputs, so repeat calls, and S-only, A-only or both, give the same bits.  Tiles without a
// sample in a chunk's states are skipped (with the default labels every state's samples are contiguous).
//
// Replicate sums (mbar_b200_bspline_replicate_sums): R_bi = sum_n V_bn B_i(x_n) for B weight rows V uploaded once,
// the sample terms of B bootstrap replicates of the fit.  A pass serves a batch of replicates: each warp evaluates a
// tile's Cox-de Boor triangle once, groups its lanes by first basis index once, and then for every replicate of the
// batch reads 32 consecutive V_bn and adds the segmented sums of V_bn B_{first + a} to its own [batch x nb]
// accumulator, so the warps of a CTA never wait for each other.  Each CTA adds its warps' accumulators in warp order
// and the CTAs are summed in CTA order.  The tiles a warp owns are fixed by N and the warps per CTA by nb, so row b's
// sum is ordered by (N, nb) alone: it does not depend on B, on the batch it falls in or on the other rows.
#include <algorithm>
#include <cmath>
#include <memory>
#include <vector>

#include "internal.cuh"

namespace mbar {

constexpr int BSP_THREADS = 128;
constexpr int BSP_WARPS = BSP_THREADS / 32;
constexpr int BSP_MAX_DEGREE = 7;
constexpr int BSP_ACC_DOUBLES = (108 * 1024) / 8;   // shared accumulator per CTA
constexpr int64_t BSP_MAX_GROUPS = 264;              // CTAs per chunk: two per SM on an H100 SXM
constexpr int BSP_REP_MAX_WARPS = 8;                 // warps per CTA of the replicate kernel (fewer for a large nb)

}  // namespace mbar

struct mbar_b200_bspline : mbar::Resident {
    int64_t N = 0;
    int64_t nTiles = 0;        // ceil(N / 32)
    int K = 0;                 // states (0: no labels)
    int nGroups = 1;           // CTAs per chunk, a function of N alone
    mbar::DevArray<double> d_x;      // [nTiles * 32], 0 in the padding
    mbar::DevArray<double> d_w;      // [nTiles * 32] or NULL
    mbar::DevArray<int32_t> d_s;     // [nTiles * 32], -1 in the padding, or NULL
    mbar::DevArray<int32_t> d_tmin;  // [nTiles] smallest / largest label of a tile (padding excluded)
    mbar::DevArray<int32_t> d_tmax;
    int64_t B = 0;                   // replicate rows uploaded by mbar_b200_bspline_set_replicates
    mbar::DevArray<double> d_V;      // [B][nTiles * 32], 0 in the padding
    int lastChunks = 0;
};

namespace mbar {

struct BspParams {
    const double* x;
    const double* w;
    const int32_t* s;
    const int32_t* tmin;
    const int32_t* tmax;
    const double* t;        // knots [nKnots]
    double* partial;        // [nGroups][rows][nb]
    int64_t N, nTiles;
    int nKnots, nb;
    int nGroups;
    int hasA;               // this chunk's row 0 is A
    int k0, k1;             // states [k0, k1) in rows hasA .. hasA + k1 - k0
    int rows;
};

// The lanes with key >= 0 grouped by key: perm[] gathers each group contiguously (groups in the order of their
// lowest lane, lanes in order within a group).  Returns src (the lane this lane reads in sorted order), and sets
// skey (the sorted key), same (bit s: the lane 2^s below has the same key) and steps.
__device__ __forceinline__ int bsp_sort(int key, int lane, int* perm, int& skey, unsigned& same, int& steps) {
    const unsigned FULL = 0xffffffffu;
    const unsigned grp = __match_any_sync(FULL, key);
    const int leader = __ffs(grp) - 1;
    const int gsize = __popc(grp);
    const int own = (lane == leader) ? gsize : 0;
    int incl = own;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(FULL, incl, d);
        if (lane >= d) incl += y;
    }
    const int start = __shfl_sync(FULL, incl - own, leader);
    perm[start + __popc(grp & ((1u << lane) - 1u))] = lane;
    __syncwarp();
    const int src = perm[lane];
    __syncwarp();
    skey = __shfl_sync(FULL, key, src);
    const int maxg = (int)__reduce_max_sync(FULL, (unsigned)gsize);
    steps = 0;
    while ((1 << steps) < maxg) ++steps;
    same = 0;
    for (int s = 0; s < steps; ++s) {
        const int kd = __shfl_up_sync(FULL, skey, 1 << s);
        if (lane >= (1 << s) && kd == skey) same |= 1u << s;
    }
    return src;
}

// segmented inclusive sum, in sorted order, of v over the lanes' groups
__device__ __forceinline__ double bsp_segsum(double v, int src, unsigned same, int steps) {
    const unsigned FULL = 0xffffffffu;
    v = __shfl_sync(FULL, v, src);
    for (int s = 0; s < steps; ++s) {
        const double y = __shfl_up_sync(FULL, v, 1 << s);
        if ((same >> s) & 1u) v += y;
    }
    return v;
}

// scipy's interval and Cox-de Boor triangle (_bspl.pyx find_interval / _deBoor_D with m = 0), in the same fp64
// operations: h[a] = B_{l - k + a}(x)
template <int KD>
__device__ __forceinline__ int bsp_basis(const double* __restrict__ t, int nKnots, int nb, double x, double* h) {
    // number of knots <= x, by binary search
    int lo = 0, hi = nKnots;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (t[mid] <= x) lo = mid + 1;
        else hi = mid;
    }
    const int l = min(max(lo - 1, KD), nb - 1);
    h[0] = 1.0;
#pragma unroll
    for (int j = 1; j <= KD; ++j) {
        double hh[KD > 0 ? KD : 1];
#pragma unroll
        for (int i = 0; i < j; ++i) hh[i] = h[i];
        h[0] = 0.0;
#pragma unroll
        for (int n = 1; n <= j; ++n) {
            const double xb = t[l + n], xa = t[l + n - j];
            if (xb == xa) {
                h[n] = 0.0;
                continue;
            }
            const double w = __ddiv_rn(hh[n - 1], __dsub_rn(xb, xa));
            h[n - 1] = __dadd_rn(h[n - 1], __dmul_rn(w, __dsub_rn(xb, x)));
            h[n] = __dmul_rn(w, __dsub_rn(x, xa));
        }
    }
    return l - KD;
}

template <int KD>
__global__ void __launch_bounds__(BSP_THREADS) bsp_accum_kernel(BspParams p) {
    extern __shared__ double smem[];
    double* acc = smem;                                 // [rows][nb]
    double* st = smem + (size_t)p.rows * p.nb;          // knots
    __shared__ int perm[BSP_WARPS][32];
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < p.rows * p.nb; i += BSP_THREADS) acc[i] = 0.0;
    for (int i = threadIdx.x; i < p.nKnots; i += BSP_THREADS) st[i] = p.t[i];
    __syncthreads();
    const int64_t g = blockIdx.x;
    const int64_t t0 = g * p.nTiles / p.nGroups, t1 = (g + 1) * p.nTiles / p.nGroups;
    const int sBase = p.hasA;
    for (int64_t base = t0; base < t1; base += BSP_WARPS) {
        const int64_t tile = base + warp;
        bool active = tile < t1;
        if (active && !p.hasA) active = p.tmax[tile] >= p.k0 && p.tmin[tile] < p.k1;
        if (!__syncthreads_or(active)) continue;
        double h[KD + 1];
        int first = 0, keyS = -1, keyA = -1, srcS = 0, srcA = 0, stS = 0, stA = 0, skS = -1, skA = -1;
        unsigned sameS = 0, sameA = 0;
        double wn = 0.0;
        if (active) {
            const int64_t n = tile * TILE_N + lane;
            first = bsp_basis<KD>(st, p.nKnots, p.nb, p.x[n], h);
            const int s = p.s ? p.s[n] : -1;
            if (p.s && s >= p.k0 && s < p.k1) keyS = (s - p.k0) * p.nb + first;
            if (p.hasA && n < p.N) {
                keyA = first;
                wn = p.w[n];
            }
            srcS = bsp_sort(keyS, lane, perm[warp], skS, sameS, stS);
            if (p.hasA) srcA = bsp_sort(keyA, lane, perm[warp], skA, sameA, stA);
        }
        // the warps write one after the other, each tile's k + 1 rounds in order
        for (int wv = 0; wv < BSP_WARPS; ++wv) {
            if (warp == wv && active) {
                // every lane takes part in the shuffles (a full-mask shuffle skipped by one lane never completes)
                const int nextS = __shfl_down_sync(FULL, skS, 1);
                const int nextA = __shfl_down_sync(FULL, skA, 1);
                const bool tailS = (lane == 31) || nextS != skS;
                const bool tailA = (lane == 31) || nextA != skA;
#pragma unroll
                for (int r = 0; r <= KD; ++r) {
                    const double vS = bsp_segsum(keyS >= 0 ? h[r] : 0.0, srcS, sameS, stS);
                    if (tailS && skS >= 0) acc[(size_t)(sBase + skS / p.nb) * p.nb + skS % p.nb + r] += vS;
                    if (p.hasA) {
                        const double vA = bsp_segsum(keyA >= 0 ? __dmul_rn(wn, h[r]) : 0.0, srcA, sameA, stA);
                        if (tailA && skA >= 0) acc[skA + r] += vA;
                    }
                    __syncwarp();
                }
            }
            __syncthreads();
        }
    }
    __syncthreads();
    double* dst = p.partial + g * p.rows * p.nb;
    for (int i = threadIdx.x; i < p.rows * p.nb; i += BSP_THREADS) dst[i] = acc[i];
}

// out rows: row r of the chunk goes to S[(k0 + r - hasA) * nb] or to A; partials summed in CTA order
__global__ void bsp_reduce_kernel(const double* __restrict__ partial, int nGroups, int rows, int nb, int hasA, int k0,
                                  double* __restrict__ S, double* __restrict__ A) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)rows * nb) return;
    double s = 0.0;
    for (int g = 0; g < nGroups; ++g) s += partial[(int64_t)g * rows * nb + i];
    const int r = (int)(i / nb), b = (int)(i % nb);
    if (hasA && r == 0) A[b] = s;
    else S[(int64_t)(k0 + r - hasA) * nb + b] = s;
}

struct BspRepParams {
    const double* x;
    const double* V;        // [B][nPad]
    const double* t;        // knots [nKnots]
    double* partial;        // [nGroups][rows][nb]
    int64_t N, nTiles, nPad;
    int64_t b0;             // first replicate of this pass
    int nKnots, nb;
    int nGroups;
    int rows;               // replicates in this pass
};

// One pass over the samples for replicates [b0, b0 + rows): blockDim.x / 32 warps, each with its own accumulator.
template <int KD>
__global__ void __launch_bounds__(BSP_REP_MAX_WARPS * 32) bsp_replicate_kernel(BspRepParams p) {
    extern __shared__ double smem[];
    __shared__ int perm[BSP_REP_MAX_WARPS][32];
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nWarps = blockDim.x >> 5;
    const int cells = p.rows * p.nb;
    double* st = smem;                                   // knots
    double* acc = smem + p.nKnots;                       // [nWarps][rows][nb]
    for (int i = threadIdx.x; i < nWarps * cells; i += blockDim.x) acc[i] = 0.0;
    for (int i = threadIdx.x; i < p.nKnots; i += blockDim.x) st[i] = p.t[i];
    __syncthreads();
    double* wacc = acc + (size_t)warp * cells;
    const int64_t g = blockIdx.x;
    const int64_t t0 = g * p.nTiles / p.nGroups, t1 = (g + 1) * p.nTiles / p.nGroups;
    for (int64_t tile = t0 + warp; tile < t1; tile += nWarps) {
        const int64_t n = tile * TILE_N + lane;
        double h[KD + 1];
        const int first = bsp_basis<KD>(st, p.nKnots, p.nb, p.x[n], h);
        int skey, steps;
        unsigned same;
        const int src = bsp_sort(n < p.N ? first : -1, lane, perm[warp], skey, same, steps);
        // the basis values in sorted order, once per tile
        double hs[KD + 1];
#pragma unroll
        for (int a = 0; a <= KD; ++a) hs[a] = __shfl_sync(FULL, h[a], src);
        const int next = __shfl_down_sync(FULL, skey, 1);
        const bool tail = skey >= 0 && (lane == 31 || next != skey);
        const double* vrow = p.V + p.b0 * p.nPad + n;
        for (int r = 0; r < p.rows; ++r) {
            const double v = __shfl_sync(FULL, vrow[(int64_t)r * p.nPad], src);
            const int cell = r * p.nb + skey;
#pragma unroll
            for (int a = 0; a <= KD; ++a) {
                double y = __dmul_rn(v, hs[a]);
                // segmented inclusive sum over the sorted groups: the group's last lane holds its total
                for (int s = 0; s < steps; ++s) {
                    const double z = __shfl_up_sync(FULL, y, 1 << s);
                    if ((same >> s) & 1u) y += z;
                }
                if (tail) wacc[cell + a] += y;
                __syncwarp();
            }
        }
    }
    __syncthreads();
    double* dst = p.partial + g * cells;
    for (int i = threadIdx.x; i < cells; i += blockDim.x) {
        double s = 0.0;
        for (int w = 0; w < nWarps; ++w) s += acc[(size_t)w * cells + i];
        dst[i] = s;
    }
}

// out[(b0 + r) * nb + i] = partials of (r, i) summed in CTA order
__global__ void bsp_replicate_reduce_kernel(const double* __restrict__ partial, int nGroups, int cells, int64_t b0,
                                            int nb, double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cells) return;
    double s = 0.0;
    for (int g = 0; g < nGroups; ++g) s += partial[(int64_t)g * cells + i];
    out[b0 * nb + i] = s;
}

typedef void (*BspRepKernelFn)(BspRepParams);

static BspRepKernelFn bsp_replicate_kernel_for(int degree) {
    switch (degree) {
        case 0: return bsp_replicate_kernel<0>;
        case 1: return bsp_replicate_kernel<1>;
        case 2: return bsp_replicate_kernel<2>;
        case 3: return bsp_replicate_kernel<3>;
        case 4: return bsp_replicate_kernel<4>;
        case 5: return bsp_replicate_kernel<5>;
        case 6: return bsp_replicate_kernel<6>;
        default: return bsp_replicate_kernel<7>;
    }
}

typedef void (*BspKernelFn)(BspParams);

static BspKernelFn bsp_kernel_for(int degree) {
    switch (degree) {
        case 0: return bsp_accum_kernel<0>;
        case 1: return bsp_accum_kernel<1>;
        case 2: return bsp_accum_kernel<2>;
        case 3: return bsp_accum_kernel<3>;
        case 4: return bsp_accum_kernel<4>;
        case 5: return bsp_accum_kernel<5>;
        case 6: return bsp_accum_kernel<6>;
        default: return bsp_accum_kernel<7>;
    }
}

}  // namespace mbar

using namespace mbar;

int mbar_b200_bspline_create(int device, int64_t N, const double* x, const double* w, const int32_t* s, int32_t K,
                             mbar_b200_bspline** out) {
    MBAR_REQUIRE(out && x, MBAR_B200_ERR_INVALID, "bspline_create: NULL argument");
    *out = nullptr;
    MBAR_REQUIRE(N >= 1, MBAR_B200_ERR_INVALID, "bspline_create: N=%lld must be >= 1", (long long)N);
    MBAR_REQUIRE(!s || K >= 1, MBAR_B200_ERR_INVALID, "bspline_create: K=%d must be >= 1 with labels", (int)K);
    for (int64_t n = 0; n < N; ++n) {
        MBAR_REQUIRE(!w || (w[n] >= 0.0 && w[n] < INFINITY), MBAR_B200_ERR_INVALID,
                     "bspline_create: weight %lld is %g (negative, NaN or infinite)", (long long)n, w ? w[n] : 0.0);
        MBAR_REQUIRE(!s || (s[n] >= 0 && s[n] < K), MBAR_B200_ERR_INVALID, "bspline_create: label %lld is %d, outside "
                     "[0, %d)", (long long)n, s ? (int)s[n] : 0, (int)K);
        MBAR_REQUIRE(std::isfinite(x[n]), MBAR_B200_ERR_NAN, "bspline_create: x[%lld] is %g", (long long)n, x[n]);
    }
    MBAR_TRY(open_device(device, nullptr));
    std::unique_ptr<mbar_b200_bspline> b(new mbar_b200_bspline());
    b->N = N;
    b->nTiles = (N + TILE_N - 1) / TILE_N;
    b->K = s ? K : 0;
    b->nGroups = (int)std::max<int64_t>(1, std::min<int64_t>(BSP_MAX_GROUPS, b->nTiles / 4));
    const int64_t nPad = b->nTiles * TILE_N;
    std::vector<double> hx((size_t)nPad, 0.0);
    std::copy(x, x + N, hx.begin());
    std::vector<double> hw;
    std::vector<int32_t> hs, tmin, tmax;
    if (w) {
        hw.assign((size_t)nPad, 0.0);
        std::copy(w, w + N, hw.begin());
    }
    if (s) {
        hs.assign((size_t)nPad, -1);
        std::copy(s, s + N, hs.begin());
        tmin.assign((size_t)b->nTiles, INT32_MAX);
        tmax.assign((size_t)b->nTiles, -1);
        for (int64_t n = 0; n < N; ++n) {
            tmin[n / TILE_N] = std::min(tmin[n / TILE_N], s[n]);
            tmax[n / TILE_N] = std::max(tmax[n / TILE_N], s[n]);
        }
    }
    const char* who = "bspline_create";
    MBAR_TRY(b->open(device, who));
    MBAR_TRY(b->upload(b->d_x, hx.data(), hx.size(), who));
    if (w) MBAR_TRY(b->upload(b->d_w, hw.data(), hw.size(), who));
    if (s) {
        MBAR_TRY(b->upload(b->d_s, hs.data(), hs.size(), who));
        MBAR_TRY(b->upload(b->d_tmin, tmin.data(), tmin.size(), who));
        MBAR_TRY(b->upload(b->d_tmax, tmax.data(), tmax.size(), who));
    }
    *out = b.release();
    return MBAR_B200_OK;
}

int mbar_b200_bspline_destroy(mbar_b200_bspline* b) { return destroy_resident(b); }

// The degree and knot checks of mbar_b200_bspline_moments and mbar_b200_bspline_replicate_sums.
static int bsp_check_knots(const char* fn, int32_t degree, int64_t n_knots, const double* t) {
    MBAR_REQUIRE(degree >= 0 && degree <= BSP_MAX_DEGREE, MBAR_B200_ERR_INVALID, "%s: degree %d outside [0, %d]", fn,
                 (int)degree, BSP_MAX_DEGREE);
    MBAR_REQUIRE(t, MBAR_B200_ERR_INVALID, "%s: NULL knots", fn);
    MBAR_REQUIRE(n_knots >= 2 * (int64_t)(degree + 1), MBAR_B200_ERR_INVALID,
                 "%s: %lld knots, degree %d needs at least %d", fn, (long long)n_knots, (int)degree, 2 * (degree + 1));
    for (int64_t i = 0; i < n_knots; ++i) {
        MBAR_REQUIRE(std::isfinite(t[i]), MBAR_B200_ERR_INVALID, "%s: knot %lld is %g", fn, (long long)i, t[i]);
        MBAR_REQUIRE(i == 0 || t[i] >= t[i - 1], MBAR_B200_ERR_INVALID, "%s: knots decrease at %lld", fn,
                     (long long)i);
    }
    const int64_t nb64 = n_knots - degree - 1;
    MBAR_REQUIRE(t[degree] < t[nb64], MBAR_B200_ERR_INVALID, "%s: t[k] = t[nb] = %g (empty base interval)", fn,
                 t[degree]);
    MBAR_REQUIRE(nb64 <= BSP_ACC_DOUBLES - n_knots, MBAR_B200_ERR_INVALID,
                 "%s: %lld basis functions exceed one accumulator", fn, (long long)nb64);
    return MBAR_B200_OK;
}

int mbar_b200_bspline_moments(mbar_b200_bspline* b, int32_t degree, int64_t n_knots, const double* t, double* S,
                              double* A) {
    MBAR_REQUIRE(b, MBAR_B200_ERR_INVALID, "bspline_moments: NULL object");
    MBAR_TRY(bsp_check_knots("bspline_moments", degree, n_knots, t));
    const int64_t nb64 = n_knots - degree - 1;
    MBAR_REQUIRE(!S || b->d_s, MBAR_B200_ERR_INVALID, "bspline_moments: S requested but no labels were uploaded");
    MBAR_REQUIRE(!A || b->d_w, MBAR_B200_ERR_INVALID, "bspline_moments: A requested but no weights were uploaded");
    MBAR_REQUIRE((int64_t)b->K * nb64 < INT32_MAX, MBAR_B200_ERR_INVALID, "bspline_moments: K * nb too large");
    const int nb = (int)nb64, nk = (int)n_knots;
    if (!S && !A) return MBAR_B200_OK;
    MBAR_CUDA(cudaSetDevice(b->device));
    NvtxRange nvtx_("mbar_b200::bspline_moments");
    const int Kw = S ? b->K : 0;
    const int totalRows = (A ? 1 : 0) + Kw;
    const int rowsPer = std::max(1, std::min(totalRows, (BSP_ACC_DOUBLES - nk) / nb));
    CallBuffers buf("bspline");
    double *d_t, *d_partial, *d_S = nullptr, *d_A = nullptr;
    MBAR_TRY(buf.alloc(&d_t, (size_t)nk));
    MBAR_TRY(buf.alloc(&d_partial, (size_t)b->nGroups * rowsPer * nb));
    if (S) MBAR_TRY(buf.alloc(&d_S, (size_t)Kw * nb));
    if (A) MBAR_TRY(buf.alloc(&d_A, (size_t)nb));
    MBAR_CUDA(cudaMemcpyAsync(d_t, t, (size_t)nk * sizeof(double), cudaMemcpyHostToDevice, b->stream));
    const BspKernelFn fn = bsp_kernel_for(degree);
    const size_t smem = ((size_t)rowsPer * nb + nk) * sizeof(double);
    MBAR_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    BspParams p{};
    p.x = b->d_x;
    p.w = b->d_w;
    p.s = b->d_s;
    p.tmin = b->d_tmin;
    p.tmax = b->d_tmax;
    p.t = d_t;
    p.partial = d_partial;
    p.N = b->N;
    p.nTiles = b->nTiles;
    p.nKnots = nk;
    p.nb = nb;
    p.nGroups = b->nGroups;
    MBAR_CUDA(cudaEventRecord(b->ev0, b->stream));
    int chunks = 0;
    // chunk c holds rows [r0, r0 + rows) of (A, states 0..Kw-1)
    for (int r0 = 0; r0 < totalRows; r0 += rowsPer) {
        const int rows = std::min(rowsPer, totalRows - r0);
        p.hasA = (A && r0 == 0) ? 1 : 0;
        p.k0 = r0 - (A ? 1 : 0) + p.hasA;
        p.k1 = p.k0 + rows - p.hasA;
        p.rows = rows;
        fn<<<b->nGroups, BSP_THREADS, smem, b->stream>>>(p);
        const int64_t cells = (int64_t)rows * nb;
        bsp_reduce_kernel<<<(unsigned)((cells + 255) / 256), 256, 0, b->stream>>>(d_partial, b->nGroups, rows, nb,
                                                                                 p.hasA, p.k0, d_S, d_A);
        MBAR_CUDA(cudaGetLastError());
        ++chunks;
    }
    MBAR_CUDA(cudaEventRecord(b->ev1, b->stream));
    if (S) MBAR_CUDA(cudaMemcpyAsync(S, d_S, (size_t)Kw * nb * sizeof(double), cudaMemcpyDeviceToHost, b->stream));
    if (A) MBAR_CUDA(cudaMemcpyAsync(A, d_A, (size_t)nb * sizeof(double), cudaMemcpyDeviceToHost, b->stream));
    MBAR_CUDA(cudaStreamSynchronize(b->stream));
    float e = 0.f;
    b->lastMs = event_ms(b->ev0, b->ev1, &e) ? e : 0.0;
    b->lastChunks = chunks;
    return MBAR_B200_OK;
}

int mbar_b200_bspline_set_replicates(mbar_b200_bspline* b, int64_t B, const double* V_host) {
    MBAR_REQUIRE(b, MBAR_B200_ERR_INVALID, "bspline_set_replicates: NULL object");
    MBAR_CUDA(cudaSetDevice(b->device));
    // a failed upload leaves no replicates
    if (b->d_V) {
        cudaStreamSynchronize(b->stream);
        b->d_V.reset();
    }
    b->B = 0;
    MBAR_TRY(check_replicate_weights("bspline_set_replicates", B, b->N, V_host));
    const int64_t N = b->N, nPad = b->nTiles * TILE_N;
    MBAR_TRY(b->d_V.reserve((size_t)B * nPad, "bspline_set_replicates"));
    // rows of N into rows of nPad, the padding zeroed
    bool ok = cudaMemcpy2DAsync(b->d_V, nPad * sizeof(double), V_host, N * sizeof(double), N * sizeof(double),
                                (size_t)B, cudaMemcpyHostToDevice, b->stream) == cudaSuccess;
    if (ok && nPad > N)
        ok = cudaMemset2DAsync(b->d_V + N, nPad * sizeof(double), 0, (nPad - N) * sizeof(double), (size_t)B,
                               b->stream) == cudaSuccess;
    if (!ok || cudaStreamSynchronize(b->stream) != cudaSuccess) {
        set_error("bspline_set_replicates: %s", cudaGetErrorString(cudaGetLastError()));
        b->d_V.reset();
        return MBAR_B200_ERR_CUDA;
    }
    b->B = B;
    return MBAR_B200_OK;
}

int mbar_b200_bspline_replicate_sums(mbar_b200_bspline* b, int32_t degree, int64_t n_knots, const double* t,
                                     double* out) {
    MBAR_REQUIRE(b, MBAR_B200_ERR_INVALID, "bspline_replicate_sums: NULL object");
    MBAR_TRY(bsp_check_knots("bspline_replicate_sums", degree, n_knots, t));
    MBAR_REQUIRE(out, MBAR_B200_ERR_INVALID, "bspline_replicate_sums: NULL output");
    MBAR_REQUIRE(b->d_V && b->B >= 1, MBAR_B200_ERR_NOT_READY, "bspline_replicate_sums: no replicates uploaded");
    const int nb = (int)(n_knots - degree - 1), nk = (int)n_knots;
    MBAR_CUDA(cudaSetDevice(b->device));
    NvtxRange nvtx_("mbar_b200::bspline_replicate_sums");
    // warps per CTA from nb alone (each warp holds a [rows x nb] accumulator), then as many replicates per pass as
    // the shared accumulator holds
    int warps = BSP_REP_MAX_WARPS;
    while (warps > 1 && (int64_t)warps * nb + nk > BSP_ACC_DOUBLES) warps >>= 1;
    const int rowsPer = (int)std::max<int64_t>(1, std::min<int64_t>(b->B, (BSP_ACC_DOUBLES - nk) / ((int64_t)warps * nb)));
    CallBuffers buf("bspline");
    double *d_t, *d_partial, *d_out;
    MBAR_TRY(buf.alloc(&d_t, (size_t)nk));
    MBAR_TRY(buf.alloc(&d_partial, (size_t)b->nGroups * rowsPer * nb));
    MBAR_TRY(buf.alloc(&d_out, (size_t)b->B * nb));
    MBAR_CUDA(cudaMemcpyAsync(d_t, t, (size_t)nk * sizeof(double), cudaMemcpyHostToDevice, b->stream));
    const BspRepKernelFn fn = bsp_replicate_kernel_for(degree);
    const size_t smem = ((size_t)warps * rowsPer * nb + nk) * sizeof(double);
    MBAR_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    BspRepParams p{};
    p.x = b->d_x;
    p.V = b->d_V;
    p.t = d_t;
    p.partial = d_partial;
    p.N = b->N;
    p.nTiles = b->nTiles;
    p.nPad = b->nTiles * TILE_N;
    p.nKnots = nk;
    p.nb = nb;
    p.nGroups = b->nGroups;
    MBAR_CUDA(cudaEventRecord(b->ev0, b->stream));
    int passes = 0;
    for (int64_t b0 = 0; b0 < b->B; b0 += rowsPer) {
        p.b0 = b0;
        p.rows = (int)std::min<int64_t>(rowsPer, b->B - b0);
        fn<<<b->nGroups, warps * 32, smem, b->stream>>>(p);
        const int cells = p.rows * nb;
        bsp_replicate_reduce_kernel<<<(unsigned)((cells + 255) / 256), 256, 0, b->stream>>>(d_partial, b->nGroups,
                                                                                           cells, b0, nb, d_out);
        MBAR_CUDA(cudaGetLastError());
        ++passes;
    }
    MBAR_CUDA(cudaEventRecord(b->ev1, b->stream));
    MBAR_CUDA(cudaMemcpyAsync(out, d_out, (size_t)b->B * nb * sizeof(double), cudaMemcpyDeviceToHost, b->stream));
    MBAR_CUDA(cudaStreamSynchronize(b->stream));
    float e = 0.f;
    b->lastMs = event_ms(b->ev0, b->ev1, &e) ? e : 0.0;
    b->lastChunks = passes;
    return MBAR_B200_OK;
}

int mbar_b200_last_bspline_stats(mbar_b200_bspline* b, double* ms, int32_t* chunks) {
    MBAR_REQUIRE(b, MBAR_B200_ERR_INVALID, "NULL bspline object");
    if (ms) *ms = b->lastMs;
    if (chunks) *chunks = b->lastChunks;
    return MBAR_B200_OK;
}

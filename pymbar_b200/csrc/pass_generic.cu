// Generic streaming pass: any K (<= 8192), any spread of f_k, log-domain sums for unsampled states.
//
// This is the robust kernel: exact per-sample max, three sweeps over the tile through L1/L2.  It is
// the fallback of the fused kernel (pass_fused.cu) and the ONLY kernel that produces values for
// states with N_k == 0 — the final all-state self-consistent update of mbar_solvers.py:1012, where
// the numerators exp(f_k - u_kn - L_n) of an unsampled state are unbounded and the reference uses a
// second logsumexp over n (mbar_solvers.py:240).
//
// Quantities (shifted frame u' = u - x_n, L' = L + x_n; W is invariant):
//   L'_n = log sum_{k sampled} exp(c_k - u'_kn),  c_k = f_k + log N_k         mbar_solvers.py:238
//   sampled k:    S_k = (1/N_k) sum_n exp(c_k - u'_kn - L'_n)                 = sum_n W_nk
//   unsampled k:  logS_k = logsumexp_n(f_k - u'_kn - L'_n)                    = log sum_n W_nk
#include <cmath>

#include "internal.cuh"

namespace mbar {

__device__ __forceinline__ bool row_active(const unsigned long long* __restrict__ mask, int k) {
    return (mask[k >> 6] >> (k & 63)) & 1ull;
}

template <bool kNeedUnsampled>
__global__ void __launch_bounds__(256)
pass_generic_kernel(const double* __restrict__ u, int K, int64_t N, int64_t nTiles,
                    const double* __restrict__ c, const double* __restrict__ f,
                    const unsigned long long* __restrict__ rowmask,
                    const unsigned long long* __restrict__ linmask,
                    const double* __restrict__ Nk, double* __restrict__ partial,
                    double* __restrict__ out, unsigned int* __restrict__ ticket,
                    double* __restrict__ Lout, const double* __restrict__ wgt, int warpsPerCta) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* tab = reinterpret_cast<double*>(smem_raw);                 // [32]
    double* trans = tab + 32;                                          // [W][32*33]
    double* acc = trans + (size_t)warpsPerCta * 32 * 33;               // [W][K][2]
    __shared__ double s_sumL[8];
    __shared__ bool s_last;

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int W = warpsPerCta;
    if (threadIdx.x < 32) tab[threadIdx.x] = MBAR_EXP_TABLE[threadIdx.x];
    for (int i = threadIdx.x; i < W * K; i += blockDim.x) {
        const int k = i % K;
        const bool act = row_active(linmask, k);
        acc[2 * i] = act ? 0.0 : -INFINITY;
        acc[2 * i + 1] = 0.0;
    }
    __syncthreads();

    double sumL = 0.0;
    double* T = trans + (size_t)warp * 32 * 33;
    double* A = acc + (size_t)warp * K * 2;
    for (int64_t tile = (int64_t)blockIdx.x * W + warp; tile < nTiles; tile += (int64_t)gridDim.x * W) {
        const double* tp = u + tile * (int64_t)K * TILE_N + lane;
        const bool valid = tile * TILE_N + lane < N;
        const double wn = wgt ? __ldg(wgt + tile * TILE_N + lane) : 1.0;   // bootstrap multiplicity
        const double logwn = wgt ? log(wn) : 0.0;
        // Sweeps 1 and 2 (per-sample max, then the shifted sum) with 8 rows in flight per thread: this kernel is
        // bound by the bytes it keeps in flight, not by its arithmetic.  `c` carries -1e300 for rows that do not
        // enter the denominator, so no mask is consulted here (exp(-1e300 - ...) is clamped to e^-800 = 0).
        double m = -INFINITY;
        int k = 0;
        for (; k + 8 <= K; k += 8) {
            double v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = tp[(int64_t)(k + i) * TILE_N];
#pragma unroll
            for (int i = 0; i < 8; ++i) m = fmax(m, __ldg(c + k + i) - v[i]);
        }
        for (; k < K; ++k) m = fmax(m, __ldg(c + k) - tp[(int64_t)k * TILE_N]);
        double D = 0.0;
        k = 0;
        for (; k + 8 <= K; k += 8) {
            double v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = tp[(int64_t)(k + i) * TILE_N];
#pragma unroll
            for (int i = 0; i < 8; ++i) D += exp_fast(fmax(__ldg(c + k + i) - v[i] - m, -800.0), tab);
        }
        for (; k < K; ++k) D += exp_fast(fmax(__ldg(c + k) - tp[(int64_t)k * TILE_N] - m, -800.0), tab);
        const double Lp = m + log(D);
        if (Lout) Lout[tile * TILE_N + lane] = Lp;
        if (valid) sumL += wn * Lp;
        for (int k0 = 0; k0 < K; k0 += 32) {
            const int kmax = min(32, K - k0);
            for (int kb = 0; kb < kmax; kb += 8) {
                double uv8[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) uv8[i] = (kb + i < kmax) ? tp[(int64_t)(k0 + kb + i) * TILE_N] : 0.0;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int kk = kb + i;
                    if (kk < kmax) {
                        const int k = k0 + kk;
                        const double uv = uv8[i];
                        double val;
                        if (row_active(linmask, k))
                            val = valid ? wn * exp_fast(fmax(__ldg(c + k) - uv - Lp, -800.0), tab) : 0.0;
                        else
                            val = (kNeedUnsampled && valid) ? (__ldg(f + k) - uv - Lp + logwn) : -INFINITY;
                        T[kk * 33 + lane] = val;
                    }
                }
            }
            __syncwarp();
            const int k = k0 + lane;
            if (k < K) {
                if (row_active(linmask, k)) {
                    double s = 0.0;
#pragma unroll 8
                    for (int j = 0; j < 32; ++j) s += T[lane * 33 + j];
                    A[2 * k] += s;
                } else if (kNeedUnsampled) {
                    double mx = -INFINITY;
                    for (int j = 0; j < 32; ++j) mx = fmax(mx, T[lane * 33 + j]);
                    if (mx > -INFINITY) {
                        if (mx == INFINITY) {  // +inf log-weight: saturate
                            A[2 * k] = INFINITY;
                            A[2 * k + 1] = 1.0;
                        } else {
                            double s = 0.0;
                            for (int j = 0; j < 32; ++j) s += exp(T[lane * 33 + j] - mx);
                            const double M = A[2 * k], a = A[2 * k + 1];
                            if (M == -INFINITY) {
                                A[2 * k] = mx;
                                A[2 * k + 1] = s;
                            } else if (mx > M) {
                                A[2 * k + 1] = a * exp(M - mx) + s;
                                A[2 * k] = mx;
                            } else {
                                A[2 * k + 1] = a + s * exp(mx - M);
                            }
                        }
                    }
                }
            }
            __syncwarp();
        }
    }
    sumL = warp_sum(sumL);
    if (lane == 0) s_sumL[warp] = sumL;
    __syncthreads();

    // merge the warps of this CTA -> partial[cta][0..K) = S or M, [K..2K) = A, [2K] = sumL
    double* P = partial + (size_t)blockIdx.x * (3 * (size_t)K + 2);
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        if (row_active(linmask, k)) {
            double s = 0.0;
            for (int w = 0; w < W; ++w) s += acc[((size_t)w * K + k) * 2];
            P[k] = s;
            P[K + k] = 0.0;
        } else {
            double M = -INFINITY;
            for (int w = 0; w < W; ++w) M = fmax(M, acc[((size_t)w * K + k) * 2]);
            double a = 0.0;
            if (M > -INFINITY && M < INFINITY)
                for (int w = 0; w < W; ++w) {
                    const double Mw = acc[((size_t)w * K + k) * 2];
                    if (Mw > -INFINITY) a += acc[((size_t)w * K + k) * 2 + 1] * exp(Mw - M);
                }
            else if (M == INFINITY)
                a = 1.0;
            P[k] = M;
            P[K + k] = a;
        }
    }
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < W; ++w) t += s_sumL[w];
        P[2 * K] = t;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicInc(ticket, gridDim.x - 1);  // wraps to 0 after the last CTA
        s_last = (prev == gridDim.x - 1);
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    // last CTA: deterministic reduction over CTAs in index order
    const PassLayout lay{K};
    const size_t stride = 3 * (size_t)K + 2;
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        if (row_active(linmask, k)) {
            double s = 0.0;
            for (unsigned b = 0; b < gridDim.x; ++b) s += partial[b * stride + k];
            out[lay.S() + k] = s / Nk[k];
            out[lay.logS() + k] = 0.0;
        } else {
            double M = -INFINITY;
            for (unsigned b = 0; b < gridDim.x; ++b) M = fmax(M, partial[b * stride + k]);
            double a = 0.0;
            if (M > -INFINITY && M < INFINITY) {
                for (unsigned b = 0; b < gridDim.x; ++b) {
                    const double Mb = partial[b * stride + k];
                    if (Mb > -INFINITY) a += partial[b * stride + K + k] * exp(Mb - M);
                }
            } else if (M == INFINITY) {
                a = 1.0;
            }
            out[lay.S() + k] = 0.0;
            out[lay.logS() + k] = (M > -INFINITY) ? M + log(a) : -INFINITY;
        }
    }
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (unsigned b = 0; b < gridDim.x; ++b) t += partial[b * stride + 2 * K];
        out[lay.sumL()] = t;
        out[lay.flag()] = 0.0;
    }
}

int launch_pass_generic(mbar_b200_ctx* ctx, const double* h_f, bool wantL, bool logAll) {
    const int K = ctx->K;
    // c (sampled) and f (all) to the device
    double* c = ctx->hf(ROW_C);
    double* f = ctx->hf(ROW_GEN_F);
    for (int k = 0; k < K; ++k) {
        const double fk = h_f[k];
        c[k] = std::isinf(ctx->h_logNk[k]) ? -1.0e300 : fk + ctx->h_logNk[k];   // (-1e300: not in the denominator)
        f[k] = fk;
    }
    static_assert(ROW_GEN_F == ROW_C + 1, "one copy uploads c and f");
    MBAR_CUDA(cudaMemcpyAsync(ctx->dc(ROW_C), c, 2 * (size_t)K * sizeof(double), cudaMemcpyHostToDevice,
                              ctx->stream));
    ctx->h2dBytes += 2 * K * 8;
    const size_t perWarp = 32 * 33 * 8 + (size_t)K * 16;
    int W = (int)((200 * 1024 - 256) / perWarp);
    if (W > 8) W = 8;
    MBAR_REQUIRE(W >= 1, MBAR_B200_ERR_INVALID, "K=%d too large for the generic kernel", K);
    const size_t smem = 256 + (size_t)W * perWarp;
    const bool needUnsampled = logAll || (int)ctx->active.size() < K;
    if (wantL) MBAR_TRY(ensure_L(ctx));
    int64_t grid = (ctx->nTiles + W - 1) / W;
    const int64_t maxGrid = (int64_t)ctx->smCount * (smem > 100 * 1024 ? 1 : 2);
    if (grid > maxGrid) grid = maxGrid;
    if (grid > MAX_GRID) grid = MAX_GRID;
    auto kern = needUnsampled ? pass_generic_kernel<true> : pass_generic_kernel<false>;
    MBAR_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    snprintf(ctx->lastKernel, sizeof(ctx->lastKernel), "pass_generic_kernel<%s> grid=%lld warps=%d",
             needUnsampled ? "log-domain rows" : "linear rows", (long long)grid, W);
    MBAR_CUDA(cudaEventRecord(ctx->ev0, ctx->stream));
    kern<<<(unsigned)grid, W * 32, smem, ctx->stream>>>(ctx->d_u, K, ctx->N, ctx->nTiles, ctx->dc(ROW_C),
                                                       ctx->dc(ROW_GEN_F), ctx->d_rowmask,
                                                       logAll ? ctx->d_zeromask : ctx->d_rowmask, ctx->d_Nk,
                                                       ctx->d_partial, ctx->d_out, ctx->d_ticket,
                                                       wantL ? ctx->d_L.ptr : nullptr, ctx->d_wgt, W);
    MBAR_CUDA(cudaEventRecord(ctx->ev1, ctx->stream));
    ctx->launches++;
    ctx->passes++;
    MBAR_CUDA(cudaGetLastError());
    return MBAR_B200_OK;
}

}  // namespace mbar

// mbar_log_W_nk / mbar_W_nk (mbar_solvers.py:439-507): logW[n, k] = f_k - u_kn - L_n, [N, K] row-major.
// Reads the tile-major u' once (+ the stored L'_n) and writes the transposed [N, K] layout through a
// 32 x 33 shared-memory transposition buffer per warp, so both the read and the write are coalesced.
#include <sys/mman.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <thread>
#include <vector>

#include "internal.cuh"

namespace mbar {

__global__ void __launch_bounds__(128)
logw_kernel(const double* __restrict__ u, const double* __restrict__ Lp, const double* __restrict__ f,
            int K, int64_t N, int64_t tile0, double* __restrict__ out, int expo) {
    __shared__ double T[4][32 * 33];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t tile = tile0 + blockIdx.x;
    const double* tp = u + tile * (int64_t)K * TILE_N + lane;
    const double L = Lp[tile * TILE_N + lane];
    double* t = T[warp];
    for (int k0 = warp * 32; k0 < K; k0 += 4 * 32) {
        const int kmax = min(32, K - k0);
        for (int kk = 0; kk < kmax; ++kk) {
            const double uu = tp[(int64_t)(k0 + kk) * TILE_N];
            // energies clamped at upload (+inf in the caller's array) have weight exactly 0, as in the reference
            double v = (uu >= U_CLAMP) ? -INFINITY : f[k0 + kk] - uu - L;
            if (expo) v = exp(v);
            t[kk * 33 + lane] = v;
        }
        __syncwarp();
        if (lane < kmax) {
            for (int n = 0; n < 32; ++n) {
                const int64_t row = (int64_t)blockIdx.x * TILE_N + n;       // row inside this chunk
                if (tile * TILE_N + n < N) out[row * K + k0 + lane] = t[lane * 33 + n];
            }
        }
        __syncwarp();
    }
}

// Requires ctx->d_L from a pass at the same f.  Streams rows [n0, n0 + n) of the [N, K] result to the host in
// chunks (n0 must be a multiple of 32).  A pinned destination is written by DMA directly; a pageable one (what
// numpy hands over) goes through two pinned staging buffers that several host threads drain in parallel while the
// next chunk is computed and copied — the driver's own pageable path is a single synchronous bounce.
int launch_logw(mbar_b200_ctx* ctx, const double* h_f, double* logW_host, int64_t ld, int expo, int64_t n0,
                int64_t n) {
    const int K = ctx->K;
    MBAR_REQUIRE(ctx->d_L, MBAR_B200_ERR_NOT_READY, "log_W: per-sample L not available");
    MBAR_TRY(check_unsampled_clamp(ctx));
    MBAR_REQUIRE(n0 >= 0 && n >= 1 && n0 + n <= ctx->N && n0 % TILE_N == 0, MBAR_B200_ERR_INVALID,
                 "log_W rows [%lld, +%lld): n0 must be a multiple of 32 inside [0, N)", (long long)n0, (long long)n);
    NvtxRange nvtx_("mbar_b200::log_W download");
    std::memcpy(ctx->hf(ROW_LOGW_F), h_f, (size_t)K * sizeof(double));
    MBAR_CUDA(cudaMemcpyAsync(ctx->dc(ROW_LOGW_F), ctx->hf(ROW_LOGW_F), (size_t)K * sizeof(double),
                              cudaMemcpyHostToDevice, ctx->stream));
    cudaPointerAttributes attr;
    bool pinnedDst = false;
    if (cudaPointerGetAttributes(&attr, logW_host) == cudaSuccess)
        pinnedDst = (attr.type == cudaMemoryTypeHost);
    else
        cudaGetLastError();
#if defined(MADV_HUGEPAGE)
    if (!pinnedDst) {
        // a freshly allocated destination is faulted in page by page while it is filled: ask for huge pages
        const uintptr_t a0 = (reinterpret_cast<uintptr_t>(logW_host) + 4095) & ~(uintptr_t)4095;
        const uintptr_t a1 = (reinterpret_cast<uintptr_t>(logW_host + (n - 1) * ld + K)) & ~(uintptr_t)4095;
        if (a1 > a0 + (8u << 20)) madvise(reinterpret_cast<void*>(a0), a1 - a0, MADV_HUGEPAGE);
    }
#endif
    const int64_t tileFirst = n0 / TILE_N;
    const int64_t tilesTotal = (n + TILE_N - 1) / TILE_N;
    int64_t tilesPerChunk = (64ll << 20) / ((int64_t)K * TILE_N * 8);
    if (tilesPerChunk < 1) tilesPerChunk = 1;
    if (tilesPerChunk > tilesTotal) tilesPerChunk = tilesTotal;
    const size_t chunkElems = (size_t)tilesPerChunk * TILE_N * K;
    DevArray<double> d_out[2];
    HostPinned<double> h_stage[2];
    for (int i = 0; i < 2; ++i) {
        MBAR_TRY(d_out[i].reserve(chunkElems, "log_W"));
        if (!pinnedDst) MBAR_TRY(h_stage[i].reserve(chunkElems, "log_W", ctx->device));
    }
    Events done;
    MBAR_TRY(done.create(2, cudaEventDisableTiming));
    StreamDrain guard{ctx};
    int rc = MBAR_B200_OK;
    struct Pending { int64_t row0 = 0, rows = 0; bool live = false; } pend[2];
    // drain staging buffer `b` into the caller's (pageable) array with several threads
    auto drain = [&](int b) {
        if (!pend[b].live) return;
        cudaEventSynchronize(done[b]);
        const int64_t rows = pend[b].rows;
        double* dst = logW_host + (pend[b].row0 - n0) * ld;
        const double* src = h_stage[b];
        const int64_t rowsPer = std::max<int64_t>(1, (128 * 1024) / ((int64_t)K * 8));     // ~128 KB per task
        const int nTasks = (int)((rows + rowsPer - 1) / rowsPer);
        host_parallel(nTasks, [&](int t) {
            const int64_t r0 = (int64_t)t * rowsPer, r1 = std::min(rows, r0 + rowsPer);
            if (ld == K) {
                std::memcpy(dst + r0 * K, src + r0 * K, (size_t)(r1 - r0) * K * sizeof(double));
            } else {
                for (int64_t r = r0; r < r1; ++r) std::memcpy(dst + r * ld, src + r * K, (size_t)K * sizeof(double));
            }
        });
        pend[b].live = false;
    };
    int buf = 0;
    for (int64_t t0 = 0; t0 < tilesTotal; t0 += tilesPerChunk, buf ^= 1) {
        const int64_t nt = (tilesTotal - t0 < tilesPerChunk) ? (tilesTotal - t0) : tilesPerChunk;
        const int64_t row0 = n0 + t0 * TILE_N;
        const int64_t rows = ((row0 + nt * TILE_N > n0 + n) ? n0 + n : row0 + nt * TILE_N) - row0;
        if (!pinnedDst) drain(buf);     // the staging buffer of two chunks ago must be empty again
        // kernel on `stream` must wait until the previous D2H out of this buffer finished
        cudaStreamWaitEvent(ctx->stream, done[buf], 0);
        logw_kernel<<<(unsigned)nt, 128, 0, ctx->stream>>>(ctx->d_u, ctx->d_L, ctx->dc(ROW_LOGW_F), K, ctx->N,
                                                          tileFirst + t0, d_out[buf], expo);
        ctx->launches++;
        Events ready;
        MBAR_TRY(ready.create(1, cudaEventDisableTiming));
        cudaEventRecord(ready[0], ctx->stream);
        cudaStreamWaitEvent(ctx->copyStream, ready[0], 0);
        cudaError_t e;
        if (pinnedDst) {
            e = cudaMemcpy2DAsync(logW_host + (row0 - n0) * ld, (size_t)ld * sizeof(double), d_out[buf],
                                  (size_t)K * sizeof(double), (size_t)K * sizeof(double), (size_t)rows,
                                  cudaMemcpyDeviceToHost, ctx->copyStream);
        } else {
            e = cudaMemcpyAsync(h_stage[buf], d_out[buf], (size_t)rows * K * sizeof(double), cudaMemcpyDeviceToHost,
                                ctx->copyStream);
            pend[buf].row0 = row0;
            pend[buf].rows = rows;
            pend[buf].live = true;
        }
        cudaEventRecord(done[buf], ctx->copyStream);
        ctx->d2hBytes += rows * K * 8;
        if (e != cudaSuccess) {
            set_error("log_W download failed: %s", cudaGetErrorString(e));
            rc = MBAR_B200_ERR_CUDA;
            break;
        }
    }
    cudaError_t e = cudaStreamSynchronize(ctx->copyStream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess && rc == MBAR_B200_OK) {
        set_error("log_W failed: %s", cudaGetErrorString(e));
        rc = MBAR_B200_ERR_CUDA;
    }
    if (!pinnedDst && rc == MBAR_B200_OK) {
        drain(0);
        drain(1);
    }
    return rc;
}

}  // namespace mbar

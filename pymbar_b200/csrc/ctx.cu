// Context, HBM layout and data movement for libmbar_b200.so.
//
// HBM layout ("tile-major"): u_kn [K, N] row-major on the host (mbar.py:243) is stored on device as
//   d_u[tile][k][lane],  tile = n / 32, lane = n % 32,
// so the K x 32 block of one group of 32 samples is ONE contiguous K*256-byte extent: a streaming
// pass is a sequence of large contiguous bulk copies, and each warp lane owns one sample.
// At upload every sample is shifted by x_n = min over SAMPLED states of u_kn (the first step of
// precondition_u_kn, mbar_solvers.py:705) and clamped to <= 1e6; gradient, Hessian, weights and
// the self-consistent update are invariant under a per-sample shift (SURVEY.md 8a, row a6), the
// objective changes by the constant sum_n x_n which the context carries.
#include <cmath>
#include <cstring>
#include <algorithm>
#include <cstdlib>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>

#include <sys/syscall.h>
#include <unistd.h>

#include "internal.cuh"

namespace mbar {

static thread_local char g_err[512] = "";

// ------------------------------------------------------------------------------------------
// NUMA placement of pinned staging memory.  cudaHostAlloc takes its pages from wherever the calling
// thread's memory policy points; on a two-socket host half of the boxes put the staging buffers on the
// socket that is NOT attached to the GPU and every H2D/D2H byte crosses the inter-socket link (round 1
// saw 0.445-0.635 s for the same 20.48 GB upload on different boxes).  While a pinned buffer is being
// allocated the thread prefers the GPU's own node (sysfs numa_node of its PCI function); hosts without
// NUMA information (-1) are left alone.  Raw syscalls: libnuma is not part of the image.
// ------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------
// host worker pool (see internal.cuh)
// ------------------------------------------------------------------------------------------
namespace {
struct HostPool {
    std::vector<std::thread> workers;
    std::mutex m;
    std::condition_variable cvStart, cvDone;
    const std::function<void(int)>* fn = nullptr;
    int nTasks = 0, next = 0, running = 0;
    uint64_t generation = 0;
    bool stop = false;
    int width = 1;

    HostPool() {
        int hw = (int)std::thread::hardware_concurrency();
        width = std::max(1, std::min(16, hw));
        if (const char* v = std::getenv("MBAR_B200_HOST_THREADS")) width = std::max(1, std::min(64, std::atoi(v)));
        for (int t = 1; t < width; ++t) workers.emplace_back([this] { loop(); });
    }
    ~HostPool() {
        {
            std::lock_guard<std::mutex> g(m);
            stop = true;
        }
        cvStart.notify_all();
        for (auto& w : workers) w.join();
    }
    void drain(std::unique_lock<std::mutex>& lk) {
        while (next < nTasks) {
            const int i = next++;
            ++running;
            lk.unlock();
            (*fn)(i);
            lk.lock();
            --running;
        }
    }
    void loop() {
        std::unique_lock<std::mutex> lk(m);
        uint64_t seen = 0;
        for (;;) {
            cvStart.wait(lk, [&] { return stop || generation != seen; });
            if (stop) return;
            seen = generation;
            drain(lk);
            if (running == 0 && next >= nTasks) cvDone.notify_all();
        }
    }
    void run(int n, const std::function<void(int)>& f) {
        std::unique_lock<std::mutex> lk(m);
        fn = &f;
        nTasks = n;
        next = 0;
        ++generation;
        cvStart.notify_all();
        drain(lk);
        cvDone.wait(lk, [&] { return running == 0 && next >= nTasks; });
        fn = nullptr;
    }
};
HostPool& pool() {
    static HostPool p;
    return p;
}
std::mutex g_poolUse;      // one parallel region at a time
}  // namespace

void host_parallel(int nTasks, const std::function<void(int)>& fn) {
    if (nTasks <= 1) {
        for (int i = 0; i < nTasks; ++i) fn(i);
        return;
    }
    std::lock_guard<std::mutex> g(g_poolUse);
    pool().run(nTasks, fn);
}
int host_parallel_width() { return pool().width; }

int gpu_numa_node(int device) {
    static int cache[16] = {-2, -2, -2, -2, -2, -2, -2, -2, -2, -2, -2, -2, -2, -2, -2, -2};
    int& c = cache[device & 15];
    if (c != -2) return c;
    c = -1;
    char bus[32] = "";
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) {
        cudaGetLastError();
        return c;
    }
    for (char* q = bus; *q; ++q)
        if (*q >= 'A' && *q <= 'F') *q = (char)(*q - 'A' + 'a');
    char path[128];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    if (FILE* fh = fopen(path, "r")) {
        int node = -1;
        if (fscanf(fh, "%d", &node) == 1) c = node;
        fclose(fh);
    }
    return c;
}
NumaPrefer::NumaPrefer(int device) {
#if defined(SYS_set_mempolicy)
    const int node = gpu_numa_node(device);
    if (node < 0 || node >= 1024) return;
    unsigned long mask[16] = {0};
    mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
    // MPOL_PREFERRED = 1
    if (syscall(SYS_set_mempolicy, 1, mask, (unsigned long)(sizeof(mask) * 8)) == 0) active = true;
#else
    (void)device;
#endif
}
NumaPrefer::~NumaPrefer() {
#if defined(SYS_set_mempolicy)
    if (active) syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0ul);
#endif
}

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// ------------------------------------------------------------------------------------------
// Buffer pool.  The reference's primitives are pure functions of host arrays, so a binding without
// residency creates and destroys a context per call; cudaFree/cudaMalloc of a 20 GB buffer and
// cudaHostAlloc of the pinned staging area cost tens to hundreds of ms each.  The largest buffers of a
// destroyed context are therefore parked (at most one u_kn buffer and one staging set per device) and
// handed to the next context that fits.  mbar_b200_trim() / MBAR_B200_NO_POOL=1 give the memory back.
// ------------------------------------------------------------------------------------------
struct Parked {
    void* ptr = nullptr;
    size_t bytes = 0;
};
static Parked g_pool[16][POOL_KINDS];   // per device: POOL_U, POOL_STAGE_DEV + i, POOL_STAGE_PIN + i
static std::mutex g_poolMutex;
bool pool_enabled() {
    static const bool off = std::getenv("MBAR_B200_NO_POOL") != nullptr;
    return !off;
}
// take a parked buffer of at least `bytes` (and at most 2x, so a small problem never pins a huge buffer)
void* pool_take(int device, int kind, size_t bytes, size_t* got) {
    std::lock_guard<std::mutex> g(g_poolMutex);
    Parked& slot = g_pool[device & 15][kind];
    if (slot.ptr && slot.bytes >= bytes && slot.bytes <= 2 * bytes + (1u << 20)) {
        void* p = slot.ptr;
        *got = slot.bytes;
        slot = Parked{};
        return p;
    }
    return nullptr;
}
// park `ptr`; whatever was parked there before is returned to the caller for release
void* pool_park(int device, int kind, void* ptr, size_t bytes) {
    std::lock_guard<std::mutex> g(g_poolMutex);
    Parked& slot = g_pool[device & 15][kind];
    void* old = slot.ptr;
    slot.ptr = ptr;
    slot.bytes = bytes;
    return old;
}

// Running minimum of one row's negative shifted energies (rounded down), one atomic per warp and row at most.
// Sampled rows are >= 0 after the shift, so in practice only unsampled rows below the sampled minimum report.
__device__ __forceinline__ void row_min_push(int* rowMin, double v, int lane) {
    int vi = v < 0.0 ? (int)fmax(floor(v), -1073741824.0) : 0;
    vi = __reduce_min_sync(0xffffffffu, vi);
    if (lane == 0 && vi < 0) atomicMin(rowMin, vi);
}
// Per row, from d = u - x before the clamp: a flag when a finite d reaches U_NEAR_CLAMP, and the count of entries at or
// above U_NEAR_CLAMP, +inf included (a row that counts every sample holds clamped or near-clamp entries only, see
// h_ufar).  The atomics are issued only by warps that hold such an entry.
__device__ __forceinline__ void row_clamp_push(int* rowClamp, unsigned long long* rowFar, double d, bool valid,
                                               int lane) {
    const unsigned far = __ballot_sync(0xffffffffu, valid && d >= U_NEAR_CLAMP);
    if (far == 0u) return;
    const bool finite = __any_sync(0xffffffffu, valid && d >= U_NEAR_CLAMP && d < INFINITY);
    if (lane == 0) {
        atomicAdd(rowFar, (unsigned long long)__popc(far));
        if (finite) atomicOr(rowClamp, 1);
    }
}

// Upload flags (d_flag[0]): NaN anywhere; a sample without a finite energy in any sampled state; -inf in an unsampled
// row (the reference would return f = -inf for that state; the library rejects the input instead)
enum { BAD_NAN = 1, BAD_NO_FINITE = 2, BAD_NEG_INF = 4 };
static const char* upload_error(int flags) {
    return flags & BAD_NAN ? "u_kn contains NaN"
         : flags & BAD_NO_FINITE ? "a sample has no finite energy in any sampled state"
                                 : "an unsampled state has an energy of -inf (its free energy would be -inf)";
}

// ------------------------------------------------------------------------------------------
// Re-tile + shift kernel.  One CTA (8 warps) per tile; lane = sample, warp w owns rows w, w+8, ...
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) retile_kernel(const double* __restrict__ src, int64_t ld,
                                                     int K, int64_t tile0, int64_t validCols,
                                                     const unsigned long long* __restrict__ rowmask,
                                                     double* __restrict__ dst,
                                                     double* __restrict__ xshift,
                                                     int* __restrict__ flags, int* __restrict__ urowmin,
                                                     unsigned long long* __restrict__ urowfar) {
    __shared__ double s_min[8][TILE_N];
    __shared__ int s_bad[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t tileLocal = blockIdx.x;
    const int64_t col = tileLocal * TILE_N + lane;
    const bool valid = col < validCols;
    const double* colp = src + col;

    double mn = INFINITY;
    unsigned bad = 0;
    for (int k = warp; k < K; k += 8) {
        double v = valid ? colp[(int64_t)k * ld] : 0.0;
        if (v != v) bad |= BAD_NAN;
        const bool act = (rowmask[k >> 6] >> (k & 63)) & 1ull;
        if (act) mn = fmin(mn, v);
        else if (v == -INFINITY) bad |= BAD_NEG_INF;
    }
    s_min[warp][lane] = mn;
    bad = __reduce_or_sync(0xffffffffu, bad);
    if (lane == 0) s_bad[warp] = (int)bad;
    __syncthreads();
    double x = s_min[0][lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) x = fmin(x, s_min[w][lane]);
    int anyBad = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) anyBad |= s_bad[w];
    // a sample whose sampled-state energies are all +inf (or contain -inf) has no finite weight
    const bool finiteShift = isfinite(x);
    // (a per-lane condition: every lane reports its own sample; warp 0 suffices, all warps hold the same x)
    if (valid && !finiteShift && warp == 0) atomicOr(&flags[0], BAD_NO_FINITE);
    if (!valid || !finiteShift) x = 0.0;

    double* out = dst + (tile0 + tileLocal) * (int64_t)K * TILE_N + lane;
    for (int k = warp; k < K; k += 8) {
        double v = valid ? colp[(int64_t)k * ld] : 0.0;
        const double d = v - x;
        row_clamp_push(urowmin + K + k, urowfar + k, d, valid, lane);
        v = fmin(d, U_CLAMP);
        row_min_push(urowmin + k, valid ? v : 0.0, lane);
        out[(int64_t)k * TILE_N] = valid ? v : 0.0;
    }
    if (warp == 0) xshift[(tile0 + tileLocal) * TILE_N + lane] = x;
    if (anyBad && threadIdx.x == 0) atomicOr(&flags[0], anyBad);
}

int retile_chunk(mbar_b200_ctx* ctx, const double* d_rowmajor, int64_t ldCols, int64_t tile0,
                 int64_t nTilesChunk, int64_t validCols, cudaStream_t s) {
    if (nTilesChunk <= 0) return MBAR_B200_OK;
    retile_kernel<<<(unsigned)nTilesChunk, 256, 0, s>>>(d_rowmajor, ldCols, ctx->K, tile0, validCols,
                                                       ctx->d_rowmask, ctx->d_u, ctx->d_xshift,
                                                       ctx->d_flag, ctx->d_urowmin, ctx->d_urowfar);
    ctx->launches++;
    MBAR_CUDA(cudaGetLastError());
    return MBAR_B200_OK;
}

// Inverse of the re-tile for verification: original-frame u = u' + x_n, row-major [K, n].
__global__ void __launch_bounds__(256) untile_kernel(const double* __restrict__ u,
                                                     const double* __restrict__ xshift, int K,
                                                     int64_t n0, int64_t n, double* __restrict__ dst,
                                                     int64_t ld) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t j = (int64_t)blockIdx.x * TILE_N + lane;  // column in the output
    if (j >= n) return;
    const int64_t g = n0 + j;
    const int64_t tile = g / TILE_N;
    const int l = (int)(g % TILE_N);
    const double x = xshift[g];
    for (int k = warp; k < K; k += 8)
        dst[(int64_t)k * ld + j] = u[(tile * K + k) * TILE_N + l] + x;
}

int launch_untile(mbar_b200_ctx* ctx, int64_t n0, int64_t n, double* d_dst, int64_t ld) {
    const unsigned grid = (unsigned)((n + TILE_N - 1) / TILE_N);
    untile_kernel<<<grid, 256, 0, ctx->stream>>>(ctx->d_u, ctx->d_xshift, ctx->K, n0, n, d_dst, ld);
    ctx->launches++;
    MBAR_CUDA(cudaGetLastError());
    return MBAR_B200_OK;
}

// sum of the per-sample shifts (valid samples only) -> one double
__global__ void __launch_bounds__(256) sumx_kernel(const double* __restrict__ x, int64_t N,
                                                   double* __restrict__ partial) {
    __shared__ double s[8];
    double acc = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N;
         i += (int64_t)gridDim.x * blockDim.x)
        acc += x[i];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += s[w];
        partial[blockIdx.x] = t;
    }
}

// sqrt(w_n) and the partial sums of w_n x_n (weighted counterpart of sumx_kernel)
__global__ void __launch_bounds__(256) wprep_kernel(const double* __restrict__ w, const double* __restrict__ x,
                                                    int64_t N, double* __restrict__ sqrtw,
                                                    double* __restrict__ partial) {
    __shared__ double s[8];
    double acc = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N;
         i += (int64_t)gridDim.x * blockDim.x) {
        const double wi = w[i];
        sqrtw[i] = sqrt(wi);
        acc += wi * x[i];
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < 8; ++i) t += s[i];
        partial[blockIdx.x] = t;
    }
}

// d_wgt and d_sqrtw exist together or not at all: reduce_sumxw writes d_sqrtw whenever d_wgt is set
static int reserve_weights(mbar_b200_ctx* ctx) {
    const size_t nPad = (size_t)ctx->nTiles * TILE_N;
    int rc = ctx->d_wgt.reserve(nPad, "sample weights");
    if (rc == MBAR_B200_OK) rc = ctx->d_sqrtw.reserve(nPad, "sample weights");
    if (rc != MBAR_B200_OK) {
        ctx->d_wgt.reset();
        ctx->d_sqrtw.reset();
    }
    return rc;
}

int set_weights(mbar_b200_ctx* ctx, const double* w_host) {
    if (!w_host) {
        ctx->d_wgt.reset();
        ctx->d_sqrtw.reset();
        return MBAR_B200_OK;
    }
    const size_t nPad = (size_t)ctx->nTiles * TILE_N;
    double sw = 0.0;
    for (int64_t i = 0; i < ctx->N; ++i) {
        MBAR_REQUIRE(w_host[i] >= 0.0, MBAR_B200_ERR_INVALID, "sample weight %lld is negative or NaN", (long long)i);
        sw += w_host[i];
    }
    MBAR_TRY(reserve_weights(ctx));
    ctx->sumW = sw;
    MBAR_CUDA(cudaMemsetAsync(ctx->d_wgt, 0, nPad * sizeof(double), ctx->stream));
    MBAR_CUDA(cudaMemsetAsync(ctx->d_sqrtw, 0, nPad * sizeof(double), ctx->stream));
    MBAR_CUDA(cudaMemcpyAsync(ctx->d_wgt, w_host, (size_t)ctx->N * sizeof(double), cudaMemcpyHostToDevice,
                              ctx->stream));
    ctx->h2dBytes += ctx->N * 8;
    return reduce_sumxw(ctx);
}

// sum_n w_n x_n depends on the shifts: every upload or synthesis into a weighted context recomputes it
int reduce_sumxw(mbar_b200_ctx* ctx) {
    if (!ctx->d_wgt) return MBAR_B200_OK;
    const int grid = 256;
    wprep_kernel<<<grid, 256, 0, ctx->stream>>>(ctx->d_wgt, ctx->d_xshift, ctx->N, ctx->d_sqrtw, ctx->d_scratch);
    ctx->launches++;
    MBAR_CUDA(cudaGetLastError());
    std::vector<double> h(grid);
    MBAR_CUDA(cudaMemcpyAsync(h.data(), ctx->d_scratch, grid * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    MBAR_CUDA(cudaStreamSynchronize(ctx->stream));
    double t = 0.0;
    for (double v : h) t += v;
    ctx->sumXw = t;
    return MBAR_B200_OK;
}

int reduce_sumx(mbar_b200_ctx* ctx) {
    const int grid = 256;
    sumx_kernel<<<grid, 256, 0, ctx->stream>>>(ctx->d_xshift, ctx->N, ctx->d_scratch);
    ctx->launches++;
    MBAR_CUDA(cudaGetLastError());
    std::vector<double> h(grid);
    MBAR_CUDA(cudaMemcpyAsync(h.data(), ctx->d_scratch, grid * sizeof(double), cudaMemcpyDeviceToHost,
                              ctx->stream));
    MBAR_CUDA(cudaStreamSynchronize(ctx->stream));
    double t = 0.0;
    for (double v : h) t += v;
    ctx->sumX = t;
    return MBAR_B200_OK;
}

// ------------------------------------------------------------------------------------------
// Synthetic harmonic-oscillator inputs generated in place (SURVEY.md 8d): Philox-4x32-10 keyed by
// the seed with the GLOBAL sample index as counter, so every shard regenerates exactly its slice.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                              uint32_t k0, uint32_t k1, uint32_t out[4]) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

__global__ void __launch_bounds__(256) synth_kernel(int K, int64_t N, int64_t nOffset, uint64_t seed,
                                                    const double* __restrict__ O_k,
                                                    const double* __restrict__ k_k,
                                                    const double* __restrict__ cumN,  // [K+1]
                                                    const unsigned long long* __restrict__ rowmask,
                                                    double* __restrict__ dst,
                                                    double* __restrict__ xshift, int* __restrict__ urowmin,
                                                    unsigned long long* __restrict__ urowfar) {
    __shared__ double s_min[8][TILE_N];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t tile = blockIdx.x;
    const int64_t nl = tile * TILE_N + lane;
    const bool valid = nl < N;
    const int64_t g = nOffset + nl;
    // state of origin: largest s with cumN[s] <= g
    int lo = 0, hi = K;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (cumN[mid] <= (double)g) lo = mid; else hi = mid;
    }
    uint32_t r[4];
    philox4x32_10((uint32_t)g, (uint32_t)((uint64_t)g >> 32), 0u, 0u, (uint32_t)seed,
                  (uint32_t)(seed >> 32), r);
    const double u1 = ((double)((((uint64_t)r[0] << 32) | r[1]) >> 11) + 0.5) * 0x1.0p-53;
    const double u2 = ((double)((((uint64_t)r[2] << 32) | r[3]) >> 11) + 0.5) * 0x1.0p-53;
    const double z = sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);
    const double x = O_k[lo] + z * rsqrt(k_k[lo]);

    double mn = INFINITY;
    for (int k = warp; k < K; k += 8) {
        const bool act = (rowmask[k >> 6] >> (k & 63)) & 1ull;
        const double d = x - O_k[k];
        if (act) mn = fmin(mn, 0.5 * k_k[k] * d * d);
    }
    s_min[warp][lane] = mn;
    __syncthreads();
    double sh = s_min[0][lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) sh = fmin(sh, s_min[w][lane]);
    if (!valid) sh = 0.0;
    double* out = dst + tile * (int64_t)K * TILE_N + lane;
    for (int k = warp; k < K; k += 8) {
        const double d = x - O_k[k];
        const double e = 0.5 * k_k[k] * d * d - sh;
        row_clamp_push(urowmin + K + k, urowfar + k, e, valid, lane);
        const double v = fmin(e, U_CLAMP);
        row_min_push(urowmin + k, valid ? v : 0.0, lane);
        out[(int64_t)k * TILE_N] = valid ? v : 0.0;
    }
    if (warp == 0) xshift[nl] = sh;
}

int launch_synth(mbar_b200_ctx* ctx, const mbar_b200_synth* spec) {
    const int K = ctx->K;
    std::vector<double> h(3 * (size_t)K + 1);
    for (int k = 0; k < K; ++k) {
        h[k] = spec->O_k[k];
        h[K + k] = spec->k_k[k];
        MBAR_REQUIRE(spec->k_k[k] > 0, MBAR_B200_ERR_INVALID, "synth: k_k[%d] must be > 0", k);
    }
    double c = 0.0;
    for (int k = 0; k <= K; ++k) {
        h[2 * K + k] = c;
        if (k < K) c += ctx->h_Nk[k];
    }
    double* d = ctx->d_scratch;  // >= K*K + 4K doubles
    MBAR_CUDA(cudaMemcpyAsync(d, h.data(), h.size() * sizeof(double), cudaMemcpyHostToDevice,
                              ctx->stream));
    synth_kernel<<<(unsigned)ctx->nTiles, 256, 0, ctx->stream>>>(
        K, ctx->N, spec->n_offset, spec->seed, d, d + K, d + 2 * K, ctx->d_rowmask, ctx->d_u,
        ctx->d_xshift, ctx->d_urowmin, ctx->d_urowfar);
    ctx->launches++;
    MBAR_CUDA(cudaGetLastError());
    MBAR_CUDA(cudaStreamSynchronize(ctx->stream));
    return MBAR_B200_OK;
}

int open_device(int device, cudaDeviceProp* propOut) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        set_error("no CUDA device visible: libmbar_b200 has no CPU fallback");
        return MBAR_B200_ERR_NO_DEVICE;
    }
    MBAR_REQUIRE(device >= 0 && device < ndev, MBAR_B200_ERR_INVALID, "device %d of %d", device, ndev);
    MBAR_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    MBAR_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_error("device %d is sm_%d%d; this library is built for sm_90a (H100) only", device,
                  prop.major, prop.minor);
        return MBAR_B200_ERR_NO_DEVICE;
    }
    if (propOut) *propOut = prop;
    return MBAR_B200_OK;
}

}  // namespace mbar

using namespace mbar;

// ------------------------------------------------------------------------------------------
// C ABI: library + context + data movement
// ------------------------------------------------------------------------------------------
extern "C" {

int mbar_b200_abi_version(void) { return MBAR_B200_ABI_VERSION; }
const char* mbar_b200_last_error(void) { return g_err; }

int mbar_b200_device_count(int* count) {
    MBAR_REQUIRE(count, MBAR_B200_ERR_INVALID, "count is NULL");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
        cudaGetLastError();
        n = 0;
    }
    *count = n;
    return MBAR_B200_OK;
}

int mbar_b200_host_alloc(void** ptr, uint64_t bytes) {
    MBAR_REQUIRE(ptr, MBAR_B200_ERR_INVALID, "ptr is NULL");
    int dev = 0;
    cudaGetDevice(&dev);
    unsigned char* p = nullptr;
    MBAR_TRY(host_alloc(&p, (size_t)bytes, "mbar_b200_host_alloc", dev));
    *ptr = p;
    return MBAR_B200_OK;
}
int mbar_b200_host_free(void* ptr) {
    MBAR_CUDA(mem_free(ptr, true));
    return MBAR_B200_OK;
}

// 64-bit content hash of a strided host matrix (rows x row_bytes, row stride stride_bytes), computed by several
// threads at memory bandwidth: the residency cache of the Python mirror keys on it, so that an in-place edit of
// u_kn between two calls can never be served from the stale device copy (a sampled probe could miss it).
static inline uint64_t mix64(uint64_t h, uint64_t w) {
    h ^= w;
    h *= 0x9E3779B97F4A7C15ull;
    return h ^ (h >> 29);
}
static uint64_t hash_span(const unsigned char* p, size_t bytes, uint64_t seed) {
    uint64_t h0 = seed, h1 = seed ^ 0xD6E8FEB86659FD93ull, h2 = seed + 0xA0761D6478BD642Full, h3 = ~seed;
    size_t i = 0;
    for (; i + 32 <= bytes; i += 32) {        // four independent lanes: the multiply chains overlap
        uint64_t w[4];
        std::memcpy(w, p + i, 32);
        h0 = mix64(h0, w[0]);
        h1 = mix64(h1, w[1]);
        h2 = mix64(h2, w[2]);
        h3 = mix64(h3, w[3]);
    }
    for (; i < bytes; ++i) h0 = mix64(h0, p[i]);
    return mix64(mix64(mix64(h0, h1), h2), h3);
}

int mbar_b200_host_hash(const void* base, int64_t rows, int64_t row_bytes, int64_t stride_bytes, uint64_t* out) {
    MBAR_REQUIRE(base && out && rows >= 0 && row_bytes >= 0 && stride_bytes >= row_bytes, MBAR_B200_ERR_INVALID,
                 "bad argument");
    const unsigned char* b = static_cast<const unsigned char*>(base);
    // split every row into fixed 4 MiB blocks; block hashes are combined in block order (thread-count independent)
    const int64_t blk = 4ll << 20;
    const int64_t perRow = row_bytes ? (row_bytes + blk - 1) / blk : 0;
    const int64_t nBlocks = rows * perRow;
    std::vector<uint64_t> part((size_t)nBlocks);
    host_parallel((int)std::min<int64_t>(nBlocks, 1 << 30), [&](int i) {
        const int64_t r = i / perRow, c = i % perRow;
        const int64_t off = c * blk, len = std::min(blk, row_bytes - off);
        part[(size_t)i] = hash_span(b + r * stride_bytes + off, (size_t)len, 0x243F6A8885A308D3ull + (uint64_t)i);
    });
    uint64_t h = 0x13198A2E03707344ull ^ (uint64_t)rows ^ ((uint64_t)row_bytes << 20);
    for (uint64_t v : part) h = mix64(h, v);
    *out = h;
    return MBAR_B200_OK;
}

int mbar_b200_create(mbar_b200_ctx** out, int device, int32_t K, int64_t N_local, const double* N_k) {
    MBAR_REQUIRE(out && N_k, MBAR_B200_ERR_INVALID, "NULL argument");
    *out = nullptr;
    MBAR_REQUIRE(K >= 1 && K <= MBAR_B200_MAX_STATES, MBAR_B200_ERR_INVALID, "K=%d outside [1, %d]", K,
                 MBAR_B200_MAX_STATES);
    MBAR_REQUIRE(N_local >= 1, MBAR_B200_ERR_INVALID, "N_local=%lld must be >= 1", (long long)N_local);
    cudaDeviceProp prop;
    MBAR_TRY(open_device(device, &prop));
    std::unique_ptr<mbar_b200_ctx> c(new mbar_b200_ctx());
    c->K = K;
    c->N = N_local;
    c->nTiles = (N_local + TILE_N - 1) / TILE_N;
    c->smCount = prop.multiProcessorCount;
    c->h_Nk.assign(N_k, N_k + K);
    c->h_logNk.resize(K);
    c->h_logNkEff.resize(K);
    std::vector<unsigned long long> mask((K + 63) / 64, 0ull);
    for (int k = 0; k < K; ++k) {
        MBAR_REQUIRE(N_k[k] >= 0.0, MBAR_B200_ERR_INVALID, "N_k[%d]=%g is negative or NaN", k, N_k[k]);
        c->N_total_states += N_k[k];
        if (N_k[k] > 0) {
            c->active.push_back(k);
            mask[k >> 6] |= 1ull << (k & 63);
            c->h_logNk[k] = std::log(N_k[k]);
            c->h_logNkEff[k] = c->h_logNk[k];
        } else {
            c->h_logNk[k] = -INFINITY;
            c->h_logNkEff[k] = LOG_EPS_UNSAMPLED;
        }
    }
    MBAR_REQUIRE(!c->active.empty(), MBAR_B200_ERR_INVALID, "all N_k are zero");
    c->firstActive = c->active[0];

    const size_t nPad = (size_t)c->nTiles * TILE_N;
    const PassLayout lay{K};
    const char* who = "mbar_b200_create";
    MBAR_TRY(c->d_u.acquire(device, POOL_U, (size_t)c->nTiles * K * TILE_N, who));
    MBAR_TRY(c->d_xshift.reserve(nPad, who));
    MBAR_TRY(c->d_c.reserve(DC_ROWS * (size_t)K, who));
    MBAR_TRY(c->d_Nk.reserve((size_t)K, who));
    MBAR_TRY(c->d_NkEff.reserve((size_t)K, who));
    MBAR_TRY(c->d_rowmask.reserve(mask.size(), who));
    MBAR_TRY(c->d_zeromask.reserve(mask.size(), who));
    MBAR_TRY(c->d_onesmask.reserve(mask.size(), who));
    MBAR_TRY(c->d_partial.reserve((size_t)MAX_GRID * (3 * (size_t)K + 2), who));
    MBAR_TRY(c->d_out.reserve((size_t)lay.size(true), who));
    MBAR_TRY(c->d_ticket.reserve(4, who));
    MBAR_TRY(c->d_flag.reserve(4, who));
    MBAR_TRY(c->d_urowmin.reserve(2 * (size_t)K, who));
    MBAR_TRY(c->d_urowfar.reserve((size_t)K, who));
    c->h_urowmin.assign(K, 0.0);
    c->h_uclamp.assign(K, 0.0);
    c->h_ufar.assign(K, 0.0);
    MBAR_TRY(c->d_f.reserve((size_t)K, who));
    MBAR_TRY(c->d_scratch.reserve(scratch_rendezvous(K) + 1024, who));
    MBAR_TRY(c->d_loop.reserve(1, who));
    MBAR_TRY(c->d_av.reserve(8 * (size_t)K, who));
    MBAR_TRY(c->d_outM.reserve(2 * (size_t)lay.size(false), who));
    MBAR_TRY(c->d_A.reserve((size_t)K * K, who));
    MBAR_TRY(c->d_active.reserve((size_t)K, who));
    MBAR_TRY(c->d_seq.reserve(1, who));
    MBAR_TRY(c->h_loop.reserve(1, who));
    MBAR_CUDA(cudaMemset(c->d_loop, 0, sizeof(mbar::LoopState)));
    MBAR_CUDA(cudaMemset(c->d_seq, 0, sizeof(unsigned long long)));
    MBAR_CUDA(cudaMemcpy(c->d_active, c->active.data(), c->active.size() * sizeof(int), cudaMemcpyHostToDevice));
    MBAR_TRY(c->evH.create(3));
    // (holds one packed result with G, or the two candidate results of mbar_b200_pass_multi)
    MBAR_TRY(c->h_out.reserve((size_t)std::max(lay.size(true), 2 * lay.size(false)), who));
    MBAR_TRY(c->h_f.reserve(HF_ROWS * (size_t)K, who));
    MBAR_TRY(c->open(device, who));
    MBAR_TRY(c->copyStream.create(who));
    MBAR_TRY(c->evCopy.create(2, cudaEventDisableTiming));
    MBAR_CUDA(cudaMemcpy(c->d_Nk, N_k, (size_t)K * sizeof(double), cudaMemcpyHostToDevice));
    {
        std::vector<double> eff(K);
        for (int k = 0; k < K; ++k) eff[k] = std::exp(c->h_logNkEff[k]);
        MBAR_CUDA(cudaMemcpy(c->d_NkEff, eff.data(), (size_t)K * sizeof(double), cudaMemcpyHostToDevice));
    }
    MBAR_CUDA(cudaMemcpy(c->d_rowmask, mask.data(), mask.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice));
    MBAR_CUDA(cudaMemset(c->d_zeromask, 0, mask.size() * sizeof(unsigned long long)));
    MBAR_CUDA(cudaMemset(c->d_onesmask, 0xff, mask.size() * sizeof(unsigned long long)));
    MBAR_CUDA(cudaMemset(c->d_ticket, 0, 4 * sizeof(unsigned int)));
    MBAR_CUDA(cudaMemset(c->d_flag, 0, 4 * sizeof(int)));
    MBAR_CUDA(cudaMemset(c->d_urowmin, 0, 2 * (size_t)K * sizeof(int)));
    MBAR_CUDA(cudaMemset(c->d_urowfar, 0, (size_t)K * sizeof(unsigned long long)));
    *out = c.release();
    return MBAR_B200_OK;
}

// Members free themselves (the pooled ones go back to the pool); what remains is what no member can own: the
// communicator and the peers' mappings go first, and the stream drains before any buffer is released.
int mbar_b200_destroy(mbar_b200_ctx* c) {
    if (!c) return MBAR_B200_OK;
    cudaSetDevice(c->device);
    if (c->comm) mbar_b200_comm_destroy(c);
    for (void* pm : c->peerMapped) cudaIpcCloseMemHandle(pm);
    if (c->loopGraph) cudaGraphExecDestroy(c->loopGraph);
    destroy_resident(c);
    cudaGetLastError();
    return MBAR_B200_OK;
}

int mbar_b200_trim(void) {
    int cur = 0;
    cudaGetDevice(&cur);
    for (int d = 0; d < 16; ++d) {
        Parked old[POOL_KINDS];
        bool any = false;
        {
            std::lock_guard<std::mutex> g(g_poolMutex);
            for (int k = 0; k < POOL_KINDS; ++k) {
                old[k] = g_pool[d][k];
                g_pool[d][k] = Parked{};
                any |= old[k].ptr != nullptr;
            }
        }
        if (!any) continue;
        cudaSetDevice(d);
        for (int k = 0; k < POOL_KINDS; ++k) mem_free(old[k].ptr, k >= POOL_STAGE_PIN);
    }
    cudaSetDevice(cur);
    cudaGetLastError();
    return MBAR_B200_OK;
}

int mbar_b200_get_shape(const mbar_b200_ctx* c, int32_t* K, int64_t* N_local) {
    MBAR_REQUIRE(c, MBAR_B200_ERR_INVALID, "ctx is NULL");
    if (K) *K = c->K;
    if (N_local) *N_local = c->N;
    return MBAR_B200_OK;
}

int mbar_b200_set_pass_kernel(mbar_b200_ctx* c, int kernel) {
    MBAR_REQUIRE(c, MBAR_B200_ERR_INVALID, "ctx is NULL");
    MBAR_REQUIRE(kernel >= 0 && kernel <= 2, MBAR_B200_ERR_INVALID, "kernel=%d", kernel);
    c->kernelChoice = kernel;
    return MBAR_B200_OK;
}

int mbar_b200_get_counters(const mbar_b200_ctx* c, int64_t* launches, int64_t* passes,
                           int64_t* h2d, int64_t* d2h) {
    MBAR_REQUIRE(c, MBAR_B200_ERR_INVALID, "ctx is NULL");
    if (launches) *launches = c->launches;
    if (passes) *passes = c->passes;
    if (h2d) *h2d = c->h2dBytes;
    if (d2h) *d2h = c->d2hBytes;
    return MBAR_B200_OK;
}

int mbar_b200_last_pass_ms(mbar_b200_ctx* c, double* ms) {
    MBAR_REQUIRE(c && ms, MBAR_B200_ERR_INVALID, "NULL argument");
    // events recorded around the most recent pass-kernel launch on the context's stream (whichever entry point
    // launched it)
    cudaSetDevice(c->device);
    float t = 0.f;
    if (c->stream && cudaStreamSynchronize(c->stream) == cudaSuccess && event_ms(c->ev0, c->ev1, &t))
        c->lastPassMs = t;
    else
        cudaGetLastError();
    *ms = c->lastPassMs;
    return MBAR_B200_OK;
}

static int ensure_staging(mbar_b200_ctx* c, bool needPinned) {
    if (c->stageCols == 0) {
        // ~64 MiB per staging buffer, whole tiles
        int64_t cols = (64ll << 20) / (8ll * c->K);
        cols = (cols / TILE_N) * TILE_N;
        if (cols < TILE_N) cols = TILE_N;
        const int64_t padN = c->nTiles * TILE_N;
        if (cols > padN) cols = padN;
        c->stageCols = cols;
    }
    const size_t count = (size_t)c->stageCols * c->K;
    for (int i = 0; i < 2; ++i) {
        MBAR_TRY(c->stage_dev[i].acquire(c->device, POOL_STAGE_DEV + i, count, "upload_u_kn"));
        if (needPinned) MBAR_TRY(c->stage_pinned[i].acquire(c->device, POOL_STAGE_PIN + i, count, "upload_u_kn"));
    }
    return MBAR_B200_OK;
}

static int reset_row_stats(mbar_b200_ctx* c) {
    MBAR_CUDA(cudaMemset(c->d_urowmin, 0, 2 * (size_t)c->K * sizeof(int)));
    MBAR_CUDA(cudaMemset(c->d_urowfar, 0, (size_t)c->K * sizeof(unsigned long long)));
    return MBAR_B200_OK;
}

// Row minima, clamp flags and far rows of the shifted energies written by the last upload: to the host, agreed
// over the shards (the upload is collective once a communicator is attached), device accumulators reset.
static int collect_row_minima(mbar_b200_ctx* c) {
    std::vector<int> m(2 * (size_t)c->K);
    std::vector<unsigned long long> far(c->K);
    MBAR_CUDA(cudaMemcpy(m.data(), c->d_urowmin, m.size() * sizeof(int), cudaMemcpyDeviceToHost));
    MBAR_CUDA(cudaMemcpy(far.data(), c->d_urowfar, far.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    MBAR_TRY(reset_row_stats(c));
    for (int k = 0; k < c->K; ++k) {
        c->h_urowmin[k] = (double)m[k];
        c->h_uclamp[k] = (double)m[c->K + k];
        c->h_ufar[k] = far[k] == (unsigned long long)c->N ? 1.0 : 0.0;
    }
    return agree_row_minima(c);
}

// After the copies of an upload or a synthesis: on success the sums over the new shifts and the row minima; on a
// rejected input every accumulator is reset, so the next upload starts from the state of a fresh context.
static int finish_upload(mbar_b200_ctx* c) {
    int flags[4];
    MBAR_CUDA(cudaStreamSynchronize(c->copyStream));
    MBAR_CUDA(cudaStreamSynchronize(c->stream));
    MBAR_CUDA(cudaMemcpy(flags, c->d_flag, sizeof(flags), cudaMemcpyDeviceToHost));
    if (flags[0]) {
        MBAR_CUDA(cudaMemset(c->d_flag, 0, 4 * sizeof(int)));
        MBAR_TRY(reset_row_stats(c));
        c->ready = false;
        set_error("%s", upload_error(flags[0]));
        return MBAR_B200_ERR_NAN;
    }
    MBAR_TRY(reduce_sumx(c));
    MBAR_TRY(reduce_sumxw(c));
    MBAR_TRY(collect_row_minima(c));
    c->ready = true;
    return MBAR_B200_OK;
}

int mbar_b200_gpu_numa_node(int device, int* node) {
    MBAR_REQUIRE(node, MBAR_B200_ERR_INVALID, "node is NULL");
    *node = gpu_numa_node(device);
    return MBAR_B200_OK;
}

int mbar_b200_upload_u_kn(mbar_b200_ctx* c, const double* u_host, int64_t ld) {
    MBAR_REQUIRE(c && u_host, MBAR_B200_ERR_INVALID, "NULL argument");
    NvtxRange nvtx_("mbar_b200::upload_u_kn");
    MBAR_REQUIRE(ld >= c->N, MBAR_B200_ERR_INVALID, "ld=%lld < N_local=%lld", (long long)ld,
                 (long long)c->N);
    MBAR_CUDA(cudaSetDevice(c->device));
    cudaPointerAttributes attr;
    bool pinned = false;
    if (cudaPointerGetAttributes(&attr, u_host) == cudaSuccess)
        pinned = (attr.type == cudaMemoryTypeHost);
    else
        cudaGetLastError();
    MBAR_TRY(ensure_staging(c, !pinned));
    const int K = c->K;
    const int64_t cols = c->stageCols;
    int buf = 0;
    // double-buffered: copy chunk i+1 (copyStream) while chunk i is re-tiled (stream)
    for (int64_t n0 = 0; n0 < c->N; n0 += cols, buf ^= 1) {
        const int64_t w = (c->N - n0 < cols) ? (c->N - n0) : cols;
        // the re-tile that last read stage_dev[buf] must be done before we overwrite it
        MBAR_CUDA(cudaStreamWaitEvent(c->copyStream, c->evCopy[buf], 0));
        const double* src = u_host + n0;
        int64_t srcLd = ld;
        if (!pinned) {
            // pageable memory: pack the chunk into the pinned staging buffer on the CPU
            MBAR_CUDA(cudaEventSynchronize(c->evCopy[buf]));
            // (numpy arrays are pageable: pack with several threads so the packing keeps up with PCIe)
            double* p = c->stage_pinned[buf];
            if ((size_t)w * K < (1u << 16)) {
                for (int k = 0; k < K; ++k)
                    std::memcpy(p + (size_t)k * w, u_host + (size_t)k * ld + n0, (size_t)w * sizeof(double));
            } else {
                // row segments in pieces of <= 128 KB so that small K still spreads over the pool
                const int64_t piece = 16384;
                const int64_t perRow = (w + piece - 1) / piece;
                host_parallel((int)(K * perRow), [&](int task) {
                    const int64_t k = task / perRow, c0 = (task % perRow) * piece;
                    const int64_t len = std::min(piece, w - c0);
                    std::memcpy(p + (size_t)k * w + c0, u_host + (size_t)k * ld + n0 + c0, (size_t)len * sizeof(double));
                });
            }
            src = p;
            srcLd = w;
        }
        MBAR_CUDA(cudaMemcpy2DAsync(c->stage_dev[buf], (size_t)cols * sizeof(double), src,
                                    (size_t)srcLd * sizeof(double), (size_t)w * sizeof(double), K,
                                    cudaMemcpyHostToDevice, c->copyStream));
        c->h2dBytes += (int64_t)w * K * 8;
        Events copied;
        MBAR_TRY(copied.create(1, cudaEventDisableTiming));
        MBAR_CUDA(cudaEventRecord(copied[0], c->copyStream));
        MBAR_CUDA(cudaStreamWaitEvent(c->stream, copied[0], 0));
        const int64_t nT = (w + TILE_N - 1) / TILE_N;
        MBAR_TRY(retile_chunk(c, c->stage_dev[buf], cols, n0 / TILE_N, nT, w, c->stream));
        MBAR_CUDA(cudaEventRecord(c->evCopy[buf], c->stream));
    }
    return finish_upload(c);
}

// ------------------------------------------------------------------------------------------
// Appended (unsampled) states on top of a resident problem.
// Every column the reference appends to Log_W_nk for an expectation or a perturbed free energy
// (mbar.py:886-940) is an unsampled state of an augmented problem with the SAME samples.  Instead of uploading
// the augmented (K + E) x N matrix again, the resident tiles are copied device-to-device into the wider tile
// stride and only the E new rows cross PCIe.  The per-sample shift x_n (min over SAMPLED states) is unchanged.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) widen_tiles_kernel(const double* __restrict__ src, int K, int Knew,
                                                          int64_t nTiles, double* __restrict__ dst) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t tile = blockIdx.x; tile < nTiles; tile += gridDim.x) {
        const double* s = src + tile * (int64_t)K * TILE_N + lane;
        double* d = dst + tile * (int64_t)Knew * TILE_N + lane;
#pragma unroll 4
        for (int k = warp; k < K; k += 8) d[(int64_t)k * TILE_N] = s[(int64_t)k * TILE_N];
    }
}
// rows [K, K + E) of tiles [tile0, tile0 + nT) from a row-major staging block [E, ldCols]
__global__ void __launch_bounds__(256) append_rows_kernel(const double* __restrict__ stage, int64_t ldCols, int E,
                                                          int K, int Knew, int64_t tile0, int64_t validCols,
                                                          const double* __restrict__ xshift,
                                                          double* __restrict__ dst, int* __restrict__ flags,
                                                          int* __restrict__ urowmin,
                                                          unsigned long long* __restrict__ urowfar) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t tl = blockIdx.x;
    const int64_t col = tl * TILE_N + lane;
    const bool valid = col < validCols;
    const double x = xshift[(tile0 + tl) * TILE_N + lane];
    double* out = dst + (tile0 + tl) * (int64_t)Knew * TILE_N + (int64_t)K * TILE_N + lane;
    unsigned bad = 0;
    for (int r = warp; r < E; r += 8) {
        double v = valid ? stage[(int64_t)r * ldCols + col] : 0.0;
        if (v != v) bad |= BAD_NAN;
        if (v == -INFINITY) bad |= BAD_NEG_INF;
        const double d = v - x;
        row_clamp_push(urowmin + Knew + K + r, urowfar + K + r, d, valid, lane);
        v = fmin(d, U_CLAMP);
        row_min_push(urowmin + K + r, valid ? v : 0.0, lane);
        out[(int64_t)r * TILE_N] = valid ? v : 0.0;
    }
    bad = __reduce_or_sync(0xffffffffu, bad);
    if (bad && lane == 0) atomicOr(&flags[0], (int)bad);
}

int mbar_b200_create_augmented(mbar_b200_ctx* base, int32_t n_extra, const double* u_extra_host, int64_t ld,
                               mbar_b200_ctx** out) {
    MBAR_REQUIRE(base && u_extra_host && out, MBAR_B200_ERR_INVALID, "NULL argument");
    *out = nullptr;
    MBAR_REQUIRE(base->ready, MBAR_B200_ERR_NOT_READY, "base problem has no u_kn yet");
    MBAR_REQUIRE(n_extra >= 1 && base->K + n_extra <= MBAR_B200_MAX_STATES, MBAR_B200_ERR_INVALID,
                 "n_extra=%d: K + n_extra must lie in [K + 1, %d]", n_extra, MBAR_B200_MAX_STATES);
    MBAR_REQUIRE(ld >= base->N, MBAR_B200_ERR_INVALID, "ld=%lld < N_local", (long long)ld);
    NvtxRange nvtx_("mbar_b200::create_augmented");
    const int K = base->K, E = n_extra, Kn = K + E;
    std::vector<double> Nk(base->h_Nk);
    Nk.resize(Kn, 0.0);
    mbar_b200_ctx* raw = nullptr;
    MBAR_TRY(mbar_b200_create(&raw, base->device, Kn, base->N, Nk.data()));
    std::unique_ptr<mbar_b200_ctx, int (*)(mbar_b200_ctx*)> c(raw, mbar_b200_destroy);
    MBAR_CUDA(cudaStreamSynchronize(base->stream));
    const size_t nPad = (size_t)c->nTiles * TILE_N;
    MBAR_CUDA(cudaMemcpyAsync(c->d_xshift, base->d_xshift, nPad * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    c->sumX = base->sumX;
    {
        int64_t grid = (int64_t)c->smCount * 8;
        if (grid > c->nTiles) grid = c->nTiles;
        widen_tiles_kernel<<<(unsigned)grid, 256, 0, c->stream>>>(base->d_u, K, Kn, c->nTiles, c->d_u);
        c->launches++;
        MBAR_CUDA(cudaGetLastError());
    }
    // the E new rows: column chunks through a pinned + a device staging block (pageable sources are packed by
    // the host first, exactly like mbar_b200_upload_u_kn)
    int64_t cols = (32ll << 20) / (8ll * E);
    cols = (cols / TILE_N) * TILE_N;
    if (cols < TILE_N) cols = TILE_N;
    if (cols > (int64_t)nPad) cols = (int64_t)nPad;
    cudaPointerAttributes attr;
    bool pinned = false;
    if (cudaPointerGetAttributes(&attr, u_extra_host) == cudaSuccess)
        pinned = (attr.type == cudaMemoryTypeHost);
    else
        cudaGetLastError();
    {
        CallBuffers buf("create_augmented");
        double* d_stage = nullptr;
        HostPinned<double> h_stage;
        StreamDrain guard{c.get()};
        MBAR_TRY(buf.alloc(&d_stage, (size_t)cols * E));
        if (!pinned) MBAR_TRY(h_stage.reserve((size_t)cols * E, "create_augmented", c->device));
        for (int64_t n0 = 0; n0 < c->N; n0 += cols) {
            const int64_t w = (c->N - n0 < cols) ? (c->N - n0) : cols;
            const double* src = u_extra_host + n0;
            int64_t srcLd = ld;
            if (!pinned) {
                cudaStreamSynchronize(c->stream);        // the staging block of the previous chunk has been consumed
                for (int r = 0; r < E; ++r)
                    std::memcpy(h_stage + (size_t)r * w, u_extra_host + (size_t)r * ld + n0, (size_t)w * sizeof(double));
                src = h_stage;
                srcLd = w;
            }
            cudaError_t e = cudaMemcpy2DAsync(d_stage, (size_t)cols * sizeof(double), src, (size_t)srcLd * sizeof(double),
                                              (size_t)w * sizeof(double), E, cudaMemcpyHostToDevice, c->stream);
            MBAR_REQUIRE(e == cudaSuccess, MBAR_B200_ERR_CUDA, "append rows: H2D failed: %s", cudaGetErrorString(e));
            c->h2dBytes += (int64_t)w * E * 8;
            const int64_t nT = (w + TILE_N - 1) / TILE_N;
            append_rows_kernel<<<(unsigned)nT, 256, 0, c->stream>>>(d_stage, cols, E, K, Kn, n0 / TILE_N, w,
                                                                  c->d_xshift, c->d_u, c->d_flag, c->d_urowmin,
                                                                  c->d_urowfar);
            c->launches++;
            if (pinned) cudaStreamSynchronize(c->stream);   // one device staging block: consume before refilling
        }
    }
    int flags[4] = {0, 0, 0, 0};   // (the appends have drained with the staging)
    MBAR_CUDA(cudaMemcpy(flags, c->d_flag, sizeof(flags), cudaMemcpyDeviceToHost));
    MBAR_CUDA(cudaMemset(c->d_flag, 0, 4 * sizeof(int)));
    MBAR_REQUIRE(!flags[0], MBAR_B200_ERR_NAN, "%s",
                 flags[0] & BAD_NAN ? "appended energies contain NaN"
                                    : "an appended state has an energy of -inf (its free energy would be -inf)");
    {
        std::vector<int> m(2 * (size_t)Kn);
        std::vector<unsigned long long> far(Kn);
        MBAR_CUDA(cudaMemcpy(m.data(), c->d_urowmin, m.size() * sizeof(int), cudaMemcpyDeviceToHost));
        MBAR_CUDA(cudaMemcpy(far.data(), c->d_urowfar, far.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        MBAR_TRY(reset_row_stats(c.get()));
        for (int k = 0; k < K; ++k) {
            c->h_urowmin[k] = base->h_urowmin[k];
            c->h_uclamp[k] = base->h_uclamp[k];
            c->h_ufar[k] = base->h_ufar[k];
        }
        for (int r = 0; r < E; ++r) {
            c->h_urowmin[K + r] = (double)m[K + r];
            c->h_uclamp[K + r] = (double)m[Kn + K + r];
            c->h_ufar[K + r] = far[K + r] == (unsigned long long)c->N ? 1.0 : 0.0;
        }
    }
    if (base->d_wgt) {
        // bootstrap multiplicities travel with the samples
        MBAR_TRY(reserve_weights(c.get()));
        MBAR_CUDA(cudaMemcpy(c->d_wgt, base->d_wgt, nPad * sizeof(double), cudaMemcpyDeviceToDevice));
        MBAR_CUDA(cudaMemcpy(c->d_sqrtw, base->d_sqrtw, nPad * sizeof(double), cudaMemcpyDeviceToDevice));
        c->sumW = base->sumW;
        c->sumXw = base->sumXw;
    }
    c->ready = true;
    *out = c.release();
    return MBAR_B200_OK;
}

int mbar_b200_upload_u_kn_dev(mbar_b200_ctx* c, const double* u_dev, int64_t ld) {
    MBAR_REQUIRE(c && u_dev, MBAR_B200_ERR_INVALID, "NULL argument");
    MBAR_REQUIRE(ld >= c->N, MBAR_B200_ERR_INVALID, "ld=%lld < N_local", (long long)ld);
    MBAR_CUDA(cudaSetDevice(c->device));
    // the context's stream does not wait for the legacy default stream (it is non-blocking), which is where torch
    // writes a tensor unless told otherwise: finish all prior work on the device before the re-tile reads u_dev
    MBAR_CUDA(cudaDeviceSynchronize());
    MBAR_TRY(retile_chunk(c, u_dev, ld, 0, c->nTiles, c->N, c->stream));
    return finish_upload(c);
}

int mbar_b200_synthesize(mbar_b200_ctx* c, const mbar_b200_synth* spec) {
    MBAR_REQUIRE(c && spec && spec->O_k && spec->k_k, MBAR_B200_ERR_INVALID, "NULL argument");
    MBAR_CUDA(cudaSetDevice(c->device));
    MBAR_TRY(launch_synth(c, spec));
    MBAR_TRY(reduce_sumx(c));
    MBAR_TRY(reduce_sumxw(c));
    MBAR_TRY(collect_row_minima(c));
    c->ready = true;
    return MBAR_B200_OK;
}

int mbar_b200_set_sample_weights(mbar_b200_ctx* c, const double* w_host) {
    MBAR_REQUIRE(c, MBAR_B200_ERR_INVALID, "ctx is NULL");
    MBAR_REQUIRE(c->ready, MBAR_B200_ERR_NOT_READY, "u_kn not uploaded");
    MBAR_CUDA(cudaSetDevice(c->device));
    return set_weights(c, w_host);
}

int mbar_b200_download_u_kn(mbar_b200_ctx* c, int64_t n0, int64_t n, double* u_host, int64_t ld) {
    MBAR_REQUIRE(c && u_host, MBAR_B200_ERR_INVALID, "NULL argument");
    MBAR_REQUIRE(c->ready, MBAR_B200_ERR_NOT_READY, "u_kn not uploaded");
    MBAR_REQUIRE(n0 >= 0 && n >= 1 && n0 + n <= c->N && ld >= n, MBAR_B200_ERR_INVALID,
                 "bad slice [%lld, +%lld) ld=%lld", (long long)n0, (long long)n, (long long)ld);
    MBAR_CUDA(cudaSetDevice(c->device));
    // chunked through a device row-major buffer
    const int64_t maxCols = (32ll << 20) / (8ll * c->K) / TILE_N * TILE_N + TILE_N;
    double* d_tmp = nullptr;
    const int64_t cols = n < maxCols ? n : maxCols;
    CallBuffers buf("download_u_kn");
    MBAR_TRY(buf.alloc(&d_tmp, (size_t)cols * c->K));
    int rc = MBAR_B200_OK;
    for (int64_t j = 0; j < n && rc == MBAR_B200_OK; j += cols) {
        const int64_t w = (n - j < cols) ? (n - j) : cols;
        rc = launch_untile(c, n0 + j, w, d_tmp, cols);
        if (rc != MBAR_B200_OK) break;
        cudaError_t e = cudaMemcpy2DAsync(u_host + j, (size_t)ld * sizeof(double), d_tmp,
                                          (size_t)cols * sizeof(double), (size_t)w * sizeof(double),
                                          c->K, cudaMemcpyDeviceToHost, c->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        if (e != cudaSuccess) {
            set_error("download failed: %s", cudaGetErrorString(e));
            rc = MBAR_B200_ERR_CUDA;
        }
        c->d2hBytes += (int64_t)w * c->K * 8;
    }
    return rc;
}

}  // extern "C"

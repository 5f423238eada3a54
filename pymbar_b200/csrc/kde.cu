// mbar_b200_kde_*: kernel-density log sums over resident weighted samples, the part of sklearn's
// KernelDensity.score_samples that grows with N x Q (pymbar FES with fes_type="kde", fes.py:650-699, :1523-1609).
//
//   l_q = log sum_n w_n k(d_qn / h),   d_qn = sqrt(sum_j (y_qj - x_nj)^2)   (rounded squares added in dimension order)
//
// The host adds sklearn's kernel normalisation and subtracts log sum_n w_n (pymbar_b200/fes.py).
//
// Decomposition.  The samples are cut into chunks whose length depends on N alone (mbar_b200_kde_create).  CTA (b, c) holds 128
// queries, one per thread, and streams chunk c through shared memory once, 256 samples (SoA, plus log w_n) per tile;
// every thread keeps a running (m, s) with s = sum exp(a_n - m), a_n = log w_n + log k_qn.  The partials of all
// chunks are then combined per query in chunk order (kde_combine_kernel).  Which samples a thread adds, and in which
// order, is a function of N only, so a query's result does not depend on Q, on the other queries or on their order,
// and there are no atomics: repeat calls are bit-identical.
//
// Per pair: the distance, the kernel, one exp.  m is raised only when a term exceeds it by more than KDE_RESCALE (a branch
// almost never taken), so every exp argument lies in [-1000, KDE_RESCALE] (clamped from
// below; arguments below about -708 return exactly 0, far less than 2^-1020 relative to s >= the kernel value of the
// term that last set m).  The compact kernels (epanechnikov, linear, cosine) enter as a factor, w_n k = exp(log w_n -
// m) k, so a pair costs one exp and no log; k is evaluated with sklearn's own fp64 operations (d*d/(h*h), d/h,
// cos(pi/2 * d / h)), so that a sample next to the edge of the support gets sklearn's value, not one that rounds
// to 0.  Support is sklearn's test: d = correctly rounded sqrt of the sum of rounded squares (no FMA contraction),
// then d < h; the tophat kernel, which needs no d, uses the equivalent r < T with T the least double whose rounded
// square root reaches h (computed on the host).
#include <algorithm>
#include <cmath>
#include <vector>

#include "internal.cuh"

struct mbar_b200_kde {
    int device = 0;
    int D = 0;
    int64_t N = 0;
    int64_t nPad = 0;            // N rounded up to a tile
    int64_t chunkLen = 0;        // samples per chunk (a multiple of KDE_TILE)
    int nChunks = 0;
    double* d_x = nullptr;       // [D][nPad] coordinates, 0 in the padding
    double* d_lw = nullptr;      // [nPad] log w_n, -inf for zero weights and the padding
    double* d_y = nullptr;       // [D][qCap] queries of one batch
    double* d_pm = nullptr;      // [nChunks][qCap] running maxima
    double* d_ps = nullptr;      // [nChunks][qCap] sums relative to them
    double* d_out = nullptr;     // [qCap]
    int64_t qCap = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    double lastMs = 0.0;
    int lastChunks = 0;
};

namespace mbar {

constexpr int KDE_THREADS = 128;              // queries per CTA
constexpr int KDE_TILE = 256;                 // samples per shared-memory tile
constexpr int64_t KDE_MIN_CHUNK = 4096;       // samples per chunk, at least
constexpr int KDE_MAX_CHUNKS = 1024;
constexpr size_t KDE_PART_BYTES = 64ull << 20;   // cap of the (m, s) partials of one query batch
constexpr double KDE_RESCALE = 128.0;         // raise m when a term exceeds it by more than this
constexpr double KDE_FLOOR = -1000.0;         // exp arguments are clamped here (result exactly 0)
constexpr double KDE_HALF_PI = 1.5707963267948966;   // 0.5 * pi as sklearn's 0.5 * PI folds it

enum { KDE_GAUSSIAN = 0, KDE_TOPHAT, KDE_EPANECHNIKOV, KDE_EXPONENTIAL, KDE_LINEAR, KDE_COSINE, KDE_NKERNELS };

struct KdeParams {
    const double* x;      // [D][nPad]
    const double* lw;     // [nPad]
    const double* y;      // [D][Qb]
    double* pm;           // [nChunks][Qb]
    double* ps;
    int64_t nPad, chunkLen;
    int Qb;
    double h;             // bandwidth
    double hh;            // h * h (epanechnikov, as sklearn rounds it)
    double c;             // 0.5 / h^2 (gaussian) | 1 / h (exponential)
    double T;             // least r with sqrt(r) >= h (tophat)
};

// exp(a) for a in [KDE_FLOOR, KDE_RESCALE]: exp_split as everywhere in the library (DESIGN 3.1), and exactly 0 where
// the binary exponent leaves the normal range
__device__ __forceinline__ double exp_flush(double a, const double* __restrict__ tab) {
    double v;
    int q;
    exp_split(a, tab, v, q);
    const int hi = __double2hiint(v) + (q << 20);
    return q < -1021 ? 0.0 : __hiloint2double(hi, __double2loint(v));
}

template <int D, int KERN>
__global__ void __launch_bounds__(KDE_THREADS) kde_partial_kernel(KdeParams p) {
    __shared__ double sx[D][KDE_TILE];
    __shared__ double slw[KDE_TILE];
    __shared__ double tab[MBAR_EXP_NT];
    if (threadIdx.x < MBAR_EXP_NT) tab[threadIdx.x] = MBAR_EXP_TABLE[threadIdx.x];
    const int q = blockIdx.x * KDE_THREADS + threadIdx.x;
    const int64_t n0 = (int64_t)blockIdx.y * p.chunkLen, n1 = min(n0 + p.chunkLen, p.nPad);
    double y[D];
#pragma unroll
    for (int j = 0; j < D; ++j) y[j] = q < p.Qb ? p.y[(int64_t)j * p.Qb + q] : 0.0;
    double m = -INFINITY, s = 0.0;
    for (int64_t t0 = n0; t0 < n1; t0 += KDE_TILE) {
        __syncthreads();
        for (int i = threadIdx.x; i < KDE_TILE; i += KDE_THREADS) {
#pragma unroll
            for (int j = 0; j < D; ++j) sx[j][i] = p.x[(int64_t)j * p.nPad + t0 + i];
            slw[i] = p.lw[t0 + i];
        }
        __syncthreads();
#pragma unroll 4
        for (int i = 0; i < KDE_TILE; ++i) {
            // sklearn's euclidean distance: rounded squares summed in dimension order, no contraction
            double t = __dsub_rn(y[0], sx[0][i]);
            double r = __dmul_rn(t, t);
#pragma unroll
            for (int j = 1; j < D; ++j) {
                t = __dsub_rn(y[j], sx[j][i]);
                r = __dadd_rn(r, __dmul_rn(t, t));
            }
            const double lw = slw[i];
            double a, k = 1.0;
            if (KERN == KDE_GAUSSIAN) {
                a = fma(-r, p.c, lw);
            } else if (KERN == KDE_TOPHAT) {
                a = r < p.T ? lw : -INFINITY;
            } else if (KERN == KDE_EXPONENTIAL) {
                a = fma(-__dsqrt_rn(r), p.c, lw);
            } else {
                const double d = __dsqrt_rn(r);
                const bool in = d < p.h;
                a = in ? lw : -INFINITY;
                if (KERN == KDE_EPANECHNIKOV) k = __dsub_rn(1.0, __ddiv_rn(__dmul_rn(d, d), p.hh));
                if (KERN == KDE_LINEAR) k = __dsub_rn(1.0, __ddiv_rn(d, p.h));
                if (KERN == KDE_COSINE) k = cos(__ddiv_rn(__dmul_rn(KDE_HALF_PI, d), p.h));
                k = in ? k : 0.0;            // outside the support k may be -inf or NaN (d = inf)
            }
            double dl = a - m;               // NaN when both are -inf: clamped to KDE_FLOOR below
            if (dl > KDE_RESCALE) {
                s *= exp_flush(fmax(m - a, KDE_FLOOR), tab);
                m = a;
                dl = 0.0;
            }
            const double e = exp_flush(fmax(dl, KDE_FLOOR), tab);
            s = (KERN == KDE_EPANECHNIKOV || KERN == KDE_LINEAR || KERN == KDE_COSINE) ? fma(e, k, s) : s + e;
        }
    }
    if (q < p.Qb) {
        p.pm[(int64_t)blockIdx.y * p.Qb + q] = m;
        p.ps[(int64_t)blockIdx.y * p.Qb + q] = s;
    }
}

// l_q = M + log sum_c s_c exp(m_c - M), M = max_c m_c, chunks in order; -inf when no term is nonzero
__global__ void kde_combine_kernel(const double* __restrict__ pm, const double* __restrict__ ps, int nChunks, int Qb,
                                   double* __restrict__ out) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= Qb) return;
    double M = -INFINITY;
    for (int c = 0; c < nChunks; ++c) M = fmax(M, pm[(int64_t)c * Qb + q]);
    if (M == -INFINITY) {
        out[q] = -INFINITY;
        return;
    }
    double S = 0.0;
    for (int c = 0; c < nChunks; ++c) S += ps[(int64_t)c * Qb + q] * exp(pm[(int64_t)c * Qb + q] - M);
    out[q] = M + log(S);
}

typedef void (*KdeKernelFn)(KdeParams);

template <int D>
static KdeKernelFn kde_kernel_for(int kernel) {
    switch (kernel) {
        case KDE_GAUSSIAN: return kde_partial_kernel<D, KDE_GAUSSIAN>;
        case KDE_TOPHAT: return kde_partial_kernel<D, KDE_TOPHAT>;
        case KDE_EPANECHNIKOV: return kde_partial_kernel<D, KDE_EPANECHNIKOV>;
        case KDE_EXPONENTIAL: return kde_partial_kernel<D, KDE_EXPONENTIAL>;
        case KDE_LINEAR: return kde_partial_kernel<D, KDE_LINEAR>;
        default: return kde_partial_kernel<D, KDE_COSINE>;
    }
}

static KdeKernelFn kde_kernel_for(int D, int kernel) {
    switch (D) {
        case 1: return kde_kernel_for<1>(kernel);
        case 2: return kde_kernel_for<2>(kernel);
        case 3: return kde_kernel_for<3>(kernel);
        default: return kde_kernel_for<4>(kernel);
    }
}

// least double r with sqrt(r) >= h: sqrt is correctly rounded and monotone, so sqrt(r) < h exactly when r < T
static double sqrt_threshold(double h) {
    double r = h * h;
    if (std::isinf(r)) return r;
    while (r > 0.0 && std::sqrt(r) >= h) r = std::nextafter(r, 0.0);
    while (std::sqrt(r) < h) r = std::nextafter(r, INFINITY);
    return r;
}

static void kde_release(mbar_b200_kde* k) {
    for (double* p : {k->d_x, k->d_lw, k->d_y, k->d_pm, k->d_ps, k->d_out})
        if (p) cudaFree(p);
    if (k->ev0) cudaEventDestroy(k->ev0);
    if (k->ev1) cudaEventDestroy(k->ev1);
    if (k->stream) cudaStreamDestroy(k->stream);
    delete k;
}

static int kde_alloc(double** p, size_t count) {
    const cudaError_t e = cudaMalloc((void**)p, std::max<size_t>(count, 1) * sizeof(double));
    if (e != cudaSuccess) {
        *p = nullptr;
        cudaGetLastError();
        set_error("kde: cannot allocate %zu bytes", count * sizeof(double));
        return e == cudaErrorMemoryAllocation ? MBAR_B200_ERR_NOMEM : MBAR_B200_ERR_CUDA;
    }
    return MBAR_B200_OK;
}

// per-batch buffers for up to qb queries; on failure the object keeps no (or its previous) buffers and stays usable
static int kde_reserve(mbar_b200_kde* k, int64_t qb) {
    if (qb <= k->qCap) return MBAR_B200_OK;
    for (double** p : {&k->d_y, &k->d_pm, &k->d_ps, &k->d_out}) {
        if (*p) cudaFree(*p);
        *p = nullptr;
    }
    k->qCap = 0;
    MBAR_TRY(kde_alloc(&k->d_y, (size_t)k->D * qb));
    MBAR_TRY(kde_alloc(&k->d_pm, (size_t)k->nChunks * qb));
    MBAR_TRY(kde_alloc(&k->d_ps, (size_t)k->nChunks * qb));
    MBAR_TRY(kde_alloc(&k->d_out, (size_t)qb));
    k->qCap = qb;
    return MBAR_B200_OK;
}

}  // namespace mbar

using namespace mbar;

int mbar_b200_kde_create(int device, int64_t N, int32_t D, const double* x_host, const double* w_host,
                         mbar_b200_kde** out) {
    MBAR_REQUIRE(out && x_host && w_host, MBAR_B200_ERR_INVALID, "kde_create: NULL argument");
    *out = nullptr;
    MBAR_REQUIRE(N >= 1, MBAR_B200_ERR_INVALID, "kde_create: N=%lld must be >= 1", (long long)N);
    MBAR_REQUIRE(D >= 1 && D <= 4, MBAR_B200_ERR_INVALID, "kde_create: D=%d outside [1, 4]", (int)D);
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
        set_error("device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
        return MBAR_B200_ERR_NO_DEVICE;
    }
    const int64_t nPad = (N + KDE_TILE - 1) / KDE_TILE * KDE_TILE;
    std::vector<double> hx((size_t)D * nPad, 0.0), hlw((size_t)nPad, -INFINITY);
    bool any = false;
    for (int64_t n = 0; n < N; ++n) {
        const double w = w_host[n];
        MBAR_REQUIRE(w >= 0.0 && w < INFINITY, MBAR_B200_ERR_INVALID, "kde_create: weight %lld is %g (negative, "
                     "NaN or infinite)", (long long)n, w);
        any |= w > 0.0;
        hlw[n] = std::log(w);
        for (int j = 0; j < D; ++j) {
            const double v = x_host[n * D + j];
            MBAR_REQUIRE(std::isfinite(v), MBAR_B200_ERR_NAN, "kde_create: coordinate (%lld, %d) is %g",
                         (long long)n, j, v);
            hx[(size_t)j * nPad + n] = v;
        }
    }
    MBAR_REQUIRE(any, MBAR_B200_ERR_INVALID, "kde_create: the weights sum to 0");
    mbar_b200_kde* k = new mbar_b200_kde();
    k->device = device;
    k->D = D;
    k->N = N;
    k->nPad = nPad;
    // chunks: a function of N alone (batch independence); at least KDE_MIN_CHUNK samples, at most KDE_MAX_CHUNKS
    int64_t nc = std::min<int64_t>(KDE_MAX_CHUNKS, std::max<int64_t>(1, (N + KDE_MIN_CHUNK - 1) / KDE_MIN_CHUNK));
    k->chunkLen = ((N + nc - 1) / nc + KDE_TILE - 1) / KDE_TILE * KDE_TILE;
    k->nChunks = (int)((nPad + k->chunkLen - 1) / k->chunkLen);
    int rc = MBAR_B200_OK;
    auto fail = [&](int status) {
        kde_release(k);
        return status;
    };
    if ((rc = kde_alloc(&k->d_x, hx.size())) || (rc = kde_alloc(&k->d_lw, hlw.size()))) return fail(rc);
    // the copies go on the object's own (non-blocking) stream and are waited for: a pageable cudaMemcpy on the legacy
    // stream may return before its DMA lands, and the kernels' stream would not wait for it
    if (cudaStreamCreateWithFlags(&k->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreate(&k->ev0) != cudaSuccess || cudaEventCreate(&k->ev1) != cudaSuccess ||
        cudaMemcpyAsync(k->d_x, hx.data(), hx.size() * sizeof(double), cudaMemcpyHostToDevice, k->stream) !=
            cudaSuccess ||
        cudaMemcpyAsync(k->d_lw, hlw.data(), hlw.size() * sizeof(double), cudaMemcpyHostToDevice, k->stream) !=
            cudaSuccess ||
        cudaStreamSynchronize(k->stream) != cudaSuccess) {
        set_error("kde_create: %s", cudaGetErrorString(cudaGetLastError()));
        return fail(MBAR_B200_ERR_CUDA);
    }
    *out = k;
    return MBAR_B200_OK;
}

int mbar_b200_kde_destroy(mbar_b200_kde* k) {
    if (!k) return MBAR_B200_OK;
    cudaSetDevice(k->device);
    if (k->stream) cudaStreamSynchronize(k->stream);
    kde_release(k);
    return MBAR_B200_OK;
}

int mbar_b200_kde_log_sum(mbar_b200_kde* k, int32_t kernel, double h, int64_t Q, const double* y_host,
                          double* out) {
    MBAR_REQUIRE(k, MBAR_B200_ERR_INVALID, "kde_log_sum: NULL object");
    MBAR_REQUIRE(kernel >= 0 && kernel < KDE_NKERNELS, MBAR_B200_ERR_INVALID, "kde_log_sum: unknown kernel %d",
                 (int)kernel);
    MBAR_REQUIRE(std::isfinite(h) && h > 0.0, MBAR_B200_ERR_INVALID, "kde_log_sum: bandwidth %g must be finite and "
                 "positive", h);
    MBAR_REQUIRE(Q >= 0, MBAR_B200_ERR_INVALID, "kde_log_sum: Q=%lld", (long long)Q);
    if (Q == 0) return MBAR_B200_OK;
    MBAR_REQUIRE(y_host && out, MBAR_B200_ERR_INVALID, "kde_log_sum: NULL argument");
    const int D = k->D;
    for (int64_t i = 0; i < Q * D; ++i)
        MBAR_REQUIRE(std::isfinite(y_host[i]), MBAR_B200_ERR_NAN, "kde_log_sum: query coordinate (%lld, %d) is %g",
                     (long long)(i / D), (int)(i % D), y_host[i]);
    MBAR_CUDA(cudaSetDevice(k->device));
    NvtxRange nvtx_("mbar_b200::kde_log_sum");
    // query batches: only the size of the partials depends on them, never a query's result
    int64_t cap = (int64_t)(KDE_PART_BYTES / (2 * sizeof(double) * (size_t)k->nChunks));
    cap = std::max<int64_t>(KDE_THREADS, cap / KDE_THREADS * KDE_THREADS);
    const int64_t qb = std::min(Q, cap);
    MBAR_TRY(kde_reserve(k, qb));
    KdeParams p{};
    p.x = k->d_x;
    p.lw = k->d_lw;
    p.y = k->d_y;
    p.pm = k->d_pm;
    p.ps = k->d_ps;
    p.nPad = k->nPad;
    p.chunkLen = k->chunkLen;
    p.h = h;
    p.hh = h * h;
    p.c = kernel == KDE_GAUSSIAN ? 0.5 / (h * h) : 1.0 / h;
    p.T = sqrt_threshold(h);
    const KdeKernelFn fn = kde_kernel_for(D, kernel);
    std::vector<double> hy((size_t)D * qb);
    double ms = 0.0;
    for (int64_t q0 = 0; q0 < Q; q0 += qb) {
        const int Qb = (int)std::min(qb, Q - q0);
        for (int64_t i = 0; i < Qb; ++i)
            for (int j = 0; j < D; ++j) hy[(size_t)j * Qb + i] = y_host[(q0 + i) * D + j];
        MBAR_CUDA(cudaMemcpyAsync(k->d_y, hy.data(), (size_t)D * Qb * sizeof(double), cudaMemcpyHostToDevice,
                                  k->stream));
        p.Qb = Qb;
        MBAR_CUDA(cudaEventRecord(k->ev0, k->stream));
        const dim3 grid((unsigned)((Qb + KDE_THREADS - 1) / KDE_THREADS), (unsigned)k->nChunks);
        fn<<<grid, KDE_THREADS, 0, k->stream>>>(p);
        kde_combine_kernel<<<(Qb + 127) / 128, 128, 0, k->stream>>>(k->d_pm, k->d_ps, k->nChunks, Qb, k->d_out);
        MBAR_CUDA(cudaGetLastError());
        MBAR_CUDA(cudaEventRecord(k->ev1, k->stream));
        MBAR_CUDA(cudaMemcpyAsync(out + q0, k->d_out, (size_t)Qb * sizeof(double), cudaMemcpyDeviceToHost,
                                  k->stream));
        MBAR_CUDA(cudaStreamSynchronize(k->stream));
        float e = 0.f;
        if (event_ms(k->ev0, k->ev1, &e)) ms += e;
    }
    k->lastMs = ms;
    k->lastChunks = k->nChunks;
    return MBAR_B200_OK;
}

int mbar_b200_last_kde_stats(mbar_b200_kde* k, double* ms, int32_t* chunks) {
    MBAR_REQUIRE(k, MBAR_B200_ERR_INVALID, "NULL kde object");
    if (ms) *ms = k->lastMs;
    if (chunks) *chunks = k->lastChunks;
    return MBAR_B200_OK;
}

// mbar_b200_work_*: the sums behind pymbar.other_estimators (bar_zero, bar's uncertainty, exp, exp_gauss;
// other_estimators.py:56-153, :478-504, :572-719) over V resident work vectors.  A request names a vector, a kind and
// two constants; for its terms x_i the reference evaluates, in fp64,
//
//   fermi:          a_i = (w_i + c1) + c2,  m_i = max(a_i, 0),  t_i = -m_i - log(exp(-m_i) + exp(a_i - m_i)),
//                   out = logsumexp(t)
//   fermi moments:  a_i = w_i + c1,  A = max(a),  t_i = -log(exp(-A) + exp(a_i - A)),
//                   out = logsumexp(t), logsumexp(2 t), A
//   exp:            x_i = exp(-w_i - max(-w)),  out = log(sum x) + max(-w), sum x, sum (x - sum x / n)^2
//   gauss:          out = sum w, sum (w - sum w / n)^2
//
// where logsumexp(t) = log(sum exp(t - M)) + M with M = max(t), and M = 0 when it is not finite (pymbar's
// utils.logsumexp).  Every term is the reference's formula with its own max shifts, so where the reference overflows
// the device gives the same inf or NaN.  Because rounding is monotone, max(w + c1) = fl(max w + c1) and
// max(-w) = -min w exactly: the vector's min and max are taken once at create time.
//
// Passes.  A call makes two passes over each requested vector: pass 1 gives the shift (the max of the terms) or the
// plain sum whose mean the second pass centres by, pass 2 the shifted or centred sums.  Each pass writes one partial
// per (request, chunk) and a finalize kernel adds a request's partials in chunk order.
//
// Determinism.  A vector of n values is cut into chunks of CL = max(4096, ceil(n / 2048)) values, a function of n
// alone.  A CTA owns one (request, chunk): thread j adds the chunk's values j, j + 256, ... sequentially from 0.0, and
// the 256 thread sums are combined by a fixed shared-memory tree.  Nothing depends on the other requests of the call,
// there are no atomics, and repeat calls are bit-identical.
#include <algorithm>
#include <cmath>
#include <memory>
#include <vector>

#include "internal.cuh"

namespace mbar {

constexpr int WORK_THREADS = 256;
constexpr int64_t WORK_MIN_CL = 4096;
constexpr int64_t WORK_MAX_CHUNKS = 2048;

__host__ __device__ __forceinline__ int64_t work_chunk_len(int64_t n) {
    return n > WORK_MIN_CL * WORK_MAX_CHUNKS ? (n + WORK_MAX_CHUNKS - 1) / WORK_MAX_CHUNKS : WORK_MIN_CL;
}

struct WorkReq {
    int64_t off, n, cl, item0;     // vector offset and length, chunk length, first (request, chunk) item
    double c1, c2;
    double vmin, vmax;
    int32_t kind;
};

}  // namespace mbar

struct mbar_b200_work : mbar::Resident {
    int64_t nTotal = 0;
    int nVec = 0;
    std::vector<int64_t> offsets;
    std::vector<double> vmin, vmax;
    mbar::DevArray<double> d_w;
    // per-call buffers, grown on demand
    mbar::DevArray<mbar::WorkReq> d_req;
    mbar::DevArray<double> d_part;   // [items][2]
    mbar::DevArray<double> d_shift;  // [requests][2]: pass-1 results (shifts, or sum and mean)
    mbar::DevArray<double> d_out;    // [requests][3]
    int32_t lastLaunches = 0;
    int64_t lastValues = 0;
};

namespace mbar {

// max that keeps a NaN once it has seen one (np.amax propagates NaN)
__device__ __forceinline__ double nan_max(double m, double x) { return (x > m || x != x) && !(m != m) ? x : m; }

__device__ __forceinline__ double fermi_term(double w, double c1, double c2) {
    const double a = __dadd_rn(__dadd_rn(w, c1), c2);
    const double m = 0.0 < a ? a : 0.0;
    return __dsub_rn(-m, log(__dadd_rn(exp(-m), exp(__dsub_rn(a, m)))));
}

__device__ __forceinline__ double moments_term(double w, double c1, double A) {
    const double a = __dadd_rn(w, c1);
    return -log(__dadd_rn(exp(-A), exp(__dsub_rn(a, A))));
}

__device__ __forceinline__ int work_find(const WorkReq* __restrict__ req, int nReq, int64_t item) {
    int lo = 0, hi = nReq - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (req[mid].item0 <= item) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// fixed-order CTA combination of the 256 thread values (sum or NaN-keeping max)
template <bool MAX>
__device__ __forceinline__ double cta_reduce(double v, double* sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
#pragma unroll
    for (int s = WORK_THREADS / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) sh[threadIdx.x] = MAX ? nan_max(sh[threadIdx.x], sh[threadIdx.x + s])
                                                   : __dadd_rn(sh[threadIdx.x], sh[threadIdx.x + s]);
        __syncthreads();
    }
    return sh[0];
}

// pass 1: per (request, chunk) the max of the terms (fermi kinds) or the plain sum (exp: x, gauss: w)
__global__ void __launch_bounds__(WORK_THREADS) work_pass1_kernel(const double* __restrict__ w,
                                                                  const WorkReq* __restrict__ req, int nReq,
                                                                  double* part) {
    __shared__ double sh[WORK_THREADS];
    const int64_t item = blockIdx.x;
    const int r = work_find(req, nReq, item);
    const WorkReq q = req[r];
    const int64_t c = item - q.item0;
    const int64_t i0 = c * q.cl, i1 = min(q.n, i0 + q.cl);
    const double* v = w + q.off;
    double acc;
    if (q.kind == MBAR_B200_WORK_FERMI || q.kind == MBAR_B200_WORK_FERMI_MOMENTS) {
        const double A = __dadd_rn(q.vmax, q.c1);
        acc = -INFINITY;
        for (int64_t i = i0 + threadIdx.x; i < i1; i += WORK_THREADS) {
            const double t = q.kind == MBAR_B200_WORK_FERMI ? fermi_term(__ldg(v + i), q.c1, q.c2)
                                                            : moments_term(__ldg(v + i), q.c1, A);
            acc = nan_max(acc, t);
        }
        acc = cta_reduce<true>(acc, sh);
    } else {
        const double amax = -q.vmin;
        acc = 0.0;
        for (int64_t i = i0 + threadIdx.x; i < i1; i += WORK_THREADS) {
            const double x = q.kind == MBAR_B200_WORK_EXP ? exp(__dsub_rn(-__ldg(v + i), amax)) : __ldg(v + i);
            acc = __dadd_rn(acc, x);
        }
        acc = cta_reduce<false>(acc, sh);
    }
    if (threadIdx.x == 0) part[2 * item] = acc;
}

// per request: the chunk partials of pass 1 in chunk order -> shift (non-finite max -> 0) or mean
__global__ void work_finalize1_kernel(const WorkReq* __restrict__ req, int nReq, const double* __restrict__ part,
                                      double* shift) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nReq) return;
    const WorkReq q = req[r];
    const int64_t nc = (q.n + q.cl - 1) / q.cl;
    if (q.kind == MBAR_B200_WORK_FERMI || q.kind == MBAR_B200_WORK_FERMI_MOMENTS) {
        double m = -INFINITY;
        for (int64_t c = 0; c < nc; ++c) m = nan_max(m, part[2 * (q.item0 + c)]);
        const double m2 = __dmul_rn(2.0, m);
        shift[2 * r] = isfinite(m) ? m : 0.0;
        shift[2 * r + 1] = isfinite(m2) ? m2 : 0.0;
    } else {
        double s = 0.0;
        for (int64_t c = 0; c < nc; ++c) s = __dadd_rn(s, part[2 * (q.item0 + c)]);
        shift[2 * r] = s;
        shift[2 * r + 1] = __ddiv_rn(s, (double)q.n);
    }
}

// pass 2: per (request, chunk) the shifted exponential sums (fermi kinds) or the centred squares
__global__ void __launch_bounds__(WORK_THREADS) work_pass2_kernel(const double* __restrict__ w,
                                                                  const WorkReq* __restrict__ req, int nReq,
                                                                  const double* __restrict__ shift, double* part) {
    __shared__ double sh[WORK_THREADS];
    const int64_t item = blockIdx.x;
    const int r = work_find(req, nReq, item);
    const WorkReq q = req[r];
    const int64_t c = item - q.item0;
    const int64_t i0 = c * q.cl, i1 = min(q.n, i0 + q.cl);
    const double* v = w + q.off;
    double s0 = 0.0, s1 = 0.0;
    if (q.kind == MBAR_B200_WORK_FERMI) {
        const double M = shift[2 * r];
        for (int64_t i = i0 + threadIdx.x; i < i1; i += WORK_THREADS)
            s0 = __dadd_rn(s0, exp(__dsub_rn(fermi_term(__ldg(v + i), q.c1, q.c2), M)));
    } else if (q.kind == MBAR_B200_WORK_FERMI_MOMENTS) {
        const double A = __dadd_rn(q.vmax, q.c1);
        const double M = shift[2 * r], M2 = shift[2 * r + 1];
        for (int64_t i = i0 + threadIdx.x; i < i1; i += WORK_THREADS) {
            const double t = moments_term(__ldg(v + i), q.c1, A);
            s0 = __dadd_rn(s0, exp(__dsub_rn(t, M)));
            s1 = __dadd_rn(s1, exp(__dsub_rn(__dmul_rn(2.0, t), M2)));
        }
    } else {
        const double mean = shift[2 * r + 1], amax = -q.vmin;
        for (int64_t i = i0 + threadIdx.x; i < i1; i += WORK_THREADS) {
            const double x = q.kind == MBAR_B200_WORK_EXP ? exp(__dsub_rn(-__ldg(v + i), amax)) : __ldg(v + i);
            const double d = __dsub_rn(x, mean);
            s0 = __dadd_rn(s0, __dmul_rn(d, d));
        }
    }
    s0 = cta_reduce<false>(s0, sh);
    if (q.kind == MBAR_B200_WORK_FERMI_MOMENTS) {
        __syncthreads();
        s1 = cta_reduce<false>(s1, sh);
    }
    if (threadIdx.x == 0) {
        part[2 * item] = s0;
        part[2 * item + 1] = s1;
    }
}

// per request: the pass-2 partials in chunk order -> out [3]
__global__ void work_finalize2_kernel(const WorkReq* __restrict__ req, int nReq, const double* __restrict__ part,
                                      const double* __restrict__ shift, double* out) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nReq) return;
    const WorkReq q = req[r];
    const int64_t nc = (q.n + q.cl - 1) / q.cl;
    double s0 = 0.0, s1 = 0.0;
    for (int64_t c = 0; c < nc; ++c) {
        s0 = __dadd_rn(s0, part[2 * (q.item0 + c)]);
        s1 = __dadd_rn(s1, part[2 * (q.item0 + c) + 1]);
    }
    double* o = out + 3 * r;
    switch (q.kind) {
        case MBAR_B200_WORK_FERMI:
            o[0] = __dadd_rn(log(s0), shift[2 * r]);
            o[1] = o[2] = 0.0;
            break;
        case MBAR_B200_WORK_FERMI_MOMENTS:
            o[0] = __dadd_rn(log(s0), shift[2 * r]);
            o[1] = __dadd_rn(log(s1), shift[2 * r + 1]);
            o[2] = __dadd_rn(q.vmax, q.c1);
            break;
        case MBAR_B200_WORK_EXP:
            o[0] = __dadd_rn(log(shift[2 * r]), -q.vmin);
            o[1] = shift[2 * r];
            o[2] = s0;
            break;
        default:
            o[0] = shift[2 * r];
            o[1] = s0;
            o[2] = 0.0;
    }
}

}  // namespace mbar

using namespace mbar;

int mbar_b200_work_create(int device, int64_t n_total, const double* w, int32_t n_vectors, const int64_t* offsets,
                          mbar_b200_work** out) {
    MBAR_REQUIRE(out && w && offsets, MBAR_B200_ERR_INVALID, "work_create: NULL argument");
    *out = nullptr;
    MBAR_REQUIRE(n_vectors >= 1, MBAR_B200_ERR_INVALID, "work_create: %d vectors", (int)n_vectors);
    MBAR_REQUIRE(n_total >= 1 && n_total < (int64_t(1) << 40), MBAR_B200_ERR_INVALID, "work_create: n_total=%lld",
                 (long long)n_total);
    MBAR_REQUIRE(offsets[0] == 0 && offsets[n_vectors] == n_total, MBAR_B200_ERR_INVALID,
                 "work_create: offsets must run from 0 to n_total=%lld", (long long)n_total);
    for (int v = 0; v < n_vectors; ++v)
        MBAR_REQUIRE(offsets[v + 1] > offsets[v], MBAR_B200_ERR_INVALID,
                     "work_create: vector %d is empty or offsets decrease", v);
    std::vector<double> vmin((size_t)n_vectors), vmax((size_t)n_vectors);
    for (int v = 0; v < n_vectors; ++v) {
        double lo = INFINITY, hi = -INFINITY;
        for (int64_t i = offsets[v]; i < offsets[v + 1]; ++i) {
            MBAR_REQUIRE(std::isfinite(w[i]), MBAR_B200_ERR_NAN, "work_create: w[%lld] is %g", (long long)i, w[i]);
            lo = std::min(lo, w[i]);
            hi = std::max(hi, w[i]);
        }
        vmin[v] = lo;
        vmax[v] = hi;
    }
    MBAR_TRY(open_device(device, nullptr));
    std::unique_ptr<mbar_b200_work> o(new mbar_b200_work());
    o->nTotal = n_total;
    o->nVec = n_vectors;
    o->offsets.assign(offsets, offsets + n_vectors + 1);
    o->vmin.swap(vmin);
    o->vmax.swap(vmax);
    MBAR_TRY(o->open(device, "work_create"));
    MBAR_TRY(o->upload(o->d_w, w, (size_t)n_total, "work_create"));
    *out = o.release();
    return MBAR_B200_OK;
}

int mbar_b200_work_destroy(mbar_b200_work* o) { return destroy_resident(o); }

int mbar_b200_work_evaluate(mbar_b200_work* o, int32_t n_requests, const int32_t* vector, const int32_t* kind,
                            const double* c1, const double* c2, double* out) {
    MBAR_REQUIRE(o, MBAR_B200_ERR_INVALID, "work_evaluate: NULL object");
    MBAR_REQUIRE(n_requests >= 1, MBAR_B200_ERR_INVALID, "work_evaluate: %d requests", (int)n_requests);
    MBAR_REQUIRE(vector && kind && c1 && c2 && out, MBAR_B200_ERR_INVALID, "work_evaluate: NULL argument");
    std::vector<WorkReq> req((size_t)n_requests);
    int64_t items = 0, values = 0;
    for (int r = 0; r < n_requests; ++r) {
        const int v = vector[r];
        MBAR_REQUIRE(v >= 0 && v < o->nVec, MBAR_B200_ERR_INVALID, "work_evaluate: request %d names vector %d of %d", r,
                     v, o->nVec);
        MBAR_REQUIRE(kind[r] >= MBAR_B200_WORK_FERMI && kind[r] <= MBAR_B200_WORK_GAUSS, MBAR_B200_ERR_INVALID,
                     "work_evaluate: request %d has unknown kind %d", r, (int)kind[r]);
        WorkReq& q = req[r];
        q.off = o->offsets[v];
        q.n = o->offsets[v + 1] - o->offsets[v];
        q.cl = work_chunk_len(q.n);
        q.item0 = items;
        q.c1 = c1[r];
        q.c2 = c2[r];
        q.vmin = o->vmin[v];
        q.vmax = o->vmax[v];
        q.kind = kind[r];
        items += (q.n + q.cl - 1) / q.cl;
        values += 2 * q.n;
    }
    MBAR_REQUIRE(items < INT32_MAX, MBAR_B200_ERR_INVALID, "work_evaluate: %lld chunks in one call", (long long)items);
    MBAR_CUDA(cudaSetDevice(o->device));
    NvtxRange nvtx_("mbar_b200::work_evaluate");
    MBAR_TRY(o->d_req.grow(n_requests, "work"));
    MBAR_TRY(o->d_part.grow(2 * items, "work"));
    MBAR_TRY(o->d_shift.grow(2 * (int64_t)n_requests, "work"));
    MBAR_TRY(o->d_out.grow(3 * (int64_t)n_requests, "work"));
    MBAR_CUDA(cudaMemcpyAsync(o->d_req, req.data(), req.size() * sizeof(WorkReq), cudaMemcpyHostToDevice, o->stream));
    const unsigned rb = (unsigned)((n_requests + 127) / 128);
    MBAR_CUDA(cudaEventRecord(o->ev0, o->stream));
    work_pass1_kernel<<<(unsigned)items, WORK_THREADS, 0, o->stream>>>(o->d_w, o->d_req, n_requests, o->d_part);
    work_finalize1_kernel<<<rb, 128, 0, o->stream>>>(o->d_req, n_requests, o->d_part, o->d_shift);
    work_pass2_kernel<<<(unsigned)items, WORK_THREADS, 0, o->stream>>>(o->d_w, o->d_req, n_requests, o->d_shift,
                                                                        o->d_part);
    work_finalize2_kernel<<<rb, 128, 0, o->stream>>>(o->d_req, n_requests, o->d_part, o->d_shift, o->d_out);
    MBAR_CUDA(cudaGetLastError());
    MBAR_CUDA(cudaEventRecord(o->ev1, o->stream));
    MBAR_CUDA(cudaMemcpyAsync(out, o->d_out, (size_t)n_requests * 3 * sizeof(double), cudaMemcpyDeviceToHost,
                              o->stream));
    MBAR_CUDA(cudaStreamSynchronize(o->stream));
    float e = 0.f;
    o->lastMs = event_ms(o->ev0, o->ev1, &e) ? e : 0.0;
    o->lastLaunches = 4;
    o->lastValues = values;
    return MBAR_B200_OK;
}

int mbar_b200_last_work_stats(mbar_b200_work* o, double* ms, int32_t* launches, int64_t* values_read) {
    MBAR_REQUIRE(o, MBAR_B200_ERR_INVALID, "NULL work object");
    if (ms) *ms = o->lastMs;
    if (launches) *launches = o->lastLaunches;
    if (values_read) *values_read = o->lastValues;
    return MBAR_B200_OK;
}

// mbar_b200_acf_*: the centred lag sums behind pymbar.timeseries (statistical_inefficiency, _multiple,
// normalized_fluctuation_correlation_function and detect_equilibration, timeseries.py:83-836).  For a start s of a
// series of length T (m = T - s) and a lag t the reference evaluates
//
//   S(s, t) = sum_{n = s}^{T - 1 - t} dA[n] dB[n + t] (+ dB[n] dA[n + t] for a cross-correlation),
//   dA[n] = A[n] - mean(A[s:]),
//
// and walks t = 1, 2, ... (fast: increments 1, 2, 3, ...) until C(t) = S / (2 (m - t) sigma^2) <= 0 past mintime.
//
// Decomposition.  A call works on a grid: a list of series, series k the samples [off_k, off_k + N_k) cut into chunks
// of NC_k = max(512, ceil(N_k / 1024)) samples from off_k (acf_grid).  An unsegmented object, and the pooled rule 1 of
// a segmented one, is the one-series grid of the whole object; mbar_b200_acf_inefficiency_series and
// correlation_multiple use the grid of the object's segments, so no chunk straddles two series.  A request is a
// (series, start) pair.  The partial of one (request, lag, chunk) is a sequential sum, from 0.0, over the chunk's
// n >= s with n + t inside the series (or, rule 1, inside its segment), and a (request, lag) sum adds the partials of
// chunks chunk(s), chunk(s) + 1, ... of its series in that order, from 0.0.  The means are the same construction with
// the term A[n].  Every term is the reference's, rounded as numpy rounds it (__dmul_rn / __dadd_rn, no contraction);
// only the order of the sums differs from numpy's pairwise one.  Nothing depends on the other requests of a call, on
// the lag batches or on the launch shapes: a request's results are the same bits in any call, and the same as those of
// its series alone in an unsegmented object.
//
// Rounds.  The stop rule is sequential, so each round evaluates a batch of lag indices for every active request, and
// acf_walk_kernel then walks each request's batch in lag order, applies the rule, accumulates g and retires the
// request at its own limit.  The batches are 8, 8, 16, 32, ... lag indices, so the lags evaluated never exceed twice
// those needed plus 8, and the host polls once per round: the number of rounds grows like log L.
//
// Ragged launch.  A request has cnt = (chunks of its series) - chunk(s) chunks to sum.  The lag launch orders its
// requests by cnt, largest first, and row r of the launch holds the requests with cnt > r at the r-th chunk from the
// end of their series; one thread owns a (row, request) item and ACF_RL consecutive lags.  The launch covers exactly
// the (request, chunk) pairs the sums read, and the threads of a row that belong to one series read the same chunk.
#include <algorithm>
#include <cmath>
#include <memory>
#include <vector>

#include "internal.cuh"

namespace mbar {

constexpr int ACF_THREADS = 256;
constexpr int ACF_RL = 4;                          // lags per thread
constexpr int ACF_B0 = 8;                          // lag indices of the first round
constexpr int64_t ACF_MAX_CHUNKS = 1024;           // NC = max(512, ceil(N / 1024))
constexpr int64_t ACF_MIN_NC = 512;
constexpr int64_t ACF_PART_BUDGET = int64_t(1) << 25;   // doubles of (request, lag, chunk) partials per launch

inline int64_t acf_chunk_size(int64_t N) { return std::max<int64_t>(ACF_MIN_NC, (N + ACF_MAX_CHUNKS - 1) / ACF_MAX_CHUNKS); }

// The chunks of a list of series: series k is [off[k], off[k + 1]), cut into its chunks [chunkOff[k], chunkOff[k + 1])
// of NC[k] samples; chunk c is [lo[c], hi[c]).
// On the device the five arrays sit in one buffer, d_all (one upload).
struct AcfGrid {
    int K = 0;
    std::vector<int64_t> off, NC, chunkOff, lo, hi;
    DevArray<int64_t> d_all;
    const int64_t *d_off = nullptr, *d_NC = nullptr, *d_chunkOff = nullptr, *d_lo = nullptr, *d_hi = nullptr;
    int64_t nChunks() const { return (int64_t)lo.size(); }
};

// the grid of K series of the given lengths, the one construction behind every call
inline void acf_grid(const int64_t* lengths, int K, AcfGrid& g) {
    g.K = K;
    g.off.assign((size_t)K + 1, 0);
    g.NC.assign((size_t)K, 0);
    g.chunkOff.assign((size_t)K + 1, 0);
    g.lo.clear();
    g.hi.clear();
    for (int k = 0; k < K; ++k) {
        const int64_t L = lengths[k], o = g.off[k];
        g.NC[k] = acf_chunk_size(L);
        for (int64_t x = 0; x < L; x += g.NC[k]) {
            g.lo.push_back(o + x);
            g.hi.push_back(o + std::min(L, x + g.NC[k]));
        }
        g.off[k + 1] = o + L;
        g.chunkOff[k + 1] = (int64_t)g.lo.size();
    }
}

}  // namespace mbar

struct mbar_b200_acf : mbar::Resident {
    int64_t T = 0;
    int64_t NC = 0, nChunks = 0;        // of the whole-object grid
    int cross = 0;
    int nSeg = 0;                       // 0: one series
    mbar::DevArray<double> d_a;
    mbar::DevArray<double> d_bOwn;      // B of a cross-correlation
    double* d_b = nullptr;              // the B the kernels read: d_bOwn, or d_a for an autocorrelation
    mbar::DevArray<int64_t> d_segEnd;   // [T] end of the segment holding n, or NULL
    mbar::DevArray<int64_t> d_segLen;   // [nSeg]
    std::vector<int64_t> segLen;
    mbar::AcfGrid whole;                // the object as one series
    mbar::AcfGrid series;               // its segments (nSeg > 0)
    int lastRounds = 0;
    int64_t lastTerms = 0, lastUseful = 0;
};

namespace mbar {

__host__ __device__ __forceinline__ int64_t acf_lag(int64_t i, int fast) {
    return fast ? 1 + i * (i + 1) / 2 : i + 1;
}

// A grid on the device and the series of each request (NULL: every request is on series 0)
struct AcfSeries {
    const int64_t* off;         // [K + 1]
    const int64_t* NC;          // [K]
    const int64_t* chunkOff;    // [K + 1]
    const int32_t* ser;         // [requests] or NULL
};

struct AcfReq {
    int64_t off, len, NC, c0, nck;   // series samples [off, off + len), its chunks [c0, c0 + nck) of NC samples
};

__device__ __forceinline__ AcfReq acf_req(const AcfSeries& v, int64_t j) {
    const int k = v.ser ? v.ser[j] : 0;
    AcfReq r;
    r.off = v.off[k];
    r.len = v.off[k + 1] - r.off;
    r.NC = v.NC[k];
    r.c0 = v.chunkOff[k];
    r.nck = v.chunkOff[k + 1] - r.c0;
    return r;
}

// chunk totals of A and B: tot[c] = 0.0 + sum over [lo[c], hi[c]) in n order
__global__ void acf_total_kernel(const double* __restrict__ a, const double* __restrict__ b,
                                 const int64_t* __restrict__ lo, const int64_t* __restrict__ hi, int64_t nChunks,
                                 double* totA, double* totB) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nChunks) return;
    double sa = 0.0, sb = 0.0;
    for (int64_t n = lo[c]; n < hi[c]; ++n) {
        sa = __dadd_rn(sa, a[n]);
        sb = __dadd_rn(sb, b[n]);
    }
    totA[c] = sa;
    totB[c] = sb;
}

// means of A[s:] and B[s:] of each request's series: the head of chunk(s) from s, then the series' following chunk
// totals in order
__global__ void acf_mean_kernel(const double* __restrict__ a, const double* __restrict__ b, AcfSeries v,
                                const double* __restrict__ totA, const double* __restrict__ totB,
                                const int64_t* __restrict__ starts, int64_t nStarts, double* muA, double* muB) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nStarts) return;
    const int64_t s = starts[j];
    const AcfReq R = acf_req(v, j);
    const int64_t c = s / R.NC, c1 = R.off + min(R.len, (c + 1) * R.NC);
    double ha = 0.0, hb = 0.0;
    for (int64_t n = R.off + s; n < c1; ++n) {
        ha = __dadd_rn(ha, a[n]);
        hb = __dadd_rn(hb, b[n]);
    }
    double sa = __dadd_rn(0.0, ha), sb = __dadd_rn(0.0, hb);
    for (int64_t k = R.c0 + c + 1; k < R.c0 + R.nck; ++k) {
        sa = __dadd_rn(sa, totA[k]);
        sb = __dadd_rn(sb, totB[k]);
    }
    muA[j] = __ddiv_rn(sa, (double)(R.len - s));
    muB[j] = __ddiv_rn(sb, (double)(R.len - s));
}

struct AcfLagParams {
    const double* a;
    const double* b;
    const int64_t* segEnd;      // SEG: [T] end of the segment holding n
    AcfSeries v;
    const int64_t* starts;      // [call requests], from the start of each request's series
    const double* muA;
    const double* muB;
    const int32_t* act;         // this launch's requests, chunk counts non-increasing: act[0 .. nAct)
    const int64_t* rowOff;      // [rows + 1] first item of each row; row r holds act[0 .. rowOff[r + 1] - rowOff[r])
    const int64_t* lags;        // this launch's lags, ascending: lags[0 .. nLags)
    double* partial;            // [items][nLags], item rowOff[r] + si
    int rows, nLags, LG;        // LG = ceil(nLags / ACF_RL) lag groups per item
};

// one (item, ACF_RL lags) per thread; item rowOff[r] + si is request act[si] at the r-th chunk from the end of its
// series
template <bool CROSS, bool SEG>
__global__ void __launch_bounds__(ACF_THREADS) acf_lag_partial_kernel(AcfLagParams p) {
    const int64_t q = (int64_t)blockIdx.x * ACF_THREADS + threadIdx.x;
    const int64_t item = q / p.LG;
    const int lg = (int)(q % p.LG);
    if (item >= p.rowOff[p.rows]) return;
    int rlo = 0, rhi = p.rows;                 // rowOff[rlo] <= item < rowOff[rhi]
    while (rhi - rlo > 1) {
        const int mid = (rlo + rhi) >> 1;
        if (p.rowOff[mid] <= item) rlo = mid;
        else rhi = mid;
    }
    const int64_t si = item - p.rowOff[rlo];
    const int j = p.act[si];
    const int64_t s = p.starts[j];
    const AcfReq R = acf_req(p.v, j);
    const int64_t c0 = R.off + (R.nck - 1 - rlo) * R.NC, c1 = min(R.off + R.len, c0 + R.NC);
    const double mua = p.muA[j], mub = p.muB[j];
    int64_t t[ACF_RL];
    double acc[ACF_RL];
    const int jl0 = lg * ACF_RL;
#pragma unroll
    for (int r = 0; r < ACF_RL; ++r) {
        t[r] = (jl0 + r < p.nLags) ? p.lags[jl0 + r] : INT64_MAX / 2;
        acc[r] = 0.0;
    }
    const int64_t send = R.off + R.len;
    const int64_t lo = max(c0, R.off + s);
    const int64_t hi = SEG ? c1 : min(c1, send - t[0]);
    for (int64_t n = lo; n < hi; ++n) {
        const double da = __dsub_rn(__ldg(p.a + n), mua);
        const double db = CROSS ? __dsub_rn(__ldg(p.b + n), mub) : da;
        const int64_t end = SEG ? __ldg(p.segEnd + n) : send;
#pragma unroll
        for (int r = 0; r < ACF_RL; ++r) {
            if (n + t[r] < end) {
                double term = __dmul_rn(da, __dsub_rn(__ldg(p.b + n + t[r]), mub));
                if (CROSS) term = __dadd_rn(term, __dmul_rn(db, __dsub_rn(__ldg(p.a + n + t[r]), mua)));
                acc[r] = __dadd_rn(acc[r], term);
            }
        }
    }
#pragma unroll
    for (int r = 0; r < ACF_RL; ++r)
        if (jl0 + r < p.nLags) p.partial[item * p.nLags + jl0 + r] = acc[r];
}

// S[row[si] * ldS + col0 + jl] (row NULL: row0 + si) = 0.0 + partials of chunks chunk(s), chunk(s) + 1, ... in
// order (rows cnt - 1 .. 0)
__global__ void acf_reduce_kernel(const double* __restrict__ partial, AcfSeries v, const int64_t* __restrict__ starts,
                                  const int32_t* __restrict__ act, const int32_t* __restrict__ row, int row0,
                                  const int64_t* __restrict__ rowOff, int nAct, int nLags, double* S, int ldS,
                                  int col0) {
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t pairs = (int64_t)nAct * nLags;
    if (q >= pairs) return;
    const int si = (int)(q / nLags), jl = (int)(q % nLags);
    const int j = act[si];
    const AcfReq R = acf_req(v, j);
    const int64_t cnt = R.nck - starts[j] / R.NC;
    double sum = 0.0;
    for (int64_t r = cnt - 1; r >= 0; --r) sum = __dadd_rn(sum, partial[(rowOff[r] + si) * nLags + jl]);
    S[(int64_t)(row ? row[si] : row0 + si) * ldS + col0 + jl] = sum;
}

// sigma^2 from the lag-0 sums; status 1 where it is 0 (the reference's ParameterError)
__global__ void acf_sigma_kernel(const double* __restrict__ S0, AcfSeries v, const int64_t* __restrict__ starts,
                                 int64_t nStarts, int cross, double* sigma2, int32_t* status, int8_t* done) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nStarts) return;
    const AcfReq R = acf_req(v, j);
    const double sum = cross ? __dmul_rn(0.5, S0[j]) : S0[j];
    const double s2 = __ddiv_rn(sum, (double)(R.len - starts[j]));
    sigma2[j] = s2;
    status[j] = s2 == 0.0 ? 1 : 0;
    done[j] = s2 == 0.0 ? 1 : 0;
}

struct AcfWalkParams {
    AcfSeries v;
    const int64_t* starts;
    const int32_t* act;
    const double* S;            // [nAct][B]
    const double* sigma2;
    const int64_t* segLen;      // multiple rule
    int nSeg;
    int nAct, B;
    int64_t i0;                 // first lag index of the batch
    int fast, multiple, cross;
    int fft;                    // rule 2: statistical_inefficiency_fft's acf and its lags 1 .. m - 1
    int64_t mintime;
    double navg;
    int64_t limitMultiple;      // max N_k (multiple rule)
    double* g;
    int64_t* lastLag;
    int8_t* done;
    double* trace;
    int64_t traceCap;
};

// the reference's loop over this batch's lags, for one request, in the reference's fp64 operations
__global__ void acf_walk_kernel(AcfWalkParams p) {
    const int si = blockIdx.x * blockDim.x + threadIdx.x;
    if (si >= p.nAct) return;
    const int j = p.act[si];
    const int64_t s = p.starts[j];
    const int64_t m = acf_req(p.v, j).len - s;
    const int64_t limit = p.multiple ? p.limitMultiple : (p.fft ? m + 1 : m);
    const double s2 = p.sigma2[j];
    double g = p.g[j];
    int64_t last = p.lastLag[j];
    int8_t fin = 0;
    for (int k = 0; k < p.B && !fin; ++k) {
        const int64_t i = p.i0 + k;
        const int64_t t = acf_lag(i, p.fast);
        if (t >= limit - 1) {
            fin = 1;
            break;
        }
        const double sum = p.S[(int64_t)si * p.B + k];
        double C;
        if (p.multiple) {
            int64_t den = 0;
            for (int q = 0; q < p.nSeg; ++q)
                if (t < p.segLen[q]) den += p.segLen[q] - t;
            C = __ddiv_rn(__ddiv_rn(sum, (double)den), s2);
        } else if (p.fft) {
            C = __ddiv_rn(__ddiv_rn(sum, (double)(m - t)), s2);       // acov(t) / acov(0), acov(0) = sigma^2
        } else {
            const double num = p.cross ? sum : __dmul_rn(2.0, sum);
            C = __ddiv_rn(num, __dmul_rn(__dmul_rn(2.0, (double)(m - t)), s2));
        }
        if (p.trace && i < p.traceCap) p.trace[(int64_t)j * p.traceCap + i] = C;
        last = t;
        if (C <= 0.0 && t > (p.multiple ? 10 : p.mintime)) {
            fin = 1;
            break;
        }
        const double frac = p.multiple ? __ddiv_rn((double)t, p.navg) : __ddiv_rn((double)t, (double)m);
        const double inc = p.fast ? (double)(i + 1) : 1.0;
        g = __dadd_rn(g, __dmul_rn(__dmul_rn(__dmul_rn(2.0, C), __dsub_rn(1.0, frac)), inc));
    }
    if (!fin && acf_lag(p.i0 + p.B, p.fast) >= limit - 1) fin = 1;
    p.g[j] = g;
    p.lastLag[j] = last;
    p.done[j] = fin;
}

// C(t) = S / (2 (m - t) sigma^2) for the lags of one start
__global__ void acf_corr_kernel(const double* __restrict__ S, const int64_t* __restrict__ lags, int nLags, int64_t m,
                                int cross, const double* __restrict__ sigma2, double* C) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nLags) return;
    const double num = cross ? S[k] : __dmul_rn(2.0, S[k]);
    C[k] = __ddiv_rn(num, __dmul_rn(__dmul_rn(2.0, (double)(m - lags[k])), sigma2[0]));
}

// Lag sums of the call requests act_h[] (indices into the call's starts) for the ascending lags lags_h[], into
// d_S [nAct][ldS] at columns col0.. (row k of d_S: act_h[k]).  Orders the requests by chunk count, largest first, and
// splits lags and requests so that one launch's partials, counted over each request's own chunks, fit the budget.
// alloc() makes the device arrays of a call: the requests' starts and series (uploaded), their means (the caller
// computes them) and room for lag batches of up to lagCap lags.
struct AcfLagRunner {
    mbar_b200_acf* o;
    const AcfGrid* grid;
    bool cross;                 // the symmetrised term dA[n] dB[n + t] + dB[n] dA[n + t]; else dA[n] dB[n + t] alone
    bool seg;                   // bound the terms by the segment of n (rule 1 on the whole-object grid)
    const int64_t* hs;          // [call requests] host starts and series (NULL: series 0)
    const int32_t* hser;
    AcfSeries v{};
    int64_t* d_starts = nullptr;
    double* d_muA = nullptr;
    double* d_muB = nullptr;
    int32_t* d_act = nullptr;       // [n] act_h as given (the walk kernel reads it)
    int32_t* d_sact = nullptr;      // [2 n] act_h ordered by chunk count, then the d_S row of each entry
    int64_t* d_lags = nullptr;      // [lagCap]
    int64_t* d_rowOff = nullptr;    // [ACF_MAX_CHUNKS + 1]
    double* d_partial = nullptr;    // [partCap]
    int64_t partCap = 0;
    std::vector<int32_t> sact;       // [2 nAct]: order, then rows
    std::vector<int64_t> cnt, rowOff, bucket;

    int alloc(CallBuffers& buf, int64_t n, int64_t lagCap, int64_t partCap_) {
        int32_t* d_ser = nullptr;
        MBAR_TRY(buf.alloc(&d_starts, (size_t)n));
        if (hser) MBAR_TRY(buf.alloc(&d_ser, (size_t)n));
        MBAR_TRY(buf.alloc(&d_muA, (size_t)n));
        MBAR_TRY(buf.alloc(&d_muB, (size_t)n));
        MBAR_TRY(buf.alloc(&d_act, 3 * (size_t)n));
        MBAR_TRY(buf.alloc(&d_lags, (size_t)lagCap + ACF_MAX_CHUNKS + 1));
        MBAR_TRY(buf.alloc(&d_partial, (size_t)partCap_));
        d_sact = d_act + n;
        d_rowOff = d_lags + lagCap;
        partCap = partCap_;
        v = AcfSeries{grid->d_off, grid->d_NC, grid->d_chunkOff, d_ser};
        MBAR_CUDA(cudaMemcpyAsync(d_starts, hs, (size_t)n * sizeof(int64_t), cudaMemcpyHostToDevice, o->stream));
        if (hser)
            MBAR_CUDA(cudaMemcpyAsync(d_ser, hser, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, o->stream));
        return MBAR_B200_OK;
    }

    int64_t count(int32_t j) const {
        const int k = hser ? hser[j] : 0;
        return (grid->chunkOff[k + 1] - grid->chunkOff[k]) - hs[j] / grid->NC[k];
    }

    template <bool CROSS, bool SEG>
    void launch(const AcfLagParams& p, int64_t items) {
        const int64_t threads = items * p.LG;
        acf_lag_partial_kernel<CROSS, SEG>
            <<<(unsigned)((threads + ACF_THREADS - 1) / ACF_THREADS), ACF_THREADS, 0, o->stream>>>(p);
    }

    int run(const int32_t* act_h, int nAct, const int64_t* lags_h, int nLags, double* d_S, int ldS) {
        // counting sort by chunk count, largest first, stable; none where act_h is in that order already (one series
        // with ascending starts): the launch then reads d_act, and the rows are the identity
        cnt.resize((size_t)nAct);
        int64_t maxCnt = 0;
        bool sorted = true;
        for (int k = 0; k < nAct; ++k) {
            cnt[k] = count(act_h[k]);
            maxCnt = std::max(maxCnt, cnt[k]);
            sorted = sorted && (k == 0 || cnt[k] <= cnt[k - 1]);
        }
        const int32_t* d_order = d_act;
        const int32_t* d_row = nullptr;
        if (!sorted) {
            bucket.assign((size_t)maxCnt + 2, 0);
            for (int k = 0; k < nAct; ++k) ++bucket[maxCnt - cnt[k] + 1];
            for (int64_t c = 1; c <= maxCnt + 1; ++c) bucket[c] += bucket[c - 1];
            sact.resize(2 * (size_t)nAct);
            for (int k = 0; k < nAct; ++k) {
                const int64_t at = bucket[maxCnt - cnt[k]]++;
                sact[at] = act_h[k];
                sact[nAct + at] = k;
            }
            for (int k = 0; k < nAct; ++k) cnt[k] = count(sact[k]);
            d_order = d_sact;
            d_row = d_sact + nAct;
        }
        const int64_t pairsMax = std::max<int64_t>(ACF_RL, partCap / std::max<int64_t>(maxCnt, 1));
        const int lagStep = (int)std::min<int64_t>(nLags, std::max<int64_t>(ACF_RL, pairsMax / ACF_RL * ACF_RL));
        MBAR_CUDA(cudaMemcpyAsync(d_lags, lags_h, (size_t)nLags * sizeof(int64_t), cudaMemcpyHostToDevice, o->stream));
        MBAR_CUDA(cudaMemcpyAsync(d_act, act_h, (size_t)nAct * sizeof(int32_t), cudaMemcpyHostToDevice, o->stream));
        if (!sorted)
            MBAR_CUDA(cudaMemcpyAsync(d_sact, sact.data(), 2 * (size_t)nAct * sizeof(int32_t),
                                      cudaMemcpyHostToDevice, o->stream));
        // groups of consecutive requests whose items times lagStep fit the budget (at least one request)
        for (int a0 = 0; a0 < nAct;) {
            int a1 = a0;
            int64_t items = 0;
            while (a1 < nAct && (a1 == a0 || (items + cnt[a1]) * lagStep <= partCap)) items += cnt[a1++];
            const int na = a1 - a0;
            const int rows = (int)cnt[a0];
            rowOff.assign((size_t)rows + 1, 0);
            {
                int k = na;        // requests with cnt > r: a prefix of the group
                for (int r = 0; r < rows; ++r) {
                    while (k > 0 && cnt[a0 + k - 1] <= r) --k;
                    rowOff[r + 1] = rowOff[r] + k;
                }
            }
            MBAR_CUDA(cudaMemcpyAsync(d_rowOff, rowOff.data(), (size_t)(rows + 1) * sizeof(int64_t),
                                      cudaMemcpyHostToDevice, o->stream));
            for (int l0 = 0; l0 < nLags; l0 += lagStep) {
                const int nl = std::min(lagStep, nLags - l0);
                AcfLagParams p{};
                p.a = o->d_a;
                p.b = o->d_b;
                p.segEnd = o->d_segEnd;
                p.v = v;
                p.starts = d_starts;
                p.muA = d_muA;
                p.muB = d_muB;
                p.act = d_order + a0;
                p.rowOff = d_rowOff;
                p.lags = d_lags + l0;
                p.partial = d_partial;
                p.rows = rows;
                p.nLags = nl;
                p.LG = (nl + ACF_RL - 1) / ACF_RL;
                if (cross) {
                    if (seg) launch<true, true>(p, items);
                    else launch<true, false>(p, items);
                } else {
                    if (seg) launch<false, true>(p, items);
                    else launch<false, false>(p, items);
                }
                const int64_t pairs = (int64_t)na * nl;
                acf_reduce_kernel<<<(unsigned)((pairs + 255) / 256), 256, 0, o->stream>>>(
                    d_partial, v, d_starts, d_order + a0, d_row ? d_row + a0 : nullptr, a0, d_rowOff, na, nl, d_S,
                    ldS, l0);
                MBAR_CUDA(cudaGetLastError());
            }
            a0 = a1;
        }
        return MBAR_B200_OK;
    }
};

// the number of lag indices i with lag(i) <= last, and the sum of those lags
inline int64_t acf_lag_count(int64_t last, int fast) {
    if (last <= 0) return 0;
    if (!fast) return last;
    int64_t i = (int64_t)std::sqrt(2.0 * (double)last);
    while (i > 0 && acf_lag(i, 1) > last) --i;
    while (acf_lag(i + 1, 1) <= last) ++i;
    return i + 1;
}

inline int64_t acf_lag_total(int64_t count, int fast) {
    return fast ? count + (count - 1) * count * (count + 1) / 6 : count * (count + 1) / 2;
}

}  // namespace mbar

using namespace mbar;

int mbar_b200_acf_create(int device, int64_t T, const double* a, const double* b, int32_t n_segments,
                         const int64_t* offsets, mbar_b200_acf** out) {
    MBAR_REQUIRE(out && a, MBAR_B200_ERR_INVALID, "acf_create: NULL argument");
    *out = nullptr;
    MBAR_REQUIRE(T >= 1, MBAR_B200_ERR_INVALID, "acf_create: T=%lld must be >= 1", (long long)T);
    MBAR_REQUIRE(T < (int64_t(1) << 40), MBAR_B200_ERR_INVALID, "acf_create: T=%lld too large", (long long)T);
    MBAR_REQUIRE(n_segments >= 0, MBAR_B200_ERR_INVALID, "acf_create: %d segments", (int)n_segments);
    MBAR_REQUIRE(n_segments == 0 || offsets, MBAR_B200_ERR_INVALID, "acf_create: NULL segment offsets");
    if (n_segments > 0) {
        MBAR_REQUIRE(offsets[0] == 0 && offsets[n_segments] == T, MBAR_B200_ERR_INVALID,
                     "acf_create: segment offsets must run from 0 to T=%lld", (long long)T);
        for (int k = 0; k < n_segments; ++k)
            MBAR_REQUIRE(offsets[k + 1] > offsets[k], MBAR_B200_ERR_INVALID,
                         "acf_create: segment %d is empty or offsets decrease", k);
    }
    for (int64_t n = 0; n < T; ++n) {
        MBAR_REQUIRE(std::isfinite(a[n]), MBAR_B200_ERR_NAN, "acf_create: A[%lld] is %g", (long long)n, a[n]);
        MBAR_REQUIRE(!b || std::isfinite(b[n]), MBAR_B200_ERR_NAN, "acf_create: B[%lld] is %g", (long long)n,
                     b ? b[n] : 0.0);
    }
    MBAR_TRY(open_device(device, nullptr));
    std::unique_ptr<mbar_b200_acf> o(new mbar_b200_acf());
    o->T = T;
    o->NC = acf_chunk_size(T);
    o->nChunks = (T + o->NC - 1) / o->NC;
    o->cross = b ? 1 : 0;
    o->nSeg = n_segments;
    const char* who = "acf_create";
    MBAR_TRY(o->open(device, who));
    MBAR_TRY(o->upload(o->d_a, a, (size_t)T, who));
    if (b) MBAR_TRY(o->upload(o->d_bOwn, b, (size_t)T, who));
    o->d_b = b ? o->d_bOwn : o->d_a;
    auto uploadGrid = [&](AcfGrid& g) -> int {
        std::vector<int64_t> all;
        for (const std::vector<int64_t>* v : {&g.off, &g.NC, &g.chunkOff, &g.lo, &g.hi})
            all.insert(all.end(), v->begin(), v->end());
        MBAR_TRY(o->upload(g.d_all, all.data(), all.size(), who));
        g.d_off = g.d_all;
        g.d_NC = g.d_off + g.off.size();
        g.d_chunkOff = g.d_NC + g.NC.size();
        g.d_lo = g.d_chunkOff + g.chunkOff.size();
        g.d_hi = g.d_lo + g.lo.size();
        return MBAR_B200_OK;
    };
    acf_grid(&T, 1, o->whole);
    MBAR_TRY(uploadGrid(o->whole));
    if (n_segments > 0) {
        std::vector<int64_t> segEnd((size_t)T);
        o->segLen.resize((size_t)n_segments);
        for (int k = 0; k < n_segments; ++k) {
            o->segLen[k] = offsets[k + 1] - offsets[k];
            for (int64_t n = offsets[k]; n < offsets[k + 1]; ++n) segEnd[n] = offsets[k + 1];
        }
        MBAR_TRY(o->upload(o->d_segEnd, segEnd.data(), (size_t)T, who));
        MBAR_TRY(o->upload(o->d_segLen, o->segLen.data(), (size_t)n_segments, who));
        acf_grid(o->segLen.data(), n_segments, o->series);
        MBAR_TRY(uploadGrid(o->series));
    }
    *out = o.release();
    return MBAR_B200_OK;
}

int mbar_b200_acf_destroy(mbar_b200_acf* o) { return destroy_resident(o); }

// means (into the runner's) and sigma^2 of the call's n requests; done[j] = 1 where sigma^2 == 0
static int acf_moments(mbar_b200_acf* o, CallBuffers& buf, int64_t n, AcfLagRunner& run, double* d_s2,
                       int32_t* d_status, int8_t* d_done) {
    const AcfGrid& grid = *run.grid;
    const int64_t nc = grid.nChunks();
    double *d_totA, *d_totB, *d_S0;
    MBAR_TRY(buf.alloc(&d_totA, (size_t)nc));
    MBAR_TRY(buf.alloc(&d_totB, (size_t)nc));
    MBAR_TRY(buf.alloc(&d_S0, (size_t)n));
    acf_total_kernel<<<(unsigned)((nc + 127) / 128), 128, 0, o->stream>>>(o->d_a, o->d_b, grid.d_lo, grid.d_hi, nc,
                                                                        d_totA, d_totB);
    acf_mean_kernel<<<(unsigned)((n + 127) / 128), 128, 0, o->stream>>>(o->d_a, o->d_b, run.v, d_totA, d_totB,
                                                                      run.d_starts, n, run.d_muA, run.d_muB);
    MBAR_CUDA(cudaGetLastError());
    std::vector<int32_t> all((size_t)n);
    for (int64_t j = 0; j < n; ++j) all[j] = (int32_t)j;
    const int64_t zero = 0;
    MBAR_TRY(run.run(all.data(), (int)n, &zero, 1, d_S0, 1));
    acf_sigma_kernel<<<(unsigned)((n + 127) / 128), 128, 0, o->stream>>>(d_S0, run.v, run.d_starts, n, o->cross,
                                                                       d_s2, d_status, d_done);
    MBAR_CUDA(cudaGetLastError());
    return MBAR_B200_OK;
}

// The statistical-inefficiency loop of every request (series ser[j] of the grid, or series 0 where ser is NULL, from
// starts[j]); the arguments are checked by the caller.
static int acf_run(mbar_b200_acf* o, const AcfGrid& grid, int64_t n, const int64_t* starts, const int32_t* ser,
                   int32_t fast, int32_t mintime, int32_t rule, double navg, int64_t trace_cap, double* mean_a,
                   double* mean_b, double* sigma2, double* g, int64_t* last_lag, int32_t* status, double* trace) {
    MBAR_CUDA(cudaSetDevice(o->device));
    const std::vector<int64_t> hs(starts, starts + n);
    auto lenOf = [&](int64_t j) -> int64_t {
        const int k = ser ? ser[j] : 0;
        return grid.off[k + 1] - grid.off[k];
    };
    int64_t limitMultiple = 0;
    for (int64_t L : o->segLen) limitMultiple = std::max(limitMultiple, L);
    int64_t maxLimit = 0;
    // lags run while t < limit - 1: limit = m for rule 0, m + 1 for rule 2 (its lags include m - 1)
    for (int64_t j = 0; j < n; ++j)
        maxLimit = std::max(maxLimit, rule == 1 ? limitMultiple : lenOf(j) - hs[j] + (rule == 2 ? 1 : 0));
    CallBuffers buf("acf");
    double *d_s2, *d_g, *d_S, *d_trace = nullptr;
    int64_t* d_last;
    int32_t* d_status;
    int8_t* d_done;
    // the largest round: every request active, one batch of B lags; keep the [active][B] sums within the budget by
    // walking the requests in groups
    const int64_t partCap = std::min<int64_t>(ACF_PART_BUDGET, grid.nChunks() * std::max<int64_t>(n, 1) * 4096);
    MBAR_TRY(buf.alloc(&d_s2, (size_t)n));
    MBAR_TRY(buf.alloc(&d_g, (size_t)n));
    MBAR_TRY(buf.alloc(&d_last, (size_t)n));
    MBAR_TRY(buf.alloc(&d_status, (size_t)n));
    MBAR_TRY(buf.alloc(&d_done, (size_t)n));
    if (trace_cap > 0) MBAR_TRY(buf.alloc(&d_trace, (size_t)(n * trace_cap)));
    if (d_trace) MBAR_CUDA(cudaMemsetAsync(d_trace, 0xff, (size_t)(n * trace_cap) * sizeof(double), o->stream));
    std::vector<double> ones((size_t)n, 1.0);
    std::vector<int64_t> zeros((size_t)n, 0);
    MBAR_CUDA(cudaMemcpyAsync(d_g, ones.data(), (size_t)n * sizeof(double), cudaMemcpyHostToDevice, o->stream));
    MBAR_CUDA(cudaMemcpyAsync(d_last, zeros.data(), (size_t)n * sizeof(int64_t), cudaMemcpyHostToDevice, o->stream));
    // lag batches: 8, 8, 16, 32, ... indices; the walk groups hold at most budget / B requests
    int64_t Bmax = ACF_B0;
    {
        int64_t cum = ACF_B0;
        while (acf_lag(cum, fast) < maxLimit - 1) {
            Bmax = cum;
            cum *= 2;
        }
    }
    const int64_t walkCap = std::max<int64_t>(Bmax, std::min<int64_t>(n * Bmax, ACF_PART_BUDGET / 4));
    MBAR_TRY(buf.alloc(&d_S, (size_t)walkCap));
    AcfLagRunner run{o, &grid, o->cross != 0, rule == 1, hs.data(), ser};
    MBAR_TRY(run.alloc(buf, n, Bmax + 1, partCap));
    MBAR_CUDA(cudaEventRecord(o->ev0, o->stream));
    MBAR_TRY(acf_moments(o, buf, n, run, d_s2, d_status, d_done));
    std::vector<int8_t> done((size_t)n);
    MBAR_CUDA(cudaMemcpyAsync(done.data(), d_done, (size_t)n, cudaMemcpyDeviceToHost, o->stream));
    MBAR_CUDA(cudaStreamSynchronize(o->stream));
    std::vector<int32_t> active;
    for (int64_t j = 0; j < n; ++j)
        if (!done[j]) active.push_back((int32_t)j);
    int rounds = 0;
    int64_t terms = 0;
    int64_t i0 = 0, B = ACF_B0;
    std::vector<int64_t> lags, lagPrefix;
    // the (request, lag, n) terms of this round's lags: sum over lags t < m of m - t (rule 1: over the segments)
    auto roundTerms = [&](int64_t j) -> int64_t {
        if (rule == 1) {
            int64_t c = 0;
            for (int64_t t : lags)
                for (int64_t L : o->segLen) c += std::max<int64_t>(L - t, 0);
            return c;
        }
        const int64_t m = lenOf(j) - hs[j];
        const int64_t k = std::lower_bound(lags.begin(), lags.end(), m) - lags.begin();
        return k * m - lagPrefix[k];
    };
    while (!active.empty()) {
        lags.clear();
        for (int64_t i = i0; i < i0 + B && acf_lag(i, fast) < maxLimit - 1; ++i) lags.push_back(acf_lag(i, fast));
        lagPrefix.assign(lags.size() + 1, 0);
        for (size_t k = 0; k < lags.size(); ++k) lagPrefix[k + 1] = lagPrefix[k] + lags[k];
        const int nl = (int)lags.size();
        const int groupMax = (int)std::max<int64_t>(1, walkCap / std::max(nl, 1));
        for (size_t a0 = 0; a0 < active.size(); a0 += groupMax) {
            const int na = (int)std::min<size_t>(groupMax, active.size() - a0);
            if (nl > 0) MBAR_TRY(run.run(active.data() + a0, na, lags.data(), nl, d_S, nl));
            else MBAR_CUDA(cudaMemcpyAsync(run.d_act, active.data() + a0, (size_t)na * sizeof(int32_t),
                                           cudaMemcpyHostToDevice, o->stream));
            AcfWalkParams w{};
            w.v = run.v;
            w.starts = run.d_starts;
            w.act = run.d_act;
            w.S = d_S;
            w.sigma2 = d_s2;
            w.segLen = o->d_segLen;
            w.nSeg = o->nSeg;
            w.nAct = na;
            w.B = nl;
            w.i0 = i0;
            w.fast = fast ? 1 : 0;
            w.multiple = rule == 1;
            w.cross = o->cross;
            w.fft = rule == 2;
            w.mintime = mintime;
            w.navg = navg;
            w.limitMultiple = limitMultiple;
            w.g = d_g;
            w.lastLag = d_last;
            w.done = d_done;
            w.trace = d_trace;
            w.traceCap = trace_cap;
            // run() copied this group's active list to d_act[0..na)
            acf_walk_kernel<<<(unsigned)((na + 127) / 128), 128, 0, o->stream>>>(w);
            MBAR_CUDA(cudaGetLastError());
            for (int k = 0; k < na; ++k) terms += roundTerms(active[a0 + k]);
        }
        MBAR_CUDA(cudaMemcpyAsync(done.data(), d_done, (size_t)n, cudaMemcpyDeviceToHost, o->stream));
        MBAR_CUDA(cudaStreamSynchronize(o->stream));
        ++rounds;
        std::vector<int32_t> next;
        for (int32_t j : active)
            if (!done[j]) next.push_back(j);
        active.swap(next);
        i0 += B;
        if (rounds > 1) B *= 2;
    }
    MBAR_CUDA(cudaEventRecord(o->ev1, o->stream));
    if (mean_a)
        MBAR_CUDA(cudaMemcpyAsync(mean_a, run.d_muA, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    if (mean_b)
        MBAR_CUDA(cudaMemcpyAsync(mean_b, run.d_muB, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    if (sigma2) MBAR_CUDA(cudaMemcpyAsync(sigma2, d_s2, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    MBAR_CUDA(cudaMemcpyAsync(g, d_g, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    MBAR_CUDA(cudaMemcpyAsync(last_lag, d_last, (size_t)n * sizeof(int64_t), cudaMemcpyDeviceToHost, o->stream));
    MBAR_CUDA(cudaMemcpyAsync(status, d_status, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, o->stream));
    if (d_trace)
        MBAR_CUDA(cudaMemcpyAsync(trace, d_trace, (size_t)(n * trace_cap) * sizeof(double), cudaMemcpyDeviceToHost,
                                  o->stream));
    MBAR_CUDA(cudaStreamSynchronize(o->stream));
    // the lag terms the stop rule needed: every lag up to each request's last evaluated one (all below m - 1)
    int64_t useful = 0;
    for (int64_t j = 0; j < n; ++j) {
        if (status[j]) continue;
        const int64_t cnt = acf_lag_count(last_lag[j], fast);
        if (rule == 1) {
            for (int64_t i = 0; i < cnt; ++i)
                for (int64_t L : o->segLen) useful += std::max<int64_t>(L - acf_lag(i, fast), 0);
        } else {
            useful += cnt * (lenOf(j) - hs[j]) - acf_lag_total(cnt, fast);
        }
    }
    float e = 0.f;
    o->lastMs = event_ms(o->ev0, o->ev1, &e) ? e : 0.0;
    o->lastRounds = rounds;
    o->lastTerms = terms;
    o->lastUseful = useful;
    return MBAR_B200_OK;
}

int mbar_b200_acf_inefficiency(mbar_b200_acf* o, int64_t n_starts, const int64_t* starts, int32_t fast,
                               int32_t mintime, int32_t rule, double navg, int64_t trace_cap, double* mean_a,
                               double* mean_b, double* sigma2, double* g, int64_t* last_lag, int32_t* status,
                               double* trace) {
    MBAR_REQUIRE(o, MBAR_B200_ERR_INVALID, "acf_inefficiency: NULL object");
    MBAR_REQUIRE(n_starts >= 1 && n_starts < INT32_MAX && starts, MBAR_B200_ERR_INVALID,
                 "acf_inefficiency: %lld starts", (long long)n_starts);
    MBAR_REQUIRE(g && last_lag && status, MBAR_B200_ERR_INVALID, "acf_inefficiency: NULL output");
    MBAR_REQUIRE(rule >= 0 && rule <= 2, MBAR_B200_ERR_INVALID, "acf_inefficiency: unknown rule %d", (int)rule);
    MBAR_REQUIRE(trace_cap >= 0 && (trace_cap == 0 || trace), MBAR_B200_ERR_INVALID,
                 "acf_inefficiency: trace_cap %lld without a trace buffer", (long long)trace_cap);
    MBAR_REQUIRE(trace_cap <= (int64_t(1) << 31) / n_starts, MBAR_B200_ERR_INVALID,
                 "acf_inefficiency: trace of %lld x %lld too large", (long long)n_starts, (long long)trace_cap);
    if (rule == 1) {
        MBAR_REQUIRE(o->nSeg > 0 && !o->cross, MBAR_B200_ERR_INVALID,
                     "acf_inefficiency: the multiple-series rule needs segments and an autocorrelation");
        MBAR_REQUIRE(n_starts == 1 && starts[0] == 0, MBAR_B200_ERR_INVALID,
                     "acf_inefficiency: the multiple-series rule takes the single start 0");
        MBAR_REQUIRE(std::isfinite(navg) && navg > 0.0, MBAR_B200_ERR_INVALID, "acf_inefficiency: Navg = %g", navg);
    } else {
        MBAR_REQUIRE(o->nSeg == 0, MBAR_B200_ERR_INVALID, "acf_inefficiency: a segmented object takes rule 1");
    }
    if (rule == 2)
        MBAR_REQUIRE(!o->cross && !fast, MBAR_B200_ERR_INVALID,
                     "acf_inefficiency: the FFT rule needs an autocorrelation and fast = 0");
    for (int64_t j = 0; j < n_starts; ++j)
        MBAR_REQUIRE(starts[j] >= 0 && starts[j] < o->T, MBAR_B200_ERR_INVALID,
                     "acf_inefficiency: start %lld outside [0, %lld)", (long long)starts[j], (long long)o->T);
    NvtxRange nvtx_("mbar_b200::acf_inefficiency");
    return acf_run(o, o->whole, n_starts, starts, nullptr, fast, mintime, rule, navg, trace_cap, mean_a, mean_b, sigma2,
                   g, last_lag, status, trace);
}

int mbar_b200_acf_inefficiency_series(mbar_b200_acf* o, int64_t n, const int32_t* series, const int64_t* starts,
                                      int32_t fast, int32_t mintime, double* mean_a, double* mean_b, double* sigma2,
                                      double* g, int64_t* last_lag, int32_t* status) {
    MBAR_REQUIRE(o, MBAR_B200_ERR_INVALID, "acf_inefficiency_series: NULL object");
    MBAR_REQUIRE(n >= 1 && n < INT32_MAX && series && starts, MBAR_B200_ERR_INVALID,
                 "acf_inefficiency_series: %lld requests", (long long)n);
    MBAR_REQUIRE(g && last_lag && status, MBAR_B200_ERR_INVALID, "acf_inefficiency_series: NULL output");
    MBAR_REQUIRE(o->nSeg > 0, MBAR_B200_ERR_INVALID, "acf_inefficiency_series: the object holds no segments");
    for (int64_t j = 0; j < n; ++j) {
        MBAR_REQUIRE(series[j] >= 0 && series[j] < o->nSeg, MBAR_B200_ERR_INVALID,
                     "acf_inefficiency_series: request %lld: series %d outside [0, %d)", (long long)j, (int)series[j],
                     o->nSeg);
        MBAR_REQUIRE(starts[j] >= 0 && starts[j] < o->segLen[series[j]], MBAR_B200_ERR_INVALID,
                     "acf_inefficiency_series: request %lld: start %lld outside [0, %lld)", (long long)j,
                     (long long)starts[j], (long long)o->segLen[series[j]]);
    }
    NvtxRange nvtx_("mbar_b200::acf_inefficiency_series");
    return acf_run(o, o->series, n, starts, series, fast, mintime, 0, 0.0, 0, mean_a, mean_b, sigma2, g, last_lag,
                   status, nullptr);
}

int mbar_b200_acf_correlation(mbar_b200_acf* o, int64_t start, int64_t n_max, double* C, double* mean_a,
                              double* mean_b, double* sigma2) {
    MBAR_REQUIRE(o, MBAR_B200_ERR_INVALID, "acf_correlation: NULL object");
    MBAR_REQUIRE(C, MBAR_B200_ERR_INVALID, "acf_correlation: NULL output");
    MBAR_REQUIRE(o->nSeg == 0, MBAR_B200_ERR_INVALID, "acf_correlation: the object holds segments");
    MBAR_REQUIRE(start >= 0 && start < o->T, MBAR_B200_ERR_INVALID, "acf_correlation: start %lld outside [0, %lld)",
                 (long long)start, (long long)o->T);
    MBAR_REQUIRE(n_max >= 0 && n_max <= o->T - start - 1, MBAR_B200_ERR_INVALID,
                 "acf_correlation: N_max %lld outside [0, %lld]", (long long)n_max, (long long)(o->T - start - 1));
    MBAR_CUDA(cudaSetDevice(o->device));
    NvtxRange nvtx_("mbar_b200::acf_correlation");
    CallBuffers buf("acf");
    double *d_s2, *d_S, *d_C;
    int32_t* d_status;
    int8_t* d_done;
    const int64_t nl = n_max + 1;
    const int64_t batch = std::min<int64_t>(nl, 1 << 20);
    const int64_t partCap = std::min<int64_t>(ACF_PART_BUDGET, o->nChunks * batch);
    MBAR_TRY(buf.alloc(&d_s2, 1));
    MBAR_TRY(buf.alloc(&d_status, 1));
    MBAR_TRY(buf.alloc(&d_done, 1));
    MBAR_TRY(buf.alloc(&d_S, (size_t)batch));
    MBAR_TRY(buf.alloc(&d_C, (size_t)nl));
    AcfLagRunner run{o, &o->whole, o->cross != 0, false, &start, nullptr};
    MBAR_TRY(run.alloc(buf, 1, batch, partCap));
    MBAR_CUDA(cudaEventRecord(o->ev0, o->stream));
    MBAR_TRY(acf_moments(o, buf, 1, run, d_s2, d_status, d_done));
    double s2 = 0.0;
    MBAR_CUDA(cudaMemcpyAsync(&s2, d_s2, sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    MBAR_CUDA(cudaStreamSynchronize(o->stream));
    MBAR_REQUIRE(s2 != 0.0, MBAR_B200_ERR_INVALID, "acf_correlation: sigma^2 = 0 (constant series)");
    const int32_t act0 = 0;
    std::vector<int64_t> lags;
    for (int64_t l0 = 0; l0 < nl; l0 += batch) {
        const int64_t b = std::min(batch, nl - l0);
        lags.resize((size_t)b);
        for (int64_t k = 0; k < b; ++k) lags[k] = l0 + k;
        MBAR_TRY(run.run(&act0, 1, lags.data(), (int)b, d_S, (int)b));
        acf_corr_kernel<<<(unsigned)((b + 255) / 256), 256, 0, o->stream>>>(d_S, run.d_lags, (int)b, o->T - start,
                                                                           o->cross, d_s2, d_C + l0);
        MBAR_CUDA(cudaGetLastError());
        MBAR_CUDA(cudaStreamSynchronize(o->stream));   // d_lags is rewritten by the next batch
    }
    MBAR_CUDA(cudaEventRecord(o->ev1, o->stream));
    MBAR_CUDA(cudaMemcpyAsync(C, d_C, (size_t)nl * sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    if (mean_a) MBAR_CUDA(cudaMemcpyAsync(mean_a, run.d_muA, sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    if (mean_b) MBAR_CUDA(cudaMemcpyAsync(mean_b, run.d_muB, sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    if (sigma2) MBAR_CUDA(cudaMemcpyAsync(sigma2, d_s2, sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    MBAR_CUDA(cudaStreamSynchronize(o->stream));
    float e = 0.f;
    o->lastMs = event_ms(o->ev0, o->ev1, &e) ? e : 0.0;
    o->lastRounds = 0;
    o->lastTerms = o->lastUseful = 0;
    for (int64_t t = 0; t < nl; ++t) o->lastTerms += o->T - start - t;
    o->lastUseful = o->lastTerms;
    return MBAR_B200_OK;
}

// ---- normalized_fluctuation_correlation_function_multiple (timeseries.py:509-658) ----------------------------------
// Request k is series k of the object's segment grid from start 0, with the pooled means in its mean slots, and its
// lag sums are the runner's one-sided dA[n] dB[n + t] (on a cross object too): the reference's np.sum of series k.
// A lag's numerator is 0.0 + those sums in list order, as the reference adds one np.sum per series; the pooled means
// are the same construction over the chunk totals.
namespace mbar {

// pooled means (one thread): each series' chunk totals in order, the series in list order, over N; written to every
// request's slot
__global__ void acf_pooled_mean_kernel(const double* __restrict__ totA, const double* __restrict__ totB,
                                       const int64_t* __restrict__ chunkOff, int K, int64_t N, double* muA,
                                       double* muB) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    double pa = 0.0, pb = 0.0;
    for (int k = 0; k < K; ++k) {
        double sa = 0.0, sb = 0.0;
        for (int64_t c = chunkOff[k]; c < chunkOff[k + 1]; ++c) {
            sa = __dadd_rn(sa, totA[c]);
            sb = __dadd_rn(sb, totB[c]);
        }
        pa = __dadd_rn(pa, sa);
        pb = __dadd_rn(pb, sb);
    }
    const double ma = __ddiv_rn(pa, (double)N), mb = __ddiv_rn(pb, (double)N);
    for (int k = 0; k < K; ++k) {
        muA[k] = ma;
        muB[k] = mb;
    }
}

// per lag t = t0 + jl: numerator = 0.0 + S[k * ldS + jl] of the series with L_k > t in list order, denominator =
// 0.0 + (double)(L_k - t) over the same series; neg[jl] = 1 when a running numerator is negative (truncate,
// timeseries.py:641); out[jl] = (numerator / denominator) / sigma2, or numerator / denominator where sigma2 is NULL
// (lag 0, whose denominator is N exactly: sigma^2)
__global__ void acf_pooled_corr_kernel(const double* __restrict__ S, int ldS, const int64_t* __restrict__ segLen,
                                       int K, int64_t t0, int nLags, const double* __restrict__ sigma2, double* out,
                                       int8_t* neg) {
    const int jl = blockIdx.x * blockDim.x + threadIdx.x;
    if (jl >= nLags) return;
    const int64_t t = t0 + jl;
    double num = 0.0, den = 0.0;
    int8_t negative = 0;
    for (int k = 0; k < K; ++k) {
        if (t >= segLen[k]) continue;
        num = __dadd_rn(num, S[(int64_t)k * ldS + jl]);
        den = __dadd_rn(den, (double)(segLen[k] - t));
        if (num < 0.0) negative = 1;
    }
    const double q = __ddiv_rn(num, den);
    out[jl] = sigma2 ? __ddiv_rn(q, sigma2[0]) : q;
    if (neg) neg[jl] = negative;
}

// sum over lags t in [t0, t1) of max(L - t, 0): the lag terms of one series
inline int64_t seg_lag_terms(int64_t L, int64_t t0, int64_t t1) {
    const int64_t hi = std::min(t1, L);
    if (hi <= t0) return 0;
    const int64_t n = hi - t0;
    return n * L - (t0 + hi - 1) * n / 2;
}

}  // namespace mbar

int mbar_b200_acf_correlation_multiple(mbar_b200_acf* o, int64_t n_max, int32_t truncate, double* C,
                                       int64_t* n_out, double* mean_a, double* mean_b, double* sigma2) {
    MBAR_REQUIRE(o, MBAR_B200_ERR_INVALID, "acf_correlation_multiple: NULL object");
    MBAR_REQUIRE(C && n_out, MBAR_B200_ERR_INVALID, "acf_correlation_multiple: NULL output");
    MBAR_REQUIRE(o->nSeg > 0, MBAR_B200_ERR_INVALID, "acf_correlation_multiple: the object holds no segments");
    const int K = o->nSeg;
    int64_t Lmax = 0;
    for (int64_t L : o->segLen) Lmax = std::max(Lmax, L);
    MBAR_REQUIRE(n_max >= 0 && n_max <= Lmax - 1, MBAR_B200_ERR_INVALID,
                 "acf_correlation_multiple: N_max %lld outside [0, %lld]", (long long)n_max, (long long)(Lmax - 1));
    MBAR_CUDA(cudaSetDevice(o->device));
    NvtxRange nvtx_("mbar_b200::acf_correlation_multiple");
    const AcfGrid& grid = o->series;
    const int64_t nc = grid.nChunks();
    const int64_t nl = n_max + 1;
    // lag sums [K][batch] within a quarter of the partial budget, as the walk's
    const int64_t batch = std::min<int64_t>(nl, std::max<int64_t>(ACF_RL, ACF_PART_BUDGET / 4 / K));
    const int64_t partCap = std::min<int64_t>(ACF_PART_BUDGET, nc * batch);
    CallBuffers buf("acf");
    double *d_totA, *d_totB, *d_S, *d_s2, *d_C;
    int8_t* d_neg;
    MBAR_TRY(buf.alloc(&d_totA, (size_t)nc));
    MBAR_TRY(buf.alloc(&d_totB, (size_t)nc));
    MBAR_TRY(buf.alloc(&d_S, (size_t)(K * batch)));
    MBAR_TRY(buf.alloc(&d_s2, 1));
    MBAR_TRY(buf.alloc(&d_C, (size_t)nl));
    MBAR_TRY(buf.alloc(&d_neg, (size_t)nl));
    // request k: series k from start 0
    const std::vector<int64_t> hs((size_t)K, 0);
    std::vector<int32_t> ser((size_t)K);
    for (int k = 0; k < K; ++k) ser[k] = k;
    AcfLagRunner run{o, &grid, false, false, hs.data(), ser.data()};
    MBAR_TRY(run.alloc(buf, K, batch, partCap));
    MBAR_CUDA(cudaMemsetAsync(d_C, 0xff, (size_t)nl * sizeof(double), o->stream));
    std::vector<int64_t> lags;
    // lags [t0, t1) in batches of lag sums; out / neg indexed from t0
    auto evalLags = [&](int64_t t0, int64_t t1, const double* s2, double* out, int8_t* neg) -> int {
        for (int64_t x = t0; x < t1; x += batch) {
            const int n = (int)std::min(batch, t1 - x);
            lags.resize((size_t)n);
            for (int k = 0; k < n; ++k) lags[k] = x + k;
            MBAR_TRY(run.run(ser.data(), K, lags.data(), n, d_S, n));
            acf_pooled_corr_kernel<<<(unsigned)((n + 127) / 128), 128, 0, o->stream>>>(
                d_S, n, o->d_segLen, K, x, n, s2, out + (x - t0), neg ? neg + (x - t0) : nullptr);
            MBAR_CUDA(cudaGetLastError());
        }
        return MBAR_B200_OK;
    };
    MBAR_CUDA(cudaEventRecord(o->ev0, o->stream));
    acf_total_kernel<<<(unsigned)((nc + 127) / 128), 128, 0, o->stream>>>(o->d_a, o->d_b, grid.d_lo, grid.d_hi, nc,
                                                                        d_totA, d_totB);
    acf_pooled_mean_kernel<<<1, 32, 0, o->stream>>>(d_totA, d_totB, grid.d_chunkOff, K, o->T, run.d_muA,
                                                    run.d_muB);
    MBAR_CUDA(cudaGetLastError());
    MBAR_TRY(evalLags(0, 1, nullptr, d_s2, nullptr));
    double s2 = 0.0;
    MBAR_CUDA(cudaMemcpyAsync(&s2, d_s2, sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    MBAR_CUDA(cudaStreamSynchronize(o->stream));
    MBAR_REQUIRE(s2 != 0.0, MBAR_B200_ERR_INVALID, "acf_correlation_multiple: sigma^2 = 0 (constant series)");
    int64_t count = n_max, evaluated = nl;
    int rounds = 0;
    if (!truncate) {
        MBAR_TRY(evalLags(0, nl, d_s2, d_C, nullptr));
    } else {
        // the reference stops at the first lag whose running numerator is negative: rounds of 8, 8, 16, 32, ... lags
        std::vector<int8_t> neg;
        int64_t t0 = 0, B = ACF_B0;
        bool stop = false;
        while (!stop && t0 < nl) {
            const int64_t t1 = std::min(nl, t0 + B);
            MBAR_TRY(evalLags(t0, t1, d_s2, d_C + t0, d_neg + t0));
            neg.resize((size_t)(t1 - t0));
            MBAR_CUDA(cudaMemcpyAsync(neg.data(), d_neg + t0, (size_t)(t1 - t0), cudaMemcpyDeviceToHost, o->stream));
            MBAR_CUDA(cudaStreamSynchronize(o->stream));
            ++rounds;
            for (int64_t t = t0; t < t1; ++t)
                if (neg[t - t0]) {
                    count = t;
                    stop = true;
                    break;
                }
            evaluated = t1;
            t0 = t1;
            if (rounds > 1) B *= 2;
        }
    }
    MBAR_CUDA(cudaEventRecord(o->ev1, o->stream));
    MBAR_CUDA(cudaMemcpyAsync(C, d_C, (size_t)nl * sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    if (mean_a) MBAR_CUDA(cudaMemcpyAsync(mean_a, run.d_muA, sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    if (mean_b) MBAR_CUDA(cudaMemcpyAsync(mean_b, run.d_muB, sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    MBAR_CUDA(cudaStreamSynchronize(o->stream));
    *n_out = count;
    if (sigma2) *sigma2 = s2;
    float e = 0.f;
    o->lastMs = event_ms(o->ev0, o->ev1, &e) ? e : 0.0;
    o->lastRounds = rounds;
    // terms: every lag evaluated after sigma^2; useful: the lags the reference evaluates (through the stop lag)
    const int64_t needed = (truncate && count < n_max) ? count + 1 : nl;
    o->lastTerms = o->lastUseful = 0;
    for (int64_t L : o->segLen) {
        o->lastTerms += seg_lag_terms(L, 0, evaluated);
        o->lastUseful += seg_lag_terms(L, 0, needed);
    }
    return MBAR_B200_OK;
}

int mbar_b200_last_acf_stats(mbar_b200_acf* o, double* ms, int32_t* rounds, int64_t* terms, int64_t* useful_terms) {
    MBAR_REQUIRE(o, MBAR_B200_ERR_INVALID, "NULL acf object");
    if (ms) *ms = o->lastMs;
    if (rounds) *rounds = o->lastRounds;
    if (terms) *terms = o->lastTerms;
    if (useful_terms) *useful_terms = o->lastUseful;
    return MBAR_B200_OK;
}

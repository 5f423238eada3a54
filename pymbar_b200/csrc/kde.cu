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
#include <memory>
#include <vector>

#include "internal.cuh"

struct mbar_b200_kde : mbar::Resident {
    int D = 0;
    int64_t N = 0;
    int64_t nPad = 0;            // N rounded up to a tile
    int64_t chunkLen = 0;        // samples per chunk (a multiple of KDE_TILE)
    int nChunks = 0;
    mbar::DevArray<double> d_x;    // [D][nPad] coordinates, 0 in the padding
    mbar::DevArray<double> d_lw;   // [nPad] log w_n, -inf for zero weights and the padding
    mbar::DevArray<double> d_y;    // [D][qb] queries of one batch
    mbar::DevArray<double> d_pm;   // [nChunks][qb] running maxima
    mbar::DevArray<double> d_ps;   // [nChunks][qb] sums relative to them
    mbar::DevArray<double> d_out;  // [qb]
    int lastChunks = 0;
    // bootstrap replicates (mbar_b200_kde_set_replicates), in batches of KDE_REP_W
    int64_t B = 0;
    mbar::DevArray<double> d_lvm;  // [nRepBatches][nPad] log vmax_n = log max_b V_bn over the batch, -inf when 0
    mbar::DevArray<double> d_rat;  // [nRepBatches * KDE_REP_W][nPad] V_bn / vmax_n (0 where vmax_n = 0, padding rows)
    mbar::DevArray<double> d_rpm;  // [nChunks][KDE_REP_W][qb] partials of one (replicate batch, query batch)
    mbar::DevArray<double> d_rps;
    mbar::DevArray<double> d_rout;   // [KDE_REP_W][qb]
    mbar::DevArray<double> d_rflag;  // [KDE_REP_W][qb] 1 where the batch's shared scale may have lost digits
    mbar::DevArray<double> d_rlw;    // [nPad] log V_bn of one replicate, for the exact pass over flagged queries
};

// Many sample sets at once (mbar_b200_kde_many_*, DESIGN.md 3.5h''): only the coordinates are resident, each set laid
// out as mbar_b200_kde lays out its own; the weights come with every request.
struct mbar_b200_kde_many : mbar::Resident {
    std::vector<int> D;
    std::vector<int64_t> N, nPad, chunkLen, xoff;   // per set; xoff: first double of its [D][nPad] block
    std::vector<int> nChunks;
    mbar::DevArray<double> d_x;
    int32_t lastLaunches = 0;
    int64_t lastPairs = 0;
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
constexpr int KDE_REP_W = 8;                  // bootstrap replicates served by one pass over the samples
// What the shared scale of a replicate batch can lose (kde_replicates_kernel): a term or a rescaled partial sum is
// flushed only when it lies below 2^-1021 ~ e^-707 of the running scale m, and a partial sum is at most (terms) e^128
// of m (KDE_RESCALE), so all that is lost at a query is below N e^(M - 579), M the batch's final scale.  A replicate
// whose log sum l >= M - (KDE_REP_EXACT - log N) therefore has lost less than e^-30 of its sum; every other entry
// is recomputed by the single-replicate pass.
constexpr double KDE_REP_EXACT = 707.0 - KDE_RESCALE - 30.0;

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

// One thread's running (m, s) over the samples [n0, n1) of one chunk for its query y: the per-pair arithmetic of every
// single-replicate KDE pass (kde_partial_kernel, kde_many_partial_kernel), stated once so that both give the same
// bits.  p holds KdeParams' x [D][nPad], lw [nPad], nPad, h, hh, c and T (the kernel's parameters, or a copy in shared
// memory); sx, slw and tab are the CTA's shared tiles and exp table.
template <int D, int KERN, class P>
__device__ __forceinline__ void kde_chunk_sum(const P& p, int64_t n0, int64_t n1, const double (&y)[D],
                                              double (&sx)[D][KDE_TILE], double (&slw)[KDE_TILE], const double* tab,
                                              double& m_out, double& s_out) {
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
            const double lwi = slw[i];
            double a, k = 1.0;
            if (KERN == KDE_GAUSSIAN) {
                a = fma(-r, p.c, lwi);
            } else if (KERN == KDE_TOPHAT) {
                a = r < p.T ? lwi : -INFINITY;
            } else if (KERN == KDE_EXPONENTIAL) {
                a = fma(-__dsqrt_rn(r), p.c, lwi);
            } else {
                const double d = __dsqrt_rn(r);
                const bool in = d < p.h;
                a = in ? lwi : -INFINITY;
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
    m_out = m;
    s_out = s;
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
    double m, s;
    kde_chunk_sum<D, KERN>(p, n0, n1, y, sx, slw, tab, m, s);
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

// ---- many sample sets (mbar_b200_kde_many_log_sum, DESIGN.md 3.5h'') ----------------------------------------------
// A piece is up to `cap` queries of one request (cap: the query batch of mbar_b200_kde_log_sum for the set's chunk
// count).  Its work items are (query block of KDE_THREADS, chunk); a piece's partials are [nChunks][Q] at poff.
struct KdeManyPiece {
    int64_t item0;     // first work item of the piece in its partial launch
    int64_t xoff;      // first double of the set's [D][nPad] coordinates
    int64_t lwoff;     // first log weight of the request ([nPad], -inf in the padding)
    int64_t yoff;      // first double of the piece's [D][Q] queries
    int64_t poff;      // first partial of the piece in its sub-batch
    int64_t ooff;      // first output of the piece in the call
    int64_t nPad, chunkLen;
    int32_t Q, nqb, nChunks;
    double h, hh, c, T;
};

// kde_partial_kernel for every piece of one (D, kernel) in a sub-batch: one CTA per work item, found by find_segment
template <int D, int KERN>
__global__ void __launch_bounds__(KDE_THREADS, 4) kde_many_partial_kernel(const KdeManyPiece* pc, int n, const double* x,
                                                                      const double* lw,
                                                                      const double* __restrict__ yAll,
                                                                      double* __restrict__ pm, double* __restrict__ ps) {
    __shared__ double sx[D][KDE_TILE];
    __shared__ double slw[KDE_TILE];
    __shared__ double tab[MBAR_EXP_NT];
    __shared__ KdeParams sp;          // the piece's samples and kernel constants, read from here by the pass
    if (threadIdx.x < MBAR_EXP_NT) tab[threadIdx.x] = MBAR_EXP_TABLE[threadIdx.x];
    const int64_t item = blockIdx.x;
    double m, s;
    {
        const KdeManyPiece& p = pc[find_segment(n, item, [&](int i) { return pc[i].item0; })];
        if (threadIdx.x == 0) {
            sp.x = x + p.xoff;
            sp.lw = lw + p.lwoff;
            sp.nPad = p.nPad;
            sp.h = p.h;
            sp.hh = p.hh;
            sp.c = p.c;
            sp.T = p.T;
        }
        const int local = (int)(item - p.item0);      // a launch has fewer than 2^31 work items
        const int chunk = local / p.nqb;
        const int q = (local - chunk * p.nqb) * KDE_THREADS + threadIdx.x;
        const int64_t n0 = (int64_t)chunk * p.chunkLen, n1 = min(n0 + p.chunkLen, p.nPad);
        double y[D];
#pragma unroll
        for (int j = 0; j < D; ++j) y[j] = q < p.Q ? yAll[p.yoff + (int64_t)j * p.Q + q] : 0.0;
        kde_chunk_sum<D, KERN>(sp, n0, n1, y, sx, slw, tab, m, s);   // its first barrier publishes sp
    }
    // the piece is found and read again after the pass, so that nothing of it stays live across the pass
    const KdeManyPiece& p = pc[find_segment(n, item, [&](int i) { return pc[i].item0; })];
    const int local = (int)(item - p.item0);
    const int chunk = local / p.nqb;
    const int q = (local - chunk * p.nqb) * KDE_THREADS + threadIdx.x;
    if (q < p.Q) {
        pm[p.poff + (int64_t)chunk * p.Q + q] = m;
        ps[p.poff + (int64_t)chunk * p.Q + q] = s;
    }
}

// kde_combine_kernel's rule for the outputs [o0, o0 + nOut) of a sub-batch's pieces (ascending ooff)
__global__ void kde_many_combine_kernel(const KdeManyPiece* __restrict__ pc, int n, int64_t o0, int64_t nOut,
                                        const double* __restrict__ pm, const double* __restrict__ ps,
                                        double* __restrict__ out) {
    const int64_t i = o0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= o0 + nOut) return;
    const KdeManyPiece& p = pc[find_segment(n, i, [&](int r) { return pc[r].ooff; })];
    const int64_t q = i - p.ooff;
    double M = -INFINITY;
    for (int c = 0; c < p.nChunks; ++c) M = fmax(M, pm[p.poff + (int64_t)c * p.Q + q]);
    if (M == -INFINITY) {
        out[i] = -INFINITY;
        return;
    }
    double S = 0.0;
    for (int c = 0; c < p.nChunks; ++c) S += ps[p.poff + (int64_t)c * p.Q + q] * exp(pm[p.poff + (int64_t)c * p.Q + q] - M);
    out[i] = M + log(S);
}

typedef void (*KdeManyKernelFn)(const KdeManyPiece*, int, const double*, const double*, const double*, double*,
                                double*);

template <int D>
static KdeManyKernelFn kde_many_kernel_for(int kernel) {
    switch (kernel) {
        case KDE_GAUSSIAN: return kde_many_partial_kernel<D, KDE_GAUSSIAN>;
        case KDE_TOPHAT: return kde_many_partial_kernel<D, KDE_TOPHAT>;
        case KDE_EPANECHNIKOV: return kde_many_partial_kernel<D, KDE_EPANECHNIKOV>;
        case KDE_EXPONENTIAL: return kde_many_partial_kernel<D, KDE_EXPONENTIAL>;
        case KDE_LINEAR: return kde_many_partial_kernel<D, KDE_LINEAR>;
        default: return kde_many_partial_kernel<D, KDE_COSINE>;
    }
}

static KdeManyKernelFn kde_many_kernel_for(int D, int kernel) {
    switch (D) {
        case 1: return kde_many_kernel_for<1>(kernel);
        case 2: return kde_many_kernel_for<2>(kernel);
        case 3: return kde_many_kernel_for<3>(kernel);
        default: return kde_many_kernel_for<4>(kernel);
    }
}

// kde_combine_kernel's rule for the W * Qb entries of a replicate batch, and flag[i] = 1 where the entry lies more
// than thr below the batch's scale M (or is -inf while M is finite): there the shared scale may have lost digits
__global__ void kde_rep_combine_kernel(const double* __restrict__ pm, const double* __restrict__ ps, int nChunks,
                                       int nOut, double thr, double* __restrict__ out, double* __restrict__ flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nOut) return;
    double M = -INFINITY;
    for (int c = 0; c < nChunks; ++c) M = fmax(M, pm[(int64_t)c * nOut + i]);
    if (M == -INFINITY) {
        out[i] = -INFINITY;
        flag[i] = 0.0;
        return;
    }
    double S = 0.0;
    for (int c = 0; c < nChunks; ++c) S += ps[(int64_t)c * nOut + i] * exp(pm[(int64_t)c * nOut + i] - M);
    const double l = M + log(S);
    out[i] = l;
    flag[i] = l >= M - thr ? 0.0 : 1.0;
}

// log V_bn of one replicate from its batch's log vmax_n and ratio r_bn (-inf where r_bn = 0)
__global__ void kde_rep_log_weight_kernel(const double* __restrict__ lvm, const double* __restrict__ rat,
                                          int64_t nPad, double* __restrict__ lw) {
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= nPad) return;
    const double r = rat[n];
    lw[n] = r > 0.0 ? lvm[n] + log(r) : -INFINITY;
}

// kde_partial_kernel for a batch of KDE_REP_W bootstrap replicates with weights V_bn on the same samples
// (mbar_b200_kde_log_sum_replicates).  p.lw holds log vmax_n, vmax_n = max_b V_bn over the batch, and rat [W][nPad]
// the ratios r_bn = V_bn / vmax_n in [0, 1].  The distance, the kernel and one exp per (query, sample) pair serve all
// W replicates: e = exp(log vmax_n + log k_qn - m) with one running scale m per query shared by the batch, and
// s_b += r_bn e (r_bn e k for the compact kernels).  Partials are written [chunk][b][Qb], so that kde_combine_kernel
// over W * Qb entries combines every replicate by its rule; m is stored once per replicate.
template <int D, int KERN>
__global__ void __launch_bounds__(KDE_THREADS) kde_replicates_kernel(KdeParams p, const double* __restrict__ rat) {
    __shared__ double sx[D][KDE_TILE];
    __shared__ double slv[KDE_TILE];
    __shared__ double sr[KDE_REP_W][KDE_TILE];
    __shared__ double tab[MBAR_EXP_NT];
    if (threadIdx.x < MBAR_EXP_NT) tab[threadIdx.x] = MBAR_EXP_TABLE[threadIdx.x];
    const int q = blockIdx.x * KDE_THREADS + threadIdx.x;
    const int64_t n0 = (int64_t)blockIdx.y * p.chunkLen, n1 = min(n0 + p.chunkLen, p.nPad);
    double y[D];
#pragma unroll
    for (int j = 0; j < D; ++j) y[j] = q < p.Qb ? p.y[(int64_t)j * p.Qb + q] : 0.0;
    double m = -INFINITY, s[KDE_REP_W];
#pragma unroll
    for (int b = 0; b < KDE_REP_W; ++b) s[b] = 0.0;
    for (int64_t t0 = n0; t0 < n1; t0 += KDE_TILE) {
        __syncthreads();
        for (int i = threadIdx.x; i < KDE_TILE; i += KDE_THREADS) {
#pragma unroll
            for (int j = 0; j < D; ++j) sx[j][i] = p.x[(int64_t)j * p.nPad + t0 + i];
            slv[i] = p.lw[t0 + i];
#pragma unroll
            for (int b = 0; b < KDE_REP_W; ++b) sr[b][i] = rat[(int64_t)b * p.nPad + t0 + i];
        }
        __syncthreads();
#pragma unroll 4
        for (int i = 0; i < KDE_TILE; ++i) {
            // distance, support and kernel exactly as kde_partial_kernel
            double t = __dsub_rn(y[0], sx[0][i]);
            double r = __dmul_rn(t, t);
#pragma unroll
            for (int j = 1; j < D; ++j) {
                t = __dsub_rn(y[j], sx[j][i]);
                r = __dadd_rn(r, __dmul_rn(t, t));
            }
            const double lv = slv[i];
            double a, k = 1.0;
            if (KERN == KDE_GAUSSIAN) {
                a = fma(-r, p.c, lv);
            } else if (KERN == KDE_TOPHAT) {
                a = r < p.T ? lv : -INFINITY;
            } else if (KERN == KDE_EXPONENTIAL) {
                a = fma(-__dsqrt_rn(r), p.c, lv);
            } else {
                const double d = __dsqrt_rn(r);
                const bool in = d < p.h;
                a = in ? lv : -INFINITY;
                if (KERN == KDE_EPANECHNIKOV) k = __dsub_rn(1.0, __ddiv_rn(__dmul_rn(d, d), p.hh));
                if (KERN == KDE_LINEAR) k = __dsub_rn(1.0, __ddiv_rn(d, p.h));
                if (KERN == KDE_COSINE) k = cos(__ddiv_rn(__dmul_rn(KDE_HALF_PI, d), p.h));
                k = in ? k : 0.0;
            }
            double dl = a - m;
            if (dl > KDE_RESCALE) {
                const double g = exp_flush(fmax(m - a, KDE_FLOOR), tab);
#pragma unroll
                for (int b = 0; b < KDE_REP_W; ++b) s[b] *= g;
                m = a;
                dl = 0.0;
            }
            double e = exp_flush(fmax(dl, KDE_FLOOR), tab);
            if (KERN == KDE_EPANECHNIKOV || KERN == KDE_LINEAR || KERN == KDE_COSINE) e *= k;
#pragma unroll
            for (int b = 0; b < KDE_REP_W; ++b) s[b] = fma(sr[b][i], e, s[b]);
        }
    }
    if (q < p.Qb) {
#pragma unroll
        for (int b = 0; b < KDE_REP_W; ++b) {
            const int64_t o = ((int64_t)blockIdx.y * KDE_REP_W + b) * p.Qb + q;
            p.pm[o] = m;
            p.ps[o] = s[b];
        }
    }
}

typedef void (*KdeRepKernelFn)(KdeParams, const double*);

template <int D>
static KdeRepKernelFn kde_rep_kernel_for(int kernel) {
    switch (kernel) {
        case KDE_GAUSSIAN: return kde_replicates_kernel<D, KDE_GAUSSIAN>;
        case KDE_TOPHAT: return kde_replicates_kernel<D, KDE_TOPHAT>;
        case KDE_EPANECHNIKOV: return kde_replicates_kernel<D, KDE_EPANECHNIKOV>;
        case KDE_EXPONENTIAL: return kde_replicates_kernel<D, KDE_EXPONENTIAL>;
        case KDE_LINEAR: return kde_replicates_kernel<D, KDE_LINEAR>;
        default: return kde_replicates_kernel<D, KDE_COSINE>;
    }
}

static KdeRepKernelFn kde_rep_kernel_for(int D, int kernel) {
    switch (D) {
        case 1: return kde_rep_kernel_for<1>(kernel);
        case 2: return kde_rep_kernel_for<2>(kernel);
        case 3: return kde_rep_kernel_for<3>(kernel);
        default: return kde_rep_kernel_for<4>(kernel);
    }
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

// chunks: a function of N alone (batch independence); at least KDE_MIN_CHUNK samples, at most KDE_MAX_CHUNKS
static void kde_chunking(int64_t N, int64_t* chunkLen, int* nChunks) {
    const int64_t nPad = (N + KDE_TILE - 1) / KDE_TILE * KDE_TILE;
    const int64_t nc = std::min<int64_t>(KDE_MAX_CHUNKS, std::max<int64_t>(1, (N + KDE_MIN_CHUNK - 1) / KDE_MIN_CHUNK));
    *chunkLen = ((N + nc - 1) / nc + KDE_TILE - 1) / KDE_TILE * KDE_TILE;
    *nChunks = (int)((nPad + *chunkLen - 1) / *chunkLen);
}

// the query batch of one call for a sample set cut into nChunks chunks: the partials of a batch stay under
// KDE_PART_BYTES (one block of KDE_THREADS queries at least); it decides the size of the partials, never a result
static int64_t kde_query_cap(int nChunks, int64_t perQuery) {
    const int64_t cap = (int64_t)(KDE_PART_BYTES / (2 * sizeof(double) * (size_t)perQuery * (size_t)nChunks));
    return std::max<int64_t>(KDE_THREADS, cap / KDE_THREADS * KDE_THREADS);
}

// per-batch buffers for up to qb queries; on failure the object keeps no (or its previous) buffers and stays usable
static int kde_reserve(mbar_b200_kde* k, int64_t qb) {
    MBAR_TRY(k->d_y.reserve((size_t)k->D * qb, "kde"));
    MBAR_TRY(k->d_pm.reserve((size_t)k->nChunks * qb, "kde"));
    MBAR_TRY(k->d_ps.reserve((size_t)k->nChunks * qb, "kde"));
    return k->d_out.reserve((size_t)qb, "kde");
}

// the replicate pass's partials and results for up to qb queries, as kde_reserve
static int kde_rep_reserve(mbar_b200_kde* k, int64_t qb) {
    MBAR_TRY(k->d_rpm.reserve((size_t)k->nChunks * KDE_REP_W * qb, "kde"));
    MBAR_TRY(k->d_rps.reserve((size_t)k->nChunks * KDE_REP_W * qb, "kde"));
    MBAR_TRY(k->d_rout.reserve((size_t)KDE_REP_W * qb, "kde"));
    return k->d_rflag.reserve((size_t)KDE_REP_W * qb, "kde");
}

static void kde_drop_replicates(mbar_b200_kde* k) {
    k->d_lvm.reset();
    k->d_rat.reset();
    k->d_rlw.reset();
    k->B = 0;
}

}  // namespace mbar

using namespace mbar;

int mbar_b200_kde_create(int device, int64_t N, int32_t D, const double* x_host, const double* w_host,
                         mbar_b200_kde** out) {
    MBAR_REQUIRE(out && x_host && w_host, MBAR_B200_ERR_INVALID, "kde_create: NULL argument");
    *out = nullptr;
    MBAR_REQUIRE(N >= 1, MBAR_B200_ERR_INVALID, "kde_create: N=%lld must be >= 1", (long long)N);
    MBAR_REQUIRE(D >= 1 && D <= 4, MBAR_B200_ERR_INVALID, "kde_create: D=%d outside [1, 4]", (int)D);
    MBAR_TRY(open_device(device, nullptr));
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
    std::unique_ptr<mbar_b200_kde> k(new mbar_b200_kde());
    k->D = D;
    k->N = N;
    k->nPad = nPad;
    kde_chunking(N, &k->chunkLen, &k->nChunks);
    MBAR_TRY(k->open(device, "kde_create"));
    MBAR_TRY(k->upload(k->d_x, hx.data(), hx.size(), "kde_create"));
    MBAR_TRY(k->upload(k->d_lw, hlw.data(), hlw.size(), "kde_create"));
    *out = k.release();
    return MBAR_B200_OK;
}

int mbar_b200_kde_destroy(mbar_b200_kde* k) { return destroy_resident(k); }

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
    const int64_t qb = std::min(Q, kde_query_cap(k->nChunks, 1));
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

int mbar_b200_kde_set_replicates(mbar_b200_kde* k, int64_t B, const double* V_host) {
    MBAR_REQUIRE(k, MBAR_B200_ERR_INVALID, "kde_set_replicates: NULL object");
    MBAR_CUDA(cudaSetDevice(k->device));
    kde_drop_replicates(k);
    MBAR_TRY(check_replicate_weights("kde_set_replicates", B, k->N, V_host));
    const int64_t N = k->N, nPad = k->nPad;
    // device: log vmax_n per batch of KDE_REP_W replicates, the ratios V_bn / vmax_n (rows past B stay 0), and one
    // replicate's log weights for the exact pass: 8 nPad (9 nRB + 1) bytes
    const int64_t nRB = (B + KDE_REP_W - 1) / KDE_REP_W;
    int rc = MBAR_B200_OK;
    if ((rc = k->d_lvm.reserve((size_t)(nRB * nPad), "kde")) ||
        (rc = k->d_rat.reserve((size_t)(nRB * KDE_REP_W * nPad), "kde")) ||
        (rc = k->d_rlw.reserve((size_t)nPad, "kde"))) {
        kde_drop_replicates(k);
        return rc;
    }
    // host: one batch at a time (8 nPad (1 + KDE_REP_W) bytes), rows read in order
    std::vector<double> hl((size_t)nPad), hr((size_t)(KDE_REP_W * nPad));
    for (int64_t rb = 0; rb < nRB; ++rb) {
        const int64_t b0 = rb * KDE_REP_W, b1 = std::min(B, b0 + KDE_REP_W);
        std::fill(hl.begin(), hl.end(), 0.0);
        std::fill(hr.begin(), hr.end(), 0.0);
        for (int64_t b = b0; b < b1; ++b)
            for (int64_t n = 0; n < N; ++n) hl[(size_t)n] = std::max(hl[(size_t)n], V_host[b * N + n]);
        for (int64_t b = b0; b < b1; ++b) {
            double* r = hr.data() + (b - b0) * nPad;
            for (int64_t n = 0; n < N; ++n)
                if (hl[(size_t)n] > 0.0) r[n] = V_host[b * N + n] / hl[(size_t)n];
        }
        for (int64_t n = 0; n < nPad; ++n) hl[(size_t)n] = hl[(size_t)n] > 0.0 ? std::log(hl[(size_t)n]) : -INFINITY;
        // synchronous per batch: the host buffers are reused by the next batch
        if (cudaMemcpyAsync(k->d_lvm + rb * nPad, hl.data(), hl.size() * sizeof(double), cudaMemcpyHostToDevice,
                            k->stream) != cudaSuccess ||
            cudaMemcpyAsync(k->d_rat + rb * KDE_REP_W * nPad, hr.data(), hr.size() * sizeof(double),
                            cudaMemcpyHostToDevice, k->stream) != cudaSuccess ||
            cudaStreamSynchronize(k->stream) != cudaSuccess) {
            set_error("kde_set_replicates: %s", cudaGetErrorString(cudaGetLastError()));
            kde_drop_replicates(k);
            return MBAR_B200_ERR_CUDA;
        }
    }
    k->B = B;
    return MBAR_B200_OK;
}

int mbar_b200_kde_log_sum_replicates(mbar_b200_kde* k, int32_t kernel, double h, int64_t Q, const double* y_host,
                                     double* out) {
    MBAR_REQUIRE(k, MBAR_B200_ERR_INVALID, "kde_log_sum_replicates: NULL object");
    MBAR_REQUIRE(k->B >= 1, MBAR_B200_ERR_NOT_READY, "kde_log_sum_replicates: no replicates uploaded");
    MBAR_REQUIRE(kernel >= 0 && kernel < KDE_NKERNELS, MBAR_B200_ERR_INVALID,
                 "kde_log_sum_replicates: unknown kernel %d", (int)kernel);
    MBAR_REQUIRE(std::isfinite(h) && h > 0.0, MBAR_B200_ERR_INVALID, "kde_log_sum_replicates: bandwidth %g must be "
                 "finite and positive", h);
    MBAR_REQUIRE(Q >= 0, MBAR_B200_ERR_INVALID, "kde_log_sum_replicates: Q=%lld", (long long)Q);
    if (Q == 0) return MBAR_B200_OK;
    MBAR_REQUIRE(y_host && out, MBAR_B200_ERR_INVALID, "kde_log_sum_replicates: NULL argument");
    const int D = k->D;
    for (int64_t i = 0; i < Q * D; ++i)
        MBAR_REQUIRE(std::isfinite(y_host[i]), MBAR_B200_ERR_NAN, "kde_log_sum_replicates: query coordinate "
                     "(%lld, %d) is %g", (long long)(i / D), (int)(i % D), y_host[i]);
    MBAR_CUDA(cudaSetDevice(k->device));
    NvtxRange nvtx_("mbar_b200::kde_log_sum_replicates");
    const int64_t qb = std::min(Q, kde_query_cap(k->nChunks, KDE_REP_W));
    MBAR_TRY(kde_reserve(k, qb));
    MBAR_TRY(kde_rep_reserve(k, qb));
    KdeParams p{};
    p.x = k->d_x;
    p.y = k->d_y;
    p.pm = k->d_rpm;
    p.ps = k->d_rps;
    p.nPad = k->nPad;
    p.chunkLen = k->chunkLen;
    p.h = h;
    p.hh = h * h;
    p.c = kernel == KDE_GAUSSIAN ? 0.5 / (h * h) : 1.0 / h;
    p.T = sqrt_threshold(h);
    const KdeRepKernelFn fn = kde_rep_kernel_for(D, kernel);
    const int64_t nRB = (k->B + KDE_REP_W - 1) / KDE_REP_W;
    const double thr = KDE_REP_EXACT - std::log((double)k->N);
    std::vector<double> hy((size_t)D * qb), hflag((size_t)KDE_REP_W * qb);
    std::vector<std::vector<int64_t>> redo((size_t)k->B);     // per replicate: queries for the exact pass
    double ms = 0.0;
    float e = 0.f;
    for (int64_t q0 = 0; q0 < Q; q0 += qb) {
        const int Qb = (int)std::min(qb, Q - q0);
        for (int64_t i = 0; i < Qb; ++i)
            for (int j = 0; j < D; ++j) hy[(size_t)j * Qb + i] = y_host[(q0 + i) * D + j];
        MBAR_CUDA(cudaMemcpyAsync(k->d_y, hy.data(), (size_t)D * Qb * sizeof(double), cudaMemcpyHostToDevice,
                                  k->stream));
        p.Qb = Qb;
        for (int64_t rb = 0; rb < nRB; ++rb) {
            p.lw = k->d_lvm + rb * k->nPad;
            const int64_t nb = std::min<int64_t>(KDE_REP_W, k->B - rb * KDE_REP_W);
            MBAR_CUDA(cudaEventRecord(k->ev0, k->stream));
            const dim3 grid((unsigned)((Qb + KDE_THREADS - 1) / KDE_THREADS), (unsigned)k->nChunks);
            fn<<<grid, KDE_THREADS, 0, k->stream>>>(p, k->d_rat + rb * KDE_REP_W * k->nPad);
            const int nOut = KDE_REP_W * Qb;
            kde_rep_combine_kernel<<<(nOut + 127) / 128, 128, 0, k->stream>>>(k->d_rpm, k->d_rps, k->nChunks, nOut,
                                                                              thr, k->d_rout, k->d_rflag);
            MBAR_CUDA(cudaGetLastError());
            MBAR_CUDA(cudaEventRecord(k->ev1, k->stream));
            // rows b of the batch go to out[(rb W + b) Q + q0 ...]
            MBAR_CUDA(cudaMemcpy2DAsync(out + rb * KDE_REP_W * Q + q0, (size_t)Q * sizeof(double), k->d_rout,
                                        (size_t)Qb * sizeof(double), (size_t)Qb * sizeof(double), (size_t)nb,
                                        cudaMemcpyDeviceToHost, k->stream));
            MBAR_CUDA(cudaMemcpyAsync(hflag.data(), k->d_rflag, (size_t)(nb * Qb) * sizeof(double),
                                      cudaMemcpyDeviceToHost, k->stream));
            MBAR_CUDA(cudaStreamSynchronize(k->stream));
            if (event_ms(k->ev0, k->ev1, &e)) ms += e;
            for (int64_t b = 0; b < nb; ++b)
                for (int64_t i = 0; i < Qb; ++i)
                    if (hflag[(size_t)(b * Qb + i)] != 0.0) redo[(size_t)(rb * KDE_REP_W + b)].push_back(q0 + i);
        }
    }
    // the entries the shared scale may have cut short: the single-replicate pass (kde_partial_kernel) on log V_bn
    KdeParams p1 = p;
    p1.lw = k->d_rlw;
    p1.pm = k->d_pm;
    p1.ps = k->d_ps;
    const KdeKernelFn fn1 = kde_kernel_for(D, kernel);
    std::vector<double> hout((size_t)qb);
    for (int64_t b = 0; b < k->B; ++b) {
        const std::vector<int64_t>& qs = redo[(size_t)b];
        if (qs.empty()) continue;
        const int64_t rb = b / KDE_REP_W;
        kde_rep_log_weight_kernel<<<(unsigned)((k->nPad + 255) / 256), 256, 0, k->stream>>>(
            k->d_lvm + rb * k->nPad, k->d_rat + b * k->nPad, k->nPad, k->d_rlw);
        MBAR_CUDA(cudaGetLastError());
        for (size_t i0 = 0; i0 < qs.size(); i0 += (size_t)qb) {
            const int Qb = (int)std::min<size_t>((size_t)qb, qs.size() - i0);
            for (int64_t i = 0; i < Qb; ++i)
                for (int j = 0; j < D; ++j) hy[(size_t)j * Qb + i] = y_host[qs[i0 + i] * D + j];
            MBAR_CUDA(cudaMemcpyAsync(k->d_y, hy.data(), (size_t)D * Qb * sizeof(double), cudaMemcpyHostToDevice,
                                      k->stream));
            p1.Qb = Qb;
            MBAR_CUDA(cudaEventRecord(k->ev0, k->stream));
            const dim3 grid((unsigned)((Qb + KDE_THREADS - 1) / KDE_THREADS), (unsigned)k->nChunks);
            fn1<<<grid, KDE_THREADS, 0, k->stream>>>(p1);
            kde_combine_kernel<<<(Qb + 127) / 128, 128, 0, k->stream>>>(k->d_pm, k->d_ps, k->nChunks, Qb, k->d_out);
            MBAR_CUDA(cudaGetLastError());
            MBAR_CUDA(cudaEventRecord(k->ev1, k->stream));
            MBAR_CUDA(cudaMemcpyAsync(hout.data(), k->d_out, (size_t)Qb * sizeof(double), cudaMemcpyDeviceToHost,
                                      k->stream));
            MBAR_CUDA(cudaStreamSynchronize(k->stream));
            if (event_ms(k->ev0, k->ev1, &e)) ms += e;
            for (int64_t i = 0; i < Qb; ++i) out[b * Q + qs[i0 + i]] = hout[(size_t)i];
        }
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

int mbar_b200_kde_many_create(int device, int32_t n_sets, const int32_t* D, const int64_t* N, const double* x,
                              mbar_b200_kde_many** out) {
    MBAR_REQUIRE(out && D && N && x, MBAR_B200_ERR_INVALID, "kde_many_create: NULL argument");
    *out = nullptr;
    MBAR_REQUIRE(n_sets >= 1, MBAR_B200_ERR_INVALID, "kde_many_create: %d sets", (int)n_sets);
    std::unique_ptr<mbar_b200_kde_many> k(new mbar_b200_kde_many());
    int64_t total = 0, src = 0;
    for (int s = 0; s < n_sets; ++s) {
        MBAR_REQUIRE(N[s] >= 1, MBAR_B200_ERR_INVALID, "kde_many_create: set %d has N=%lld", s, (long long)N[s]);
        MBAR_REQUIRE(D[s] >= 1 && D[s] <= 4, MBAR_B200_ERR_INVALID, "kde_many_create: set %d has D=%d outside [1, 4]",
                     s, (int)D[s]);
        for (int64_t i = 0; i < N[s] * D[s]; ++i)
            MBAR_REQUIRE(std::isfinite(x[src + i]), MBAR_B200_ERR_NAN, "kde_many_create: set %d: coordinate (%lld, %d) "
                         "is %g", s, (long long)(i / D[s]), (int)(i % D[s]), x[src + i]);
        int64_t chunkLen;
        int nChunks;
        kde_chunking(N[s], &chunkLen, &nChunks);
        const int64_t nPad = (N[s] + KDE_TILE - 1) / KDE_TILE * KDE_TILE;
        k->D.push_back(D[s]);
        k->N.push_back(N[s]);
        k->nPad.push_back(nPad);
        k->chunkLen.push_back(chunkLen);
        k->nChunks.push_back(nChunks);
        k->xoff.push_back(total);
        total += (int64_t)D[s] * nPad;
        src += N[s] * D[s];
    }
    // each set as mbar_b200_kde_create lays it out: [D][nPad], 0 in the padding
    std::vector<double> hx((size_t)total, 0.0);
    src = 0;
    for (int s = 0; s < n_sets; ++s) {
        for (int64_t n = 0; n < N[s]; ++n)
            for (int j = 0; j < D[s]; ++j) hx[(size_t)(k->xoff[s] + j * k->nPad[s] + n)] = x[src + n * D[s] + j];
        src += N[s] * D[s];
    }
    MBAR_TRY(open_device(device, nullptr));
    MBAR_TRY(k->open(device, "kde_many_create"));
    MBAR_TRY(k->upload(k->d_x, hx.data(), hx.size(), "kde_many_create"));
    *out = k.release();
    return MBAR_B200_OK;
}

int mbar_b200_kde_many_destroy(mbar_b200_kde_many* k) { return destroy_resident(k); }

int mbar_b200_kde_many_log_sum(mbar_b200_kde_many* k, int32_t n_requests, const int32_t* set, const int32_t* kernel,
                               const double* h, const double* w, const int64_t* Q, const double* y, double* out) {
    MBAR_REQUIRE(k, MBAR_B200_ERR_INVALID, "kde_many_log_sum: NULL object");
    MBAR_REQUIRE(n_requests >= 0, MBAR_B200_ERR_INVALID, "kde_many_log_sum: %d requests", (int)n_requests);
    if (n_requests == 0) return MBAR_B200_OK;
    MBAR_REQUIRE(set && kernel && h && w && Q, MBAR_B200_ERR_INVALID, "kde_many_log_sum: NULL argument");
    const int nSets = (int)k->D.size();
    // every request checked before any device work
    int64_t wsrc = 0, ysrc = 0, outs = 0, lws = 0;
    for (int r = 0; r < n_requests; ++r) {
        const int s = set[r];
        MBAR_REQUIRE(s >= 0 && s < nSets, MBAR_B200_ERR_INVALID, "kde_many_log_sum: request %d names set %d of %d", r,
                     s, nSets);
        MBAR_REQUIRE(kernel[r] >= 0 && kernel[r] < KDE_NKERNELS, MBAR_B200_ERR_INVALID,
                     "kde_many_log_sum: request %d: unknown kernel %d", r, (int)kernel[r]);
        MBAR_REQUIRE(std::isfinite(h[r]) && h[r] > 0.0, MBAR_B200_ERR_INVALID,
                     "kde_many_log_sum: request %d: bandwidth %g must be finite and positive", r, h[r]);
        MBAR_REQUIRE(Q[r] >= 0, MBAR_B200_ERR_INVALID, "kde_many_log_sum: request %d: Q=%lld", r, (long long)Q[r]);
        bool any = false;
        for (int64_t n = 0; n < k->N[s]; ++n) {
            const double v = w[wsrc + n];
            MBAR_REQUIRE(v >= 0.0 && v < INFINITY, MBAR_B200_ERR_INVALID, "kde_many_log_sum: request %d: weight %lld "
                         "is %g (negative, NaN or infinite)", r, (long long)n, v);
            any |= v > 0.0;
        }
        MBAR_REQUIRE(any, MBAR_B200_ERR_INVALID, "kde_many_log_sum: request %d: the weights sum to 0", r);
        MBAR_REQUIRE(Q[r] == 0 || (y && out), MBAR_B200_ERR_INVALID, "kde_many_log_sum: NULL queries or output");
        const int D = k->D[s];
        for (int64_t i = 0; i < Q[r] * D; ++i)
            MBAR_REQUIRE(std::isfinite(y[ysrc + i]), MBAR_B200_ERR_NAN, "kde_many_log_sum: request %d: query "
                         "coordinate (%lld, %d) is %g", r, (long long)(i / D), (int)(i % D), y[ysrc + i]);
        wsrc += k->N[s];
        ysrc += Q[r] * D;
        outs += Q[r];
        lws += k->nPad[s];
    }
    // pieces of at most kde_query_cap queries, in request order; sub-batches of pieces whose partials stay under
    // KDE_PART_BYTES (one piece at least).  Neither decides a result.
    struct Piece {
        int r;
        int64_t q0;
        int32_t Qp;
    };
    std::vector<Piece> pieces;
    std::vector<std::pair<size_t, size_t>> subs;      // [first, last) piece of each sub-batch
    size_t first = 0;
    int64_t used = 0, maxParts = 0, pairs = 0;
    for (int r = 0; r < n_requests; ++r) {
        const int s = set[r];
        const int64_t cap = kde_query_cap(k->nChunks[s], 1);
        pairs += Q[r] * k->N[s];
        for (int64_t q0 = 0; q0 < Q[r]; q0 += cap) {
            const int32_t Qp = (int32_t)std::min(cap, Q[r] - q0);
            const int64_t parts = (int64_t)k->nChunks[s] * Qp;     // (m, s) pairs
            if (pieces.size() > first && (size_t)(used + parts) * 2 * sizeof(double) > KDE_PART_BYTES) {
                subs.emplace_back(first, pieces.size());
                first = pieces.size();
                used = 0;
            }
            pieces.push_back(Piece{r, q0, Qp});
            used += parts;
            maxParts = std::max(maxParts, used);
        }
    }
    if (pieces.size() > first) subs.emplace_back(first, pieces.size());
    // host staging: log w_n of every request (std::log, as kde_create takes it; -inf in the padding), the queries of
    // every piece as [D][Qp], and the piece records: per sub-batch, grouped by (D, kernel) for the partial launches,
    // then in output order for the combine
    std::vector<double> hlw((size_t)lws, -INFINITY), hy((size_t)ysrc);
    std::vector<int64_t> lwoff((size_t)n_requests), yoff((size_t)n_requests), ooff((size_t)n_requests);
    wsrc = 0;
    ysrc = 0;
    lws = 0;
    outs = 0;
    for (int r = 0; r < n_requests; ++r) {
        const int s = set[r], D = k->D[s];
        for (int64_t n = 0; n < k->N[s]; ++n) hlw[(size_t)(lws + n)] = std::log(w[wsrc + n]);
        lwoff[r] = lws;
        yoff[r] = ysrc;
        ooff[r] = outs;
        wsrc += k->N[s];
        lws += k->nPad[s];
        ysrc += Q[r] * D;
        outs += Q[r];
    }
    auto record = [&](const Piece& pc, int64_t poff) {
        const int r = pc.r, s = set[r], D = k->D[s];
        KdeManyPiece p{};
        p.xoff = k->xoff[s];
        p.lwoff = lwoff[r];
        p.yoff = yoff[r] + (int64_t)D * pc.q0;        // the piece's own [D][Qp] block
        p.poff = poff;
        p.ooff = ooff[r] + pc.q0;
        p.nPad = k->nPad[s];
        p.chunkLen = k->chunkLen[s];
        p.Q = pc.Qp;
        p.nqb = (pc.Qp + KDE_THREADS - 1) / KDE_THREADS;
        p.nChunks = k->nChunks[s];
        p.h = h[r];
        p.hh = h[r] * h[r];
        p.c = kernel[r] == KDE_GAUSSIAN ? 0.5 / (h[r] * h[r]) : 1.0 / h[r];
        p.T = sqrt_threshold(h[r]);
        return p;
    };
    // a piece reads its queries as [D][Qp]: lay every request's queries out piece by piece
    for (const Piece& pc : pieces) {
        const int r = pc.r, D = k->D[set[r]];
        double* dst = hy.data() + yoff[r] + (int64_t)D * pc.q0;
        for (int64_t i = 0; i < pc.Qp; ++i)
            for (int j = 0; j < D; ++j) dst[(size_t)j * pc.Qp + i] = y[yoff[r] + (pc.q0 + i) * D + j];
    }
    std::vector<KdeManyPiece> hpc;                    // per sub-batch: grouped records, then ordered records
    struct Launch {
        size_t rec;       // first record
        int n;            // records
        int64_t items;    // CTAs (partial launch) or outputs (combine)
        int64_t o0;       // first output (combine)
        KdeManyKernelFn fn;   // NULL: the combine
    };
    std::vector<Launch> launches;
    for (const auto& sb : subs) {
        std::vector<int64_t> poff(sb.second - sb.first);
        int64_t parts = 0;
        for (size_t i = sb.first; i < sb.second; ++i) {
            poff[i - sb.first] = parts;
            parts += (int64_t)k->nChunks[set[pieces[i].r]] * pieces[i].Qp;
        }
        std::vector<std::pair<int, int>> groups;      // distinct (D, kernel) in order of first appearance
        for (size_t i = sb.first; i < sb.second; ++i) {
            const std::pair<int, int> g(k->D[set[pieces[i].r]], kernel[pieces[i].r]);
            if (std::find(groups.begin(), groups.end(), g) == groups.end()) groups.push_back(g);
        }
        for (const auto& g : groups) {
            Launch L{hpc.size(), 0, 0, 0, kde_many_kernel_for(g.first, g.second)};
            for (size_t i = sb.first; i < sb.second; ++i) {
                const Piece& pc = pieces[i];
                if (k->D[set[pc.r]] != g.first || kernel[pc.r] != g.second) continue;
                KdeManyPiece p = record(pc, poff[i - sb.first]);
                p.item0 = L.items;
                L.items += (int64_t)p.nqb * p.nChunks;
                hpc.push_back(p);
                ++L.n;
            }
            MBAR_REQUIRE(L.items < INT32_MAX, MBAR_B200_ERR_INVALID, "kde_many_log_sum: %lld work items in one launch",
                         (long long)L.items);
            launches.push_back(L);
        }
        Launch C{hpc.size(), 0, 0, 0, nullptr};
        for (size_t i = sb.first; i < sb.second; ++i) {
            KdeManyPiece p = record(pieces[i], poff[i - sb.first]);
            if (C.n == 0) C.o0 = p.ooff;
            C.items += p.Q;
            hpc.push_back(p);
            ++C.n;
        }
        launches.push_back(C);
    }
    MBAR_CUDA(cudaSetDevice(k->device));
    NvtxRange nvtx_("mbar_b200::kde_many_log_sum");
    CallBuffers buf("kde_many_log_sum");
    double *d_lw, *d_y, *d_pm, *d_ps, *d_out;
    KdeManyPiece* d_pc;
    MBAR_TRY(buf.alloc(&d_lw, hlw.size()));
    MBAR_TRY(buf.alloc(&d_y, hy.size()));
    MBAR_TRY(buf.alloc(&d_pm, (size_t)maxParts));
    MBAR_TRY(buf.alloc(&d_ps, (size_t)maxParts));
    MBAR_TRY(buf.alloc(&d_out, (size_t)outs));
    MBAR_TRY(buf.alloc(&d_pc, hpc.size()));
    cudaStream_t st = k->stream;
    MBAR_CUDA(cudaMemcpyAsync(d_lw, hlw.data(), hlw.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    MBAR_CUDA(cudaMemcpyAsync(d_y, hy.data(), hy.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    MBAR_CUDA(cudaMemcpyAsync(d_pc, hpc.data(), hpc.size() * sizeof(KdeManyPiece), cudaMemcpyHostToDevice, st));
    MBAR_CUDA(cudaEventRecord(k->ev0, st));
    for (const Launch& L : launches) {
        if (L.fn) {
            L.fn<<<(unsigned)L.items, KDE_THREADS, 0, st>>>(d_pc + L.rec, L.n, k->d_x, d_lw, d_y, d_pm, d_ps);
        } else if (L.items > 0) {
            kde_many_combine_kernel<<<(unsigned)((L.items + 127) / 128), 128, 0, st>>>(d_pc + L.rec, L.n, L.o0, L.items,
                                                                                      d_pm, d_ps, d_out);
        }
    }
    MBAR_CUDA(cudaGetLastError());
    MBAR_CUDA(cudaEventRecord(k->ev1, st));
    if (outs > 0) MBAR_CUDA(cudaMemcpyAsync(out, d_out, (size_t)outs * sizeof(double), cudaMemcpyDeviceToHost, st));
    MBAR_CUDA(cudaStreamSynchronize(st));
    float e = 0.f;
    k->lastMs = event_ms(k->ev0, k->ev1, &e) ? e : 0.0;
    k->lastLaunches = (int32_t)launches.size();
    k->lastPairs = pairs;
    return MBAR_B200_OK;
}

int mbar_b200_last_kde_many_stats(mbar_b200_kde_many* k, double* ms, int32_t* launches, int64_t* pairs) {
    MBAR_REQUIRE(k, MBAR_B200_ERR_INVALID, "NULL kde_many object");
    if (ms) *ms = k->lastMs;
    if (launches) *launches = k->lastLaunches;
    if (pairs) *pairs = k->lastPairs;
    return MBAR_B200_OK;
}

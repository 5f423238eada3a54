// Device-resident solver loops: no host round trip between iterations.
//
// Reference loops being replaced: adaptive() (mbar_solvers.py:510-667; one iteration = mbar_solvers.py:575-640,
// the JAX build runs that iteration as ONE jitted step, jax_core_adaptive :670-694) and the plain
// self-consistent iteration (Eq. C3).  Round 1 stepped these loops from the host: after every pass a
// cudaStreamSynchronize, a D2H copy, a K-vector update on the CPU, and for Newton a D2H of K^2 doubles plus a
// single-threaded host Cholesky.  At the sizes of BASELINE configs C2 / C4 (a pass takes 30-100 us) the loop was
// round-trip-bound.
//
// Here every quantity of an iteration lives on the device:
//   self-consistent:  pass kernel (its last CTA exchanges the sums, updates f, tests convergence)
//   adaptive:         pass(f) -> adapt_pre (g, f_sci) -> Hessian -> newton_build -> newton (Cholesky + solves,
//                     f_nr) -> pass(f_sci), pass(f_nr) -> adapt_post (step choice :607, convergence :627-640)
// Every kernel starts with `if (loop->done) return;`, so the host enqueues `loopBatch` iterations at a time and
// reads the 112-byte LoopState once per batch.  Anything the fast path cannot represent (range flag of the fused
// kernel, an underflowing S_k, non-finite candidates) sets status = 1 and the host finishes on the robust
// host-stepped loop, starting from the last good f.
//
// This file holds every solver loop and its C entry points: the device-resident loops, the host-stepped loops
// (one run_pass per step; the fallback of the device-resident ones and mbar_b200_set_loop_mode(ctx, 1)), and
// mbar_b200_sci_iterate.
#include <nvtx3/nvToolsExt.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "internal.cuh"

namespace mbar {

NvtxRange::NvtxRange(const char* name) { nvtxRangePushA(name); }
NvtxRange::~NvtxRange() { nvtxRangePop(); }

// rows of ctx->d_av
enum { AV_FSCI = 0, AV_FNR = 1, AV_G = 2, AV_CSCI = 3, AV_CNR = 4, AV_CH = 5, AV_X = 6, AV_DIAG = 7 };

__device__ __forceinline__ bool loop_done(const LoopState* loop) {
    return *reinterpret_cast<const volatile int*>(&loop->done) != 0;
}
__device__ __forceinline__ bool row_on(const unsigned long long* __restrict__ mask, int k) {
    return (mask[k >> 6] >> (k & 63)) & 1ull;
}

// Deterministic block-wide reductions (fixed tree): sum and NaN-propagating max.
__device__ double block_sum(double v, double* s_buf) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_buf[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_buf[w];
    return t;
}
__device__ double block_max_nan(double v, double* s_buf) {
    // NaN must survive (mbar_solvers.py:636 treats a NaN max_delta specially): carry it as +inf marker pairs
    double nanflag = (v != v) ? 1.0 : 0.0;
    if (v != v) v = 0.0;
    for (int o = 16; o > 0; o >>= 1) {
        v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
        nanflag = fmax(nanflag, __shfl_xor_sync(0xffffffffu, nanflag, o));
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) {
        s_buf[threadIdx.x >> 5] = v;
        s_buf[32 + (threadIdx.x >> 5)] = nanflag;
    }
    __syncthreads();
    double t = 0.0, nf = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
        t = fmax(t, s_buf[w]);
        nf = fmax(nf, s_buf[32 + w]);
    }
    return nf > 0.0 ? NAN : t;
}

// ------------------------------------------------------------------------------------------------
// self-consistent iteration, NCCL flavour (no peer memory): epilogue kernel after the all-reduce
// ------------------------------------------------------------------------------------------------
// f <- f - log S (sampled states), gauge f[first] = 0, c <- f + log N - mid, convergence test.  With loop == NULL
// (as in the fused pass's epilogue) every launch runs and nothing is tested or counted.
__global__ void __launch_bounds__(256)
sci_loop_epilogue_kernel(const double* __restrict__ out, double* __restrict__ f, double* __restrict__ c,
                         const double* __restrict__ Nk, const unsigned long long* __restrict__ rowmask, int K,
                         int first, double mid, LoopState* loop) {
    if (loop && loop_done(loop)) return;
    __shared__ double s_buf[64];
    __shared__ double s_f0;
    if (threadIdx.x == 0) s_f0 = f[first] - log(out[first]);
    __syncthreads();
    const double thr = loop ? fmin(1.0e-8, loop->tol) : 1.0e-8;
    double md = 0.0;
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        if (row_on(rowmask, k)) {
            const double fo = f[k];
            // an underflowed S_k poisons the result so the host redoes the step in the log domain
            const double fn = (out[k] > 1e-280) ? fo - log(out[k]) - s_f0 : NAN;
            f[k] = fn;
            c[k] = fn + log(Nk[k]) - mid;
            if (fn != fn) md = NAN;
            if (k != first && md == md) md = fmax(md, rel_change(fn, fo, fn, thr));
        }
    }
    if (!loop) return;
    md = block_max_nan(md, s_buf);
    if (threadIdx.x == 0) {
        const int it = loop->iterations + 1;
        loop->iterations = it;
        loop->sci_iterations = it;
        loop->max_delta = md;
        if (md != md || out[K + 1] != 0.0) {
            loop->status = 1;
            loop->done = 1;
        } else if (md < loop->tol) {
            loop->success = 1;
            loop->done = 1;
        } else if (it >= loop->maxiter) {
            loop->done = 1;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// adaptive(): K-vector kernels
// ------------------------------------------------------------------------------------------------
// After the pass at f: gradient (Eq. C6), the self-consistent candidate (Eq. C3) with the gauge of
// mbar_solvers.py:588, the constants of the next launches and the diagonal N_i S_i of the Hessian (Eq. C9).
__global__ void __launch_bounds__(256)
adapt_pre_kernel(const double* __restrict__ out, const double* __restrict__ f, const double* __restrict__ Nk,
                 const unsigned long long* __restrict__ rowmask, int K, int first, double mid,
                 double* __restrict__ av, LoopState* loop) {
    if (loop_done(loop)) return;
    __shared__ double s_buf[64];
    __shared__ double s_f0;
    if (threadIdx.x == 0) s_f0 = f[first] - log(out[first]);
    __syncthreads();
    double bad = (threadIdx.x == 0 && out[K + 1] != 0.0) ? 1.0 : 0.0;
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        const double fk = f[k];
        if (row_on(rowmask, k)) {
            const double S = out[k], n = Nk[k], ln = log(n);
            if (!(S > 1e-280) || !(S < 1e300)) bad = 1.0;
            const double fs = fk - log(S) - s_f0;
            av[AV_FSCI * K + k] = fs;
            av[AV_CSCI * K + k] = fs + ln - mid;
            av[AV_G * K + k] = n * (S - 1.0);
            av[AV_CH * K + k] = fk + ln;
            av[AV_DIAG * K + k] = n * S;
        } else {
            av[AV_FSCI * K + k] = fk;
            av[AV_CSCI * K + k] = 0.0;
            av[AV_G * K + k] = 0.0;
            av[AV_CH * K + k] = 0.0;
            av[AV_DIAG * K + k] = 0.0;
        }
    }
    bad = block_sum(bad, s_buf);
    if (threadIdx.x == 0 && bad > 0.0) {
        loop->status = out[K + 1] >= 1.0e6 ? 2 : 1;
        loop->done = 1;
    }
}

// Reduced Newton matrix A = H[1:,1:] over the sampled states (gauge state dropped, mbar_solvers.py:804-818 /
// SURVEY.md Appendix A): A_ab = delta_ab N_i S_i (1 + ridge) - Ghat_ij, stored column-major (it is symmetric).
// ridgeRel > 0 is the retry after a failed factorisation (only then: onlyIfFail).
__global__ void __launch_bounds__(256)
newton_build_kernel(const double* __restrict__ G, const double* __restrict__ av, const int* __restrict__ active,
                    int na, int K, double* __restrict__ A, double ridgeRel, int onlyIfFail, LoopState* loop) {
    if (loop_done(loop)) return;
    if (onlyIfFail && !*reinterpret_cast<volatile int*>(&loop->cholFail)) return;
    const int n = na - 1;
    const int64_t total = (int64_t)n * n;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(e / n), a = (int)(e % n);          // column b, row a
        const int i = active[a + 1], j = active[b + 1];
        double v = -G[(size_t)i * K + j];
        if (a == b) v += av[AV_DIAG * K + i] * (1.0 + ridgeRel);
        A[e] = v;
    }
}

// Cholesky factorisation A = L L^T (left-looking by columns), the two triangular solves and the Newton
// candidate f_nr = f - gamma * H^-1 g (mbar_solvers.py:581-584), all in ONE CTA.  SMEM: the matrix lives in
// shared memory (n <= 160); otherwise it stays in global memory (L2-resident: n^2 * 8 <= 32 MB) and is read with
// ld.global.cg so that no stale L1 line is ever seen.
template <bool SMEM>
__global__ void __launch_bounds__(1024)
newton_kernel(double* __restrict__ Ag, int na, int K, const int* __restrict__ active, const double* __restrict__ f,
              const double* __restrict__ Nk, double* __restrict__ av, double mid, int onlyIfFail, int lastAttempt,
              LoopState* loop) {
    if (loop_done(loop)) return;
    if (onlyIfFail && !*reinterpret_cast<volatile int*>(&loop->cholFail)) return;
    if (onlyIfFail && threadIdx.x == 0) loop->ridgeRetries++;
    extern __shared__ __align__(16) double sm[];
    const int n = na - 1;
    const int tid = threadIdx.x, nt = blockDim.x;
    double* b = sm;                       // [n] right-hand side / solution
    double* row = sm + ((n + 1) & ~1);    // [n] pivot row of L
    double* M = SMEM ? row + ((n + 1) & ~1) : Ag;
    __shared__ int s_fail;
    if (tid == 0) s_fail = 0;
    if (SMEM)
        for (int e = tid; e < n * n; e += nt) M[e] = Ag[e];
    for (int a = tid; a < n; a += nt) b[a] = av[AV_G * K + active[a + 1]];
    __syncthreads();
#define LDM(ptr) (SMEM ? *(ptr) : __ldcg(ptr))
    for (int j = 0; j < n; ++j) {
        for (int k = tid; k < j; k += nt) row[k] = LDM(M + (size_t)k * n + j);
        __syncthreads();
        // row i of the update is a dot product of length j: four lanes share it (k = ks, ks + 4, ...) so that a
        // column keeps 4 (n - j) threads busy instead of n - j — the loop is bound by the latency of its loads
        for (int base = j; base < n; base += (nt >> 2)) {     // trip count uniform over the CTA (full-mask shuffles)
            const int i0 = base + (tid >> 2);
            const int i = i0 < n ? i0 : n - 1;          // (idle quads recompute the last row)
            const int ks = tid & 3;
            double s0 = 0.0, s1 = 0.0;
            int k = ks;
            for (; k + 4 < j; k += 8) {
                s0 = fma(-LDM(M + (size_t)k * n + i), row[k], s0);
                s1 = fma(-LDM(M + (size_t)(k + 4) * n + i), row[k + 4], s1);
            }
            if (k < j) s0 = fma(-LDM(M + (size_t)k * n + i), row[k], s0);
            double t = s0 + s1;
            t += __shfl_xor_sync(0xffffffffu, t, 1);
            t += __shfl_xor_sync(0xffffffffu, t, 2);
            if (ks == 0 && i0 < n) M[(size_t)j * n + i] = LDM(M + (size_t)j * n + i) + t;
        }
        __syncthreads();
        const double d = LDM(M + (size_t)j * n + j);
        if (!(d > 0.0) || !(d < 1e300)) {       // not positive definite (or NaN): uniform exit
            if (tid == 0) s_fail = 1;
            break;
        }
        const double sq = sqrt(d), inv = 1.0 / sq;
        __syncthreads();                          // everyone has read d before the diagonal is overwritten
        for (int i = j + tid; i < n; i += nt) {
            const double v = LDM(M + (size_t)j * n + i);
            M[(size_t)j * n + i] = (i == j) ? sq : v * inv;
        }
        __syncthreads();
    }
    __syncthreads();
    if (s_fail) {
        if (tid == 0) {
            loop->cholFail = 1;
            if (lastAttempt) {
                loop->haveNr = 0;
                loop->nrFailed++;
            }
        }
        if (lastAttempt)   // no Newton candidate this iteration: it coincides with the self-consistent one
            for (int k = tid; k < K; k += nt) {
                av[AV_FNR * K + k] = av[AV_FSCI * K + k];
                av[AV_CNR * K + k] = av[AV_CSCI * K + k];
            }
        return;
    }
    // L y = g
    for (int j = 0; j < n; ++j) {
        if (tid == 0) b[j] = b[j] / LDM(M + (size_t)j * n + j);
        __syncthreads();
        const double xj = b[j];
        for (int i = j + 1 + tid; i < n; i += nt) b[i] = fma(-LDM(M + (size_t)j * n + i), xj, b[i]);
        __syncthreads();
    }
    // L^T x = y
    for (int j = n - 1; j >= 0; --j) {
        if (tid == 0) b[j] = b[j] / LDM(M + (size_t)j * n + j);
        __syncthreads();
        const double xj = b[j];
        for (int i = tid; i < j; i += nt) b[i] = fma(-LDM(M + (size_t)i * n + j), xj, b[i]);
        __syncthreads();
    }
#undef LDM
    // candidate: f_nr = f - gamma x on the free states; gauge and unsampled states untouched
    const double gamma = loop->gamma;
    __shared__ int s_badnr;
    if (tid == 0) s_badnr = 0;
    __syncthreads();
    for (int k = tid; k < K; k += nt) av[AV_FNR * K + k] = f[k];
    __syncthreads();
    for (int a = tid; a < n; a += nt) {
        const int k = active[a + 1];
        const double v = f[k] - gamma * b[a];
        av[AV_FNR * K + k] = v;
        if (!(fabs(v) < 0.5 * C_RANGE)) s_badnr = 1;     // NaN / inf / out of the supported range
    }
    __syncthreads();
    if (s_badnr) {
        for (int k = tid; k < K; k += nt) {
            av[AV_FNR * K + k] = av[AV_FSCI * K + k];
            av[AV_CNR * K + k] = av[AV_CSCI * K + k];
        }
        if (tid == 0) {
            loop->haveNr = 0;
            loop->cholFail = 0;
            loop->nrRejected++;
        }
        return;
    }
    for (int k = tid; k < K; k += nt) av[AV_CNR * K + k] = (Nk[k] > 0.0) ? av[AV_FNR * K + k] + log(Nk[k]) - mid : 0.0;
    if (tid == 0) {
        loop->haveNr = 1;
        loop->cholFail = 0;
    }
}

// After the two candidate passes: gradient norms, the step choice of mbar_solvers.py:607, the convergence rule
// of :627-640, and the vectors of the next iteration.
__global__ void __launch_bounds__(256)
adapt_post_kernel(const double* __restrict__ outS, const double* __restrict__ outN, const double* __restrict__ av,
                  double* __restrict__ f, double* __restrict__ c0, const double* __restrict__ Nk,
                  const unsigned long long* __restrict__ rowmask, int K, int first, double mid, LoopState* loop) {
    if (loop_done(loop)) return;
    __shared__ double s_buf[64];
    double gs = 0.0, gn = 0.0, badS = 0.0, badN = 0.0;
    if (threadIdx.x == 0) {
        if (outS[K + 1] != 0.0) badS = 1.0;
        if (outN[K + 1] != 0.0) badN = 1.0;
    }
    for (int k = threadIdx.x; k < K; k += blockDim.x)
        if (row_on(rowmask, k)) {
            const double a = Nk[k] * (outS[k] - 1.0), b = Nk[k] * (outN[k] - 1.0);
            if (!(outS[k] > 1e-280) || !(outS[k] < 1e300)) badS = 1.0;
            if (!(outN[k] > 1e-280) || !(outN[k] < 1e300)) badN = 1.0;
            gs += a * a;
            gn += b * b;
        }
    gs = block_sum(gs, s_buf);
    gn = block_sum(gn, s_buf);
    badS = block_sum(badS, s_buf);
    badN = block_sum(badN, s_buf);
    const int haveNr = loop->haveNr && !(badN > 0.0) && gn == gn;
    const double gnNr = haveNr ? gn : INFINITY;
    const bool takeSci = (gs < gnNr) || (loop->sci_iterations < loop->min_sc_iter);    // mbar_solvers.py:607
    const double* fnew = av + (takeSci ? AV_FSCI : AV_FNR) * K;
    const double* fsci = av + AV_FSCI * K;
    const double* fnr = haveNr ? av + AV_FNR * K : fsci;
    const double thr = fmin(1.0e-8, loop->tol);
    double md = 0.0, mx = 0.0;
    for (int k = threadIdx.x; k < K; k += blockDim.x)
        if (row_on(rowmask, k) && k != first) {
            const double v = fnew[k];
            const double d1 = rel_change(v, f[k], v, thr), d2 = rel_change(fsci[k], fnr[k], v, thr);
            if (d1 != d1 || md != md) md = NAN; else md = fmax(md, d1);
            if (d2 == d2) mx = fmax(mx, d2);
        }
    md = block_max_nan(md, s_buf);
    mx = block_max_nan(mx, s_buf);
    __syncthreads();
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        const double v = fnew[k];
        f[k] = v;
        c0[k] = row_on(rowmask, k) ? v + log(Nk[k]) - mid : 0.0;
    }
    if (threadIdx.x == 0) {
        const int it = loop->iterations + 1;
        loop->iterations = it;
        if (takeSci) loop->sci_iterations++; else loop->nr_iterations++;
        loop->gn_sci = gs;
        loop->gn_nr = gnNr;
        loop->gnorm = sqrt(takeSci ? gs : gn);
        loop->max_delta = md;
        loop->max_diff = mx;
        if (badS > 0.0 || md != md) {
            // the fused kernel's range assumption failed on the self-consistent candidate, or a non-finite
            // candidate: the host redoes this iteration on the robust stepped path
            loop->status = (outS[K + 1] >= 1.0e6 || outN[K + 1] >= 1.0e6) ? 2 : 1;
            loop->done = 1;
        } else if (md < loop->tol && mx < sqrt(loop->tol)) {
            loop->success = 1;
            loop->done = 1;
        } else if (it >= loop->maxiter) {
            loop->done = 1;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// stream-ordered rendezvous of all ranks (one tiny all-reduce) before the first in-kernel peer exchange of a loop
static int comm_rendezvous(mbar_b200_ctx* c) {
    if (!c->comm || c->nranks == 1) return MBAR_B200_OK;
    // every rank's stream reaches the first in-kernel exchange within microseconds of the others
    return comm_allreduce(c, c->d_scratch + scratch_rendezvous(c->K), 1, 0);
}

static int loop_begin(mbar_b200_ctx* c, double tol, int maxiter, int min_sc_iter, double gamma) {
    LoopState st{};
    st.tol = tol;
    st.gamma = gamma;
    st.maxiter = maxiter;
    st.min_sc_iter = min_sc_iter;
    *c->h_loop = st;
    MBAR_CUDA(cudaMemcpyAsync(c->d_loop, c->h_loop, sizeof(LoopState), cudaMemcpyHostToDevice, c->stream));
    return MBAR_B200_OK;
}

static bool device_loop_possible(const mbar_b200_ctx* c) {
    if (c->kernelChoice == MBAR_B200_KERNEL_GENERIC) return false;
    if (c->nranks > 1 && !c->comm) return false;
    return c->K <= 2048;
}

// One kernel per self-consistent iteration when the exchange can live inside the pass kernel (single GPU, or peers
// attached through mbar_b200_peer_attach); otherwise pass -> all-reduce -> sci_loop_epilogue_kernel.
static bool sci_epilogue_in_kernel(const mbar_b200_ctx* c) {
    return (c->nranks == 1 || c->peerReady) && !std::getenv("MBAR_B200_NO_FUSED_EPILOGUE");
}

// f -> pinned row ROW_F -> ctx->d_f (asynchronous)
static int upload_f(mbar_b200_ctx* c, const double* f) {
    const int K = c->K;
    std::memcpy(c->hf(ROW_F), f, K * sizeof(double));
    MBAR_CUDA(cudaMemcpyAsync(c->d_f, c->hf(ROW_F), K * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    c->h2dBytes += K * 8;
    return MBAR_B200_OK;
}

StepRows step_rows(const mbar_b200_ctx* c) { return StepRows{c->K, c->active.data(), (int)c->active.size(), c->h_Nk.data()}; }

// Largest relative change over the sampled states other than the gauge state (mbar_solvers.py:627-631), NaN if any
// entry is NaN.
double step_rel_delta(const StepRows& s, const double* fn, const double* fo, double tol) {
    double md = 0.0;
    const double thr = std::min(1e-8, tol);
    for (int i = 1; i < s.na; ++i) {
        const int k = s.active[i];
        const double d = rel_change(fn[k], fo[k], fn[k], thr);
        if (std::isnan(d)) return NAN;
        md = std::max(md, d);
    }
    return md;
}
static double rel_delta(const mbar_b200_ctx* c, const std::vector<double>& fn, const std::vector<double>& fo,
                        double tol) {
    return step_rel_delta(step_rows(c), fn.data(), fo.data(), tol);
}

// The self-consistent step (Eq. C3) from log S_k at cur: f_k - log S_k over the sampled states, gauge-fixed so that
// f[active[0]] = 0; unsampled states keep cur.  nxt may be cur.
void step_sci(const StepRows& s, const std::vector<double>& cur, const double* logS, std::vector<double>& nxt) {
    const int g0 = s.active[0];
    const double shift = cur[g0] - logS[g0];
    nxt = cur;
    for (int i = 0; i < s.na; ++i) {
        const int k = s.active[i];
        nxt[k] = (cur[k] - logS[k]) - shift;
    }
}

// The self-consistent step from the packed output of run_pass at cur.
static void sci_step(const mbar_b200_ctx* c, const std::vector<double>& cur, std::vector<double>& nxt) {
    step_sci(step_rows(c), cur, c->h_out + PassLayout{c->K}.logS(), nxt);
}

// g_k = N_k (S_k - 1) over every state (0 where N_k = 0) and its squared norm
double step_gradient(const StepRows& s, const double* S, std::vector<double>& g) {
    double gn = 0.0;
    for (int k = 0; k < s.K; ++k) {
        g[k] = s.Nk[k] > 0 ? s.Nk[k] * (S[k] - 1.0) : 0.0;
        gn += g[k] * g[k];
    }
    return gn;
}

// gradient norm at f over the sampled states (mbar_solvers.py:938-940): one more pass
static int final_gnorm(mbar_b200_ctx* c, const std::vector<double>& f, mbar_b200_solve_result* r) {
    const int rc = run_pass(c, f.data(), PassWant{});
    r->passes++;
    double gn = 0.0;
    for (int k : c->active) {
        const double g = c->h_Nk[k] * (c->h_out[k] - 1.0);
        gn += g * g;
    }
    r->gnorm = std::sqrt(gn);
    return rc;
}

// In-place Cholesky of the n x n SPD matrix A (row-major, lower); returns false if not PD.
static bool cholesky(std::vector<double>& A, int n) {
    for (int j = 0; j < n; ++j) {
        double d = A[(size_t)j * n + j];
        for (int k = 0; k < j; ++k) d -= A[(size_t)j * n + k] * A[(size_t)j * n + k];
        if (!(d > 0.0) || !std::isfinite(d)) return false;
        d = std::sqrt(d);
        A[(size_t)j * n + j] = d;
        const double inv = 1.0 / d;
        for (int i = j + 1; i < n; ++i) {
            double s = A[(size_t)i * n + j];
            const double* ai = &A[(size_t)i * n];
            const double* aj = &A[(size_t)j * n];
            for (int k = 0; k < j; ++k) s -= ai[k] * aj[k];
            A[(size_t)i * n + j] = s * inv;
        }
    }
    return true;
}
static void chol_solve(const std::vector<double>& Lc, int n, std::vector<double>& b) {
    for (int i = 0; i < n; ++i) {
        double s = b[i];
        for (int k = 0; k < i; ++k) s -= Lc[(size_t)i * n + k] * b[k];
        b[i] = s / Lc[(size_t)i * n + i];
    }
    for (int i = n - 1; i >= 0; --i) {
        double s = b[i];
        for (int k = i + 1; k < n; ++k) s -= Lc[(size_t)k * n + i] * b[k];
        b[i] = s / Lc[(size_t)i * n + i];
    }
}

// ---- host-stepped loops: one host round trip per pass.  They are the robust fallback of the device-resident loops
// (generic kernel, log-domain sums, ridge retries) and stay selectable with mbar_b200_set_loop_mode(ctx, 1).
static int solve_sci_stepped(mbar_b200_ctx* c, double* f, double tol, int32_t maxiter, mbar_b200_solve_result* res) {
    const int K = c->K;
    std::vector<double> cur(f, f + K), nxt(K);
    mbar_b200_solve_result r{};
    Events timer;
    MBAR_TRY(timer.start(c->stream));
    for (int k : c->active) cur[k] -= f[c->firstActive];
    int rc = MBAR_B200_OK;
    for (int it = 0; it < maxiter; ++it) {
        rc = run_pass(c, cur.data(), PassWant{});
        if (rc != MBAR_B200_OK) break;
        r.passes++;
        sci_step(c, cur, nxt);
        r.max_delta = rel_delta(c, nxt, cur, tol);
        cur.swap(nxt);
        r.iterations = it + 1;
        r.sci_iterations = it + 1;
        if (std::isnan(r.max_delta) || r.max_delta < tol) {
            r.success = 1;
            break;
        }
    }
    if (rc == MBAR_B200_OK) rc = final_gnorm(c, cur, &r);
    r.device_ms = timer.stop();
    if (rc == MBAR_B200_OK) std::memcpy(f, cur.data(), K * sizeof(double));
    if (res) *res = r;
    return rc;
}

// The Newton candidate of one adaptive iteration from the sums at cur, in the reduced coordinates (gauge state
// dropped): H[1:,1:] x = g[1:] with H_ab = delta_ab N_i S_i - Ghat_ij (mbar_solvers.py:581-584 uses the min-norm
// lstsq of the singular full H minus its first component — the same step in exact arithmetic, SURVEY.md Appendix A).
// A factorisation that fails is retried with a relative ridge, up to four attempts.  False: no candidate (no free
// state, H not positive definite, or f_nr non-finite or outside C_RANGE).  A and rhs are scratch.
bool step_newton(const StepRows& s, const double* S, const double* Gh, const std::vector<double>& g,
                 const std::vector<double>& cur, double gamma, std::vector<double>& A, std::vector<double>& rhs,
                 std::vector<double>& f_nr) {
    const int K = s.K, na = s.na;
    bool haveNr = false;
    if (na > 1) {
        const int n = na - 1;
        double ridge = 0.0, ridgeRel = 0.0, tr = 0.0;
        for (int a = 1; a < na; ++a) {
            const int i = s.active[a];
            tr += s.Nk[i] * S[i];
        }
        for (int attempt = 0; attempt < 4 && !haveNr; ++attempt) {
            A.assign((size_t)n * n, 0.0);
            for (int a = 1; a < na; ++a) {
                const int i = s.active[a];
                for (int b = 1; b <= a; ++b) {
                    const int j = s.active[b];
                    double v = -Gh[(size_t)i * K + j];
                    if (i == j) v += s.Nk[i] * S[i] + ridge;
                    A[(size_t)(a - 1) * n + (b - 1)] = v;
                }
            }
            if (cholesky(A, n)) {
                rhs.resize(n);
                for (int a = 1; a < na; ++a) rhs[a - 1] = g[s.active[a]];
                chol_solve(A, n, rhs);
                f_nr = cur;
                for (int a = 1; a < na; ++a) f_nr[s.active[a]] = cur[s.active[a]] - gamma * rhs[a - 1];
                haveNr = true;
                for (int a = 1; a < na; ++a)
                    if (!std::isfinite(f_nr[s.active[a]]) || std::fabs(f_nr[s.active[a]]) > 0.5 * C_RANGE)
                        haveNr = false;
            } else {
                ridgeRel = (ridgeRel == 0.0) ? 1e-12 : ridgeRel * 1e3;   // relative to the mean diagonal
                ridge = ridgeRel * (tr / n + 1e-300);
            }
        }
    }
    return haveNr;
}

// The step choice of one adaptive iteration (mbar_solvers.py:607) and its convergence rule (:627-640), given the
// squared gradient norms at both candidates (gn_nr is ignored without a Newton candidate; NaN counts as +inf).  cur
// becomes the chosen candidate; r's iteration counters, gnorm and max_delta advance.  True when converged.
bool step_choose(const StepRows& s, const std::vector<double>& f_sci, const std::vector<double>& f_nr, bool haveNr,
                 double gn_sci, double gn_nr, double tol, int32_t min_sc_iter, std::vector<double>& cur,
                 mbar_b200_solve_result& r) {
    const std::vector<double>& fnr = haveNr ? f_nr : f_sci;
    if (!haveNr || std::isnan(gn_nr)) gn_nr = INFINITY;
    std::vector<double> f_old = cur;
    if (gn_sci < gn_nr || r.sci_iterations < min_sc_iter) {     // mbar_solvers.py:607
        cur = f_sci;
        r.sci_iterations++;
        r.gnorm = std::sqrt(gn_sci);
    } else {
        cur = fnr;
        r.nr_iterations++;
        r.gnorm = std::sqrt(gn_nr);
    }
    r.iterations++;
    r.max_delta = step_rel_delta(s, cur.data(), f_old.data(), tol);
    // max |f_sci - f_nr| / |f|  (mbar_solvers.py:632)
    double max_diff = 0.0;
    const double thr = std::min(1e-8, tol);
    for (int i = 1; i < s.na; ++i) {
        const int k = s.active[i];
        max_diff = std::max(max_diff, rel_change(f_sci[k], fnr[k], cur[k], thr));
    }
    if (std::isnan(r.max_delta) || (r.max_delta < tol && max_diff < std::sqrt(tol))) {
        r.success = 1;
        return true;
    }
    return false;
}

static int solve_adaptive_stepped(mbar_b200_ctx* c, double* f, double tol, int32_t maxiter, int32_t min_sc_iter,
                                  double gamma, mbar_b200_solve_result* res) {
    const int K = c->K;
    const PassLayout lay{K};
    const StepRows rows = step_rows(c);
    std::vector<double> cur(f, f + K), f_sci(K), f_nr(K), g(K, 0.0), g_sci(K), g_nr(K);
    std::vector<double> A, rhs;
    mbar_b200_solve_result r{};
    Events timer;
    MBAR_TRY(timer.start(c->stream));
    for (int k : c->active) cur[k] -= f[c->firstActive];
    int rc = MBAR_B200_OK;
    for (int it = 0; it < maxiter && rc == MBAR_B200_OK; ++it) {
        // pass at f with the second moments: gives g, H and the self-consistent candidate at once
        PassWant w;
        w.G = true;
        rc = run_pass(c, cur.data(), w);
        if (rc != MBAR_B200_OK) break;
        r.passes++;
        r.hessian_passes++;
        step_gradient(rows, c->h_out, g);
        sci_step(c, cur, f_sci);
        const bool haveNr = step_newton(rows, c->h_out, c->h_out + lay.G(), g, cur, gamma, A, rhs, f_nr);
        rc = run_pass(c, f_sci.data(), PassWant{});
        if (rc != MBAR_B200_OK) break;
        r.passes++;
        const double gn_sci = step_gradient(rows, c->h_out, g_sci);
        double gn_nr = INFINITY;
        if (haveNr) {
            rc = run_pass(c, f_nr.data(), PassWant{});
            if (rc != MBAR_B200_OK) break;
            r.passes++;
            gn_nr = step_gradient(rows, c->h_out, g_nr);
        }
        if (step_choose(rows, f_sci, f_nr, haveNr, gn_sci, gn_nr, tol, min_sc_iter, cur, r)) break;
    }
    r.device_ms = timer.stop();
    if (rc == MBAR_B200_OK) std::memcpy(f, cur.data(), K * sizeof(double));
    if (res) *res = r;
    return rc;
}

// `iters` host-stepped self-consistent iterations, no convergence test (mbar_b200_sci_iterate's robust path)
static int sci_iterate_stepped(mbar_b200_ctx* c, double* f, int iters) {
    std::vector<double> cur(f, f + c->K);
    for (int it = 0; it < iters; ++it) {
        MBAR_TRY(run_pass(c, cur.data(), PassWant{}));
        sci_step(c, cur, cur);
    }
    std::memcpy(f, cur.data(), c->K * sizeof(double));
    return MBAR_B200_OK;
}

// ---- device-resident loops
// Enqueues `n` self-consistent iterations on the f in ctx->d_f with the pass p (from fused_prepare): the fused pass
// with its in-kernel epilogue, or pass -> all-reduce -> epilogue kernel.  loop: early exit and convergence test, or
// NULL (every iteration runs).  ev, optional: two events per iteration recorded around the pass launch.
static int enqueue_sci(mbar_b200_ctx* c, FusedParams p, bool inKernel, int n, LoopState* loop,
                       const cudaEvent_t* ev) {
    const int K = c->K;
    p.loop = loop;
    p.first = c->firstActive;
    if (inKernel) {
        p.epi = 1;
        p.f = c->d_f;
        p.cnext = c->dc(ROW_C);
        if (c->peerReady) p.peer = c->peer;
    }
    for (int it = 0; it < n; ++it) {
        if (ev) MBAR_CUDA(cudaEventRecord(ev[2 * it], c->stream));
        MBAR_TRY(fused_enqueue(c, p));
        if (ev) MBAR_CUDA(cudaEventRecord(ev[2 * it + 1], c->stream));
        if (!inKernel) {
            MBAR_TRY(comm_allreduce(c, c->d_out, K + 2, 0));
            sci_loop_epilogue_kernel<<<1, 256, 0, c->stream>>>(c->d_out, c->d_f, c->dc(ROW_C), c->d_Nk, c->d_rowmask,
                                                               K, p.first, p.mid, loop);
            c->launches++;
        }
    }
    return MBAR_B200_OK;
}

// The batches of a device-resident solver.  batch(f, &ok) configures the fused pass at f (ok = false: it does not
// apply), uploads f and enqueues one batch of iterations; then LoopState and f come back in the batch's one
// synchronisation.  On return cur holds the last f the device reported.  *fallback: the fast path gave up, cur is
// the f that batch started from and *good the LoopState polled with it (its iteration counters are the ones that
// led to cur; a failed batch's own steps are redone), and the caller finishes on its host-stepped loop.
static int poll_batches(mbar_b200_ctx* c, std::vector<double>& cur, LoopState* good, bool* fallback,
                        const std::function<int(const double*, bool*)>& batch) {
    const int K = c->K;
    *fallback = false;
    for (;;) {
        *good = *c->h_loop;
        bool ok = false;
        MBAR_TRY(batch(cur.data(), &ok));
        if (!ok) {
            *fallback = true;
            return MBAR_B200_OK;
        }
        MBAR_CUDA(cudaMemcpyAsync(c->h_loop, c->d_loop, sizeof(LoopState), cudaMemcpyDeviceToHost, c->stream));
        MBAR_CUDA(cudaMemcpyAsync(c->hf(ROW_POLL), c->d_f, (size_t)K * sizeof(double), cudaMemcpyDeviceToHost,
                                  c->stream));
        MBAR_CUDA(cudaStreamSynchronize(c->stream));
        c->d2hBytes += (int64_t)K * 8 + (int64_t)sizeof(LoopState);
        c->loopPolls++;
        MBAR_CUDA(cudaGetLastError());
        const LoopState& st = *c->h_loop;
        if (st.status != 0) {
            MBAR_REQUIRE(st.status != 2, MBAR_B200_ERR_COMM,
                         "peer exchange timed out inside the pass kernel (a rank did not arrive)");
            *fallback = true;
            return MBAR_B200_OK;
        }
        std::memcpy(cur.data(), c->hf(ROW_POLL), K * sizeof(double));
        if (st.done) return MBAR_B200_OK;
    }
}

static int solve_sci_device(mbar_b200_ctx* c, double* f, double tol, int32_t maxiter, mbar_b200_solve_result* res) {
    MBAR_REQUIRE(c->ready, MBAR_B200_ERR_NOT_READY, "u_kn has not been uploaded");
    MBAR_CUDA(cudaSetDevice(c->device));
    MBAR_TRY(check_range(c, f));
    if (!device_loop_possible(c) || maxiter < 1 || c->active.size() < 2)
        return solve_sci_stepped(c, f, tol, maxiter, res);
    std::vector<double> cur(f, f + c->K);
    for (int k : c->active) cur[k] -= f[c->firstActive];
    Events timer;
    MBAR_TRY(timer.start(c->stream));
    MBAR_TRY(loop_begin(c, tol, maxiter, 0, 1.0));
    const bool inKernel = sci_epilogue_in_kernel(c);
    if (c->peerReady && inKernel) MBAR_TRY(comm_rendezvous(c));
    LoopState good{};
    bool fallback = false;
    MBAR_TRY(poll_batches(c, cur, &good, &fallback, [&](const double* fb, bool* ok) -> int {
        FusedParams p;
        MBAR_TRY(fused_prepare(c, fb, false, false, &p, ok));
        if (!*ok) return MBAR_B200_OK;
        MBAR_TRY(upload_f(c, fb));
        return enqueue_sci(c, p, inKernel, c->loopBatch, c->d_loop, nullptr);
    }));
    mbar_b200_solve_result r{};
    int rc;
    if (fallback) {
        // redo from the last good f on the robust path (generic kernel, log-domain sums)
        const int itersBefore = good.iterations;
        rc = solve_sci_stepped(c, cur.data(), tol, std::max(maxiter - itersBefore, 1), &r);
        r.iterations += itersBefore;
        r.sci_iterations += itersBefore;
        r.passes += itersBefore;
    } else {
        const LoopState& st = *c->h_loop;
        r.iterations = r.sci_iterations = st.iterations;
        r.passes = st.iterations;
        r.success = st.success;
        r.max_delta = st.max_delta;
        rc = final_gnorm(c, cur, &r);
    }
    r.device_ms = timer.stop();
    if (rc == MBAR_B200_OK)
        for (int k : c->active) f[k] = cur[k];
    if (res) *res = r;
    return rc;
}

// Launch plan of newton_kernel for an n x n system: the matrix in shared memory when it fits (n <= 158), and a CTA of
// 256, 512 or 1024 threads (four per row of the column update).
static bool newton_in_smem(int n) { return (size_t)n * n * 8 + 2 * ((size_t)n + 2) * 8 <= 200 * 1024; }
static int newton_threads(int n) { return n >= 96 ? 1024 : n >= 32 ? 512 : 256; }

// One adaptive iteration, enqueued with no host synchronisation.
static int enqueue_adaptive_iteration(mbar_b200_ctx* c, const FusedParams& pF, const FusedParams& pS,
                                      const FusedParams& pN, const FusedParams* pM) {
    const int K = c->K;
    const PassLayout lay{K};
    const int na = (int)c->active.size();
    const int n = na - 1;
    const int g0 = c->firstActive;
    const bool nccl = c->nranks > 1 && !c->peerReady;
    double* av = c->d_av;
    // (1) pass at f: S, sum L, per-sample L'_n
    MBAR_TRY(fused_enqueue(c, pF));
    if (nccl) MBAR_TRY(comm_allreduce(c, c->d_out, K + 2, 0));
    adapt_pre_kernel<<<1, 256, 0, c->stream>>>(c->d_out, c->d_f, c->d_Nk, c->d_rowmask, K, g0, pF.mid, av, c->d_loop);
    // (2) second moments at f (reads L'_n of the pass above)
    MBAR_TRY(launch_hessian_dev(c, av + AV_CH * K, false, c->d_loop, pF.Wout != nullptr));
    if (c->nranks > 1) MBAR_TRY(comm_allreduce(c, c->d_out + lay.G(), K * K, 0));
    // (3) Newton candidate: build, factorise, solve; one retry with a relative ridge if not positive definite
    const bool smem = newton_in_smem(n);
    const size_t shBytes = 2 * ((size_t)n + 2) * 8 + (smem ? (size_t)n * n * 8 : 0);
    auto kern = smem ? newton_kernel<true> : newton_kernel<false>;
    static size_t attr[16][2] = {{0}};
    size_t& a = attr[c->device & 15][smem ? 0 : 1];
    if (a < shBytes) {
        MBAR_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shBytes));
        a = shBytes;
    }
    const int bgrid = (int)std::min<int64_t>(((int64_t)n * n + 255) / 256, 4 * c->smCount);
    const int nthreads = newton_threads(n);
    for (int attempt = 0; attempt < 2; ++attempt) {
        newton_build_kernel<<<bgrid, 256, 0, c->stream>>>(c->d_out + lay.G(), av, c->d_active, na, K, c->d_A,
                                                         attempt ? 1.0e-10 : 0.0, attempt, c->d_loop);
        kern<<<1, nthreads, shBytes, c->stream>>>(c->d_A, na, K, c->d_active, c->d_f, c->d_Nk, av, pF.mid, attempt,
                                                 attempt == 1, c->d_loop);
    }
    MBAR_CUDA(cudaGetLastError());
    // (4) both candidates: ONE launch evaluates f_sci and f_nr on the same staged tiles (M = 2) when the kernel
    //     family allows it, otherwise two launches
    if (pM) {
        MBAR_TRY(fused_enqueue(c, *pM));
        if (nccl) {
            MBAR_TRY(comm_allreduce(c, pM->out, K + 2, 0));
            MBAR_TRY(comm_allreduce(c, pM->out2, K + 2, 0));
        }
    } else {
        MBAR_TRY(fused_enqueue(c, pS));
        if (nccl) MBAR_TRY(comm_allreduce(c, pS.out, K + 2, 0));
        MBAR_TRY(fused_enqueue(c, pN));
        if (nccl) MBAR_TRY(comm_allreduce(c, pN.out, K + 2, 0));
    }
    // (5) choice + convergence + next iteration's vectors
    adapt_post_kernel<<<1, 256, 0, c->stream>>>(pS.out, pN.out, av, c->d_f, c->dc(ROW_C), c->d_Nk, c->d_rowmask, K, g0,
                                               pF.mid, c->d_loop);
    MBAR_CUDA(cudaGetLastError());
    c->launches += 6;
    return MBAR_B200_OK;
}

// Everything that distinguishes two launches of the fused kernel (the captured graph bakes these in).
static void key_push(std::vector<uint64_t>& key, const FusedParams& p) {
    auto bits = [](double v) { uint64_t u; std::memcpy(&u, &v, 8); return u; };
    const uint64_t f[] = {(uint64_t)(uintptr_t)p.u, (uint64_t)(uintptr_t)p.c, (uint64_t)(uintptr_t)p.c2,
                          (uint64_t)(uintptr_t)p.out, (uint64_t)(uintptr_t)p.out2, (uint64_t)(uintptr_t)p.Lout,
                          (uint64_t)(uintptr_t)p.Wout, (uint64_t)(uintptr_t)p.wgt, (uint64_t)(uintptr_t)p.loop,
                          (uint64_t)(uintptr_t)p.rowmask, (uint64_t)(uintptr_t)p.Nk, (uint64_t)(uintptr_t)p.peer.seq,
                          bits(p.mid), bits(p.mid2), bits(p.sumW), (uint64_t)p.N, (uint64_t)p.nStages,
                          (uint64_t)p.K | ((uint64_t)p.CL << 16) | ((uint64_t)p.M << 24) | ((uint64_t)p.mode << 28) |
                              ((uint64_t)p.NS << 32) | ((uint64_t)p.TPW << 40) | ((uint64_t)p.Wk << 48) | ((uint64_t)p.Rw << 56),
                          (uint64_t)p.peer.nranks | ((uint64_t)p.peer.rank << 8) | ((uint64_t)p.epi << 16) |
                              ((uint64_t)p.first << 24) | ((uint64_t)p.debugSkip << 56)};
    key.insert(key.end(), f, f + sizeof(f) / sizeof(f[0]));
}

// `batch` adaptive iterations.  The first batch a context ever runs is enqueued kernel by kernel (it sizes the
// buffers and sets the kernel attributes); after that ONE iteration is captured into a CUDA graph and relaunched:
// an iteration is ~11 launches and ~9 event records, which at C2 / C4 sizes (30-150 us kernels) cost as much
// as a third of the iteration when enqueued one by one.  The graph is kept across batches and across solves as
// long as the launch parameters are the same (the centring constant is quantised for that purpose).
static int run_adaptive_batch(mbar_b200_ctx* c, const FusedParams& pF, const FusedParams& pS, const FusedParams& pN,
                              const FusedParams* pM, int batch) {
    static const bool noGraph = std::getenv("MBAR_B200_NO_GRAPH") != nullptr;
    // Sharded problems keep the kernel-by-kernel path: an iteration then contains NCCL collectives (K x K
    // second moments; every pass without peer inboxes), and the 2-rank run with captured collectives did not
    // complete on the 8-GPU box this round (the same build without capture passed at 2 and 4 ranks), so the
    // graph is restricted to what has been verified: one GPU.  MBAR_B200_GRAPH_MULTI=1 re-enables it.
    static const bool graphMulti = std::getenv("MBAR_B200_GRAPH_MULTI") != nullptr;
    if (noGraph || !c->graphWarm || (c->nranks > 1 && !graphMulti)) {
        for (int b = 0; b < batch; ++b) MBAR_TRY(enqueue_adaptive_iteration(c, pF, pS, pN, pM));
        c->graphWarm = true;
        return MBAR_B200_OK;
    }
    std::vector<uint64_t> key;
    key_push(key, pF);
    key_push(key, pS);
    key_push(key, pN);
    if (pM) key_push(key, *pM);
    key.push_back((uint64_t)c->nranks | ((uint64_t)c->peerReady << 8) | ((uint64_t)(uintptr_t)c->comm << 16));
    if (!c->loopGraph || key != c->loopGraphKey) {
        if (c->loopGraph) {
            cudaGraphExecDestroy(c->loopGraph);
            c->loopGraph = nullptr;
        }
        const int64_t launches0 = c->launches, passes0 = c->passes;
        c->capturing = true;
        cudaError_t e = cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeRelaxed);
        int rc = MBAR_B200_OK;
        if (e == cudaSuccess) rc = enqueue_adaptive_iteration(c, pF, pS, pN, pM);
        cudaGraph_t g = nullptr;
        if (e == cudaSuccess) e = cudaStreamEndCapture(c->stream, &g);
        c->capturing = false;
        c->launches = launches0;
        c->passes = passes0;
        if (e == cudaSuccess && rc == MBAR_B200_OK && g) e = cudaGraphInstantiate(&c->loopGraph, g, 0);
        if (g) cudaGraphDestroy(g);
        if (e != cudaSuccess || rc != MBAR_B200_OK || !c->loopGraph) {
            // capture is an optimisation: fall back to plain launches for this batch
            cudaGetLastError();
            c->loopGraph = nullptr;
            c->loopGraphKey.clear();
            for (int b = 0; b < batch; ++b) MBAR_TRY(enqueue_adaptive_iteration(c, pF, pS, pN, pM));
            return MBAR_B200_OK;
        }
        c->loopGraphKey = key;
        c->graphCaptures++;
    }
    for (int b = 0; b < batch; ++b) {
        MBAR_CUDA(cudaGraphLaunch(c->loopGraph, c->stream));
        c->graphLaunches++;
        c->launches += 11;
        c->passes += pM ? 3 : 4;
    }
    return MBAR_B200_OK;
}

static int solve_adaptive_device(mbar_b200_ctx* c, double* f, double tol, int32_t maxiter, int32_t min_sc_iter,
                                 double gamma, mbar_b200_solve_result* res) {
    MBAR_REQUIRE(c->ready, MBAR_B200_ERR_NOT_READY, "u_kn has not been uploaded");
    MBAR_CUDA(cudaSetDevice(c->device));
    MBAR_TRY(check_range(c, f));
    const int K = c->K;
    if (!device_loop_possible(c) || maxiter < 1 || c->active.size() < 2)
        return solve_adaptive_stepped(c, f, tol, maxiter, min_sc_iter, gamma, res);
    std::vector<double> cur(f, f + K);
    for (int k : c->active) cur[k] -= f[c->firstActive];
    Events timer;
    MBAR_TRY(timer.start(c->stream));
    MBAR_TRY(loop_begin(c, tol, maxiter, min_sc_iter, gamma));
    if (c->peerReady) MBAR_TRY(comm_rendezvous(c));
    bool usedM2 = false;
    LoopState good{};
    bool fallback = false;
    MBAR_TRY(poll_batches(c, cur, &good, &fallback, [&](const double* fb, bool* ok) -> int {
        FusedParams pF;
        MBAR_TRY(fused_prepare(c, fb, true, false, &pF, ok, nullptr, nullptr, true, 1, 16.0));
        if (!*ok) return MBAR_B200_OK;
        MBAR_TRY(upload_f(c, fb));
        pF.loop = c->d_loop;
        pF.first = c->firstActive;
        if (c->peerReady) pF.peer = c->peer;
        FusedParams pS = pF, pN = pF;
        pS.Wout = pN.Wout = nullptr;
        pS.c = c->d_av + AV_CSCI * K;
        pS.out = c->d_outM;
        pS.Lout = nullptr;
        pN.c = c->d_av + AV_CNR * K;
        pN.out = c->d_outM + PassLayout{K}.size(false);
        pN.Lout = nullptr;
        // candidate-batched pass (same f -> same centring `mid` as pF; the device kernels write its constants)
        FusedParams pM;
        bool okM = false;
        static const bool noM2 = std::getenv("MBAR_B200_NO_M2") != nullptr;
        if (!noM2)
            MBAR_TRY(fused_prepare(c, fb, false, false, &pM, &okM, c->d_av + AV_CSCI * K, c->hf(ROW_C2), false, 2,
                                   16.0));
        if (okM) {
            pM.loop = c->d_loop;
            pM.first = c->firstActive;
            if (c->peerReady) pM.peer = c->peer;
            pM.c = c->d_av + AV_CSCI * K;
            pM.c2 = c->d_av + AV_CNR * K;
            pM.mid2 = pM.mid;
            pM.out = pS.out;
            pM.out2 = pN.out;
        }
        usedM2 = usedM2 || okM;
        return run_adaptive_batch(c, pF, pS, pN, okM ? &pM : nullptr, c->loopBatch);
    }));
    const int passesPerIter = usedM2 ? 2 : 3;
    const LoopState st = *c->h_loop;
    mbar_b200_solve_result r{};
    int rc = MBAR_B200_OK;
    mbar_b200_adaptive_stats& as = c->lastAdaptive;
    as.ridge_retries = st.ridgeRetries;
    as.newton_failed = st.nrFailed;
    as.newton_rejected = st.nrRejected;
    as.fell_back = fallback;
    as.device_iterations = fallback ? good.iterations : st.iterations;
    if (st.iterations > 0) {
        const int n = (int)c->active.size() - 1;
        as.newton_threads = newton_threads(n);
        as.newton_smem = newton_in_smem(n);
    }
    if (fallback) {
        // the stepped loop continues from the last good poll: its counters, and what is left of min_sc_iter,
        // start from that poll's (a failed batch's steps are redone, so they are not counted)
        const int msi = std::max(min_sc_iter - good.sci_iterations, 0);
        rc = solve_adaptive_stepped(c, cur.data(), tol, std::max(maxiter - good.iterations, 1), msi, gamma, &r);
        r.iterations += good.iterations;
        r.nr_iterations += good.nr_iterations;
        r.sci_iterations += good.sci_iterations;
        r.passes += passesPerIter * good.iterations;
        r.hessian_passes += good.iterations;
    } else {
        r.iterations = st.iterations;
        r.nr_iterations = st.nr_iterations;
        r.sci_iterations = st.sci_iterations;
        r.passes = passesPerIter * st.iterations;
        r.hessian_passes = st.iterations;
        r.success = st.success;
        r.max_delta = st.max_delta;
        r.gnorm = st.gnorm;
    }
    r.device_ms = timer.stop();
    if (rc == MBAR_B200_OK)
        for (int k : c->active) f[k] = cur[k];
    if (res) *res = r;
    return rc;
}

}  // namespace mbar

using namespace mbar;

extern "C" {

int mbar_b200_solve_sci(mbar_b200_ctx* c, double* f, double tol, int32_t maxiter, mbar_b200_solve_result* res) {
    MBAR_REQUIRE(c && f, MBAR_B200_ERR_INVALID, "NULL argument");
    NvtxRange nvtx_("mbar_b200::solve_sci");
    if (c->loopMode == 1) return solve_sci_stepped(c, f, tol, maxiter, res);
    return solve_sci_device(c, f, tol, maxiter, res);
}

int mbar_b200_solve_adaptive(mbar_b200_ctx* c, double* f, double tol, int32_t maxiter, int32_t min_sc_iter,
                             double gamma, mbar_b200_solve_result* res) {
    MBAR_REQUIRE(c && f, MBAR_B200_ERR_INVALID, "NULL argument");
    NvtxRange nvtx_("mbar_b200::solve_adaptive");
    c->lastAdaptive = mbar_b200_adaptive_stats{};
    if (c->loopMode == 1) return solve_adaptive_stepped(c, f, tol, maxiter, min_sc_iter, gamma, res);
    return solve_adaptive_device(c, f, tol, maxiter, min_sc_iter, gamma, res);
}

int mbar_b200_set_loop_mode(mbar_b200_ctx* c, int32_t mode, int32_t batch) {
    MBAR_REQUIRE(c, MBAR_B200_ERR_INVALID, "ctx is NULL");
    MBAR_REQUIRE(mode == 0 || mode == 1, MBAR_B200_ERR_INVALID, "mode=%d (0 device-resident, 1 host-stepped)", mode);
    c->loopMode = mode;
    if (batch >= 1) c->loopBatch = batch > 64 ? 64 : batch;
    return MBAR_B200_OK;
}

int mbar_b200_get_loop_stats(const mbar_b200_ctx* c, int64_t* polls, int32_t* mode, int32_t* batch) {
    MBAR_REQUIRE(c, MBAR_B200_ERR_INVALID, "ctx is NULL");
    if (polls) *polls = c->loopPolls;
    if (mode) *mode = c->loopMode;
    if (batch) *batch = c->loopBatch;
    return MBAR_B200_OK;
}

int mbar_b200_get_graph_stats(const mbar_b200_ctx* c, int64_t* captures, int64_t* launches) {
    MBAR_REQUIRE(c, MBAR_B200_ERR_INVALID, "ctx is NULL");
    if (captures) *captures = c->graphCaptures;
    if (launches) *launches = c->graphLaunches;
    return MBAR_B200_OK;
}

int mbar_b200_get_adaptive_stats(const mbar_b200_ctx* c, mbar_b200_adaptive_stats* stats) {
    MBAR_REQUIRE(c && stats, MBAR_B200_ERR_INVALID, "NULL argument");
    *stats = c->lastAdaptive;
    return MBAR_B200_OK;
}

int mbar_b200_sci_iterate(mbar_b200_ctx* c, double* f, int32_t iters) {
    MBAR_REQUIRE(c && f && iters >= 0, MBAR_B200_ERR_INVALID, "bad argument");
    MBAR_REQUIRE(c->ready, MBAR_B200_ERR_NOT_READY, "u_kn has not been uploaded");
    MBAR_CUDA(cudaSetDevice(c->device));
    MBAR_TRY(check_range(c, f));
    const int K = c->K;
    FusedParams p;
    bool ok = false;
    if (c->kernelChoice != MBAR_B200_KERNEL_GENERIC) MBAR_TRY(fused_prepare(c, f, false, false, &p, &ok));
    if (!ok) return sci_iterate_stepped(c, f, iters);
    MBAR_TRY(upload_f(c, f));
    // per-launch CUDA events of the pass kernel (bench: average launch duration over the loop)
    Events ev;
    const bool perLaunch = c->timePasses && iters > 0 && iters <= 4096;
    if (perLaunch) MBAR_TRY(ev.create(2 * (size_t)iters));
    Events timer;
    MBAR_TRY(timer.start(c->stream));
    const bool inKernel = sci_epilogue_in_kernel(c);
    MBAR_REQUIRE(c->nranks == 1 || c->comm, MBAR_B200_ERR_NOT_READY,
                 "sharded problem (%d ranks) without a communicator: call mbar_b200_comm_init", c->nranks);
    if (inKernel && c->peerReady) MBAR_TRY(comm_rendezvous(c));
    NvtxRange nvtx_("mbar_b200::sci_iterate");
    MBAR_TRY(enqueue_sci(c, p, inKernel, iters, nullptr, perLaunch ? ev.ev.data() : nullptr));
    c->lastLoopMs = timer.stop();
    double ksum = 0.0;
    for (int it = 0; perLaunch && it < iters; ++it) ksum += ev.ms(2 * it, 2 * it + 1);
    c->lastLoopKernelMs = ksum;
    c->lastLoopIters = iters;
    MBAR_CUDA(cudaGetLastError());
    double* fh = c->hf(ROW_F);
    MBAR_CUDA(cudaMemcpyAsync(fh, c->d_f, K * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    const PassLayout lay{K};
    MBAR_CUDA(cudaMemcpyAsync(c->h_out, c->d_out, (size_t)lay.size(false) * sizeof(double),
                              cudaMemcpyDeviceToHost, c->stream));
    MBAR_CUDA(cudaStreamSynchronize(c->stream));
    c->d2hBytes += K * 8 + lay.size(false) * 8;
    float ms = 0.f;
    if (event_ms(c->ev0, c->ev1, &ms)) c->lastPassMs = ms;   // (no pass has run on a fresh context with iters = 0)
    MBAR_REQUIRE(!(iters > 0 && c->h_out[lay.flag()] >= 1.0e6), MBAR_B200_ERR_COMM,
                 "peer exchange timed out inside the pass kernel (a rank did not arrive)");
    if (p.debugSkip) return MBAR_B200_OK;   // memory-pipeline probe: the arithmetic was skipped, nothing to return
    if (iters > 0 && c->h_out[lay.flag()] != 0.0) fh[c->firstActive] = NAN;  // force the robust redo
    bool finite = true;
    for (int k : c->active) finite = finite && std::isfinite(fh[k]);
    // some S_k underflowed in the linear-domain fused kernel: redo on the robust stepped path
    if (!finite) return sci_iterate_stepped(c, f, iters);
    for (int k = 0; k < K; ++k)
        if (c->h_Nk[k] > 0) f[k] = fh[k];
    return MBAR_B200_OK;
}

int mbar_b200_last_loop_ms(mbar_b200_ctx* c, double* total_ms, double* kernel_ms_sum, int32_t* iters) {
    MBAR_REQUIRE(c, MBAR_B200_ERR_INVALID, "ctx is NULL");
    if (total_ms) *total_ms = c->lastLoopMs;
    if (kernel_ms_sum) *kernel_ms_sum = c->lastLoopKernelMs;
    if (iters) *iters = c->lastLoopIters;
    return MBAR_B200_OK;
}

}  // extern "C"

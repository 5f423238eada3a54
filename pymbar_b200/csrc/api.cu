// C ABI: the streaming pass (run_pass, pass_multi), the reference primitives built on it, the communicator.
// The solver loops and their entry points are in loops.cu.
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cmath>
#include <cstring>

#include "internal.cuh"

using namespace mbar;

namespace mbar {

// ------------------------------------------------------------------------------------------
// NCCL, loaded lazily so that single-GPU use has no dependency on libnccl.
// ------------------------------------------------------------------------------------------
struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t,
                              cudaStream_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi g_nccl;

static int nccl_load() {
    if (g_nccl.handle) return MBAR_B200_OK;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    void* h = nullptr;
    for (const char* n : names) {
        h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (h) break;
    }
    MBAR_REQUIRE(h, MBAR_B200_ERR_COMM, "cannot dlopen libnccl.so.2: %s", dlerror());
#define SYM(field, name)                                                              \
    g_nccl.field = reinterpret_cast<decltype(g_nccl.field)>(dlsym(h, name));          \
    MBAR_REQUIRE(g_nccl.field, MBAR_B200_ERR_COMM, "libnccl lacks %s", name)
    SYM(GetUniqueId, "ncclGetUniqueId");
    SYM(CommInitRank, "ncclCommInitRank");
    SYM(CommDestroy, "ncclCommDestroy");
    SYM(AllReduce, "ncclAllReduce");
    SYM(GetErrorString, "ncclGetErrorString");
#undef SYM
    g_nccl.handle = h;
    return MBAR_B200_OK;
}

int comm_allreduce(mbar_b200_ctx* ctx, double* d_buf, int count, int op) {
    if (!ctx->comm || ctx->nranks == 1) return MBAR_B200_OK;
    ncclResult_t r = g_nccl.AllReduce(d_buf, d_buf, (size_t)count, ncclDouble,
                                      op == 2 ? ncclMax : ncclSum, (ncclComm_t)ctx->comm, ctx->stream);
    MBAR_REQUIRE(r == ncclSuccess, MBAR_B200_ERR_COMM, "ncclAllReduce: %s", g_nccl.GetErrorString(r));
    ctx->launches++;
    return MBAR_B200_OK;
}

// The lowest shifted energy of every row over all shards (max of its negation), so that every rank makes the same
// fused / log-domain choice for its all-state passes and issues the same collectives; likewise the clamp flags (any
// shard) and the far rows (every shard), so that every rank gives the same all-state answers.
int agree_row_minima(mbar_b200_ctx* c) {
    if (!c->comm || c->nranks == 1) return MBAR_B200_OK;
    const int K = c->K;
    std::vector<double> v(3 * (size_t)K);
    for (int k = 0; k < K; ++k) {
        v[k] = -c->h_urowmin[k];
        v[K + k] = c->h_uclamp[k];
        v[2 * K + k] = 1.0 - c->h_ufar[k];
    }
    MBAR_CUDA(cudaMemcpyAsync(c->d_scratch, v.data(), v.size() * sizeof(double), cudaMemcpyHostToDevice,
                              c->stream));
    MBAR_TRY(comm_allreduce(c, c->d_scratch, 3 * K, 2));
    MBAR_CUDA(cudaMemcpyAsync(v.data(), c->d_scratch, v.size() * sizeof(double), cudaMemcpyDeviceToHost,
                              c->stream));
    MBAR_CUDA(cudaStreamSynchronize(c->stream));
    for (int k = 0; k < K; ++k) {
        c->h_urowmin[k] = -v[k];
        c->h_uclamp[k] = v[K + k];
        c->h_ufar[k] = 1.0 - v[2 * K + k];
    }
    return MBAR_B200_OK;
}

// A row stores min(u - x, 1e6), and the passes weigh a stored 1e6 (+inf in the caller's array) e^(c - 1e6) rather than
// 0.  An unsampled row whose entries all lie at or above U_NEAR_CLAMP, some finite, is answered by those clamped values
// (f = 1e6 + const where the reference gives 2e6 for a copy u_0 + 2e6): refused.  Sampled rows are exempt: every
// sample has an entry 0 in some sampled row, so with |c| < 1e6 (check_range) such entries weigh nothing.
int check_unsampled_clamp(const mbar_b200_ctx* c) {
    for (int k = 0; k < c->K; ++k)
        MBAR_REQUIRE(c->h_Nk[k] > 0 || c->h_uclamp[k] == 0.0 || c->h_ufar[k] == 0.0, MBAR_B200_ERR_RANGE,
                     "unsampled state %d: every energy lies 999200 or more above its sample's lowest sampled-state "
                     "energy, some finite: beyond the stored range (1e6)", k);
    return MBAR_B200_OK;
}

// logS of unsampled states across ranks: logsumexp over ranks of the local log-sums.
__global__ void logs_to_scaled(double* logS, const double* mx, double* scaled, int K) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < K) scaled[k] = (logS[k] > -INFINITY && mx[k] < INFINITY) ? exp(logS[k] - mx[k]) : 0.0;
}
__global__ void scaled_to_logs(double* logS, const double* mx, const double* scaled, int K) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < K) logS[k] = (mx[k] > -INFINITY && mx[k] < INFINITY) ? mx[k] + log(scaled[k]) : mx[k];
}

}  // namespace mbar

// ------------------------------------------------------------------------------------------
// one streaming pass
// ------------------------------------------------------------------------------------------
namespace mbar {
int check_range(mbar_b200_ctx* c, const double* f) {
    for (int k : c->active) {
        const double ck = f[k] + c->h_logNk[k];
        MBAR_REQUIRE(std::isfinite(ck) && std::fabs(ck) < C_RANGE, MBAR_B200_ERR_RANGE,
                     "f_k[%d]=%g: f_k + log N_k must be finite and below 1e6 in magnitude", k, f[k]);
    }
    return MBAR_B200_OK;
}

// Runs the pass, all-reduces, downloads the packed result into ctx->h_out.
int run_pass(mbar_b200_ctx* c, const double* f, PassWant want) {
    MBAR_REQUIRE(c && f, MBAR_B200_ERR_INVALID, "NULL argument");
    MBAR_REQUIRE(c->ready, MBAR_B200_ERR_NOT_READY, "u_kn has not been uploaded");
    // a sharded problem needs a working reduction: peers attached without a communicator would silently
    // return shard-local sums from every host-stepped path
    MBAR_REQUIRE(c->nranks == 1 || c->comm, MBAR_B200_ERR_NOT_READY,
                 "sharded problem (%d ranks) without a communicator: call mbar_b200_comm_init", c->nranks);
    MBAR_CUDA(cudaSetDevice(c->device));
    MBAR_TRY(check_range(c, f));
    if (want.unsampled || want.Gall) MBAR_TRY(check_unsampled_clamp(c));
    NvtxRange nvtx_("mbar_b200::pass");
    const int K = c->K;
    const PassLayout lay{K};
    const bool needUnsampled = want.unsampled && (int)c->active.size() < K;
    const bool wantL = want.L || want.G || want.Gall;
    // attempt 0: fused (if applicable) | 1: generic, linear sums | 2: generic, log-domain sums for
    // every state (the reference's second logsumexp, mbar_solvers.py:240): taken when a sampled
    // state's S_k underflows, i.e. f_k is hundreds of kT away from self-consistency.
    bool fused = false, wroteW = false;
    for (int attempt = 0; attempt < 3; ++attempt) {
        fused = false;
        wroteW = false;
        const bool logAll = (attempt == 2);
        if (attempt == 0 && c->kernelChoice != MBAR_B200_KERNEL_GENERIC)
            MBAR_TRY(launch_pass_fused(c, f, wantL, needUnsampled, &fused, want.G && !want.Gall, &wroteW));
        if (attempt == 0 && !fused) continue;
        if (!fused) MBAR_TRY(launch_pass_generic(c, f, wantL, logAll));
        // S | sumL | flag are sums over samples -> one all-reduce
        MBAR_TRY(comm_allreduce(c, c->d_out, K + 2, 0));
        // log-domain partial sums (generic kernel only) are combined across ranks by max + rescaled sum;
        // the fused kernel's linear sums for unsampled states went through the all-reduce above
        if (((needUnsampled && !fused) || logAll) && c->comm && c->nranks > 1) {
            double* mx = c->d_scratch;
            double* sc = c->d_scratch + K;
            MBAR_CUDA(cudaMemcpyAsync(mx, c->d_out + lay.logS(), K * sizeof(double),
                                      cudaMemcpyDeviceToDevice, c->stream));
            MBAR_TRY(comm_allreduce(c, mx, K, 2));
            logs_to_scaled<<<(K + 255) / 256, 256, 0, c->stream>>>(c->d_out + lay.logS(), mx, sc, K);
            MBAR_TRY(comm_allreduce(c, sc, K, 0));
            scaled_to_logs<<<(K + 255) / 256, 256, 0, c->stream>>>(c->d_out + lay.logS(), mx, sc, K);
            c->launches += 2;
        }
        MBAR_CUDA(cudaMemcpyAsync(c->h_out, c->d_out, (size_t)lay.size(false) * sizeof(double),
                                  cudaMemcpyDeviceToHost, c->stream));
        MBAR_CUDA(cudaStreamSynchronize(c->stream));
        c->d2hBytes += (int64_t)lay.size(false) * 8;
        float ms = 0.f;
        if (event_ms(c->ev0, c->ev1, &ms)) c->lastPassMs = ms;
        if (fused && c->h_out[lay.flag()] != 0.0) continue;   // range assumption failed on a sample
        if (fused && needUnsampled) {
            // unsampled states rode along with weight e^-80: valid only while their weight sums are
            // moderate (their share of any denominator stays below 2^-53); otherwise log-domain kernel
            bool ok = true;
            for (int k = 0; k < K; ++k)
                if (!(c->h_Nk[k] > 0)) {
                    const double S = c->h_out[lay.S() + k];
                    if (!(S > 1e-250 && S < 1e12)) ok = false;
                    c->h_out[lay.logS() + k] = std::log(S);
                    c->h_out[lay.S() + k] = 0.0;           // contract: S = 0 for unsampled states
                }
            if (!ok) continue;
        }
        if (logAll) {
            for (int k : c->active) c->h_out[lay.S() + k] = std::exp(c->h_out[lay.logS() + k]);
            break;
        }
        bool underflow = false;
        for (int k : c->active) {
            const double S = c->h_out[lay.S() + k];
            if (!(S > 1e-280)) underflow = true;
            c->h_out[lay.logS() + k] = std::log(S);
        }
        if (!underflow) break;
        if (attempt == 0) ++attempt;   // skip the linear generic pass: it would underflow the same way
    }
    // an unsampled row of +inf only was weighed e^(c - 1e6) per entry; the reference's S is exactly 0 (f = +inf)
    if (needUnsampled)
        for (int k = 0; k < K; ++k)
            if (!(c->h_Nk[k] > 0) && c->h_ufar[k] != 0.0 && c->h_uclamp[k] == 0.0) c->h_out[lay.logS() + k] = -INFINITY;
    if (want.G || want.Gall) {
        NvtxRange nvtxH("mbar_b200::hessian");
        MBAR_TRY(launch_hessian(c, f, want.Gall, fused && wroteW));
        MBAR_TRY(comm_allreduce(c, c->d_out + lay.G(), K * K, 0));
        MBAR_CUDA(cudaMemcpyAsync(c->h_out + lay.G(), c->d_out + lay.G(), (size_t)K * K * sizeof(double),
                                  cudaMemcpyDeviceToHost, c->stream));
        MBAR_CUDA(cudaStreamSynchronize(c->stream));
        c->d2hBytes += (int64_t)K * K * 8;
    }
    return MBAR_B200_OK;
}

double global_sumx(mbar_b200_ctx* c, int* rc) {
    *rc = MBAR_B200_OK;
    const double mine = c->d_wgt ? c->sumXw : c->sumX;
    if (!c->comm || c->nranks == 1) return mine;
    double* d = c->d_scratch;
    cudaMemcpyAsync(d, &mine, sizeof(double), cudaMemcpyHostToDevice, c->stream);
    *rc = comm_allreduce(c, d, 1, 0);
    double v = 0.0;
    cudaMemcpyAsync(&v, d, sizeof(double), cudaMemcpyDeviceToHost, c->stream);
    cudaStreamSynchronize(c->stream);
    return v;
}

}  // namespace mbar

extern "C" {

int mbar_b200_pass(mbar_b200_ctx* c, const double* f, double* S, double* sumL, double* G) {
    PassWant w;
    w.G = (G != nullptr);
    MBAR_TRY(run_pass(c, f, w));
    const int K = c->K;
    const PassLayout lay{K};
    if (S) std::memcpy(S, c->h_out + lay.S(), K * sizeof(double));
    if (sumL) {
        int rc;
        const double sx = global_sumx(c, &rc);
        MBAR_TRY(rc);
        *sumL = c->h_out[lay.sumL()] - sx;
    }
    if (G) {
        const double* Gh = c->h_out + lay.G();
        for (int i = 0; i < K; ++i)
            for (int j = 0; j < K; ++j) {
                const double d = c->h_Nk[i] * c->h_Nk[j];
                G[(size_t)i * K + j] = d > 0 ? Gh[(size_t)i * K + j] / d : 0.0;
            }
    }
    return MBAR_B200_OK;
}

// M candidate f-vectors in one call (SURVEY.md 8b `mbar_pass(ctx, M, f[M][K], ...)`): the launches are
// enqueued back to back on the fused kernel and synchronised ONCE; anything the fused kernel cannot take
// falls back to the robust single-candidate path.
int mbar_b200_pass_multi(mbar_b200_ctx* c, int32_t M, const double* f, double* S, double* sumL) {
    MBAR_REQUIRE(c && f, MBAR_B200_ERR_INVALID, "NULL argument");
    MBAR_REQUIRE(M >= 1 && M <= 2, MBAR_B200_ERR_INVALID, "M=%d: 1 or 2 candidates", M);
    MBAR_REQUIRE(c->ready, MBAR_B200_ERR_NOT_READY, "u_kn has not been uploaded");
    MBAR_REQUIRE(c->nranks == 1 || c->comm, MBAR_B200_ERR_NOT_READY, "sharded problem without a communicator");
    MBAR_CUDA(cudaSetDevice(c->device));
    const int K = c->K;
    const PassLayout lay{K};
    NvtxRange nvtx_("mbar_b200::pass_multi");
    for (int m = 0; m < M; ++m) MBAR_TRY(check_range(c, f + (size_t)m * K));
    int rc0;
    const double sx = global_sumx(c, &rc0);
    MBAR_TRY(rc0);
    bool fast = c->kernelChoice != MBAR_B200_KERNEL_GENERIC;
    FusedParams p[2];
    bool batched = false;
    static const bool noM2 = std::getenv("MBAR_B200_NO_M2") != nullptr;
    if (fast && M == 2 && !noM2) {
        // one launch for both candidates (pass_fused_kernel<..., M = 2>): one read of u_kn, one exp per entry
        bool ok0 = false, ok1 = false;
        MBAR_TRY(fused_prepare(c, f, false, false, &p[0], &ok0, c->dc(ROW_C), c->hf(ROW_C), false, 2));
        if (ok0)
            MBAR_TRY(fused_prepare(c, f + K, false, false, &p[1], &ok1, c->dc(ROW_C2), c->hf(ROW_C2), false, 2));
        if (ok0 && ok1) {
            p[0].c2 = p[1].c;
            p[0].mid2 = p[1].mid;
            p[0].out = c->d_outM;
            p[0].out2 = c->d_outM + lay.size(false);
            batched = true;
        }
    }
    for (int m = 0; m < M && fast && !batched; ++m) {
        bool ok = false;
        // candidate m stages its constants in its own device row / pinned row (the copies are asynchronous)
        const int row = m == 0 ? ROW_C : ROW_C2;
        MBAR_TRY(fused_prepare(c, f + (size_t)m * K, false, false, &p[m], &ok, c->dc(row), c->hf(row)));
        p[m].out = c->d_outM + (size_t)m * lay.size(false);
        fast = ok;
    }
    if (fast) {
        if (batched) {
            MBAR_TRY(fused_enqueue(c, p[0]));
            MBAR_TRY(comm_allreduce(c, p[0].out, K + 2, 0));
            MBAR_TRY(comm_allreduce(c, p[0].out2, K + 2, 0));
        } else {
            for (int m = 0; m < M; ++m) {
                MBAR_TRY(fused_enqueue(c, p[m]));
                MBAR_TRY(comm_allreduce(c, p[m].out, K + 2, 0));
            }
        }
        MBAR_CUDA(cudaMemcpyAsync(c->h_out, c->d_outM, (size_t)M * lay.size(false) * sizeof(double),
                                  cudaMemcpyDeviceToHost, c->stream));
        MBAR_CUDA(cudaStreamSynchronize(c->stream));
        c->d2hBytes += (int64_t)M * lay.size(false) * 8;
        for (int m = 0; m < M && fast; ++m) {
            const double* o = c->h_out + (size_t)m * lay.size(false);
            if (o[lay.flag()] != 0.0) fast = false;
            for (int k : c->active)
                if (!(o[k] > 1e-280)) fast = false;
        }
        if (fast) {
            for (int m = 0; m < M; ++m) {
                const double* o = c->h_out + (size_t)m * lay.size(false);
                if (S)
                    for (int k = 0; k < K; ++k) S[(size_t)m * K + k] = c->h_Nk[k] > 0 ? o[k] : 0.0;
                if (sumL) sumL[m] = o[lay.sumL()] - sx;
            }
            return MBAR_B200_OK;
        }
    }
    for (int m = 0; m < M; ++m) {
        MBAR_TRY(run_pass(c, f + (size_t)m * K, PassWant{}));
        if (S) std::memcpy(S + (size_t)m * K, c->h_out + lay.S(), K * sizeof(double));
        if (sumL) sumL[m] = c->h_out[lay.sumL()] - sx;
    }
    return MBAR_B200_OK;
}

int mbar_b200_last_kernels(const mbar_b200_ctx* c, char* pass_kernel, char* hessian_kernel, int32_t len) {
    MBAR_REQUIRE(c && len > 0, MBAR_B200_ERR_INVALID, "bad argument");
    if (pass_kernel) snprintf(pass_kernel, (size_t)len, "%s", c->lastKernel);
    if (hessian_kernel) snprintf(hessian_kernel, (size_t)len, "%s", c->lastHessKernel);
    return MBAR_B200_OK;
}

int mbar_b200_last_hessian_ms(mbar_b200_ctx* c, double* weights_ms, double* hessian_ms) {
    MBAR_REQUIRE(c, MBAR_B200_ERR_INVALID, "ctx is NULL");
    MBAR_CUDA(cudaSetDevice(c->device));
    MBAR_CUDA(cudaStreamSynchronize(c->stream));
    float a = 0.f, b = 0.f;
    if (cudaEventElapsedTime(&a, c->evH[0], c->evH[1]) != cudaSuccess) { cudaGetLastError(); a = 0.f; }
    if (cudaEventElapsedTime(&b, c->evH[1], c->evH[2]) != cudaSuccess) { cudaGetLastError(); b = 0.f; }
    if (weights_ms) *weights_ms = a;
    if (hessian_ms) *hessian_ms = b;
    return MBAR_B200_OK;
}

int mbar_b200_self_consistent_update(mbar_b200_ctx* c, const double* f, double* f_out) {
    MBAR_REQUIRE(f_out, MBAR_B200_ERR_INVALID, "f_out is NULL");
    PassWant w;
    w.unsampled = true;
    MBAR_TRY(run_pass(c, f, w));
    const PassLayout lay{c->K};
    for (int k = 0; k < c->K; ++k) {
        f_out[k] = f[k] - c->h_out[lay.logS() + k];
    }
    return MBAR_B200_OK;
}

int mbar_b200_gradient(mbar_b200_ctx* c, const double* f, double* g_out) {
    MBAR_REQUIRE(g_out, MBAR_B200_ERR_INVALID, "g_out is NULL");
    MBAR_TRY(run_pass(c, f, PassWant{}));
    for (int k = 0; k < c->K; ++k) g_out[k] = c->h_Nk[k] * (c->h_out[k] - 1.0);
    return MBAR_B200_OK;
}

int mbar_b200_objective_and_gradient(mbar_b200_ctx* c, const double* f, double* obj, double* g_out) {
    MBAR_REQUIRE(obj, MBAR_B200_ERR_INVALID, "obj_out is NULL");
    MBAR_TRY(run_pass(c, f, PassWant{}));
    const PassLayout lay{c->K};
    int rc;
    const double sx = global_sumx(c, &rc);
    MBAR_TRY(rc);
    double nf = 0.0;
    for (int k = 0; k < c->K; ++k) nf += c->h_Nk[k] * f[k];
    *obj = (c->h_out[lay.sumL()] - sx) - nf;
    if (g_out)
        for (int k = 0; k < c->K; ++k) g_out[k] = c->h_Nk[k] * (c->h_out[k] - 1.0);
    return MBAR_B200_OK;
}

int mbar_b200_hessian(mbar_b200_ctx* c, const double* f, double* H) {
    MBAR_REQUIRE(H, MBAR_B200_ERR_INVALID, "H_out is NULL");
    PassWant w;
    w.G = true;
    MBAR_TRY(run_pass(c, f, w));
    const int K = c->K;
    const PassLayout lay{K};
    const double* Gh = c->h_out + lay.G();
    for (int i = 0; i < K; ++i)
        for (int j = 0; j < K; ++j) {
            double v = -Gh[(size_t)i * K + j];
            if (i == j) v += c->h_Nk[i] * c->h_out[lay.S() + i];
            H[(size_t)i * K + j] = (c->h_Nk[i] > 0 && c->h_Nk[j] > 0) ? v : 0.0;
        }
    return MBAR_B200_OK;
}

int mbar_b200_weight_moments(mbar_b200_ctx* c, const double* f, double* S, double* G) {
    MBAR_REQUIRE(G, MBAR_B200_ERR_INVALID, "G_out is NULL");
    PassWant w;
    w.unsampled = true;
    w.Gall = true;
    MBAR_TRY(run_pass(c, f, w));
    const int K = c->K;
    const PassLayout lay{K};
    const double* Gh = c->h_out + lay.G();
    for (int i = 0; i < K; ++i) {
        const double si = c->h_Nk[i] > 0 ? c->h_Nk[i] : 1.0;
        if (S) S[i] = c->h_Nk[i] > 0 ? c->h_out[lay.S() + i] : std::exp(c->h_out[lay.logS() + i]);
        for (int j = 0; j < K; ++j) {
            const double sj = c->h_Nk[j] > 0 ? c->h_Nk[j] : 1.0;
            G[(size_t)i * K + j] = Gh[(size_t)i * K + j] / (si * sj);
        }
    }
    return MBAR_B200_OK;
}

int mbar_b200_log_W_nk(mbar_b200_ctx* c, const double* f, double* logW, int64_t ld, int expo) {
    MBAR_REQUIRE(logW, MBAR_B200_ERR_INVALID, "logW_host is NULL");
    MBAR_REQUIRE(c && ld >= c->K, MBAR_B200_ERR_INVALID, "ld_out < K");
    PassWant w;
    w.L = true;
    MBAR_TRY(run_pass(c, f, w));
    return launch_logw(c, f, logW, ld, expo, 0, c->N);
}

int mbar_b200_log_W_nk_rows(mbar_b200_ctx* c, const double* f, int64_t n0, int64_t n, double* logW, int64_t ld,
                            int expo) {
    MBAR_REQUIRE(logW, MBAR_B200_ERR_INVALID, "logW_host is NULL");
    MBAR_REQUIRE(c && ld >= c->K, MBAR_B200_ERR_INVALID, "ld_out < K");
    MBAR_REQUIRE(n0 >= 0 && n >= 1 && n0 + n <= c->N && n0 % TILE_N == 0, MBAR_B200_ERR_INVALID,
                 "rows [%lld, +%lld): n0 must be a multiple of 32 inside [0, N_local)", (long long)n0, (long long)n);
    PassWant w;
    w.L = true;
    MBAR_TRY(run_pass(c, f, w));
    return launch_logw(c, f, logW, ld, expo, n0, n);
}

int mbar_b200_log_denominator(mbar_b200_ctx* c, const double* f, double* L_host) {
    MBAR_REQUIRE(L_host, MBAR_B200_ERR_INVALID, "L_host is NULL");
    PassWant w;
    w.L = true;
    MBAR_TRY(run_pass(c, f, w));
    // L_n = L'_n - x_n
    std::vector<double> x((size_t)c->N);
    MBAR_CUDA(cudaMemcpyAsync(L_host, c->d_L, (size_t)c->N * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    MBAR_CUDA(cudaMemcpyAsync(x.data(), c->d_xshift, (size_t)c->N * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    MBAR_CUDA(cudaStreamSynchronize(c->stream));
    c->d2hBytes += 2 * c->N * 8;
    for (int64_t n = 0; n < c->N; ++n) L_host[n] -= x[n];
    return MBAR_B200_OK;
}

int mbar_b200_self_consistent_update_host(int device, int32_t K, int64_t N, const double* u_host, int64_t ld,
                                          const double* N_k, const double* f_k, double* f_out) {
    mbar_b200_ctx* c = nullptr;
    MBAR_TRY(mbar_b200_create(&c, device, K, N, N_k));
    int rc = mbar_b200_upload_u_kn(c, u_host, ld);
    if (rc == MBAR_B200_OK) rc = mbar_b200_self_consistent_update(c, f_k, f_out);
    mbar_b200_destroy(c);
    return rc;
}

// ------------------------------------------------------------------------------------------
// communicator
// ------------------------------------------------------------------------------------------
int mbar_b200_comm_unique_id(void* id_out) {
    MBAR_REQUIRE(id_out, MBAR_B200_ERR_INVALID, "id_out is NULL");
    MBAR_TRY(nccl_load());
    static_assert(sizeof(ncclUniqueId) <= MBAR_B200_UNIQUE_ID_BYTES, "unique id size");
    ncclUniqueId id;
    ncclResult_t r = g_nccl.GetUniqueId(&id);
    MBAR_REQUIRE(r == ncclSuccess, MBAR_B200_ERR_COMM, "ncclGetUniqueId: %s", g_nccl.GetErrorString(r));
    std::memset(id_out, 0, MBAR_B200_UNIQUE_ID_BYTES);
    std::memcpy(id_out, &id, sizeof(id));
    return MBAR_B200_OK;
}

int mbar_b200_comm_init(mbar_b200_ctx* c, int32_t nranks, int32_t rank, const void* unique_id) {
    MBAR_REQUIRE(c && unique_id, MBAR_B200_ERR_INVALID, "NULL argument");
    MBAR_REQUIRE(nranks >= 1 && rank >= 0 && rank < nranks, MBAR_B200_ERR_INVALID, "rank %d of %d", rank, nranks);
    MBAR_TRY(nccl_load());
    MBAR_CUDA(cudaSetDevice(c->device));
    ncclUniqueId id;
    std::memcpy(&id, unique_id, sizeof(id));
    ncclComm_t comm;
    ncclResult_t r = g_nccl.CommInitRank(&comm, nranks, id, rank);
    MBAR_REQUIRE(r == ncclSuccess, MBAR_B200_ERR_COMM, "ncclCommInitRank: %s", g_nccl.GetErrorString(r));
    c->comm = comm;
    c->nranks = nranks;
    c->rank = rank;
    // kernel-selection inputs must be identical on every rank (all ranks issue the same collectives)
    return agree_row_minima(c);
}

static size_t inbox_doubles(int K) { return (size_t)2 * MAX_PEERS * 2 * (K + 2); }   // (2 candidates per launch)

int mbar_b200_peer_export(mbar_b200_ctx* c, void* handle_out) {
    MBAR_REQUIRE(c && handle_out, MBAR_B200_ERR_INVALID, "NULL argument");
    MBAR_CUDA(cudaSetDevice(c->device));
    if (!c->d_inbox) {
        // the inbox, then the [2][MAX_PEERS] flags (8 bytes each, like a double)
        const size_t count = inbox_doubles(c->K) + 2 * MAX_PEERS;
        MBAR_TRY(c->d_inbox.reserve(count, "peer_export"));
        MBAR_CUDA(cudaMemset(c->d_inbox, 0, count * sizeof(double)));
    }
    cudaIpcMemHandle_t h;
    MBAR_CUDA(cudaIpcGetMemHandle(&h, c->d_inbox));
    static_assert(sizeof(h) == MBAR_B200_IPC_HANDLE_BYTES, "ipc handle size");
    std::memcpy(handle_out, &h, sizeof(h));
    return MBAR_B200_OK;
}

int mbar_b200_peer_attach(mbar_b200_ctx* c, int32_t nranks, int32_t rank, const void* handles) {
    MBAR_REQUIRE(c && handles, MBAR_B200_ERR_INVALID, "NULL argument");
    MBAR_REQUIRE(nranks >= 1 && nranks <= MAX_PEERS && rank >= 0 && rank < nranks, MBAR_B200_ERR_INVALID,
                 "rank %d of %d (at most %d peers)", rank, nranks, MAX_PEERS);
    MBAR_REQUIRE(c->d_inbox, MBAR_B200_ERR_NOT_READY, "call mbar_b200_peer_export first");
    // The peer inbox only carries the exchange of the device-resident loops; every host-stepped path (and the
    // K x K Hessian) reduces through the communicator, so a sharded problem without one would return
    // shard-local sums.  Require it instead of guessing.
    MBAR_REQUIRE(nranks == 1 || (c->comm && c->nranks == nranks && c->rank == rank), MBAR_B200_ERR_NOT_READY,
                 "mbar_b200_peer_attach needs mbar_b200_comm_init(nranks=%d, rank=%d) first", nranks, rank);
    MBAR_CUDA(cudaSetDevice(c->device));
    c->peer = PeerCfg{};
    c->peer.nranks = nranks;
    c->peer.rank = rank;
    for (int q = 0; q < nranks; ++q) {
        void* ptr = c->d_inbox;
        if (q != rank) {
            cudaIpcMemHandle_t h;
            std::memcpy(&h, static_cast<const char*>(handles) + (size_t)q * sizeof(h), sizeof(h));
            MBAR_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
            c->peerMapped.push_back(ptr);
        }
        c->peer.inbox[q] = static_cast<double*>(ptr);
        c->peer.flags[q] = reinterpret_cast<unsigned long long*>(static_cast<double*>(ptr) + inbox_doubles(c->K));
    }
    c->peer.seq = c->d_seq;
    MBAR_CUDA(cudaMemset(c->d_seq, 0, sizeof(unsigned long long)));
    c->peerReady = nranks > 1;
    return MBAR_B200_OK;
}

int mbar_b200_comm_destroy(mbar_b200_ctx* c) {
    if (c && c->comm) {
        g_nccl.CommDestroy((ncclComm_t)c->comm);
        c->comm = nullptr;
        c->nranks = 1;
        c->rank = 0;
    }
    return MBAR_B200_OK;
}

}  // extern "C"

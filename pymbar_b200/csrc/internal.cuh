// Shared internals of libmbar_b200.so (not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdarg>
#include <cstdio>
#include <functional>
#include <vector>

#include "../../include/mbar_b200.h"
#include "exp_tables.h"

namespace mbar {

constexpr int TILE_N = 32;              // samples per tile (one warp lane each)
constexpr double U_CLAMP = 1.0e6;       // shifted energies are clamped to [.., 1e6] at upload
// +inf and everything past 1e6 are stored as U_CLAMP and weighed e^(c - 1e6) by the passes.  In a row with an entry
// below U_NEAR_CLAMP such entries are negligible next to it (e^-800 each), as in the reference; a row with none has
// only clamped or near-clamp entries, which decide its answer (h_ufar, h_uclamp).
constexpr double U_NEAR_CLAMP = U_CLAMP - 800.0;
constexpr double C_RANGE = 1.0e6;       // |f_k + log N_k| must stay below this
constexpr double FUSED_SPREAD = 1200.0; // fused kernel needs max(c) - min(c) below this
constexpr int MAX_GRID = 132 * 4;
// Unsampled states ride through the fused kernel as "sampled with weight e^-80": their share of any
// denominator is below 2^-53 as long as their sum of weights stays below 1e12 (checked by the host).
constexpr double LOG_EPS_UNSAMPLED = -80.0;
// The device exp (exp_split + scale2) is accurate for arguments in [-707.7, 709.7].  Below, the result is floored
// into [0, 2^-1020] instead of underflowing; above ~709.78 the binary exponent wraps, so the host never lets an
// argument above FUSED_MAX_ARG reach the fused pass (unsampled rows below the sampled minimum: fused_applicable).
// Sampled rows have u' >= 0 and spread(c) < 1200, so their arguments stay below 600.
constexpr double FUSED_MAX_ARG = 700.0;
// A floored entry enters S_k's raw sum sum_n e_kn / D_n divided by D_n >= e^(c_min - mid), c_min over the SAMPLED
// states (every sample has one with u' = 0): the fused pass treats a raw sum below 2^53 * N * 2^-1020 * e^(mid - c_min)
// as underflowed (S_k = NaN) and the host redoes the pass in the log domain.  log(2^53 * 2^-1020) = -967 ln 2:
constexpr double LOG_FLOOR_S = -670.273323601467;

void set_error(const char* fmt, ...);
#define MBAR_CUDA(call)                                                                     \
    do {                                                                                    \
        cudaError_t e__ = (call);                                                           \
        if (e__ != cudaSuccess) {                                                           \
            mbar::set_error("%s failed at %s:%d: %s", #call, __FILE__, __LINE__,            \
                            cudaGetErrorString(e__));                                       \
            return MBAR_B200_ERR_CUDA;                                                      \
        }                                                                                   \
    } while (0)
#define MBAR_REQUIRE(cond, status, ...)                                                     \
    do {                                                                                    \
        if (!(cond)) {                                                                      \
            mbar::set_error(__VA_ARGS__);                                                   \
            return (status);                                                                \
        }                                                                                   \
    } while (0)
#define MBAR_TRY(call)                                                                      \
    do {                                                                                    \
        int s__ = (call);                                                                   \
        if (s__ != MBAR_B200_OK) return s__;                                                \
    } while (0)

// Packed per-pass output on device / pinned host:  [0..K) S_k, [K] sumL, [K+1] flag (as double),
// [K+2 .. K+2+K) log-domain S for unsampled states (generic kernel), then K*K G when requested.
struct PassLayout {
    int K;
    __host__ __device__ int S() const { return 0; }
    __host__ __device__ int sumL() const { return K; }
    __host__ __device__ int flag() const { return K + 1; }
    __host__ __device__ int logS() const { return K + 2; }
    __host__ __device__ int G() const { return 2 * K + 2; }
    __host__ __device__ int size(bool withG) const { return 2 * K + 2 + (withG ? K * K : 0); }
};

// Peer-memory exchange of the per-pass partial sums (fused into the pass kernel's last CTA).
constexpr int MAX_PEERS = 16;
struct PeerCfg {
    int nranks = 1, rank = 0;
    double* inbox[MAX_PEERS] = {nullptr};               // inbox[q]: rank q's [2][nranks][K+2] buffer, mapped here
    unsigned long long* flags[MAX_PEERS] = {nullptr};   // flags[q]: rank q's [2][nranks] sequence numbers
    // Exchange sequence number, kept on the DEVICE and advanced by the last CTA of every launch that
    // actually runs: launches that exit early (solver already converged) must not consume a number, or two
    // executed launches could reuse an inbox parity without an exchange in between.
    unsigned long long* seq = nullptr;
};

// State of a device-resident solver loop (device memory + pinned host mirror).  Every kernel of an iteration
// starts with `if (loop->done) return;`, so the host can enqueue a batch of iterations without knowing when
// the solver converges and polls this struct once per batch: no per-iteration host round trip.
struct LoopState {
    int done;            // 1: stop (converged, failed or maxiter reached)
    int status;          // 0 ok | 1 range/underflow problem: redo on the robust host-stepped path | 2 comm
    int success;         // convergence criterion met (mbar_solvers.py:627-640)
    int iterations, nr_iterations, sci_iterations;
    int maxiter, min_sc_iter;
    int haveNr;          // this iteration has a valid Newton candidate
    int cholFail;        // last Cholesky attempt met a non-positive pivot
    // per solve, for mbar_b200_get_adaptive_stats: factorisations retried with the ridge, iterations whose retry
    // failed too, Newton candidates rejected as non-finite or out of range
    int ridgeRetries, nrFailed, nrRejected, pad_;
    double tol, gamma;
    double max_delta, max_diff, gnorm;
    double gn_sci, gn_nr;
};

// Rows of the staging buffers d_c ([DC_ROWS][K]) and h_f ([HF_ROWS][K], pinned; its row r stages d_c's row r, and is not
// rewritten while a copy out of it is in flight): c of the fused or generic pass, f of the generic pass, c of the Hessian,
// f of log W, c of a second candidate; pinned only: f to and from d_f, f of each LoopState poll.
enum { ROW_C, ROW_GEN_F, ROW_HESS_C, ROW_LOGW_F, ROW_C2, DC_ROWS, ROW_F = DC_ROWS, ROW_POLL, HF_ROWS };

// Elapsed ms between two events.  False when either was never recorded (e.g. no pass has run yet); the runtime's
// error is then cleared, or the next MBAR_CUDA(cudaGetLastError()) of an unrelated call would report it.
inline bool event_ms(cudaEvent_t a, cudaEvent_t b, float* ms) {
    if (cudaEventElapsedTime(ms, a, b) == cudaSuccess) return true;
    cudaGetLastError();
    return false;
}

// ---- host scaffold of the device objects (mbar_b200_ctx, _batch, _kde, _bspline, _acf, _work) ----
// Every device buffer, pinned buffer, event and stream of the library has an owner defined here; outside this file only
// the buffer pool of ctx.cu calls the runtime's allocator.

// Checks that `device` is visible and is an sm_90 part, makes it current and fills *prop unless it is NULL (ctx.cu).
int open_device(int device, cudaDeviceProp* prop);

// Prefer the GPU's NUMA node for host allocations made while this object lives (ctx.cu).
int gpu_numa_node(int device);
struct NumaPrefer {
    bool active = false;
    explicit NumaPrefer(int device);
    ~NumaPrefer();
};

// cudaMalloc of max(count, 1) elements.  On failure *p is NULL, the runtime's error is cleared and the status is
// ERR_NOMEM when the device is out of memory, ERR_CUDA otherwise.
template <class T>
int dev_alloc(T** p, size_t count, const char* who) {
    const cudaError_t e = cudaMalloc((void**)p, (count > 0 ? count : 1) * sizeof(T));
    if (e == cudaSuccess) return MBAR_B200_OK;
    *p = nullptr;
    cudaGetLastError();
    set_error("%s: cannot allocate %zu bytes", who, count * sizeof(T));
    return e == cudaErrorMemoryAllocation ? MBAR_B200_ERR_NOMEM : MBAR_B200_ERR_CUDA;
}

// The same for pinned host memory.  numaDevice >= 0: the pages come from that GPU's NUMA node (NumaPrefer), which
// keeps the large staging buffers of uploads and downloads off the inter-socket link.
template <class T>
int host_alloc(T** p, size_t count, const char* who, int numaDevice = -1) {
    const size_t bytes = (count > 0 ? count : 1) * sizeof(T);
    cudaError_t e;
    if (numaDevice >= 0) {
        NumaPrefer numa(numaDevice);
        e = cudaHostAlloc((void**)p, bytes, cudaHostAllocDefault);
    } else {
        e = cudaHostAlloc((void**)p, bytes, cudaHostAllocDefault);
    }
    if (e == cudaSuccess) return MBAR_B200_OK;
    *p = nullptr;
    cudaGetLastError();
    set_error("%s: cannot allocate %zu bytes of pinned host memory", who, count * sizeof(T));
    return e == cudaErrorMemoryAllocation ? MBAR_B200_ERR_NOMEM : MBAR_B200_ERR_CUDA;
}

// Releases what dev_alloc (pinned = false) or host_alloc (pinned = true) returned; NULL is a no-op.
inline cudaError_t mem_free(void* p, bool pinned) {
    if (!p) return cudaSuccess;
    return pinned ? cudaFreeHost(p) : cudaFree(p);
}

// Device buffers of one call, freed on every return path.
struct CallBuffers {
    const char* who;
    std::vector<void*> ptrs;
    explicit CallBuffers(const char* who_) : who(who_) {}
    CallBuffers(const CallBuffers&) = delete;
    CallBuffers& operator=(const CallBuffers&) = delete;
    ~CallBuffers() {
        for (void* p : ptrs) mem_free(p, false);
    }
    template <class T>
    int alloc(T** p, size_t count) {
        MBAR_TRY(dev_alloc(p, count, who));
        ptrs.push_back((void*)*p);
        return MBAR_B200_OK;
    }
};

// An array owned by an object or a call and freed with it: device memory (DevArray) or pinned host memory
// (HostPinned).  reserve(n) keeps the buffer when it already holds n elements; otherwise it drops the contents and
// allocates n, and a failure leaves the array empty with capacity 0.  grow(n) reserves with room to spare
// (n + n/2 + 64) for per-call buffers whose next call may be somewhat larger.  numaDevice: see host_alloc.
template <class T, bool Pinned>
struct OwnedArray {
    T* ptr = nullptr;
    size_t cap = 0;
    OwnedArray() = default;
    OwnedArray(OwnedArray&& o) noexcept : ptr(o.ptr), cap(o.cap) {
        o.ptr = nullptr;
        o.cap = 0;
    }
    OwnedArray& operator=(OwnedArray&& o) noexcept {
        std::swap(ptr, o.ptr);
        std::swap(cap, o.cap);
        return *this;
    }
    ~OwnedArray() { reset(); }
    void reset() {
        mem_free(ptr, Pinned);
        ptr = nullptr;
        cap = 0;
    }
    int reserve(size_t n, const char* who, int numaDevice = -1) {
        if (ptr && n <= cap) return MBAR_B200_OK;
        reset();
        MBAR_TRY(Pinned ? host_alloc(&ptr, n, who, numaDevice) : dev_alloc(&ptr, n, who));
        cap = n;
        return MBAR_B200_OK;
    }
    int grow(size_t n, const char* who) { return n <= cap ? MBAR_B200_OK : reserve(n + n / 2 + 64, who); }
    operator T*() const { return ptr; }
};
template <class T>
using DevArray = OwnedArray<T, false>;
template <class T>
using HostPinned = OwnedArray<T, true>;

// The per-device pool of the context's largest buffers (ctx.cu), one slot per kind and device.  pool_take hands out
// the parked buffer when it holds [bytes, 2 bytes + 1 MiB] (a small problem never pins a huge buffer) and sets *got to
// its size, else NULL; pool_park parks a buffer and returns the one parked there before, for the caller to release.
enum { POOL_U, POOL_STAGE_DEV, POOL_STAGE_PIN = POOL_STAGE_DEV + 2, POOL_KINDS = POOL_STAGE_PIN + 2 };
bool pool_enabled();   // false under MBAR_B200_NO_POOL
void* pool_take(int device, int kind, size_t bytes, size_t* got);
void* pool_park(int device, int kind, void* ptr, size_t bytes);

// An array of a context that comes from the pool when a parked buffer fits, and goes back to it at the size it really
// has when the context is destroyed (released instead when the pool is off).
template <class T, bool Pinned>
struct PooledArray {
    OwnedArray<T, Pinned> a;
    int device = 0, kind = 0;
    PooledArray() = default;
    PooledArray(const PooledArray&) = delete;
    PooledArray& operator=(const PooledArray&) = delete;
    ~PooledArray() {
        if (a.ptr && pool_enabled()) {
            mem_free(pool_park(device, kind, a.ptr, a.cap * sizeof(T)), Pinned);
            a.ptr = nullptr;
        }
    }
    // at least n elements, allocated once (pinned: on the GPU's NUMA node)
    int acquire(int dev, int k, size_t n, const char* who) {
        if (a.ptr) return MBAR_B200_OK;
        device = dev;
        kind = k;
        size_t got = 0;
        if (pool_enabled() && (a.ptr = static_cast<T*>(pool_take(dev, k, n * sizeof(T), &got)))) {
            a.cap = got / sizeof(T);
            return MBAR_B200_OK;
        }
        return a.reserve(n, who, Pinned ? dev : -1);
    }
    operator T*() const { return a.ptr; }
};

// CUDA events, destroyed with the object on every return path.  As the timer of a solve: start() creates two and
// records the first on the stream, stop() records the second, waits for it and returns the elapsed ms.
struct Events {
    std::vector<cudaEvent_t> ev;
    cudaStream_t s = nullptr;
    Events() = default;
    Events(const Events&) = delete;
    Events& operator=(const Events&) = delete;
    ~Events() {
        for (cudaEvent_t e : ev) cudaEventDestroy(e);
    }
    // flags: cudaEventDisableTiming for events that only order work
    int create(size_t n, unsigned flags = cudaEventDefault) {
        for (size_t i = 0; i < n; ++i) {
            cudaEvent_t e;
            MBAR_CUDA(cudaEventCreateWithFlags(&e, flags));
            ev.push_back(e);
        }
        return MBAR_B200_OK;
    }
    cudaEvent_t operator[](size_t i) const { return ev[i]; }
    float ms(size_t a, size_t b) const {
        float m = 0.f;
        event_ms(ev[a], ev[b], &m);
        return m;
    }
    int start(cudaStream_t stream) {
        s = stream;
        MBAR_TRY(create(2));
        MBAR_CUDA(cudaEventRecord(ev[0], s));
        return MBAR_B200_OK;
    }
    float stop() {
        cudaEventRecord(ev[1], s);
        cudaEventSynchronize(ev[1]);
        return ms(0, 1);
    }
};

// A non-blocking stream (work on the legacy stream does not serialise with it), destroyed with its owner.
struct Stream {
    cudaStream_t s = nullptr;
    Stream() = default;
    Stream(const Stream&) = delete;
    Stream& operator=(const Stream&) = delete;
    ~Stream() {
        if (s) cudaStreamDestroy(s);
    }
    int create(const char* who) {
        if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess) return MBAR_B200_OK;
        s = nullptr;
        set_error("%s: %s", who, cudaGetErrorString(cudaGetLastError()));
        return MBAR_B200_ERR_CUDA;
    }
    operator cudaStream_t() const { return s; }
};

// Device, stream and timing events of a resident device object.  The u_kn context and mbar_b200_batch, _kde,
// _bspline, _acf and _work derive from it and hold their memory in the owners above; each create holds its object in a
// std::unique_ptr until it succeeds, and each destroy waits for the stream before the delete (destroy_resident).
struct Resident {
    int device = 0;
    Stream stream;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr; // the timed window of the last call
    double lastMs = 0.0;

    Resident() = default;
    Resident(const Resident&) = delete;
    Resident& operator=(const Resident&) = delete;
    ~Resident() {
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
    }
    // the stream and the events, on `dev` (made current by open_device)
    int open(int dev, const char* who) {
        device = dev;
        MBAR_TRY(stream.create(who));
        if (cudaEventCreate(&ev0) != cudaSuccess || cudaEventCreate(&ev1) != cudaSuccess) {
            set_error("%s: %s", who, cudaGetErrorString(cudaGetLastError()));
            return MBAR_B200_ERR_CUDA;
        }
        return MBAR_B200_OK;
    }
    // count elements of src into dst (allocated to fit).  The copy goes on the object's own stream and is waited for:
    // a pageable cudaMemcpy on the legacy stream may return before its DMA lands, and the kernels' stream would not
    // wait for it.
    template <class T>
    int upload(DevArray<T>& dst, const T* src, size_t count, const char* who) {
        MBAR_TRY(dst.reserve(count, who));
        if (cudaMemcpyAsync(dst, src, count * sizeof(T), cudaMemcpyHostToDevice, stream) != cudaSuccess ||
            cudaStreamSynchronize(stream) != cudaSuccess) {
            set_error("%s: %s", who, cudaGetErrorString(cudaGetLastError()));
            return MBAR_B200_ERR_CUDA;
        }
        return MBAR_B200_OK;
    }
};

// Deletes a resident object once its stream has drained.  C++ destroys the derived object's arrays before ~Resident
// runs, so the wait has to come before the delete.
template <class T>
int destroy_resident(T* o) {
    if (!o) return MBAR_B200_OK;
    cudaSetDevice(o->device);
    if (o->stream) cudaStreamSynchronize(o->stream);
    delete o;
    return MBAR_B200_OK;
}

}  // namespace mbar

struct mbar_b200_ctx : mbar::Resident {
    int K = 0;
    int64_t N = 0;        // local samples
    int64_t nTiles = 0;   // ceil(N / 32)
    bool ready = false;   // u uploaded
    int kernelChoice = MBAR_B200_KERNEL_AUTO;
    int smCount = 132;

    std::vector<double> h_Nk;       // [K]
    std::vector<double> h_logNk;    // [K], -inf for unsampled
    std::vector<double> h_logNkEff; // [K], LOG_EPS_UNSAMPLED for unsampled
    mbar::DevArray<double> d_NkEff; // [K], exp(LOG_EPS_UNSAMPLED) for unsampled
    // [K] min over samples of each row's shifted energy u'_kn, rounded down, 0 when none is negative (only
    // unsampled rows can be): bounds the exp argument an unsampled row presents to the fused pass
    std::vector<double> h_urowmin;
    // [K] 1 where some sample's FINITE shifted energy reached U_NEAR_CLAMP (on any shard)
    std::vector<double> h_uclamp;
    // [K] 1 where every shifted energy of the row is at or above U_NEAR_CLAMP, +inf included (on every shard).  An
    // unsampled row with both flags cannot be answered (ERR_RANGE, check_unsampled_clamp); with this one alone it is
    // all +inf: S = 0, f = +inf
    std::vector<double> h_ufar;
    mbar::DevArray<int> d_urowmin;  // [2K] the row minima, then the clamp flags, accumulated during upload / append
    mbar::DevArray<unsigned long long> d_urowfar;  // [K] entries per row at or above U_NEAR_CLAMP (+inf included)
    std::vector<int> active;        // indices of sampled states
    int firstActive = 0;
    double N_total_states = 0;      // sum_k N_k (global N)

    mbar::PooledArray<double, false> d_u;  // [nTiles][K][32] shifted, clamped
    mbar::DevArray<double> d_xshift;  // [nTiles*32] per-sample shift x_n = min over sampled k of u_kn
    mbar::DevArray<double> d_wgt;     // [nTiles*32] per-sample multiplicities w_n (bootstrap), or NULL = all 1
    mbar::DevArray<double> d_sqrtw;   // [nTiles*32] sqrt(w_n) for the second-moment kernel (with d_wgt or neither)
    double sumW = 0.0;              // sum_n w_n over valid local samples (= N when unweighted)
    double sumXw = 0.0;             // sum_n w_n x_n
    double sumX = 0.0;              // sum_n x_n over valid local samples
    mbar::DevArray<double> d_c;     // [DC_ROWS][K] pass constants, rows ROW_*
    mbar::DevArray<double> d_Nk;    // [K]
    mbar::DevArray<unsigned long long> d_rowmask;   // [ceil(K/64)] bit per sampled state
    mbar::DevArray<unsigned long long> d_zeromask;  // same size, all zero (log-domain for every row)
    mbar::DevArray<unsigned long long> d_onesmask;  // same size, all one (second moments of every state)
    mbar::DevArray<double> d_partial;  // [MAX_GRID][K+2] per-CTA partials
    mbar::DevArray<double> d_out;   // PassLayout packed result (with G)
    mbar::HostPinned<double> h_out; // pinned mirror of d_out
    mbar::DevArray<double> d_L;     // [nTiles*32] per-sample L_n (lazy, ensure_L)
    mbar::DevArray<double> d_W;     // per-CTA partial blocks of the Hessian kernels (grown on demand)
    mbar::DevArray<unsigned int> d_ticket;
    mbar::DevArray<int> d_flag;     // [4] error/diagnostic flags
    mbar::DevArray<double> d_f;     // [K] device-resident f of the native loops
    mbar::HostPinned<double> h_f;   // pinned [HF_ROWS][K] staging, rows ROW_*
    mbar::DevArray<double> d_scratch;  // misc scratch (see scratch_rendezvous)
    // upload staging: copies on copyStream, evCopy[buf] marks the re-tile that last read stage_dev[buf]
    mbar::Stream copyStream;
    mbar::Events evCopy;
    mbar::PooledArray<double, true> stage_pinned[2];
    mbar::PooledArray<double, false> stage_dev[2];
    int64_t stageCols = 0;

    // peer-memory exchange (cudaIpc): this rank's inbox + flags and the peers' mappings
    mbar::DevArray<double> d_inbox;
    mbar::PeerCfg peer;
    bool peerReady = false;
    std::vector<void*> peerMapped;

    // communicator (NCCL, dlopen'd)
    void* comm = nullptr;
    int nranks = 1, rank = 0;

    // device-resident solver loops
    mbar::DevArray<mbar::LoopState> d_loop;    // device
    mbar::HostPinned<mbar::LoopState> h_loop;  // pinned mirror
    mbar::DevArray<double> d_av;         // [8][K] adaptive work vectors, rows AV_* (loops.cu)
    mbar::DevArray<double> d_outM;       // [2][2K+2] pass outputs of the two candidates
    mbar::DevArray<double> d_A;          // [K*K] Newton matrix / Cholesky factor
    mbar::DevArray<int> d_active;        // [K] indices of the sampled states
    mbar::DevArray<unsigned long long> d_seq;  // peer-exchange sequence number (device-side, see PeerCfg::seq)
    int loopMode = 0;                    // 0 device-resident, 1 host-stepped (round-1 behaviour)
    int loopBatch = 4;                   // iterations enqueued between two polls of LoopState
    int64_t loopPolls = 0;               // host synchronisations spent polling LoopState
    mbar_b200_adaptive_stats lastAdaptive{};   // how the last mbar_b200_solve_adaptive ran (loops.cu)
    // the adaptive iteration as a CUDA graph (captured once, relaunched per iteration; see loops.cu)
    bool capturing = false;              // stream capture in progress: no timing events, no allocations
    bool graphWarm = false;              // one uncaptured iteration has sized every buffer / kernel attribute
    cudaGraphExec_t loopGraph = nullptr;
    std::vector<uint64_t> loopGraphKey;
    int64_t graphLaunches = 0, graphCaptures = 0;
    mbar::DevArray<double> d_Wt;         // [nTiles][K][32] materialised N_k W_nk (swizzled) for the Hessian
    bool wtAllocFailed = false;
    char lastKernel[200] = "";           // description of the pass-kernel variant launched last
    char lastHessKernel[200] = "";       // ... and of the Hessian kernel path
    double lastHessMs = 0.0, lastWeightsMs = 0.0;
    double lastBinMs = 0.0;              // mbar_b200_bin_moments: kernels after the pass (CUDA events)
    int lastBinChunks = 0;               // ... and the reads of u_kn its moments step took
    double lastRepMs = 0.0;              // mbar_b200_replicate_unsampled: its kernels (CUDA events),
    int lastRepBatches = 0;              // ... its replicate batches
    int64_t lastRepExps = 0;             // ... and the exps it evaluated
    mbar::Events evH;                    // [3] bounds of the Hessian's weights and kernel windows

    // counters
    int64_t launches = 0, passes = 0, h2dBytes = 0, d2hBytes = 0;
    double lastPassMs = 0.0;
    double lastLoopMs = 0.0, lastLoopKernelMs = 0.0;
    int lastLoopIters = 0;
    bool timePasses = true;

    double* dc(int row) const { return d_c + (size_t)row * K; }
    double* hf(int row) const { return h_f + (size_t)row * K; }
};

namespace mbar {

// Waits for the context's streams when it goes out of scope.  Declared after the call-scoped staging (buffers, events)
// it protects, it runs before their destructors on every return path: staging is never freed under an in-flight copy.
struct StreamDrain {
    const mbar_b200_ctx* c;
    ~StreamDrain() {
        cudaStreamSynchronize(c->copyStream);
        cudaStreamSynchronize(c->stream);
    }
};

// The per-sample L'_n of the passes, allocated by the first pass that keeps it (never under stream capture: the
// uncaptured warm-up iteration comes first)
inline int ensure_L(mbar_b200_ctx* c) { return c->d_L.reserve((size_t)c->nTiles * TILE_N, "pass"); }

}  // namespace mbar

namespace mbar {

struct FusedParams {
    const double* u;
    const double* c;                       // [K] f_k + log N_k - mid (sampled rows)
    const double* c2;                      // second candidate (M == 2): [K] f2_k + log N_k - mid2
    double* out2;                          // ... and its packed result
    double mid2;
    int M;                                 // candidates evaluated per launch (1 or 2)
    const unsigned long long* rowmask;
    const unsigned long long* sampledmask;  // sampled states (the rows that bound D_n from below)
    const double* Nk;
    double* partial;                       // [grid][K + 2]
    double* out;
    unsigned int* ticket;
    double* Lout;                          // [nTiles*32] shifted-frame L'_n, or NULL
    double* Wout;                          // [nTiles][K][32] N_k W_nk (swizzled rows) for the Hessian kernels, or NULL
    const double* wgt;                     // [nTiles*32] sample multiplicities or NULL
    double sumW;                           // sum of the multiplicities of this shard (N if unweighted)
    double* f;                             // [K] device f_k (epilogue) or NULL
    double* cnext;                         // [K] where the epilogue writes c for the next launch
    PeerCfg peer;
    LoopState* loop;                       // device-resident loop state (early exit + convergence) or NULL
    int epi, first;
    int64_t N, nTiles, nStages;
    double mid;
    double logFloorN;                      // LOG_FLOOR_S + log N (global sample count): underflow test of S_k
    int K, Wk, Wn, Rw, TPW, NS, CW, batch, debugSkip, mode, CL, Kh, allStates;
    uint32_t tileBytes, stageBytes;
};

// What a host-driven pass should leave behind (api.cu: run_pass).
struct PassWant {
    bool L = false;          // keep per-sample L'_n on the device
    bool unsampled = false;  // need log-domain sums for N_k == 0 states
    bool G = false;          // K x K second moments
    bool Gall = false;       // ... including the unsampled states' rows and columns
};

// NVTX ranges around pass / exchange / Hessian / upload / solver loops (SURVEY.md section 5).  nvtx3 is header
// only: without an attached tool every call is a no-op through a NULL function table.
struct NvtxRange {
    explicit NvtxRange(const char* name);
    ~NvtxRange();
};

// Persistent host worker threads for the memcpy-bound staging steps (packing pageable uploads, draining log W):
// spawning threads per 64 MB chunk cost as much as a quarter of the chunk's copy time.  run(n, fn) executes
// fn(0..n-1) on the pool plus the calling thread and returns when all are done.
void host_parallel(int nTasks, const std::function<void(int)>& fn);
int host_parallel_width();

// ---- host-side helpers implemented across the .cu files ----
int check_range(mbar_b200_ctx* c, const double* f);
int run_pass(mbar_b200_ctx* c, const double* f, PassWant want);   // pass + all-reduce + D2H into ctx->h_out
double global_sumx(mbar_b200_ctx* c, int* rc);
int retile_chunk(mbar_b200_ctx* ctx, const double* d_rowmajor, int64_t ldCols, int64_t tile0,
                 int64_t nTilesChunk, int64_t validCols, cudaStream_t s);
int launch_pass_generic(mbar_b200_ctx* ctx, const double* h_f, bool wantL, bool logAll);
int launch_pass_fused(mbar_b200_ctx* ctx, const double* h_f, bool wantL, bool allStates, bool* usedOut,
                      bool wantW = false, bool* wroteW = nullptr);
// d_cdst / h_stage: where c = f + log N - mid is staged (default: row ROW_C of ctx->d_c / ctx->h_f); midForce: reuse the
// centring of a previous prepare (candidates evaluated against the same exp(c) range), NaN = derive from f
int fused_prepare(mbar_b200_ctx* ctx, const double* h_f, bool wantL, bool allStates, FusedParams* out, bool* ok,
                  double* d_cdst = nullptr, double* h_stage = nullptr, bool wantW = false, int M = 1,
                  double midQuantum = 0.0);
int fused_enqueue(mbar_b200_ctx* ctx, const FusedParams& p);
bool fused_applicable(const mbar_b200_ctx* ctx, const double* h_f, bool allStates, double* midOut, double* spreadOut);
// weightsReady: the fused pass at this f already wrote N_k W_nk into ctx->d_Wt (FusedParams::Wout)
int launch_hessian(mbar_b200_ctx* ctx, const double* h_f, bool allRows, bool weightsReady = false);
// same with c_k = f_k + log N_k already on the device (device-resident loops); loop may be NULL
int launch_hessian_dev(mbar_b200_ctx* ctx, const double* d_ch, bool allRows, LoopState* loop,
                       bool weightsReady = false);
// the 8*K*N weight buffer of the K > 64 Hessian path; false when it cannot be allocated (in-place fallback)
bool ensure_weight_buffer(mbar_b200_ctx* ctx);
int launch_logw(mbar_b200_ctx* ctx, const double* h_f, double* logW_host, int64_t ld, int expo, int64_t n0,
                int64_t n);
int launch_synth(mbar_b200_ctx* ctx, const mbar_b200_synth* spec);
int launch_untile(mbar_b200_ctx* ctx, int64_t n0, int64_t n, double* d_dst, int64_t ld);
int comm_allreduce(mbar_b200_ctx* ctx, double* d_buf, int count, int op /*0 sum, 2 max*/);
// h_urowmin and h_uclamp made identical on every rank (collective; a no-op without a communicator)
int agree_row_minima(mbar_b200_ctx* ctx);
// ERR_RANGE when an unsampled row holds a clamped finite energy (h_uclamp): for entry points that read those rows
int check_unsampled_clamp(const mbar_b200_ctx* ctx);
int reduce_sumx(mbar_b200_ctx* ctx);
int reduce_sumxw(mbar_b200_ctx* ctx);   // sum_n w_n x_n with the current shifts (no-op without multiplicities)
int set_weights(mbar_b200_ctx* ctx, const double* w_host);
int probe_exp_launch(int which, int64_t n, const double* d_a, double* d_out);   // mbar_b200_probe_exp

// ---- one adaptive iteration on the host (loops.cu): the rules the host-stepped loop and the batched loop of batch.cu
// share.  A problem is K states, the indices of its sampled ones (active[0] is the gauge state) and N_k; S, log S and
// Ghat (N-scaled second moments, row-major K x K) are the sums of a pass.
struct StepRows {
    int K;
    const int* active;
    int na;
    const double* Nk;
};
StepRows step_rows(const mbar_b200_ctx* c);
double step_rel_delta(const StepRows& s, const double* fn, const double* fo, double tol);
void step_sci(const StepRows& s, const std::vector<double>& cur, const double* logS, std::vector<double>& nxt);
double step_gradient(const StepRows& s, const double* S, std::vector<double>& g);
bool step_newton(const StepRows& s, const double* S, const double* Gh, const std::vector<double>& g,
                 const std::vector<double>& cur, double gamma, std::vector<double>& A, std::vector<double>& rhs,
                 std::vector<double>& f_nr);
bool step_choose(const StepRows& s, const std::vector<double>& f_sci, const std::vector<double>& f_nr, bool haveNr,
                 double gn_sci, double gn_nr, double tol, int32_t min_sc_iter, std::vector<double>& cur,
                 mbar_b200_solve_result& r);

// ---- device helpers ----
#ifdef __CUDACC__
static __device__ const double MBAR_EXP_TABLE[MBAR_EXP_NT] = {MBAR_EXP_TABLE_VALUES};
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar), "r"(parity)
            : "memory");
    } while (!done);
}
// Same wait for the single producer lane: back off between polls so the spin does not steal issue
// slots from the consumer warps that share its scheduler.
__device__ __forceinline__ void mbar_wait_backoff(uint32_t bar, uint32_t parity) {
    uint32_t done;
    for (;;) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar), "r"(parity), "r"(0x989680u)
            : "memory");
        if (done) break;
        __nanosleep(200);
    }
}
// 1-D bulk async copy global -> shared (TMA engine; SASS UBLKCP), completion on an mbarrier.
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
        "l"(src), "r"(bytes), "r"(bar)
        : "memory");
}
// order this thread's generic-proxy shared-memory accesses before later async-proxy (TMA) accesses
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

constexpr double EXP_MAGIC = 6755399441055744.0;  // 1.5 * 2^52

// exp(a) with the binary exponent kept apart:  exp(a) = v * 2^q,  v in [1, 2).
// a in [-5e7, 5e7]; `tab` = 32-entry table of 2^(j/32) in shared memory (conflict-free: 256 B).
// 9 fp64 pipe ops (FMA t, ADD nf, FMA r, 4 FMA Horner, MUL, FMA) + integer work on the ALU pipe.  The reduction
// subtracts n ln2/32 as ONE double (MBAR_EXP_LN2N_LO is not applied): the result is exp(a (1 + 3.35e-17)), up to
// 108 ulp off at |a| = 708 but 1.5 ulp from that (DESIGN.md 3.1: the second FMA would cost the fused pass time).
__device__ __forceinline__ void exp_split(double a, const double* __restrict__ tab, double& v, int& q) {
    const double t = fma(a, MBAR_EXP_SCALE, EXP_MAGIC);
    const int n = __double2loint(t);
    const double nf = t - EXP_MAGIC;
    const double r = fma(nf, -MBAR_EXP_LN2N, a);
    double p = fma(MBAR_EXP_C5, r, MBAR_EXP_C4);
    p = fma(p, r, MBAR_EXP_C3);
    p = fma(p, r, MBAR_EXP_C2);
    p = fma(p, r, MBAR_EXP_C1);
    p = p * r;
    const double T = tab[n & (MBAR_EXP_NT - 1)];
    v = fma(T, p, T);
    q = n >> 5;
}
// v * 2^q with q clamped to the normal range from below (result in [2^-1021, 2^-1020), never denormal: callers
// must treat sums that such entries could dominate as underflowed, see LOG_FLOOR_S) and assumed <= 1023 from
// above (arguments <= 709.7, see FUSED_MAX_ARG).
__device__ __forceinline__ double scale2(double v, int q) {
    q = max(q, -1021);
    const int hi = __double2hiint(v) + (q << 20);
    return __hiloint2double(hi, __double2loint(v));
}
__device__ __forceinline__ double exp_fast(double a, const double* __restrict__ tab) {
    double v;
    int q;
    exp_split(a, tab, v, q);
    return scale2(v, q);
}
__device__ __forceinline__ double warp_sum(double x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}

// the last of n segments whose start(s) <= i, for ascending starts with start(0) <= i
template <class Start>
__device__ __forceinline__ int find_segment(int n, int64_t i, Start start) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (start(mid) <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// The order-preserving integer form of a double, so that a per-bin maximum can be taken by an integer atomicMax (a
// maximum does not depend on the order of its operands, so the result is deterministic); 0 is below every key.
__device__ __forceinline__ unsigned long long ordered_key(double d) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(d);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double ordered_value(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// The lanes of a warp grouped by an integer key (__match_any_sync) and sorted so that every group is contiguous,
// groups in the order of their lowest lane.  Lane i of the sorted order holds lane src's value and key; `same` bit s
// says the lane 2^s below it holds the same key; `tail` marks the last lane of each group.  Computed once per tile and
// reused for every row summed over that tile; perm is the warp's 32-int shared scratch.
struct WarpGroups {
    int src, key, steps;
    unsigned same;
    bool tail;
};
__device__ __forceinline__ WarpGroups warp_groups(int b, int* perm) {
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const unsigned grp = __match_any_sync(FULL, b);
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
    WarpGroups g;
    g.src = perm[lane];
    __syncwarp();
    g.key = __shfl_sync(FULL, b, g.src);
    const int maxg = (int)__reduce_max_sync(FULL, (unsigned)gsize);
    g.steps = 0;
    while ((1 << g.steps) < maxg) ++g.steps;
    g.same = 0;
    for (int s = 0; s < g.steps; ++s) {
        const int kd = __shfl_up_sync(FULL, g.key, 1 << s);
        if (lane >= (1 << s) && kd == g.key) g.same |= 1u << s;
    }
    const int next = __shfl_down_sync(FULL, g.key, 1);
    g.tail = (lane == 31) || next != g.key;
    return g;
}
// v of lane src, summed over its group by a segmented scan of g.steps steps: a tail lane ends with its group's sum,
// added in an order fixed by the keys alone
__device__ __forceinline__ double warp_group_sum(const WarpGroups& g, double v) {
    v = __shfl_sync(0xffffffffu, v, g.src);
    for (int s = 0; s < g.steps; ++s) {
        const double y = __shfl_up_sync(0xffffffffu, v, 1 << s);
        if ((g.same >> s) & 1u) v += y;
    }
    return v;
}
#endif

// Relative change |a - b| / |ref| of one entry (mbar_solvers.py:627-632); entries with |ref| below thr = min(1e-8, tol)
// compare absolutely.  Subtraction, fabs, division and a comparison are correctly rounded on host and device alike,
// so every solver loop gets the same value.  The reduction and its NaN policy stay with each caller.
__host__ __device__ __forceinline__ double rel_change(double a, double b, double ref, double thr) {
    double div = fabs(ref);
    if (div < thr) div = 1.0;
    return fabs(a - b) / div;
}

// d_scratch holds K*K + 4K + 1024 doubles of call-local scratch; the rendezvous all-reduce of the device-resident
// loops owns the word at this offset
inline size_t scratch_rendezvous(int K) { return (size_t)K * K + 4 * (size_t)K; }

// The replicate weights V [B, N] of mbar_b200_kde_set_replicates and mbar_b200_bspline_set_replicates: B >= 1 and
// every V_bn finite and >= 0.
inline int check_replicate_weights(const char* who, int64_t B, int64_t N, const double* V) {
    MBAR_REQUIRE(B >= 1 && V, MBAR_B200_ERR_INVALID, "%s: B=%lld, V=%p", who, (long long)B, (const void*)V);
    for (int64_t i = 0; i < B * N; ++i)
        MBAR_REQUIRE(V[i] >= 0.0 && V[i] < INFINITY, MBAR_B200_ERR_INVALID,
                     "%s: weight (%lld, %lld) is %g (negative, NaN or infinite)", who, (long long)(i / N),
                     (long long)(i % N), V[i]);
    return MBAR_B200_OK;
}

}  // namespace mbar

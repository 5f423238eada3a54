"""DeviceProblem: one (u_kn, N_k) data set resident in HBM on one GPU (one shard of the samples).

Thin object wrapper over the C ABI (include/mbar_b200.h).  All math happens in libmbar_b200.so;
this file only marshals numpy buffers.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import AdaptiveStats, SolveResult, check


def _dptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _i32p(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def _i64p(a):
    return a.ctypes.data_as(C.POINTER(C.c_int64))


def _f64(a, K=None):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if K is not None and a.shape != (K,):
        raise ValueError(f"expected shape ({K},), got {a.shape}")
    return a


def _set_replicates(obj, upload, V):
    """Upload the replicate weights V [B, obj.N] with `upload` (a *_set_replicates entry point) and set obj.B."""
    V = np.ascontiguousarray(V, dtype=np.float64)
    if V.ndim != 2 or V.shape[1] != obj.N:
        raise ValueError(f"replicate weights must be [B, {obj.N}], got shape {V.shape}")
    obj.B = 0                              # a failed upload leaves none
    check(upload(obj._h, V.shape[0], _dptr(V)))
    obj.B = V.shape[0]


def _knots(t, k):
    """(t as contiguous float64, nb): the knot vector and its number of basis functions of degree k."""
    t = np.ascontiguousarray(t, dtype=np.float64)
    if t.ndim != 1:
        raise ValueError(f"knots must be one-dimensional, got shape {t.shape}")
    return t, max(t.shape[0] - int(k) - 1, 0)


class _Resident:
    """Owner of one library object: the handle `_h` and `_destroy`, the name of the entry point that frees it."""

    _destroy = None

    def close(self):
        if self._h is not None and self._h.value:
            getattr(self._lib, self._destroy)(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class PinnedArray:
    """float64 ndarray backed by cudaHostAlloc memory (mbar_b200_host_alloc)."""

    def __init__(self, shape):
        self.shape = tuple(int(s) for s in shape)
        n = int(np.prod(self.shape))
        self._ptr = C.c_void_p()
        check(_lib.load().mbar_b200_host_alloc(C.byref(self._ptr), n * 8))
        buf = (C.c_double * n).from_address(self._ptr.value)
        self.array = np.frombuffer(buf, dtype=np.float64).reshape(self.shape)

    def free(self):
        if self._ptr is not None and self._ptr.value:
            self.array = None
            _lib.load().mbar_b200_host_free(self._ptr)
            self._ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class DeviceProblem(_Resident):
    """u_kn [K, N_local] + global N_k [K] on one H100.

    Parameters
    ----------
    u_kn : ndarray [K, N_local] float64 (any strides with unit inner stride), or None to allocate
        only (fill later with :meth:`synthesize` / :meth:`upload`).
    N_k : array [K] — GLOBAL sample counts (all ranks), int or float; zeros mark unsampled states.
    device : CUDA device ordinal.
    N_local : required when u_kn is None.
    """

    _destroy = "mbar_b200_destroy"

    def __init__(self, u_kn, N_k, device=0, N_local=None):
        self._lib = _lib.load()
        self._h = C.c_void_p()
        N_k = _f64(N_k)
        if N_k.ndim != 1:
            raise ValueError("N_k must be 1-D")
        self.K = int(N_k.shape[0])
        self.N_k = N_k
        if u_kn is not None:
            if u_kn.ndim != 2 or u_kn.shape[0] != self.K:
                raise ValueError(f"u_kn must be [K={self.K}, N], got {u_kn.shape}")
            N_local = u_kn.shape[1]
        if N_local is None:
            raise ValueError("N_local is required when u_kn is None")
        self.N = int(N_local)
        self.device = int(device)
        check(self._lib.mbar_b200_create(C.byref(self._h), self.device, self.K, self.N, _dptr(N_k)))
        if u_kn is not None:
            self.upload(u_kn)

    # ---- data -------------------------------------------------------------------------------
    def upload(self, u_kn):
        u = np.asarray(u_kn)
        if u.dtype != np.float64 or u.ndim != 2 or u.strides[1] != 8 or u.strides[0] % 8 or u.strides[0] < 8 * u.shape[1]:
            u = np.ascontiguousarray(u, dtype=np.float64)
        if u.shape != (self.K, self.N):
            raise ValueError(f"u_kn must be [{self.K}, {self.N}], got {u.shape}")
        check(self._lib.mbar_b200_upload_u_kn(self._h, C.c_void_p(u.ctypes.data), u.strides[0] // 8))

    def augmented(self, u_extra):
        """New DeviceProblem = these samples + the rows of `u_extra` [E, N] as unsampled states (the resident
        tiles are copied on the device, only the new rows are uploaded)."""
        u = np.asarray(u_extra, dtype=np.float64)
        if u.ndim == 1:
            u = u.reshape(1, -1)
        if u.ndim != 2 or u.shape[1] != self.N:
            raise ValueError(f"u_extra must be [E, {self.N}], got {u.shape}")
        if u.strides[1] != 8 or u.strides[0] % 8 or u.strides[0] < 8 * u.shape[1]:
            u = np.ascontiguousarray(u)
        h = C.c_void_p()
        check(self._lib.mbar_b200_create_augmented(self._h, u.shape[0], C.c_void_p(u.ctypes.data),
                                                   u.strides[0] // 8, C.byref(h)))
        q = DeviceProblem.__new__(DeviceProblem)
        q._lib, q._h = self._lib, h
        q.K, q.N, q.device = self.K + u.shape[0], self.N, self.device
        q.N_k = np.concatenate([self.N_k, np.zeros(u.shape[0])])
        return q

    def upload_device_ptr(self, ptr, ld):
        check(self._lib.mbar_b200_upload_u_kn_dev(self._h, C.c_void_p(int(ptr)), int(ld)))

    def synthesize(self, O_k, k_k, seed=0, n_offset=0, N_global=None):
        O_k, k_k = _f64(O_k, self.K), _f64(k_k, self.K)
        spec = _lib.Synth(int(seed), int(n_offset), int(N_global if N_global is not None else self.N),
                          _dptr(O_k), _dptr(k_k))
        check(self._lib.mbar_b200_synthesize(self._h, C.byref(spec)))

    def set_sample_weights(self, w):
        """Per-sample multiplicities (bootstrap replicate without copying u_kn); None restores w = 1."""
        if w is None:
            check(self._lib.mbar_b200_set_sample_weights(self._h, None))
            return
        w = _f64(w)
        if w.shape != (self.N,):
            raise ValueError(f"weights must have shape ({self.N},)")
        check(self._lib.mbar_b200_set_sample_weights(self._h, C.c_void_p(w.ctypes.data)))

    def download(self, n0=0, n=None, out=None):
        n = self.N - n0 if n is None else n
        if out is None:
            out = np.empty((self.K, n), np.float64)
        check(self._lib.mbar_b200_download_u_kn(self._h, int(n0), int(n), C.c_void_p(out.ctypes.data),
                                                out.strides[0] // 8))
        return out

    def set_kernel(self, which):
        code = {"auto": 0, "fused": 1, "generic": 2}.get(which, which)
        check(self._lib.mbar_b200_set_pass_kernel(self._h, int(code)))

    def counters(self):
        v = [C.c_int64(0) for _ in range(4)]
        check(self._lib.mbar_b200_get_counters(self._h, *[C.byref(x) for x in v]))
        return dict(launches=v[0].value, passes=v[1].value, h2d_bytes=v[2].value, d2h_bytes=v[3].value)

    def last_pass_ms(self):
        ms = C.c_double(0)
        check(self._lib.mbar_b200_last_pass_ms(self._h, C.byref(ms)))
        return ms.value

    def last_loop_ms(self):
        tot, ker, it = C.c_double(0), C.c_double(0), C.c_int32(0)
        check(self._lib.mbar_b200_last_loop_ms(self._h, C.byref(tot), C.byref(ker), C.byref(it)))
        return dict(total_ms=tot.value, kernel_ms_sum=ker.value, iters=it.value)

    # ---- communicator -------------------------------------------------------------------------
    @staticmethod
    def comm_unique_id():
        buf = C.create_string_buffer(_lib.UNIQUE_ID_BYTES)
        check(_lib.load().mbar_b200_comm_unique_id(buf))
        return buf.raw

    def comm_init(self, nranks, rank, unique_id):
        buf = C.create_string_buffer(bytes(unique_id), _lib.UNIQUE_ID_BYTES)
        check(self._lib.mbar_b200_comm_init(self._h, int(nranks), int(rank), buf))

    def peer_export(self):
        buf = C.create_string_buffer(64)
        check(self._lib.mbar_b200_peer_export(self._h, buf))
        return buf.raw

    def peer_attach(self, nranks, rank, handles):
        blob = b"".join(bytes(h) for h in handles)
        buf = C.create_string_buffer(blob, len(blob))
        check(self._lib.mbar_b200_peer_attach(self._h, int(nranks), int(rank), buf))

    # ---- the pass and the reference primitives ----------------------------------------------------
    def _bad(self, f):
        """The reference propagates NaN through its primitives (SURVEY.md Appendix A); the C ABI
        reports ERR_RANGE instead.  Mirror the reference for optimiser trial points that left the
        representable range: non-finite (or > 1e6 in magnitude) f_k on a sampled state -> NaNs."""
        c = f[self.N_k > 0]
        return not np.all(np.isfinite(c)) or np.max(np.abs(c)) > 9.0e5

    def streaming_pass(self, f_k, want_G=False):
        f = _f64(f_k, self.K)
        S = np.empty(self.K)
        sumL = C.c_double(0)
        G = np.empty((self.K, self.K)) if want_G else None
        check(self._lib.mbar_b200_pass(self._h, _dptr(f), _dptr(S), C.byref(sumL),
                                       _dptr(G) if want_G else None))
        return S, sumL.value, G

    def pass_multi(self, f_mk):
        """One call, one synchronisation, M (1 or 2) candidate vectors: returns (S[M, K], sumL[M])."""
        f = np.ascontiguousarray(f_mk, dtype=np.float64)
        if f.ndim != 2 or f.shape[1] != self.K or not 1 <= f.shape[0] <= 2:
            raise ValueError(f"expected [M in (1, 2), {self.K}], got {f.shape}")
        S = np.empty_like(f)
        sumL = np.empty(f.shape[0])
        check(self._lib.mbar_b200_pass_multi(self._h, f.shape[0], _dptr(f), _dptr(S), _dptr(sumL)))
        return S, sumL

    def self_consistent_update(self, f_k):
        f = _f64(f_k, self.K)
        if self._bad(f):
            return np.full(self.K, np.nan)
        out = np.empty(self.K)
        check(self._lib.mbar_b200_self_consistent_update(self._h, _dptr(f), _dptr(out)))
        return out

    def gradient(self, f_k):
        f = _f64(f_k, self.K)
        if self._bad(f):
            return np.full(self.K, np.nan)
        out = np.empty(self.K)
        check(self._lib.mbar_b200_gradient(self._h, _dptr(f), _dptr(out)))
        return out

    def objective_and_gradient(self, f_k):
        f = _f64(f_k, self.K)
        if self._bad(f):
            return np.nan, np.full(self.K, np.nan)
        g = np.empty(self.K)
        obj = C.c_double(0)
        check(self._lib.mbar_b200_objective_and_gradient(self._h, _dptr(f), C.byref(obj), _dptr(g)))
        return obj.value, g

    def objective(self, f_k):
        f = _f64(f_k, self.K)
        if self._bad(f):
            return np.nan
        obj = C.c_double(0)
        check(self._lib.mbar_b200_objective_and_gradient(self._h, _dptr(f), C.byref(obj), None))
        return obj.value

    def hessian(self, f_k):
        f = _f64(f_k, self.K)
        if self._bad(f):
            return np.full((self.K, self.K), np.nan)
        H = np.empty((self.K, self.K))
        check(self._lib.mbar_b200_hessian(self._h, _dptr(f), _dptr(H)))
        return H

    def weight_moments(self, f_k):
        """(S_k, G = W^T W) over ALL states — the K x K input of pymbar_b200.estimators."""
        f = _f64(f_k, self.K)
        S = np.empty(self.K)
        G = np.empty((self.K, self.K))
        check(self._lib.mbar_b200_weight_moments(self._h, _dptr(f), _dptr(S), _dptr(G)))
        return S, G

    def log_W_nk(self, f_k, exponentiate=False, out=None, rows=None, row0=0):
        """[N, K] log weights (mbar_solvers.py:439-473); `rows` / `row0` (multiple of 32) fetch a block of rows."""
        f = _f64(f_k, self.K)
        if self._bad(f):
            n = self.N if rows is None else int(rows)
            return np.full((n, self.K), np.nan)
        if rows is None and row0 == 0:
            if out is None:
                out = np.empty((self.N, self.K), np.float64)
            check(self._lib.mbar_b200_log_W_nk(self._h, _dptr(f), C.c_void_p(out.ctypes.data),
                                               out.strides[0] // 8, int(bool(exponentiate))))
            return out
        rows = self.N - row0 if rows is None else int(rows)
        if out is None:
            out = np.empty((rows, self.K), np.float64)
        check(self._lib.mbar_b200_log_W_nk_rows(self._h, _dptr(f), int(row0), rows, C.c_void_p(out.ctypes.data),
                                                out.strides[0] // 8, int(bool(exponentiate))))
        return out

    def log_denominator(self, f_k):
        f = _f64(f_k, self.K)
        if self._bad(f):                 # the reference propagates NaN (ADVICE r1)
            return np.full(self.N, np.nan)
        out = np.empty(self.N)
        check(self._lib.mbar_b200_log_denominator(self._h, _dptr(f), _dptr(out)))
        return out

    def bin_moments(self, f_k, u_n, bin_n, nbins, want_C=True):
        """Histogram FES of the target state `u_n` [N] over the dense bin index `bin_n` [N] in [0, nbins):
        (f_bin [nbins], C [K, nbins], D [nbins]) with f_i = -log sum_{n in i} exp(-u_n - L_n),
        C_ki = sum_{n in i} W_nk w^_n, D_i = sum_{n in i} w^_n^2 and w^_n = exp(-u_n - L_n + f_i)
        (mbar_b200_bin_moments).  want_C=False skips the moments: (f_bin, None, None)."""
        f = _f64(f_k, self.K)
        u = _f64(u_n)
        b = np.ascontiguousarray(bin_n, dtype=np.int32)
        nbins = int(nbins)
        if u.shape != (self.N,) or b.shape != (self.N,):
            raise ValueError(f"u_n and bin_n must have shape ({self.N},), got {u.shape} and {b.shape}")
        f_bin = np.empty(nbins)
        C_ = np.empty((self.K, nbins)) if want_C else None
        D = np.empty(nbins) if want_C else None
        check(self._lib.mbar_b200_bin_moments(self._h, _dptr(f), _dptr(u), _i32p(b), nbins, _dptr(f_bin),
                                              _dptr(C_) if want_C else None, _dptr(D) if want_C else None))
        return f_bin, C_, D

    def last_bin_stats(self):
        """CUDA-event time of the last bin_moments' kernels after its pass, and its reads of u_kn for C / D."""
        ms, chunks = C.c_double(0), C.c_int32(0)
        check(self._lib.mbar_b200_last_bin_stats(self._h, C.byref(ms), C.byref(chunks)))
        return dict(ms=ms.value, chunks=chunks.value)

    def replicate_unsampled(self, counts, F):
        """[B, n_u]: for bootstrap replicate b with multiplicities counts[b] [N] and free energies F[b] [K], the
        unsampled states' updates -log sum_n counts[b, n] exp(-u_jn - L_bn), what set_sample_weights(counts[b]) +
        self_consistent_update(F[b]) give for those rows, every replicate in one device call
        (mbar_b200_replicate_unsampled).  Counts are sent as uint16: above 65535 (or negative) raises ValueError."""
        c = np.asarray(counts)
        if c.ndim != 2 or c.shape[1] != self.N:
            raise ValueError(f"counts must be [B, {self.N}], got shape {c.shape}")
        if c.size and (c.min() < 0 or c.max() > 65535):
            raise ValueError("replicate counts must lie in [0, 65535]")
        c = np.ascontiguousarray(c, dtype=np.uint16)
        F = np.ascontiguousarray(F, dtype=np.float64)
        if F.shape != (c.shape[0], self.K):
            raise ValueError(f"F must be [{c.shape[0]}, {self.K}], got shape {F.shape}")
        out = np.empty((c.shape[0], int(np.sum(~(self.N_k > 0)))))
        check(self._lib.mbar_b200_replicate_unsampled(self._h, c.shape[0], c.ctypes.data_as(C.POINTER(C.c_uint16)),
                                                      _dptr(F), _dptr(out)))
        return out

    def last_replicate_stats(self):
        """CUDA-event time (ms) of the last replicate_unsampled's kernels, its replicate batches and the exps it
        evaluated."""
        ms, batches, exps = C.c_double(0), C.c_int32(0), C.c_int64(0)
        check(self._lib.mbar_b200_last_replicate_stats(self._h, C.byref(ms), C.byref(batches), C.byref(exps)))
        return dict(ms=ms.value, batches=batches.value, exps=exps.value)

    # ---- native loops ---------------------------------------------------------------------------
    @staticmethod
    def _result(r):
        return {name: getattr(r, name) for name, _ in SolveResult._fields_}

    def solve_sci(self, f_k, tol=1e-12, maxiter=10000):
        f = _f64(f_k, self.K).copy()
        r = SolveResult()
        check(self._lib.mbar_b200_solve_sci(self._h, _dptr(f), float(tol), int(maxiter), C.byref(r)))
        return f, self._result(r)

    def solve_adaptive(self, f_k, tol=1e-12, maxiter=10000, min_sc_iter=2, gamma=1.0):
        f = _f64(f_k, self.K).copy()
        r = SolveResult()
        check(self._lib.mbar_b200_solve_adaptive(self._h, _dptr(f), float(tol), int(maxiter), int(min_sc_iter),
                                                 float(gamma), C.byref(r)))
        return f, self._result(r)

    def set_loop_mode(self, mode="device", batch=0):
        """'device' (default): solver iterations stay on the GPU, polled every `batch` iterations;
        'stepped': one host round trip per pass (round-1 behaviour, also the robust fallback)."""
        code = {"device": 0, "stepped": 1}.get(mode, mode)
        check(self._lib.mbar_b200_set_loop_mode(self._h, int(code), int(batch)))

    def loop_stats(self):
        polls, mode, batch = C.c_int64(0), C.c_int32(0), C.c_int32(0)
        check(self._lib.mbar_b200_get_loop_stats(self._h, C.byref(polls), C.byref(mode), C.byref(batch)))
        cap, lau = C.c_int64(0), C.c_int64(0)
        check(self._lib.mbar_b200_get_graph_stats(self._h, C.byref(cap), C.byref(lau)))
        return dict(polls=polls.value, mode="stepped" if mode.value else "device", batch=batch.value,
                    graph_captures=cap.value, graph_launches=lau.value)

    def adaptive_stats(self):
        """How the last solve_adaptive ran: iterations the device-resident loop kept, whether the host-stepped loop
        finished the solve, the device Newton step's ridge retries, failed and rejected candidates, and its launch
        plan (CTA size, matrix in shared memory or not)."""
        st = AdaptiveStats()
        check(self._lib.mbar_b200_get_adaptive_stats(self._h, C.byref(st)))
        d = {name: getattr(st, name) for name, _ in AdaptiveStats._fields_ if name != "reserved"}
        d["fell_back"] = bool(d["fell_back"])
        d["newton_smem"] = bool(d["newton_smem"])
        return d

    def last_kernels(self):
        a, b = C.create_string_buffer(256), C.create_string_buffer(256)
        check(self._lib.mbar_b200_last_kernels(self._h, a, b, 256))
        return dict(pass_kernel=a.value.decode(), hessian_kernel=b.value.decode())

    def last_hessian_ms(self):
        w, h = C.c_double(0), C.c_double(0)
        check(self._lib.mbar_b200_last_hessian_ms(self._h, C.byref(w), C.byref(h)))
        return dict(weights_ms=w.value, hessian_ms=h.value)

    def sci_iterate(self, f_k, iters):
        f = _f64(f_k, self.K).copy()
        check(self._lib.mbar_b200_sci_iterate(self._h, _dptr(f), int(iters)))
        return f


KDE_KERNELS = ("gaussian", "tophat", "epanechnikov", "exponential", "linear", "cosine")   # mbar_b200_kde_kernel


class DeviceKde(_Resident):
    """Weighted samples x_n [N, D] (D = 1..4) resident on one H100 for kernel-density sums (mbar_b200_kde_*).

    `log_sum(kernel, h, y)` returns l_q = log sum_n w_n k(|y_q - x_n| / h) for the query points y [Q, D], with
    sklearn's unnormalised kernels; pymbar_b200.fes adds the normalisation.  Independent of any DeviceProblem."""

    _destroy = "mbar_b200_kde_destroy"

    def __init__(self, x_n, w_n, device=0):
        self._lib = _lib.load()
        self._h = C.c_void_p()
        x = np.asarray(x_n, dtype=np.float64)
        if x.ndim == 1:
            x = x.reshape(-1, 1)
        if x.ndim != 2:
            raise ValueError(f"x_n must be [N] or [N, D], got shape {np.shape(x_n)}")
        x = np.ascontiguousarray(x)
        w = _f64(w_n, x.shape[0])
        self.N, self.D = x.shape
        self.B = 0                         # replicates uploaded by set_replicates
        self.device = int(device)
        check(self._lib.mbar_b200_kde_create(self.device, self.N, self.D, _dptr(x), _dptr(w), C.byref(self._h)))

    def _kernel_and_queries(self, kernel, y):
        code = KDE_KERNELS.index(kernel) if isinstance(kernel, str) and kernel in KDE_KERNELS else kernel
        if isinstance(code, str):
            code = -1                      # unknown name: the library reports ERR_INVALID
        y = np.asarray(y, dtype=np.float64)
        if y.ndim == 1 and self.D == 1:
            y = y.reshape(-1, 1)
        if y.ndim != 2 or y.shape[1] != self.D:
            raise ValueError(f"queries must be [Q, {self.D}], got shape {y.shape}")
        return code, np.ascontiguousarray(y)

    def log_sum(self, kernel, h, y):
        """l_q [Q] for the queries y [Q, D] (or [Q] when D = 1); kernel is a name of KDE_KERNELS or its code."""
        code, y = self._kernel_and_queries(kernel, y)
        out = np.empty(y.shape[0])
        check(self._lib.mbar_b200_kde_log_sum(self._h, int(code), float(h), y.shape[0], _dptr(y), _dptr(out)))
        return out

    def set_replicates(self, V):
        """Upload the weights V [B, N] of B bootstrap replicates of the resident samples (V_bn >= 0); they replace any
        uploaded before and stay on the device for log_sum_replicates."""
        _set_replicates(self, self._lib.mbar_b200_kde_set_replicates, V)

    def log_sum_replicates(self, kernel, h, y):
        """[B, Q]: log_sum with the weights of each uploaded replicate, all replicates in one device call."""
        code, y = self._kernel_and_queries(kernel, y)
        out = np.empty((self.B, y.shape[0]))
        check(self._lib.mbar_b200_kde_log_sum_replicates(self._h, int(code), float(h), y.shape[0], _dptr(y),
                                                         _dptr(out)))
        return out

    def last_stats(self):
        """CUDA-event time (ms) of the last log_sum's or log_sum_replicates' kernels and the number of sample chunks."""
        ms, chunks = C.c_double(0), C.c_int32(0)
        check(self._lib.mbar_b200_last_kde_stats(self._h, C.byref(ms), C.byref(chunks)))
        return dict(ms=ms.value, chunks=chunks.value)


class DeviceKdeMany(_Resident):
    """Many sample sets x_list[s] ([N_s] or [N_s, D_s], D_s = 1..4) resident on one H100 for kernel-density sums of
    many small problems in one call (mbar_b200_kde_many_*).  Only the coordinates are resident: every request brings
    its own weights, so a surface and each of its bootstrap replicates are requests on the same set.

    `log_sum(sets, kernels, hs, w_list, y_list)` returns, per request r, l_q = log sum_n w_n k(|y_q - x_n| / h) over
    set sets[r] with weights w_list[r] [N_s], kernel kernels[r] and bandwidth hs[r] at the queries y_list[r] [Q_r, D_s]:
    the same bits DeviceKde(x_list[s], w).log_sum gives."""

    _destroy = "mbar_b200_kde_many_destroy"

    def __init__(self, x_list, device=0):
        self._lib = _lib.load()
        self._h = C.c_void_p()
        xs = []
        for s, x in enumerate(x_list):
            x = np.asarray(x, dtype=np.float64)
            if x.ndim == 1:
                x = x.reshape(-1, 1)
            if x.ndim != 2:
                raise ValueError(f"set {s}: x_n must be [N] or [N, D], got shape {x.shape}")
            xs.append(np.ascontiguousarray(x))
        if not xs:
            raise ValueError("need at least one sample set")
        self.N = np.ascontiguousarray([x.shape[0] for x in xs], dtype=np.int64)
        self.D = np.ascontiguousarray([x.shape[1] for x in xs], dtype=np.int32)
        self.device = int(device)
        flat = np.ascontiguousarray(np.concatenate([x.ravel() for x in xs]))
        check(self._lib.mbar_b200_kde_many_create(self.device, len(xs), _i32p(self.D), _i64p(self.N), _dptr(flat),
                                                  C.byref(self._h)))

    def log_sum(self, sets, kernels, hs, w_list, y_list):
        """[l [Q_r]] per request; kernels are names of KDE_KERNELS or their codes."""
        sets = np.ascontiguousarray(sets, dtype=np.int32).reshape(-1)
        n = sets.size
        if not (len(kernels) == len(hs) == len(w_list) == len(y_list) == n):
            raise ValueError("need one set, kernel, bandwidth, weight vector and query array per request")
        codes = np.ascontiguousarray([KDE_KERNELS.index(k) if isinstance(k, str) and k in KDE_KERNELS else
                                      (-1 if isinstance(k, str) else int(k)) for k in kernels], dtype=np.int32)
        known = [0 <= s < self.N.size for s in sets]           # an unknown set is the library's error
        ws, ys = [], []
        for r, (s, ok, w, y) in enumerate(zip(sets, known, w_list, y_list)):
            w = _f64(w, int(self.N[s]) if ok else None)
            y = np.asarray(y, dtype=np.float64)
            D = int(self.D[s]) if ok else (y.shape[1] if y.ndim == 2 else 1)
            if y.ndim == 1 and D == 1:
                y = y.reshape(-1, 1)
            if y.ndim != 2 or y.shape[1] != D:
                raise ValueError(f"request {r}: queries must be [Q, {D}], got shape {y.shape}")
            ws.append(w)
            ys.append(np.ascontiguousarray(y))
        Q = np.ascontiguousarray([y.shape[0] for y in ys], dtype=np.int64)
        w = np.ascontiguousarray(np.concatenate(ws)) if ws else np.zeros(0)
        y = np.ascontiguousarray(np.concatenate([a.ravel() for a in ys])) if ys else np.zeros(0)
        h = np.ascontiguousarray(hs, dtype=np.float64).reshape(-1)
        out = np.empty(int(Q.sum()))
        check(self._lib.mbar_b200_kde_many_log_sum(self._h, n, _i32p(sets), _i32p(codes), _dptr(h), _dptr(w),
                                                   _i64p(Q), _dptr(y), _dptr(out)))
        return np.split(out, np.cumsum(Q)[:-1]) if n else []

    def last_stats(self):
        """CUDA-event time (ms) of the last log_sum's kernels, its kernel launches and (query, sample) pairs."""
        ms, launches, pairs = C.c_double(0), C.c_int32(0), C.c_int64(0)
        check(self._lib.mbar_b200_last_kde_many_stats(self._h, C.byref(ms), C.byref(launches), C.byref(pairs)))
        return dict(ms=ms.value, launches=launches.value, pairs=pairs.value)


class DeviceBSpline(_Resident):
    """Samples x_n [N] with optional weights w_n and state labels state_n in [0, K) resident on one H100 for B-spline
    basis sums (mbar_b200_bspline_*).

    `moments(t, k)` returns (S [K, nb], A [nb]) with S_ki = sum_{n: state_n = k} B_i(x_n) and A_i = sum_n w_n B_i(x_n),
    B_i the basis functions of scipy's BSpline(t, e_i, k).  One upload serves any number of knot vectors.  Independent
    of any DeviceProblem."""

    _destroy = "mbar_b200_bspline_destroy"

    def __init__(self, x_n, w_n=None, state_n=None, K=None, device=0):
        self._lib = _lib.load()
        self._h = C.c_void_p()
        x = np.ascontiguousarray(x_n, dtype=np.float64)
        if x.ndim != 1:
            raise ValueError(f"x_n must be one-dimensional, got shape {np.shape(x_n)}")
        self.N = x.shape[0]
        w = None if w_n is None else _f64(w_n, self.N)
        s = None
        if state_n is not None:
            s_raw = np.asarray(state_n)
            if s_raw.shape != (self.N,) or not np.issubdtype(s_raw.dtype, np.integer):
                raise ValueError(f"state_n must be [{self.N}] integers, got {s_raw.dtype} {s_raw.shape}")
            K = int(s_raw.max()) + 1 if K is None else int(K)
            # labels beyond int32 become -1, which the library rejects
            s = np.ascontiguousarray(np.where((s_raw >= -1) & (s_raw < 2 ** 31 - 1), s_raw, -1), dtype=np.int32)
        self.K = int(K) if s is not None else 0
        self.B = 0                         # replicates uploaded by set_replicates
        self.has_weights, self.has_labels = w is not None, s is not None
        self.device = int(device)
        check(self._lib.mbar_b200_bspline_create(
            self.device, self.N, _dptr(x), None if w is None else _dptr(w),
            None if s is None else _i32p(s), self.K, C.byref(self._h)))

    def moments(self, t, k, want_S=True, want_A=True):
        """(S [K, nb] or None, A [nb] or None) for the knots t and degree k."""
        t, nb = _knots(t, k)
        S = np.empty((self.K, nb)) if want_S else None
        A = np.empty(nb) if want_A else None
        check(self._lib.mbar_b200_bspline_moments(self._h, int(k), t.shape[0], _dptr(t),
                                                  None if S is None else _dptr(S), None if A is None else _dptr(A)))
        return S, A

    def set_replicates(self, V):
        """Upload the weights V [B, N] of B bootstrap replicates of the resident samples (V_bn >= 0); they replace any
        uploaded before and stay on the device for replicate_sums.  The weights and labels of the constructor are
        kept."""
        _set_replicates(self, self._lib.mbar_b200_bspline_set_replicates, V)

    def replicate_sums(self, t, k):
        """[B, nb]: row b is sum_n V_bn B_i(x_n), the A of moments with replicate b's weights, for every uploaded
        replicate in one device call."""
        t, nb = _knots(t, k)
        out = np.empty((self.B, nb))
        check(self._lib.mbar_b200_bspline_replicate_sums(self._h, int(k), t.shape[0], _dptr(t), _dptr(out)))
        return out

    def last_stats(self):
        """CUDA-event time (ms) of the last moments or replicate_sums call's kernels and the number of row chunks
        (moments) or replicate batches (replicate_sums)."""
        ms, chunks = C.c_double(0), C.c_int32(0)
        check(self._lib.mbar_b200_last_bspline_stats(self._h, C.byref(ms), C.byref(chunks)))
        return dict(ms=ms.value, chunks=chunks.value)


class DeviceAcf(_Resident):
    """A series A [T] (and B [T] for a cross-correlation; optionally K concatenated series given by their lengths)
    resident on one H100 for the centred lag sums of pymbar.timeseries (mbar_b200_acf_*).  Independent of any
    DeviceProblem.

    `inefficiency(starts, fast, mintime)` runs the reference's statistical-inefficiency loop for every start at once
    (rule="fft": statistical_inefficiency_fft's); `correlation(start, n_max)` returns C(t), t = 0 .. n_max, and
    `correlation_multiple(n_max, truncate)` the multiple-series correlation function of a segmented object."""

    _destroy = "mbar_b200_acf_destroy"

    def __init__(self, A_n, B_n=None, lengths=None, device=0):
        self._lib = _lib.load()
        self._h = C.c_void_p()
        a = np.ascontiguousarray(A_n, dtype=np.float64)
        if a.ndim != 1:
            raise ValueError(f"A_n must be one-dimensional, got shape {np.shape(A_n)}")
        self.T = a.shape[0]
        b = None if B_n is None else _f64(B_n, self.T)
        offsets = None
        if lengths is not None:
            offsets = np.ascontiguousarray(np.concatenate([[0], np.cumsum(np.asarray(lengths, dtype=np.int64))]),
                                           dtype=np.int64)
        self.lengths = None if lengths is None else np.asarray(lengths, dtype=np.int64)
        self.cross = b is not None
        self.device = int(device)
        check(self._lib.mbar_b200_acf_create(
            self.device, self.T, _dptr(a), None if b is None else _dptr(b), 0 if offsets is None else len(offsets) - 1,
            None if offsets is None else _i64p(offsets), C.byref(self._h)))

    def inefficiency(self, starts, fast=False, mintime=3, multiple=False, navg=0.0, trace_cap=0, rule=None):
        """dict of per-start arrays: mean_a, mean_b, sigma2, g (before the g >= 1 clamp), last_lag, status
        (1: sigma^2 == 0) and, with trace_cap > 0, trace [n, trace_cap] (C at the first lag indices, NaN after the
        last).  multiple=True: statistical_inefficiency_multiple's loop (start 0 of a segmented object, navg the
        mean series length).  rule="fft": statistical_inefficiency_fft's loop (an autocorrelation, fast=False)."""
        if rule not in (None, "fft"):
            raise ValueError(f"unknown rule {rule!r}")
        if rule == "fft" and multiple:
            raise ValueError("rule='fft' and multiple=True exclude each other")
        code = 2 if rule == "fft" else (1 if multiple else 0)
        s = np.ascontiguousarray(np.atleast_1d(starts), dtype=np.int64)
        n = s.shape[0]
        out = {k: np.empty(n) for k in ("mean_a", "mean_b", "sigma2", "g")}
        out["last_lag"] = np.empty(n, np.int64)
        out["status"] = np.empty(n, np.int32)
        trace = np.empty((n, int(trace_cap))) if trace_cap > 0 else None
        check(self._lib.mbar_b200_acf_inefficiency(
            self._h, n, _i64p(s), int(bool(fast)), int(mintime), code, float(navg), int(trace_cap),
            _dptr(out["mean_a"]), _dptr(out["mean_b"]), _dptr(out["sigma2"]), _dptr(out["g"]), _i64p(out["last_lag"]),
            _i32p(out["status"]), None if trace is None else _dptr(trace)))
        if trace is not None:
            out["trace"] = trace
        return out

    def inefficiency_series(self, series, starts, fast=False, mintime=3):
        """`inefficiency` for requests on a segmented object: request r is series series[r] alone from starts[r]
        (counted from that series' first sample), the same bits as `inefficiency([starts[r]])` on an object holding
        that series alone.  dict of per-request arrays mean_a, mean_b, sigma2, g, last_lag, status."""
        k = np.ascontiguousarray(np.atleast_1d(series), dtype=np.int32)
        s = np.ascontiguousarray(np.atleast_1d(starts), dtype=np.int64)
        if k.shape != s.shape or k.ndim != 1:
            raise ValueError(f"series {k.shape} and starts {s.shape} must be matching 1-D arrays")
        n = s.shape[0]
        out = {key: np.empty(n) for key in ("mean_a", "mean_b", "sigma2", "g")}
        out["last_lag"] = np.empty(n, np.int64)
        out["status"] = np.empty(n, np.int32)
        check(self._lib.mbar_b200_acf_inefficiency_series(
            self._h, n, _i32p(k), _i64p(s), int(bool(fast)), int(mintime), _dptr(out["mean_a"]), _dptr(out["mean_b"]),
            _dptr(out["sigma2"]), _dptr(out["g"]), _i64p(out["last_lag"]), _i32p(out["status"])))
        return out

    def correlation(self, start, n_max):
        """(C [n_max + 1], mean_a, mean_b, sigma2) of the series from `start`."""
        Cn = np.empty(int(n_max) + 1)
        ma, mb, s2 = C.c_double(0), C.c_double(0), C.c_double(0)
        check(self._lib.mbar_b200_acf_correlation(self._h, int(start), int(n_max), _dptr(Cn), C.byref(ma),
                                                  C.byref(mb), C.byref(s2)))
        return Cn, ma.value, mb.value, s2.value

    def correlation_multiple(self, n_max, truncate=False):
        """(C, mean_a, mean_b, sigma2) of normalized_fluctuation_correlation_function_multiple over the object's
        series: C holds the entries the reference returns (n_max of them, or with truncate those before the first
        lag whose running numerator is negative)."""
        Cn = np.empty(int(n_max) + 1)
        count, ma, mb, s2 = C.c_int64(0), C.c_double(0), C.c_double(0), C.c_double(0)
        check(self._lib.mbar_b200_acf_correlation_multiple(self._h, int(n_max), int(bool(truncate)), _dptr(Cn),
                                                           C.byref(count), C.byref(ma), C.byref(mb), C.byref(s2)))
        return Cn[:count.value].copy(), ma.value, mb.value, s2.value

    def last_stats(self):
        """CUDA-event time (ms) of the last call, its lag rounds, the lag terms evaluated and those the stop rule
        needed (waste = terms / useful_terms)."""
        ms, rounds, terms, useful = C.c_double(0), C.c_int32(0), C.c_int64(0), C.c_int64(0)
        check(self._lib.mbar_b200_last_acf_stats(self._h, C.byref(ms), C.byref(rounds), C.byref(terms),
                                                 C.byref(useful)))
        return dict(ms=ms.value, rounds=rounds.value, terms=terms.value, useful_terms=useful.value,
                    waste=terms.value / useful.value if useful.value else 1.0)


WORK_KINDS = ("fermi", "fermi_moments", "exp", "gauss")      # MBAR_B200_WORK_* in this order


class DeviceWork(_Resident):
    """V work vectors resident on one H100 for the sums of pymbar.other_estimators (mbar_b200_work_*).  Independent of
    any DeviceProblem.

    `evaluate(vector, kind, c1, c2)` answers R requests in one device call and returns out [R, 3]: for kind "fermi"
    logsumexp of bar_zero's term at a = (w + c1) + c2, for "fermi_moments" logsumexp(t), logsumexp(2 t) and
    A = max(w + c1) of bar's uncertainty sums, for "exp" log(sum x) + max(-w), sum x and sum (x - mean x)^2 with
    x = exp(-w - max(-w)), for "gauss" sum w and sum (w - mean w)^2 (include/mbar_b200.h)."""

    _destroy = "mbar_b200_work_destroy"

    def __init__(self, vectors, device=0):
        self._lib = _lib.load()
        self._h = C.c_void_p()
        vs = [np.asarray(v) for v in vectors]
        if not vs or any(v.ndim != 1 for v in vs):
            raise ValueError("vectors must be a non-empty list of one-dimensional arrays")
        self.lengths = np.array([v.size for v in vs], dtype=np.int64)
        offsets = np.ascontiguousarray(np.concatenate([[0], np.cumsum(self.lengths)]), dtype=np.int64)
        w = np.ascontiguousarray(np.concatenate(vs) if vs else np.zeros(0), dtype=np.float64)
        self.device = int(device)
        check(self._lib.mbar_b200_work_create(self.device, w.shape[0], _dptr(w), len(vs), _i64p(offsets),
                                              C.byref(self._h)))

    def evaluate(self, vector, kind, c1, c2):
        """out [R, 3] for the requests (vector[r], kind[r], c1[r], c2[r]); a kind is a name of WORK_KINDS or its code."""
        v = np.ascontiguousarray(np.atleast_1d(vector), dtype=np.int32)
        k = np.ascontiguousarray([WORK_KINDS.index(x) if isinstance(x, str) and x in WORK_KINDS else
                                  (-1 if isinstance(x, str) else int(x)) for x in np.atleast_1d(kind)], dtype=np.int32)
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(c1, dtype=np.float64), v.shape))
        b = np.ascontiguousarray(np.broadcast_to(np.asarray(c2, dtype=np.float64), v.shape))
        if k.shape != v.shape:
            raise ValueError("vector and kind must have the same length")
        out = np.empty((v.shape[0], 3))
        check(self._lib.mbar_b200_work_evaluate(self._h, v.shape[0], _i32p(v), _i32p(k), _dptr(a), _dptr(b),
                                                _dptr(out)))
        return out

    def last_stats(self):
        """CUDA-event time (ms) of the last evaluate's kernels, its launches, the work values and bytes it read."""
        ms, launches, values = C.c_double(0), C.c_int32(0), C.c_int64(0)
        check(self._lib.mbar_b200_last_work_stats(self._h, C.byref(ms), C.byref(launches), C.byref(values)))
        return dict(ms=ms.value, launches=launches.value, values_read=values.value, bytes_read=8 * values.value)


class DeviceMbarBatch(_Resident):
    """P small MBAR problems (u_kn [K_p, N_p], N_k [K_p], 1 <= K_p <= 64) resident on one H100 and evaluated together
    (mbar_b200_batch_*).  Independent of any DeviceProblem.

    `moments(f_list)` returns each problem's S_k, log S_k, sum_n L_n, range flag and optionally the N-scaled Gram
    Ghat (two launches and one synchronisation for all of them); `solve(f_list)` runs the adaptive solver of
    DeviceProblem.solve_adaptive on every problem in lockstep, one moments call per iteration.

    Bootstrap replicates live in replicate slots (`set_replicates`): uint16 multiplicities c_n over one problem's
    samples.  `moments(..., slots=)` and `solve_replicates` evaluate a slot exactly as
    DeviceProblem.set_sample_weights(c) followed by the matching single-problem call would, in the same batched
    launches: S_k = sum_n c_n e^{a_kn}, Ghat_ij = sum_n c_n w_in w_jn and sum_L = sum_n c_n L_n."""

    _destroy = "mbar_b200_batch_destroy"
    MAX_K = 64
    MAX_ROWS = _lib.BATCH_MAX_ROWS     # K_p + M_p of a problem with appended rows

    def __init__(self, u_kn_list, N_k_list, device=0):
        self._lib = _lib.load()
        self._h = C.c_void_p()
        us = [np.asarray(u, dtype=np.float64) for u in u_kn_list]
        nks = [_f64(n) for n in N_k_list]
        if not us or len(us) != len(nks):
            raise ValueError("u_kn_list and N_k_list must be non-empty and of the same length")
        for p, (u, n) in enumerate(zip(us, nks)):
            if u.ndim != 2 or n.shape != (u.shape[0],):
                raise ValueError(f"problem {p}: u_kn {u.shape} and N_k {n.shape} do not match")
        self.P = len(us)
        self.slot_problems = np.zeros(0, np.int32)
        self.appended = np.zeros(self.P, np.int64)     # M_p: appended rows of each problem (set_unsampled)
        self.K = np.ascontiguousarray([u.shape[0] for u in us], dtype=np.int32)
        self.N = np.ascontiguousarray([u.shape[1] for u in us], dtype=np.int64)
        self.N_k = nks
        self.device = int(device)
        flat = np.empty(int(np.sum(self.K.astype(np.int64) * self.N)))
        o = 0
        for u in us:
            flat[o:o + u.size] = u.ravel()
            o += u.size
        Nk = np.ascontiguousarray(np.concatenate(nks))
        check(self._lib.mbar_b200_batch_create(self.device, self.P, _i32p(self.K), _i64p(self.N), _dptr(Nk),
                                               _dptr(flat), C.byref(self._h)))

    def set_replicates(self, problems, counts):
        """Replace the resident replicate slots: slot s holds the multiplicities counts[s] [N_p] of problem
        problems[s] (a sequence of 1-D arrays, or one [S, N] array when every slot's problem has N samples).  Counts
        lie in [0, 65535] (ValueError before anything changes) and sum to N_p; a bad problem index or sum raises the
        library's error and leaves no slot.  Each slot's sum_n c_n x_n is computed once, here.  An empty `problems`
        drops every slot."""
        problems = np.ascontiguousarray(problems, dtype=np.int32).reshape(-1)
        if len(counts) != problems.size:
            raise ValueError(f"need one count vector per slot: {problems.size} problems, {len(counts)} count vectors")
        parts = [np.asarray(c).reshape(-1) for c in counts]
        for s, c in enumerate(parts):
            if c.size and (c.min() < 0 or c.max() > 65535):
                raise ValueError(f"slot {s}: replicate counts must lie in [0, 65535]")
        flat = np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros(0), dtype=np.uint16)
        self.slot_problems = np.zeros(0, np.int32)
        check(self._lib.mbar_b200_batch_set_replicates(self._h, problems.size, _i32p(problems),
                                                       flat.ctypes.data_as(C.POINTER(C.c_uint16))))
        self.slot_problems = problems

    def moments(self, f_list, want_G=False, all_rows=False, problems=None, slots=None):
        """One dict per request (f_list[r] at problem problems[r], by default problem r): S [K_p], log_S [K_p],
        sum_L, flag and, with want_G, G = Ghat [K_p, K_p] (rows scaled by N_k; unsampled rows by 1 when all_rows,
        0 otherwise).  Unsampled rows of S and log_S are filled only when all_rows.

        slots: the requests name replicate slots instead (f_list[r] at slot slots[r], of problem
        slot_problems[slots[r]]) and every sum counts sample n c_n times, with the same range flag.  All-ones counts
        give the bits of the unweighted request."""
        if slots is not None and problems is not None:
            raise ValueError("a moments call names problems or slots, not both")
        weighted = slots is not None
        ids = np.ascontiguousarray(np.arange(len(f_list)) if not weighted and problems is None
                                   else (slots if weighted else problems), dtype=np.int32)
        if ids.shape != (len(f_list),) or len(f_list) == 0:
            raise ValueError("need one problem or slot index per f vector, and at least one")
        owner = self.slot_problems if weighted else np.arange(self.P)
        Ks = [int(self.K[owner[i]]) if 0 <= i < len(owner) else -1 for i in ids]
        call = self._lib.mbar_b200_batch_replicate_moments if weighted else self._lib.mbar_b200_batch_moments
        return self._requests(call, ids, f_list, Ks, want_G, int(bool(all_rows)))

    def solve(self, f_list=None, tol=1e-12, maxiter=10000, min_sc_iter=0, gamma=1.0):
        """(f_list, status [P], iterations [P]): the adaptive solver from f_list (zeros by default) on every problem.
        status 0 converged, 1 maxiter reached, 2 an iterate the batched sums could not represent (see
        mbar_b200_batch_solve).  Sampled states come back with f[first sampled] = 0, unsampled ones untouched."""
        if f_list is None:
            f_list = [np.zeros(K) for K in self.K]
        f = np.ascontiguousarray(np.concatenate([_f64(v, int(K)) for v, K in zip(f_list, self.K)]))
        status = np.empty(self.P, np.int32)
        iters = np.empty(self.P, np.int32)
        check(self._lib.mbar_b200_batch_solve(self._h, _dptr(f), float(tol), int(maxiter), int(min_sc_iter),
                                              float(gamma), _i32p(status), _i32p(iters)))
        return np.split(f, np.cumsum(self.K)[:-1]), status, iters

    def solve_replicates(self, f_list, tol=1e-12, maxiter=10000, min_sc_iter=0, gamma=1.0):
        """(f_list, status, iterations), one entry per replicate slot: the loop of `solve` (the same code, with slots
        as its units) on every slot in lockstep from f_list[s] [K_p], with the same status codes.  Each iteration is
        one weighted moments call for both candidates of every unfinished slot."""
        S = self.slot_problems.size
        Ks = [int(self.K[p]) for p in self.slot_problems]
        if len(f_list) != S:
            raise ValueError(f"need one f vector per slot ({S}), got {len(f_list)}")
        status = np.empty(S, np.int32)
        iters = np.empty(S, np.int32)
        if S == 0:
            return [], status, iters
        f = np.ascontiguousarray(np.concatenate([_f64(v, K) for v, K in zip(f_list, Ks)]))
        check(self._lib.mbar_b200_batch_solve_replicates(self._h, _dptr(f), float(tol), int(maxiter),
                                                         int(min_sc_iter), float(gamma), _i32p(status),
                                                         _i32p(iters)))
        return np.split(f, np.cumsum(Ks)[:-1]), status, iters

    def set_unsampled(self, problems, rows_list):
        """Replace the resident appended rows: problem problems[i] gets the unsampled rows rows_list[i] [M_i, N_p]
        on top of its own K_p (K_p + M_i <= MAX_ROWS), stored shifted by the problem's x_n.  NaN or -inf, a bad or
        repeated problem index or too many rows raise the library's error and leave no appended rows.  An empty
        `problems` drops them all."""
        problems = np.ascontiguousarray(problems, dtype=np.int32).reshape(-1)
        if len(rows_list) != problems.size:
            raise ValueError(f"need one row block per problem: {problems.size} problems, {len(rows_list)} blocks")
        parts = [np.asarray(r, dtype=np.float64) for r in rows_list]
        parts = [r.reshape(1, -1) if r.ndim == 1 else r for r in parts]
        for i, (p, r) in enumerate(zip(problems, parts)):
            if r.ndim != 2 or (0 <= p < self.P and r.shape[1] != self.N[p]):
                raise ValueError(f"entry {i}: rows {r.shape} do not match problem {p}")
        M = np.ascontiguousarray([r.shape[0] for r in parts], dtype=np.int32)
        flat = np.ascontiguousarray(np.concatenate([r.ravel() for r in parts]) if parts else np.zeros(0))
        self.appended = np.zeros(self.P, np.int64)
        check(self._lib.mbar_b200_batch_set_unsampled(self._h, problems.size, _i32p(problems), _i32p(M),
                                                      _dptr(flat)))
        self.appended[problems] = M

    def augmented_moments(self, f_list, want_G=False, problems=None, slots=None):
        """One dict per request (f_list[r] [R_p] at problem problems[r], by default problem r; R_p = K_p + M_p rows,
        the problem's own first): S [R_p], log_S [R_p], sum_L, flag and, with want_G, G = Ghat [R_p, R_p] (rows
        scaled by N_k where sampled, by 1 otherwise).  L_n comes from the sampled rows alone.  Appended weights are not
        shifted: ask for the Gram at a normalised f.  Two launches (three with the Gram) and one synchronisation for
        all requests.

        slots: the requests name replicate slots instead (f_list[r] [R_p] at slot slots[r], whose problem
        slot_problems[slots[r]] holds appended rows) and every sum counts sample n c_n times, L_n keeping N_k: the
        appended rows' -log S are the updates DeviceProblem.replicate_unsampled gives.  No Gram; two launches.  All-ones
        counts give the bits of the unweighted request."""
        if slots is not None and problems is not None:
            raise ValueError("an augmented moments call names problems or slots, not both")
        weighted = slots is not None
        if weighted and want_G:
            raise ValueError("weighted augmented moments have no Gram")
        ids = np.ascontiguousarray(np.arange(len(f_list)) if not weighted and problems is None
                                   else (slots if weighted else problems), dtype=np.int32)
        if ids.shape != (len(f_list),) or len(f_list) == 0:
            raise ValueError("need one problem or slot index per f vector, and at least one")
        owner = self.slot_problems if weighted else np.arange(self.P)
        Rs = [int(self.K[owner[i]] + self.appended[owner[i]]) if 0 <= i < len(owner) else -1 for i in ids]
        if weighted:
            return self._requests(self._lib.mbar_b200_batch_replicate_augmented_moments, ids, f_list, Rs, False,
                                  gram=False)
        return self._requests(self._lib.mbar_b200_batch_augmented_moments, ids, f_list, Rs, want_G)

    def bin_moments(self, problems, f_list, u_n_list, bin_list, nbins_list, want_C=True):
        """Histogram FES of every request in one call (mbar_b200_batch_bin_moments): request r is problem problems[r]
        at its converged f_list[r] [K_p], with the target state's u_n_list[r] [N_p] and dense bin indices bin_list[r]
        [N_p] in [0, nbins_list[r]).  Returns ([(f_bin [nbins], C [K_p, nbins], D [nbins]) per request], flags
        [n_requests] bool) with f_i = -log sum_{n in i} exp(-u_n - L_n), C_ki = sum_{n in i} W_nk w^_n,
        D_i = sum_{n in i} w^_n^2 and w^_n = exp(-u_n - L_n + f_i), what DeviceProblem.bin_moments gives for the
        problem.  want_C=False skips C and D: (f_bin, None, None).  A flagged request (an exponent above 700, a bin
        without a sample of finite weight) holds no usable values."""
        ids = np.ascontiguousarray(problems, dtype=np.int32).reshape(-1)
        n = ids.size
        if n == 0 or not (len(f_list) == len(u_n_list) == len(bin_list) == len(nbins_list) == n):
            raise ValueError("need one problem, f, u_n, bin index vector and bin count per request, and at least one")
        known = [0 <= p < self.P for p in ids]          # an unknown problem is the library's error
        Ks = [int(self.K[p]) if ok else 0 for p, ok in zip(ids, known)]
        us = [_f64(u) for u in u_n_list]
        bs = [np.asarray(b) for b in bin_list]
        for r, (u, b, p, ok) in enumerate(zip(us, bs, ids, known)):
            N = int(self.N[p]) if ok else u.shape[0]
            if u.shape != (N,) or b.shape != (N,):
                raise ValueError(f"request {r}: u_n {u.shape} and bin_n {b.shape} must have shape ({N},)")
        nb = np.ascontiguousarray(nbins_list, dtype=np.int32)
        f = np.ascontiguousarray(np.concatenate([_f64(v, K) if ok else _f64(v) for v, K, ok in zip(f_list, Ks, known)]))
        u = np.ascontiguousarray(np.concatenate(us))
        b = np.ascontiguousarray(np.concatenate(bs), dtype=np.int32)
        f_bin = np.empty(int(nb.astype(np.int64).sum()))
        C_ = np.empty(int(np.dot(np.asarray(Ks, np.int64), nb))) if want_C else None
        D = np.empty(f_bin.size) if want_C else None
        flag = np.empty(n, np.int32)
        check(self._lib.mbar_b200_batch_bin_moments(self._h, n, _i32p(ids), _dptr(f), _dptr(u), _i32p(b), _i32p(nb),
                                                    _dptr(f_bin), _dptr(C_) if want_C else None,
                                                    _dptr(D) if want_C else None, _i32p(flag)))
        out, o, c = [], 0, 0
        for K, m in zip(Ks, nb.tolist()):
            out.append((f_bin[o:o + m], C_[c:c + K * m].reshape(K, m), D[o:o + m]) if want_C else
                       (f_bin[o:o + m], None, None))
            o += m
            c += K * m
        return out, flag.astype(bool)

    def replicate_bin_moments(self, target_problems, u_n_list, bin_list, nbins_list, slots, targets, f_list):
        """Histogram FES of replicate slots in one call (mbar_b200_batch_replicate_bin_moments).  Target t is problem
        target_problems[t] with the target state's u_n_list[t] [N_p] and dense bin indices bin_list[t] [N_p] in
        [0, nbins_list[t]), uploaded once; request r is slot slots[r] at its replicate's converged f_list[r] [K_p]
        against target targets[r] of the slot's problem.  Returns ([f_bin [nbins]] per request, flags bool) with
        f_i = -log sum_{n in i} c_n exp(-u_n - L_n), L_n keeping N_k: what set_sample_weights(c) and
        DeviceProblem.bin_moments(want_C=False) give.  A flagged request holds no usable values."""
        tp = np.ascontiguousarray(target_problems, dtype=np.int32).reshape(-1)
        if tp.size == 0 or not (len(u_n_list) == len(bin_list) == len(nbins_list) == tp.size):
            raise ValueError("need one problem, u_n, bin index vector and bin count per target, and at least one")
        sl = np.ascontiguousarray(slots, dtype=np.int32).reshape(-1)
        tg = np.ascontiguousarray(targets, dtype=np.int32).reshape(-1)
        if sl.size == 0 or not (tg.size == len(f_list) == sl.size):
            raise ValueError("need one slot, target and f vector per request, and at least one")
        us = [_f64(u) for u in u_n_list]
        bs = [np.asarray(b) for b in bin_list]
        for t, (u, b, p) in enumerate(zip(us, bs, tp)):
            N = int(self.N[p]) if 0 <= p < self.P else u.shape[0]   # an unknown problem is the library's error
            if u.shape != (N,) or b.shape != (N,):
                raise ValueError(f"target {t}: u_n {u.shape} and bin_n {b.shape} must have shape ({N},)")
        nb = np.ascontiguousarray(nbins_list, dtype=np.int32)
        owner = self.slot_problems
        Ks = [int(self.K[owner[s]]) if 0 <= s < len(owner) else None for s in sl]
        f = np.ascontiguousarray(np.concatenate([_f64(v) if K is None else _f64(v, K) for v, K in zip(f_list, Ks)]))
        out_nb = [int(nb[t]) if 0 <= t < nb.size else 0 for t in tg]
        f_bin = np.empty(sum(out_nb))
        flag = np.empty(sl.size, np.int32)
        check(self._lib.mbar_b200_batch_replicate_bin_moments(
            self._h, tp.size, _i32p(tp), _dptr(np.ascontiguousarray(np.concatenate(us))),
            _i32p(np.ascontiguousarray(np.concatenate(bs), dtype=np.int32)), _i32p(nb), sl.size, _i32p(sl), _i32p(tg),
            _dptr(f), _dptr(f_bin), _i32p(flag)))
        return np.split(f_bin, np.cumsum(out_nb)[:-1]), flag.astype(bool)

    def log_weights(self, problems, f_list, u_n_list):
        """Target-state log weights of every request in one call (mbar_b200_batch_log_weights): request r is problem
        problems[r] at its converged f_list[r] [K_p] with the target state's u_n_list[r] [N_p].  Returns ([log_w [N_p]
        per request], flags bool) with log w_n = -u_n - L_n, L_n = log sum_{k sampled} N_k exp(f_k - u_kn); u_n = +inf
        gives -inf.  A flagged request holds a NaN log w_n."""
        ids = np.ascontiguousarray(problems, dtype=np.int32).reshape(-1)
        n = ids.size
        if n == 0 or not (len(f_list) == len(u_n_list) == n):
            raise ValueError("need one problem, f and u_n per request, and at least one")
        known = [0 <= p < self.P for p in ids]          # an unknown problem is the library's error
        us = [_f64(u) for u in u_n_list]
        for r, (u, p, ok) in enumerate(zip(us, ids, known)):
            if ok and u.shape != (int(self.N[p]),):
                raise ValueError(f"request {r}: u_n {u.shape} must have shape ({int(self.N[p])},)")
        f = np.ascontiguousarray(np.concatenate([_f64(v, int(self.K[p])) if ok else _f64(v)
                                                 for v, p, ok in zip(f_list, ids, known)]))
        u = np.ascontiguousarray(np.concatenate(us))
        out = np.empty(u.size)
        flag = np.empty(n, np.int32)
        check(self._lib.mbar_b200_batch_log_weights(self._h, n, _i32p(ids), _dptr(f), _dptr(u), _dptr(out),
                                                    _i32p(flag)))
        return np.split(out, np.cumsum([u.size for u in us])[:-1]), flag.astype(bool)

    def _requests(self, call, ids, f_list, rows, want_G, *flags, gram=True):
        """One batched moments call on requests f_list[r] [rows[r]] at units ids[r], `flags` passed after f; one dict
        per request: S, log_S, sum_L, flag and, with want_G, G [rows[r], rows[r]].  gram=False: `call` takes no Gram
        argument."""
        f = np.ascontiguousarray(np.concatenate([_f64(v, R) for v, R in zip(f_list, rows)]))
        S, logS = np.empty(f.size), np.empty(f.size)
        sumL = np.empty(len(rows))
        flag = np.empty(len(rows), np.int32)
        G = np.empty(sum(R * R for R in rows)) if want_G else None
        check(call(self._h, len(rows), _i32p(ids), _dptr(f), *flags, _dptr(S), _dptr(logS), _dptr(sumL), _i32p(flag),
                   *((_dptr(G) if want_G else None,) if gram else ())))
        out, o, g = [], 0, 0
        for r, R in enumerate(rows):
            d = dict(S=S[o:o + R], log_S=logS[o:o + R], sum_L=float(sumL[r]), flag=bool(flag[r]))
            if want_G:
                d["G"] = G[g:g + R * R].reshape(R, R)
            out.append(d)
            o += R
            g += R * R
        return out

    def last_stats(self):
        """CUDA-event time (ms) of the last moments, solve, solve_replicates or augmented_moments call's kernels,
        its launches, iterations and the bytes of u_kn tiles (appended tiles, replicate counts) it read."""
        ms, launches, iters, nbytes = C.c_double(0), C.c_int32(0), C.c_int32(0), C.c_int64(0)
        check(self._lib.mbar_b200_last_batch_stats(self._h, C.byref(ms), C.byref(launches), C.byref(iters),
                                                   C.byref(nbytes)))
        return dict(ms=ms.value, launches=launches.value, iterations=iters.value, bytes_read=nbytes.value)


def measure_fp64_peak(device=0):
    """(DMMA TFLOP/s, DFMA TFLOP/s) of this GPU from register-only loops (mbar_b200_measure_fp64_peak)."""
    a, b = C.c_double(0), C.c_double(0)
    check(_lib.load().mbar_b200_measure_fp64_peak(int(device), C.byref(a), C.byref(b)))
    return a.value, b.value


def probe_exp(a, which=0, device=0):
    """exp(a) through the device's own exp (mbar_b200_probe_exp): which = 0 exp_fast, 1 the fused pass with the
    constant in the exponent (MODE=1), 2 the fused pass's multiplicative form (MODE=3).  Development aid."""
    a = np.ascontiguousarray(a, dtype=np.float64).ravel()
    out = np.empty_like(a)
    check(_lib.load().mbar_b200_probe_exp(int(device), int(which), a.size, _dptr(a), _dptr(out)))
    return out


def gpu_numa_node(device=0):
    """NUMA node of the GPU's PCI function (-1: the host exposes none)."""
    n = C.c_int(-1)
    check(_lib.load().mbar_b200_gpu_numa_node(int(device), C.byref(n)))
    return n.value

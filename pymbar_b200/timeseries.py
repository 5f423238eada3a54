"""The host side of pymbar.timeseries (timeseries.py:83-836) over the lag sums of a `DeviceAcf`.

`statistical_inefficiency`, `statistical_inefficiency_multiple`, `normalized_fluctuation_correlation_function` and
`detect_equilibration` take the reference's arguments and return what it returns.  The device evaluates every
centred lag sum, the stop rule and the g accumulation in the reference's fp64 operations; only the order of the sums
differs from numpy's pairwise one, so g, C and sigma^2 agree to a few ulps times the chunk length (DESIGN.md §3.5d),
and `detect_equilibration` gets every start of the series in one device call instead of one numpy pass per start
and lag.

Starts whose remaining series is constant are the one place where the order of a sum changes the answer: the
reference raises ParameterError (sigma^2 = 0, g = T - t + 1 in detect_equilibration, pymbar issue #122) when numpy's
mean of the repeated value is exact, and otherwise runs its loop on the rounding noise of that mean.  Such starts are
answered on the host: g = T - t + 1 when the mean is exact in any order (the value has at most 53 - ceil(log2 T)
significant bits), else `_host_inefficiency`, the reference's loop in the reference's numpy operations.  They have
Neff close to 1, and a long inexact constant tail costs what it costs in the reference.

`normalized_fluctuation_correlation_function_multiple`, `statistical_inefficiency_fft` and
`detect_equilibration_binary_search` (timeseries.py:509-658, :839-970) take the reference's arguments and return its
values and types.  The FFT functions need no statsmodels: the device evaluates statsmodels' acf(adjusted=True) by
direct lag sums up to the stop lag, which is the same C(t) in exact arithmetic and the more accurate of the two in
fp64.  Where the reference's answer is not reproducible (a constant remaining series, whose statsmodels acf divides
rounding noise by rounding noise, or sigma^2 = 0) or the input is not a 1-D float64 or integer array, these raise
`NotOnDevice`, and the facade calls the original.

`detect_equilibration_many`, `statistical_inefficiency_many` and `subsample_correlated_data_many` return what a loop
of the single-series functions returns, with every start of every series in one segmented device call per wave
(DESIGN.md §3.5d′).  The single and many-series functions share their host halves (`_si_plan` / `_si_finish`,
`_eq_plan` / `_EqPlan.finish`).
"""
from __future__ import annotations

import math

import numpy as np

from . import utils as _u

DeviceAcf = None          # the device class; resolved on first use (a test may put a stand-in here)


def _device(A, B=None, lengths=None):
    global DeviceAcf
    from . import mbar_solvers as ms

    if DeviceAcf is None:
        DeviceAcf = ms.DeviceAcf
    return DeviceAcf(A, B, lengths=lengths, device=ms._DEVICE)


def _parameter_error(msg):
    # looked up at raise time: install() makes it pymbar's own ParameterError
    return _u.ParameterError(msg)


class NotOnDevice(Exception):
    """The input has no device answer that reproduces the reference's; the caller runs the reference instead."""


def _device_series(x):
    """x as float64 if it is a 1-D float64 or integer ndarray, else NotOnDevice."""
    if not isinstance(x, np.ndarray) or x.ndim != 1 or not (x.dtype == np.float64 or x.dtype.kind in "iu"):
        raise NotOnDevice("input is not a 1-D float64 or integer array")
    return np.ascontiguousarray(x, dtype=np.float64)


def lag(i, fast):
    """The lag of lag index i (0, 1, ...): 1, 2, 3, ... or, fast, 1, 2, 4, 7, 11, ... (increments 1, 2, 3, ...)."""
    i = np.asarray(i, dtype=np.int64)
    return 1 + i * (i + 1) // 2 if fast else i + 1


def lag_count(last_lag, fast):
    """How many lags the loop evaluated when the last one was last_lag (0: none)."""
    if last_lag <= 0:
        return 0
    if not fast:
        return int(last_lag)
    i = int(math.isqrt(2 * int(last_lag)))
    while lag(i, True) > last_lag:
        i -= 1
    while lag(i + 1, True) <= last_lag:
        i += 1
    return i + 1


def mean_is_exact(value, T):
    """True when the mean of up to T copies of `value` is exact whatever the order of the sum: its significand has at
    most 53 - ceil(log2 T) significant bits, so every partial sum k * value is representable."""
    if value == 0.0:
        return True
    mant, _ = math.frexp(float(value))
    bits = int(abs(mant) * 2 ** 53)
    sig = 53 - ((bits & -bits).bit_length() - 1)
    return sig <= 53 - math.ceil(math.log2(max(int(T), 2)))


def _constant(x):
    return x.size > 0 and bool(np.all(x == x[0]))


def _host_inefficiency(A, B, fast, mintime):
    """The reference's statistical_inefficiency loop (timeseries.py:152-196) in its own numpy operations, for series
    whose device answer would differ only because of the order of a sum (constant series).  g before the clamp, or
    None where sigma^2 == 0."""
    B = A if B is None else B
    N = A.size
    dA = A.astype(np.float64) - A.mean()
    dB = B.astype(np.float64) - B.mean()
    s2 = (dA * dB).mean()
    if s2 == 0:
        return None
    g, t, inc = 1.0, 1, 1
    while t < N - 1:
        C = np.sum(dA[0:N - t] * dB[t:N] + dB[0:N - t] * dA[t:N]) / (2.0 * float(N - t) * s2)
        if C <= 0.0 and t > mintime:
            break
        g += 2.0 * C * (1.0 - float(t) / float(N)) * float(inc)
        t += inc
        if fast:
            inc += 1
    return g


def neff(count, g32):
    """(T - t + 1) / g_t[t] as detect_equilibration evaluates it (a Python int over a float32 scalar), elementwise:
    a float32 division under numpy >= 2 (NEP 50); under numpy 1 a float32 division for counts below 2**16 and a
    float64 one, rounded to float32, above."""
    count = np.asarray(count, dtype=np.int64)
    g32 = np.asarray(g32, dtype=np.float32)
    if int(np.__version__.split(".")[0]) >= 2:
        return count.astype(np.float32) / g32
    small = count < 2 ** 16
    out = (count.astype(np.float64) / g32.astype(np.float64)).astype(np.float32)
    out[small] = count[small].astype(np.float32) / g32[small]
    return out


def _si_plan(A_n, B_n, fast, mintime):
    """statistical_inefficiency up to the device call: (a, b, None) with the float64 series the device answers, or
    (None, None, [g]) where the host answers (a constant series; g None where sigma^2 == 0)."""
    A = np.array(A_n)
    B = None if B_n is None else np.array(B_n)
    if B is not None and A.shape != B.shape:
        raise _parameter_error("A_n and B_n must have same dimensions.")
    a = np.ascontiguousarray(A.ravel(), dtype=np.float64)
    b = None if B is None else np.ascontiguousarray(B.ravel(), dtype=np.float64)
    if _constant(a) or (b is not None and _constant(b)):
        return None, None, [_host_inefficiency(A.ravel(), None if B is None else B.ravel(), fast, mintime)]
    return a, b, None


def _si_finish(g):
    """statistical_inefficiency's answer from g before the clamp (None: sigma^2 == 0)."""
    if g is None:
        raise _parameter_error("Sample covariance sigma_AB^2 = 0 -- cannot compute statistical inefficiency")
    return 1.0 if g < 1.0 else g


def _device_g(r, k):
    return None if r["status"][k] else float(r["g"][k])


def statistical_inefficiency(A_n, B_n=None, fast=False, mintime=3):
    """statistical_inefficiency (timeseries.py:83-203) without fft: g >= 1 of one series, or of two."""
    a, b, host = _si_plan(A_n, B_n, fast, mintime)
    if host is not None:
        return _si_finish(host[0])
    with _device(a, b) as dev:
        r = dev.inefficiency([0], fast=fast, mintime=mintime)
    return _si_finish(_device_g(r, 0))


def _series_list(A_kn):
    if isinstance(A_kn, np.ndarray):
        return [A_kn.copy()] if A_kn.ndim == 1 else [A_kn[k, :].copy() for k in range(A_kn.shape[0])]
    return list(A_kn)


def statistical_inefficiency_multiple(A_kn, fast=False, return_correlation_function=False):
    """statistical_inefficiency_multiple (timeseries.py:209-365): g of K series of possibly different lengths, and
    with return_correlation_function the reference's [(t, C), ...].  A constant input (sigma^2 = 0 or rounding noise
    in the reference) raises ParameterError."""
    series = _series_list(A_kn)
    N_k = np.array([np.asarray(x).size for x in series], np.int32)
    navg = np.array(N_k, np.float64).mean()
    a = np.concatenate([np.asarray(x, dtype=np.float64).ravel() for x in series])
    if _constant(a):
        raise _parameter_error("constant series: sigma^2 is 0 or rounding noise")
    nmax = int(N_k.max())
    cap = 0
    if return_correlation_function:
        cap = lag_count(nmax - 2, fast) if nmax > 2 else 0
    with _device(a, lengths=N_k.astype(np.int64)) as dev:
        r = dev.inefficiency([0], fast=fast, multiple=True, navg=navg, trace_cap=cap)
    if r["status"][0]:
        raise _parameter_error("Sample covariance sigma^2 = 0 -- cannot compute statistical inefficiency")
    g = float(r["g"][0])
    g = 1.0 if g < 1.0 else g
    if not return_correlation_function:
        return g
    n = lag_count(int(r["last_lag"][0]), fast)
    ts = lag(np.arange(n), fast)
    return g, [(int(t), np.float64(C)) for t, C in zip(ts, r["trace"][0, :n])] if cap else []


def normalized_fluctuation_correlation_function(A_n, B_n=None, N_max=None, norm=True):
    """normalized_fluctuation_correlation_function (timeseries.py:405-503): C(t), t = 0 .. N_max, or with
    norm=False C(t) sigma^2 + mu_A mu_B."""
    A = np.array(A_n)
    B = None if B_n is None else np.array(B_n)
    N = A.size
    if (not N_max) or (N_max > N - 1):
        N_max = N - 1
    if B is not None and A.shape != B.shape:
        raise _parameter_error("A_n and B_n must have same dimensions.")
    a = np.ascontiguousarray(A.ravel(), dtype=np.float64)
    b = None if B is None else np.ascontiguousarray(B.ravel(), dtype=np.float64)
    if _constant(a) or (b is not None and _constant(b)):
        Bh = A if B is None else B
        dA = A.astype(np.float64) - A.mean()
        dB = Bh.astype(np.float64) - Bh.mean()
        s2 = (dA * dB).mean()
        if s2 == 0:
            raise _parameter_error("Sample covariance sigma_AB^2 = 0 -- cannot compute statistical inefficiency")
        dA, dB = dA.ravel(), dB.ravel()
        C = np.array([np.sum(dA[0:N - t] * dB[t:N] + dB[0:N - t] * dA[t:N]) / (2.0 * float(N - t) * s2)
                      for t in range(N_max + 1)])
        mu_a, mu_b = A.mean(), Bh.mean()
    else:
        with _device(a, b) as dev:
            C, mu_a, mu_b, s2 = dev.correlation(0, N_max)
    return C if norm else C * s2 + mu_a * mu_b


class _EqPlan:
    """detect_equilibration up to the device call: the starts, which of them go to the device (`on_dev`), and g /
    sigma^2 == 0 (`zero`) of those answered on the host (a constant remaining series)."""

    def __init__(self, A_t, fast, nskip):
        T = self.T = A_t.size
        self.a = np.ascontiguousarray(np.asarray(A_t).ravel(), dtype=np.float64)
        a = self.a
        self.g_t = np.ones([T - 1], np.float32)
        self.starts = np.arange(0, T - 1, nskip, dtype=np.int64)
        differs = np.flatnonzero(a != a[-1])
        tail = int(differs[-1]) + 1 if differs.size else 0          # A[t:] is constant for t >= tail
        self.g = np.ones(self.starts.size)
        self.zero = np.zeros(self.starts.size, bool)
        self.on_dev = self.starts < tail
        exact = mean_is_exact(a[-1], T)
        for k in np.flatnonzero(~self.on_dev):
            t = int(self.starts[k])
            gk = None if exact else _host_inefficiency(np.asarray(A_t).ravel()[t:T], None, fast, 3)
            if gk is None:
                self.zero[k] = True
            else:
                self.g[k] = gk

    def finish(self, r=None):
        """(t, g, Neff_max) from the device's answers r (a dict of g and status over starts[on_dev])."""
        T, starts, g, zero, g_t = self.T, self.starts, self.g, self.zero, self.g_t
        if r is not None:
            g[self.on_dev] = r["g"]
            zero[self.on_dev] = r["status"] != 0
        Neff_t = np.ones([T - 1], np.float32)
        g_t[starts] = np.where(g < 1.0, 1.0, g)
        g_t[starts[zero]] = T - starts[zero] + 1
        Neff_t[starts] = neff(T - starts + 1, g_t[starts])
        Neff_max = Neff_t.max()
        t = Neff_t.argmax()
        return t, g_t[t], Neff_max


def _eq_plan(A_t, fast, nskip):
    """detect_equilibration's early answer (a series whose numpy std is 0) or its _EqPlan."""
    if A_t.std() == 0.0:
        return 0, 1, 1
    return _EqPlan(A_t, fast, nskip)


def detect_equilibration(A_t, fast=True, nskip=1):
    """detect_equilibration (timeseries.py:771-836): (t, g, Neff_max) as np.int64, np.float32, np.float32, every
    start in one device call."""
    plan = _eq_plan(A_t, fast, nskip)
    if isinstance(plan, tuple):
        return plan
    r = None
    if plan.on_dev.any():
        with _device(plan.a) as dev:
            r = dev.inefficiency(plan.starts[plan.on_dev], fast=fast, mintime=3)
    return plan.finish(r)


def normalized_fluctuation_correlation_function_multiple(A_kn, B_kn=None, N_max=None, norm=True, truncate=False):
    """normalized_fluctuation_correlation_function_multiple (timeseries.py:509-658): C(t) over K series with pooled
    means, in one device call; the reference's C_n[:t] (with norm=False C sigma^2 + mu_A mu_B)."""
    cross = B_kn is not None
    if B_kn is None:
        B_kn = A_kn
    if (type(A_kn) is not list) or (type(B_kn) is not list):
        raise _parameter_error("A_kn and B_kn must each be a list of numpy arrays.")
    if len(A_kn) != len(B_kn):
        raise _parameter_error("A_kn and B_kn must contain corresponding timeseries -- different numbers of "
                               "timeseries detected in each.")
    A = [_device_series(x) for x in A_kn]
    B = [_device_series(x) for x in B_kn] if cross else A
    if any(x.size != y.size for x, y in zip(A, B)):
        raise _parameter_error("A_kn and B_kn must contain corresponding timeseries -- lack of correspondence in "
                               "timeseries lenghts detected.")
    N_k = np.array([x.size for x in A], np.int64)
    if N_k.size == 0 or N_k.sum() == 0:
        raise NotOnDevice("no samples")
    if (not N_max) or (N_max > N_k.max() - 1):
        N_max = int(N_k.max()) - 1
    if not isinstance(N_max, (int, np.integer)) or N_max < 0:
        raise NotOnDevice(f"N_max = {N_max!r}")
    keep = [k for k in range(N_k.size) if N_k[k] > 0]        # empty series add nothing to any sum
    a = np.concatenate([A[k] for k in keep])
    b = np.concatenate([B[k] for k in keep]) if cross else None
    if _constant(a) or (b is not None and _constant(b)):
        raise NotOnDevice("constant series: sigma^2 is 0 or rounding noise")
    with _device(a, b, lengths=N_k[keep]) as dev:
        C, mu_a, mu_b, s2 = dev.correlation_multiple(int(N_max), truncate=bool(truncate))
    return C if norm else C * s2 + mu_a * mu_b


def _fft_g(dev, starts, mintime):
    """g before the clamp of statistical_inefficiency_fft for each start of the device series."""
    mintime = min(max(int(mintime), -1), 2 ** 31 - 1)          # t >= 1: every mintime < 0 acts as -1
    r = dev.inefficiency(starts, mintime=mintime, rule="fft")
    if np.any(r["status"] != 0):
        raise NotOnDevice("sigma^2 = 0")
    return r["g"]


def statistical_inefficiency_fft(A_n, mintime=3):
    """statistical_inefficiency_fft (timeseries.py:839-898) without statsmodels: max(1.0, g)."""
    a = _device_series(np.array(A_n))
    if a.size < 2 or _constant(a):
        raise NotOnDevice("fewer than 2 samples or a constant series")
    if isinstance(mintime, bool) or not isinstance(mintime, (int, np.integer)):
        raise NotOnDevice(f"mintime = {mintime!r}")
    with _device(a) as dev:
        g = np.float64(_fft_g(dev, [0], mintime)[0])
    return max(1.0, g)


def detect_equilibration_binary_search(A_t, bs_nodes=10):
    """detect_equilibration_binary_search (timeseries.py:901-970): the reference's grid and window updates on the
    host, each round's starts in one device call; (t, g, Neff_max) as np.int64, np.float64, np.float64."""
    assert bs_nodes > 4, "Number of nodes for binary search must be > 4"
    a = _device_series(A_t)
    T = A_t.size
    if T < 2:
        raise NotOnDevice("fewer than 2 samples")
    if A_t.std() == 0.0:
        return 0, 1, T
    if _constant(a):                 # numpy's std of a constant series is rounding noise when its mean is inexact
        raise NotOnDevice("constant series")
    tail = int(np.flatnonzero(a != a[-1])[-1]) + 1               # A[t:] is constant for t >= tail
    start = 1
    end = T - 1
    n_grid = min(bs_nodes, T)
    with _device(a) as dev:
        while True:
            time_grid = np.unique((10 ** np.linspace(np.log10(start), np.log10(end), n_grid)).round().astype("int"))
            g_t = np.ones(time_grid.size)
            Neff_t = np.ones(time_grid.size)
            on = time_grid < T - 1
            if on.any():
                s = time_grid[on]
                if s.max() >= tail:
                    raise NotOnDevice("constant remaining series")
                g = _fft_g(dev, s, 3)
                g_t[on] = np.where(g > 1.0, g, 1.0)
                Neff_t[on] = (T - s + 1) / g_t[on]
            Neff_max = Neff_t.max()
            k = Neff_t.argmax()
            t = time_grid[k]
            g = g_t[k]
            if end - start < 4:
                break
            if k == 0:
                start = time_grid[0]
                end = time_grid[1]
            elif k == time_grid.size - 1:
                start = time_grid[-2]
                end = time_grid[-1]
            else:
                start = time_grid[k - 1]
                end = time_grid[k + 1]
    return t, g, Neff_max


# ---- many series in lockstep ----------------------------------------------------------------------------------------
# The _many functions return what a list comprehension over the single-series function returns, and raise the
# exception of the lowest-index failing series.  Every device request (series, start) of every series goes to one
# segmented DeviceAcf and its `inefficiency_series`, whose answers are the single-series call's bits; requests go in
# waves of at most WAVE_BYTES // REQUEST_BYTES, which changes no bits.  A series that cannot be a segment (empty, or
# with a non-finite value) is answered by the single-series function, so that its own error is the one raised.

WAVE_BYTES = 1 << 30        # device footprint of the requests of one inefficiency_series call
REQUEST_BYTES = 96          # device bytes per request (starts, series, means, sigma^2, g, last lag, status, order)
LAST_MANY_STATS = {}        # waves, rounds, kernel ms, lag terms and requests of the last _many device work


def _segmentable(a, b):
    return a.size > 0 and bool(np.all(np.isfinite(a))) and (b is None or bool(np.all(np.isfinite(b))))


def _many_requests(series, cross, ser, starts, fast, mintime):
    """(g, status) of requests (series ser[r], start starts[r]) over the float64 series [(a, b)], one segmented
    DeviceAcf (autocorrelation, or cross when `cross`) and one inefficiency_series call per wave."""
    n = ser.size
    g = np.empty(n)
    status = np.empty(n, np.int32)
    a = np.concatenate([x for x, _ in series])
    b = np.concatenate([y for _, y in series]) if cross else None
    lengths = np.array([x.size for x, _ in series], np.int64)
    per = max(1, int(WAVE_BYTES) // REQUEST_BYTES)
    st = LAST_MANY_STATS
    with _device(a, b, lengths=lengths) as dev:
        for w0 in range(0, n, per):
            r = dev.inefficiency_series(ser[w0:w0 + per], starts[w0:w0 + per], fast=fast, mintime=mintime)
            g[w0:w0 + per] = r["g"]
            status[w0:w0 + per] = r["status"]
            s = dev.last_stats() if hasattr(dev, "last_stats") else {}
            st["waves"] = st.get("waves", 0) + 1
            for k in ("rounds", "ms", "terms"):
                st[k] = st.get(k, 0) + s.get(k, 0)
    st["requests"] = st.get("requests", 0) + n
    return g, status


def _raise_lowest(errors):
    if errors:
        raise errors[min(errors)]


def statistical_inefficiency_many(A_list, B_list=None, fast=False, mintime=3):
    """`statistical_inefficiency(A_list[i], B_list[i], fast, mintime)` for every series: a float64 array of g >= 1,
    every device series in one call per wave (autocorrelations and cross-correlations in one object each)."""
    LAST_MANY_STATS.clear()
    n = len(A_list)
    if B_list is not None and len(B_list) != n:
        raise ValueError(f"{n} series A but {len(B_list)} series B")
    out = np.ones(n)
    errors = {}
    groups = {False: [], True: []}                 # cross -> [(i, a, b)]
    for i in range(n):
        B_i = None if B_list is None else B_list[i]
        try:
            a, b, host = _si_plan(A_list[i], B_i, fast, mintime)
            if host is not None:
                out[i] = _si_finish(host[0])
            elif not _segmentable(a, b):
                out[i] = statistical_inefficiency(A_list[i], B_i, fast, mintime)
            else:
                groups[b is not None].append((i, a, b))
        except Exception as e:                  # noqa: BLE001  (re-raised below, lowest index first)
            errors[i] = e
            break                               # the series after it cannot change what is raised
    first = min(errors) if errors else n
    for cross, items in groups.items():
        items = [x for x in items if x[0] < first]
        if not items:
            continue
        k = np.arange(len(items), dtype=np.int32)
        g, status = _many_requests([(a, b) for _, a, b in items], cross, k, np.zeros(k.size, np.int64), fast,
                                   mintime)
        for (i, _, _), gi, si in zip(items, g, status):
            try:
                out[i] = _si_finish(None if si else float(gi))
            except Exception as e:              # noqa: BLE001
                errors[i] = e
    _raise_lowest(errors)
    return out


def detect_equilibration_many(A_list, fast=True, nskip=1):
    """`detect_equilibration(A, fast, nskip)` for every series: a list of (t, g, Neff_max), every start of every series
    in one device call per wave, with the lag rounds shared by all series."""
    LAST_MANY_STATS.clear()
    n = len(A_list)
    out = [None] * n
    errors = {}
    plans = []                                  # (i, plan) of the series with device starts
    for i in range(n):
        try:
            plan = _eq_plan(A_list[i], fast, nskip)
            if isinstance(plan, tuple):
                out[i] = plan
            elif not plan.on_dev.any():
                out[i] = plan.finish()
            elif not _segmentable(plan.a, None):
                out[i] = detect_equilibration(A_list[i], fast, nskip)
            else:
                plans.append((i, plan))
        except Exception as e:                  # noqa: BLE001  (re-raised below, lowest index first)
            errors[i] = e
            break
    if plans:
        counts = np.array([int(p.on_dev.sum()) for _, p in plans], np.int64)
        ser = np.repeat(np.arange(len(plans), dtype=np.int32), counts)
        starts = np.concatenate([p.starts[p.on_dev] for _, p in plans])
        g, status = _many_requests([(p.a, None) for _, p in plans], False, ser, starts, fast, 3)
        off = np.concatenate([[0], np.cumsum(counts)])
        for k, (i, p) in enumerate(plans):
            out[i] = p.finish(dict(g=g[off[k]:off[k + 1]], status=status[off[k]:off[k + 1]]))
    _raise_lowest(errors)
    return out


def _subsample_indices(T, g, conservative):
    """The indices subsample_correlated_data keeps of T samples for a statistical inefficiency g: stride ceil(g) when
    conservative, else round(n g) for n = 0, 1, 2, ... while below T, each index once."""
    if conservative:
        return list(range(0, T, int(math.ceil(g))))
    if not g > 0:
        raise ValueError(f"g = {g!r}: the indices round(n g) never reach T")
    # n g as Python evaluates it for a scalar g: float64, or g's own precision for a numpy float
    dtype = g.dtype if isinstance(g, np.floating) else np.float64
    n = np.arange(int(math.floor((T + 0.5) / float(g))) + 2).astype(dtype)
    t = np.round(n * g)
    t = t[t < T]
    return np.unique(t).astype(np.int64).tolist()


def subsample_correlated_data_many(A_list, g=None, fast=False, conservative=False):
    """`pymbar.timeseries.subsample_correlated_data(A_list[i], g_i, fast, conservative)` for every series: one index
    list per series.  g is None, one value for every series or one value per series; the series whose g is falsy get
    g from one statistical_inefficiency_many call (the reference's statistical_inefficiency(A, A, fast): a
    cross-correlation of a series with itself is its autocorrelation, bit for bit)."""
    A = [np.array(x) for x in A_list]
    n = len(A)
    gs = [g] * n if g is None or np.ndim(g) == 0 else list(g)
    if len(gs) != n:
        raise ValueError(f"{len(gs)} values of g for {n} series")
    need = [i for i in range(n) if not gs[i]]
    if need:
        for i, gi in zip(need, statistical_inefficiency_many([A[i] for i in need], fast=fast)):
            gs[i] = float(gi)
    return [_subsample_indices(A[i].size, gs[i], conservative) for i in range(n)]

"""Host restatements for the multiple-series correlation function and the FFT rule (tests/_timeseries.py's
conventions).

* `NumpyAcfExtra` adds `correlation_multiple` and `inefficiency(rule="fft")` to the numpy stand-in `NumpyAcf`, in the
  device's order: each series cut into its own chunks of max(512, ceil(N_k / 1024)) samples, summed sequentially from
  0.0, the chunk partials in order, then the series in list order.  Its results are the device's bits.
* `ld_corr_multiple` and `ld_walk_fft` are the reference's loops in long double, with a bound per C on how far an
  fp64 result in any summation order may lie from them; `ld_walk_fft` adds a bound on the FFT's rounding.
* `sm_acf` restates statsmodels' acf(adjusted=True, fft=True) (acovf: demean, FFT of length >= 2N + 1, divide by
  N - t, then by lag 0).
"""
import hashlib
import math

import numpy as np

from tests import _timeseries as tsr
from tests._timeseries import EPS, _ld, _seq, chunk_size


def digest(x):
    """sha256 of a series as little-endian float64 (the fixture's check that the seeded series are unchanged)"""
    return hashlib.sha256(np.ascontiguousarray(x, dtype="<f8").tobytes()).hexdigest()


def _error(status, msg):
    from pymbar_b200 import _lib

    return _lib.MbarB200Error(status, msg)


def _series_sum(x, L=None):
    """the device's sum of the terms x of a series of length L (x.size when None; x covers its first x.size
    samples, the rest add nothing): chunks of chunk_size(L), sequential, then the chunks in order"""
    L = x.size if L is None else L
    NC = chunk_size(L)
    n = -(-L // NC)
    pad = np.zeros(n * NC)
    pad[:x.size] = x
    parts = np.cumsum(np.concatenate([np.zeros((n, 1)), pad.reshape(n, NC)], axis=1), axis=1)[:, -1]
    return _seq(parts)


class NumpyAcfExtra(tsr.NumpyAcf):
    """mbar_b200_acf in numpy, in the device's summation order, with the multiple-series correlation function and
    the FFT rule."""

    def inefficiency(self, starts, fast=False, mintime=3, multiple=False, navg=0.0, trace_cap=0, rule=None):
        if rule is None:
            return super().inefficiency(starts, fast=fast, mintime=mintime, multiple=multiple, navg=navg,
                                        trace_cap=trace_cap)
        if rule != "fft":
            raise ValueError(rule)
        if self.cross or self.lengths is not None or fast:
            raise _error(-1, "the FFT rule needs an unsegmented autocorrelation and fast = 0")
        self.calls += 1
        starts = np.atleast_1d(starts).astype(np.int64)
        n = starts.size
        out = {k: np.empty(n) for k in ("mean_a", "mean_b", "sigma2", "g")}
        out["last_lag"] = np.zeros(n, np.int64)
        out["status"] = np.zeros(n, np.int32)
        if trace_cap:
            out["trace"] = np.full((n, trace_cap), np.nan)
        for j, s in enumerate(starts):
            s = int(s)
            mua, mub = self._means(s)
            s2 = self._sigma2(s, mua, mub)
            out["mean_a"][j], out["mean_b"][j], out["sigma2"][j] = mua, mub, s2
            out["g"][j] = 1.0
            if s2 == 0.0:
                out["status"][j] = 1
                continue
            m = self.T - s
            g, t, last = 1.0, 1, 0
            while t <= m - 1:
                C = self.lag_sum(s, t, mua, mub) / float(m - t) / s2
                if trace_cap and t - 1 < trace_cap:
                    out["trace"][j, t - 1] = C
                last = t
                if C <= 0.0 and t > mintime:
                    break
                g += 2.0 * C * (1.0 - t / m) * 1.0
                t += 1
            out["g"][j], out["last_lag"][j] = g, last
        return out

    # ---- multiple-series correlation function ----
    def _segments(self):
        if self.lengths is None:
            raise _error(-1, "the object holds no segments")
        off = np.concatenate([[0], np.cumsum(self.lengths)])
        return [(int(o), int(L)) for o, L in zip(off[:-1], self.lengths)]

    def multi_moments(self):
        """(mu_A, mu_B, sigma2) of the multiple-series correlation function"""
        seg = self._segments()
        mua = _seq([_series_sum(self.a[o:o + L]) for o, L in seg]) / float(self.T)
        mub = _seq([_series_sum(self.b[o:o + L]) for o, L in seg]) / float(self.T)
        s2 = self.multi_numerator(0, mua, mub)[0] / float(self.T)
        return mua, mub, s2

    def multi_numerator(self, t, mua, mub):
        """(numerator, denominator, some running numerator < 0) at lag t"""
        vals, dens = [], []
        for o, L in self._segments():
            if t >= L:
                continue
            vals.append(_series_sum((self.a[o:o + L - t] - mua) * (self.b[o + t:o + L] - mub), L))
            dens.append(float(L - t))
        running = np.cumsum(np.concatenate([[0.0], vals]))[1:]
        return _seq(vals), _seq(dens), bool(np.any(running < 0.0))

    def correlation_multiple(self, n_max, truncate=False):
        self.calls += 1
        seg = self._segments()
        if n_max < 0 or n_max > max(L for _, L in seg) - 1:
            raise _error(-1, "N_max out of range")
        mua, mub, s2 = self.multi_moments()
        if s2 == 0.0:
            raise _error(-1, "sigma^2 = 0")
        C = np.full(n_max + 1, np.nan)
        count = n_max
        for t in range(n_max + 1):
            num, den, neg = self.multi_numerator(t, mua, mub)
            C[t] = num / den / s2
            if truncate and neg:
                count = t
                break
        return C[:count].copy(), mua, mub, s2


# ---- long double ---------------------------------------------------------------------------------------------------

def ld_corr_multiple(A_kn, B_kn=None, n_max=None):
    """The multiple-series correlation function in long double for t = 0 .. n_max: dict with C, C_bound, the running
    numerators after each series with N_k > t (run [n_lags][...]) and a bound on any of them (run_bound)."""
    L = np.array([x.size for x in A_kn])
    a = _ld(np.concatenate(A_kn))
    b = a if B_kn is None else _ld(np.concatenate(B_kn))
    N = a.size
    n_max = int(L.max()) - 1 if n_max is None else n_max
    mua, mub = np.sum(a) / N, np.sum(b) / N
    da, db = a - mua, b - mub
    off = np.concatenate([[0], np.cumsum(L)])
    seg_end = np.repeat(off[1:], L)
    k = max(chunk_size(int(x)) for x in L) + sum(-(-int(x) // chunk_size(int(x))) for x in L) + L.size + 4
    dA = k * EPS * np.sum(np.abs(a)) / N
    dB = k * EPS * np.sum(np.abs(b)) / N
    s2 = np.sum(da * db) / N
    s2_err = tsr._sum_bound(da, db, 0, None, k, dA, dB, False) / N
    res = dict(mean_a=mua, mean_b=mub, sigma2=s2, C=[], C_bound=[], run=[], run_bound=[])
    for t in range(n_max + 1):
        n = np.arange(0, N - t)
        n = n[n + t < seg_end[n]]
        prod = da[n] * db[n + t]
        den = int(np.sum(np.maximum(L - t, 0)))
        C = np.sum(prod) / den / s2
        Sb = tsr._sum_bound(da, db, t, n, k, dA, dB, False)
        res["C"].append(C)
        res["C_bound"].append((Sb / den + abs(C) * s2_err) / abs(s2) * 1.01 + 8 * EPS * abs(C))
        run, acc = [], np.longdouble(0)
        for o, Lk in zip(off[:-1], L):
            if t < Lk:
                acc += np.sum(da[o:o + Lk - t] * db[o + t:o + Lk])
                run.append(acc)
        res["run"].append(run)
        # any running numerator: |x||y| terms and the mean errors against sums of |x|, |y| (not their window sums)
        x, y = np.abs(da[n]), np.abs(db[n + t])
        res["run_bound"].append((k + 3) * EPS * np.sum((x + dA) * (y + dB)) + dA * np.sum(y) + dB * np.sum(x)
                                + n.size * dA * dB)
    return res


def corr_multiple_stop(res, n_max):
    """the reference's returned length from the long-double running numerators with truncate"""
    for t, run in enumerate(res["run"][:n_max + 1]):
        if any(v < 0 for v in run):
            return t
    return n_max


def corr_multiple_margin(res, stop):
    """smallest |running numerator| / bound over the truncate decisions through lag `stop`"""
    r = [abs(float(v)) / float(b) for run, b in zip(res["run"][:stop + 1], res["run_bound"][:stop + 1]) for v in run]
    return min(r) if r else math.inf


def next_regular(n):
    """the smallest 5-smooth integer >= n (statsmodels' FFT length)"""
    m = n
    while True:
        x = m
        for p in (2, 3, 5):
            while x % p == 0:
                x //= p
        if x == 1:
            return m
        m += 1


def sm_acf(x, adjusted=True, fft=True, nlags=None, **kwargs):
    """statsmodels.tsa.stattools.acf(x, adjusted=True, fft=True, nlags) restated: acovf demeans x, takes the FFT of
    length next_regular(2 N + 1), ifft(F conj(F))[:N].real / (N - t), and acf divides by lag 0."""
    assert adjusted and fft
    x = np.asarray(x, dtype=np.float64)
    n = x.size
    xo = x - x.mean()
    F = np.fft.fft(xo, n=next_regular(2 * n + 1))
    acov = (np.fft.ifft(F * np.conjugate(F))[:n] / (n - np.arange(n))).real
    return (acov / acov[0])[:(n if nlags is None else nlags) + 1]


def ld_walk_fft(A, start=0, mintime=3):
    """statistical_inefficiency_fft's loop in long double from `start`: dict with lags, C, C_bound (fp64 direct sums
    in any order), fft_bound (statsmodels' FFT), g and g_bound (|g_fp64 - g_ld| for either evaluation), last_lag."""
    T = np.asarray(A).size
    a = _ld(A)[start:]
    m = a.size
    mu = np.sum(a) / m
    d = a - mu
    ss = np.sum(d * d)
    s2 = ss / m
    k = chunk_size(T) + -(-T // chunk_size(T)) + 4
    dA = k * EPS * np.sum(np.abs(a)) / m
    s2_err = tsr._sum_bound(d, d, 0, None, k, dA, dA, False) / m
    E = 10 * math.log2(next_regular(2 * m + 1)) * EPS * ss            # the FFT's error on any S(t)
    res = dict(lags=[], C=[], C_bound=[], fft_bound=[], g=np.longdouble(1.0), last_lag=0, sigma2=s2)
    terms, tb = [], []
    for t in range(1, m):
        n = np.arange(0, m - t)
        C = np.sum(d[n] * d[n + t]) / (m - t) / s2
        Sb = tsr._sum_bound(d, d, t, n, k, dA, dA, False) / (m - t)
        cb = (Sb + abs(C) * s2_err) / abs(s2) * 1.01 + 8 * EPS * abs(C)
        fb = (E / (m - t) + abs(C) * E / m) / abs(s2) * 1.01 + 8 * EPS * abs(C)
        res["lags"].append(t)
        res["C"].append(C)
        res["C_bound"].append(cb)
        res["fft_bound"].append(fb)
        res["last_lag"] = t
        if C <= 0 and t > mintime:
            break
        frac = np.longdouble(t) / m
        terms.append(2 * C * (1 - frac))
        tb.append(2 * (cb + fb) * abs(1 - frac))
        res["g"] += 2 * C * (1 - frac)
    tv = np.array([float(v) for v in terms])
    res["g_bound"] = float(np.sum(np.array(tb, dtype=np.float64)) * 1.01
                           + 2 * (len(tv) + 6) * EPS * (1.0 + np.sum(np.abs(tv))))
    return res


def fft_margins(res):
    """(smallest |C| / C_bound, smallest |C| / fft_bound) over the evaluated lags"""
    c = np.array([abs(float(v)) for v in res["C"]])
    if c.size == 0:
        return math.inf, math.inf
    return (float(np.min(c / np.array([float(b) for b in res["C_bound"]]))),
            float(np.min(c / np.array([float(b) for b in res["fft_bound"]]))))

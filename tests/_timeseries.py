"""Host restatements for the timeseries tests.

* `NumpyAcf` is a numpy stand-in for `pymbar_b200.DeviceAcf`: the device's algorithm in the device's order (chunks of
  NC = max(512, ceil(T / 1024)) samples summed sequentially from 0.0, the chunk partials from the start's chunk on in
  order, every term and quotient in the reference's fp64 operations), so its results are the device's bits.
* `ld_walk` is the reference's loop in long double with long-double means: the "exact" answer.
* the `C_bound` entries of `ld_walk` and `g_bound` state how far the fp64 result may lie from it (DESIGN.md §3.5d).
"""
import math

import numpy as np

EPS = np.finfo(np.float64).eps / 2          # unit roundoff of fp64


def chunk_size(T):
    return max(512, -(-T // 1024))


def lag(i, fast):
    return 1 + i * (i + 1) // 2 if fast else i + 1


def _seq(x):
    """0.0 + x[0] + x[1] + ... left to right."""
    return float(np.cumsum(np.concatenate([[0.0], x]))[-1]) if len(x) else 0.0


class NumpyAcf:
    """mbar_b200_acf in numpy, in the device's summation order."""

    def __init__(self, A_n, B_n=None, lengths=None, device=0):
        self.a = np.ascontiguousarray(A_n, dtype=np.float64)
        if self.a.ndim != 1 or self.a.size < 1:
            raise ValueError("A_n must be one-dimensional and not empty")
        if not np.all(np.isfinite(self.a)) or (B_n is not None and not np.all(np.isfinite(B_n))):
            from pymbar_b200 import _lib

            raise _lib.MbarB200Error(-5, "non-finite value")
        self.cross = B_n is not None
        self.b = self.a if B_n is None else np.ascontiguousarray(B_n, dtype=np.float64)
        self.T = self.a.size
        self.NC = chunk_size(self.T)
        self.nChunks = -(-self.T // self.NC)
        self.lengths = None if lengths is None else np.asarray(lengths, dtype=np.int64)
        if self.lengths is not None:
            off = np.concatenate([[0], np.cumsum(self.lengths)])
            self.seg_end = np.repeat(off[1:], self.lengths)
        self.calls = 0

    def close(self):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        pass

    def _sum(self, terms, s):
        """the device's sum of terms [T] (zero outside the support) for a start s"""
        pad = np.zeros(self.nChunks * self.NC)
        pad[:self.T] = terms
        blocks = pad.reshape(self.nChunks, self.NC)
        parts = np.cumsum(np.concatenate([np.zeros((self.nChunks, 1)), blocks], axis=1), axis=1)[:, -1]
        return _seq(parts[s // self.NC:])

    def _means(self, s):
        ta = np.where(np.arange(self.T) >= s, self.a, 0.0)
        tb = np.where(np.arange(self.T) >= s, self.b, 0.0)
        m = float(self.T - s)
        return self._sum(ta, s) / m, self._sum(tb, s) / m

    def lag_sum(self, s, t, mua, mub):
        T = self.T
        n = np.arange(s, T - t)
        if self.lengths is not None:
            n = n[n + t < self.seg_end[n]]
        da, db_t = self.a[n] - mua, self.b[n + t] - mub
        term = da * db_t
        if self.cross:
            term = term + (self.b[n] - mub) * (self.a[n + t] - mua)
        full = np.zeros(T)
        full[n] = term
        return self._sum(full, s)

    def _sigma2(self, s, mua, mub):
        S0 = self.lag_sum(s, 0, mua, mub)
        return (0.5 * S0 if self.cross else S0) / float(self.T - s)

    def inefficiency(self, starts, fast=False, mintime=3, multiple=False, navg=0.0, trace_cap=0):
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
            limit = int(self.lengths.max()) if multiple else m
            g, i, last = 1.0, 0, 0
            while True:
                t = lag(i, fast)
                if t >= limit - 1:
                    break
                S = self.lag_sum(s, t, mua, mub)
                if multiple:
                    den = int(np.sum(np.maximum(self.lengths - t, 0)))
                    C = S / float(den) / s2
                else:
                    C = (S if self.cross else 2.0 * S) / (2.0 * float(m - t) * s2)
                if trace_cap and i < trace_cap:
                    out["trace"][j, i] = C
                last = t
                if C <= 0.0 and t > (10 if multiple else mintime):
                    break
                frac = t / navg if multiple else t / m
                g += 2.0 * C * (1.0 - frac) * float(i + 1 if fast else 1)
                i += 1
            out["g"][j], out["last_lag"][j] = g, last
        return out

    def correlation(self, start, n_max):
        self.calls += 1
        mua, mub = self._means(start)
        s2 = self._sigma2(start, mua, mub)
        if s2 == 0.0:
            from pymbar_b200 import _lib

            raise _lib.MbarB200Error(-1, "sigma^2 = 0")
        m = self.T - start
        C = np.array([(S if self.cross else 2.0 * S) / (2.0 * float(m - t) * s2)
                      for t, S in ((t, self.lag_sum(start, t, mua, mub)) for t in range(n_max + 1))])
        return C, mua, mub, s2


# ---- long double ---------------------------------------------------------------------------------------------------

def _ld(x):
    return np.asarray(x, dtype=np.longdouble)


def ld_walk(A, B=None, start=0, fast=False, mintime=3, lengths=None, navg=None):
    """The reference's loop in long double from `start` (lengths: the multiple-series rule): dict with mean_a, mean_b,
    sigma2, lags, C (one per evaluated lag), g (before the clamp), last_lag, and the bound inputs."""
    a = _ld(A)[start:]
    b = a if B is None else _ld(B)[start:]
    m = a.size
    mua, mub = a.mean(dtype=np.longdouble), b.mean(dtype=np.longdouble)
    da, db = a - mua, b - mub
    s2 = np.sum(da * db) / m
    res = dict(mean_a=mua, mean_b=mub, sigma2=s2, lags=[], C=[], g=np.longdouble(1.0), last_lag=0, m=m,
               abs_a=np.sum(np.abs(a)), abs_b=np.sum(np.abs(b)), C_bound=[], g_terms=[])
    if s2 == 0:
        return res
    if lengths is not None:
        off = np.concatenate([[0], np.cumsum(lengths)])
        seg_end = np.repeat(off[1:], lengths)
        limit = int(np.max(lengths))
    else:
        seg_end, limit = None, m
    T = np.asarray(A).size
    k = chunk_size(T) + -(-T // chunk_size(T)) + 4
    dA_mean = k * EPS * res["abs_a"] / m
    dB_mean = k * EPS * res["abs_b"] / m
    s2_err = _sum_bound(da, db, 0, None, k, dA_mean, dB_mean, B is not None) / m
    res["sigma2_bound"] = s2_err
    g, i = np.longdouble(1.0), 0
    while True:
        t = lag(i, fast)
        if t >= limit - 1:
            break
        n = np.arange(0, m - t)
        if seg_end is not None:
            n = n[n + t < seg_end[n]]
        prod = da[n] * db[n + t]
        if lengths is not None:
            den = int(np.sum(np.maximum(np.asarray(lengths) - t, 0)))
            C = np.sum(prod) / den / s2
            Sb = _sum_bound(da, db, t, n, k, dA_mean, dB_mean, False) / den
        else:
            num = np.sum(prod + db[n] * da[n + t])
            C = num / (2 * (m - t) * s2)
            Sb = _sum_bound(da, db, t, n, k, dA_mean, dB_mean, True) / (2 * (m - t))
        cb = (Sb + abs(C) * s2_err) / abs(s2) * 1.01 + 8 * EPS * abs(C)
        res["lags"].append(t)
        res["C"].append(C)
        res["C_bound"].append(cb)
        res["last_lag"] = t
        if C <= 0 and t > (10 if lengths is not None else mintime):
            break
        frac = np.longdouble(t) / (navg if lengths is not None else m)
        inc = (i + 1) if fast else 1
        res["g_terms"].append((2 * C * (1 - frac) * inc, 2 * cb * abs(1 - frac) * inc))
        g += 2 * C * (1 - frac) * inc
        i += 1
    res["g"] = g
    return res


def _sum_bound(da, db, t, n, k, dA, dB, both):
    """bound on |fp64 sum - exact| of sum_n da[n] db[n + t] (+ db[n] da[n + t] when both): k roundings of the
    sequential sums and the products on |terms| with the centring errors, plus the mean errors dA, dB times the
    window sums they multiply."""
    if n is None:
        n = np.arange(da.size - t)
    x, y = da[n], db[n + t]
    b = (k + 3) * EPS * np.sum((np.abs(x) + dA) * (np.abs(y) + dB)) + dA * abs(np.sum(y)) + dB * abs(np.sum(x)) \
        + n.size * dA * dB
    if both:
        x2, y2 = db[n], da[n + t]
        b = b + (k + 3) * EPS * np.sum((np.abs(x2) + dB) * (np.abs(y2) + dA)) + dB * abs(np.sum(y2)) \
            + dA * abs(np.sum(x2)) + n.size * dA * dB
    return b


def g_bound(res):
    """bound on |g_fp64 - g_exact|: the C bounds carried through g's terms, and the roundings of its accumulation."""
    if not res["g_terms"]:
        return 0.0
    terms = np.array([float(v) for v, _ in res["g_terms"]])
    cb = np.array([float(e) for _, e in res["g_terms"]])
    return float(np.sum(cb) * 1.01 + (len(terms) + 6) * EPS * (1.0 + np.sum(np.abs(terms))))


def stop_margin(res):
    """the smallest |C| / C_bound among the stop decisions past mintime (how far each is from flipping)."""
    if not res["C"]:
        return math.inf
    r = [abs(float(c)) / float(b) for c, b in zip(res["C"], res["C_bound"]) if float(b) > 0]
    return min(r) if r else math.inf

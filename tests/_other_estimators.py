"""Host restatements for the other_estimators tests.

* `NumpyWork` is a numpy stand-in for `pymbar_b200.DeviceWork`: every request evaluated with the reference's formulas
  in numpy's own operations and summation order (other_estimators.py:120-145, :489-504, :617-636, :694-696 and
  pymbar.utils.logsumexp), so the host drivers over it reproduce the reference's bits.
* `ld_request` evaluates a request in long double from the same fp64 work values, and `bound` states how far the
  device's fp64 result may lie from it (DESIGN.md §3.5e): a few ulps of each term's arguments, carried into the
  shifted exponentials, plus (chunk length + number of chunks + 4) roundings over the chunked sums.
"""
import numpy as np

EPS = np.finfo(np.float64).eps / 2          # unit roundoff of fp64
FERMI, FERMI_MOMENTS, EXP, GAUSS = 0, 1, 2, 3


def chunk_len(n):
    return max(4096, -(-n // 2048))


def n_chunks(n):
    return -(-n // chunk_len(n))


def logsumexp(a):
    """pymbar.utils.logsumexp (utils.py:313-337) for a 1-D array: a non-finite max is replaced by 0."""
    a_max = np.amax(a, keepdims=True)
    a_max[~np.isfinite(a_max)] = 0
    out = np.log(np.exp(a - a_max).sum(None))
    return out + np.squeeze(a_max)


def request(w, kind, c1, c2):
    """out [3] of one request in the reference's numpy operations."""
    w = np.asarray(w, dtype=np.float64)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        if kind == FERMI:
            a = w + c1 + c2
            m = np.choose(np.less(0.0, a), (0.0, a))
            t = -m - np.log(np.exp(-m) + np.exp(a - m))
            lse = logsumexp(t)
            return np.array([lse, 0.0, 0.0])
        if kind == FERMI_MOMENTS:
            a = w + c1
            A = np.max(a)
            t = -np.log(np.exp(-A) + np.exp(a - A))
            return np.array([logsumexp(t), logsumexp(2 * t), A])
        if kind == EXP:
            amax = np.max(-w)
            x = np.exp(-w - amax)
            S = np.sum(x)
            d = x - S / w.size
            return np.array([np.log(S) + amax, S, np.sum(d * d)])
        if kind == GAUSS:
            S = np.sum(w)
            d = w - S / w.size
            return np.array([S, np.sum(d * d), 0.0])
    raise ValueError(kind)


class NumpyWork:
    """mbar_b200_work in numpy, in the reference's operations and numpy's summation order."""

    def __init__(self, vectors, device=0):
        from pymbar_b200 import _lib

        self.w = [np.asarray(v, dtype=np.float64) for v in vectors]
        if not self.w or any(v.ndim != 1 or v.size == 0 for v in self.w):
            raise _lib.MbarB200Error(-1, "empty vector")
        if not all(np.all(np.isfinite(v)) for v in self.w):
            raise _lib.MbarB200Error(-5, "non-finite value")
        self.calls = 0
        self.requests = 0

    def close(self):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        pass

    def evaluate(self, vector, kind, c1, c2):
        from pymbar_b200 import _lib

        v, k = np.atleast_1d(vector), np.atleast_1d(kind)
        a = np.broadcast_to(np.asarray(c1, dtype=np.float64), v.shape)
        b = np.broadcast_to(np.asarray(c2, dtype=np.float64), v.shape)
        for vi, ki in zip(v, k):
            if not 0 <= vi < len(self.w) or ki not in (0, 1, 2, 3):
                raise _lib.MbarB200Error(-1, "bad request")
        self.calls += 1
        self.requests += v.size
        return np.array([request(self.w[int(vi)], int(ki), float(ai), float(bi)) for vi, ki, ai, bi in zip(v, k, a, b)])


# ---- long double ---------------------------------------------------------------------------------------------------

def _ld(x):
    return np.asarray(x, dtype=np.longdouble)


def _lse_ld(t):
    M = np.max(t)
    return np.log(np.sum(np.exp(t - M))) + M


def ld_request(w, kind, c1, c2, A=None):
    """The request in long double from the fp64 values w, c1, c2 (for FERMI_MOMENTS the shift A is the fp64 one, the
    value the host then divides out).  Returns (values [3] as long double, bound [3])."""
    w64 = np.asarray(w, dtype=np.float64)
    w = _ld(w64)
    n = w.size
    k = chunk_len(n) + n_chunks(n) + 4
    if kind == FERMI:
        a = (w + _ld(c1)) + _ld(c2)
        m = np.maximum(a, 0)
        t = -m - np.log(np.exp(-m) + np.exp(a - m))
        lse = _lse_ld(t)
        eps = 8 * EPS * float(np.max(np.abs(w)) + abs(c1) + abs(c2) + 2) + EPS * float(np.max(t) - np.min(t))
        b = eps + (k + 2) * EPS + EPS * abs(float(lse)) + 2 * EPS
        return np.array([lse, 0, 0], dtype=np.longdouble), np.array([b, 0.0, 0.0])
    if kind == FERMI_MOMENTS:
        A = float(np.max(w64 + c1)) if A is None else A
        a = w + _ld(c1)
        t = -np.log(np.exp(-_ld(A)) + np.exp(a - _ld(A)))
        l1, l2 = _lse_ld(t), _lse_ld(2 * t)
        eps = 8 * EPS * float(np.max(np.abs(w)) + abs(c1) + abs(A) + 2) + EPS * float(np.max(t) - np.min(t))
        b1 = eps + (k + 2) * EPS + EPS * abs(float(l1)) + 2 * EPS
        b2 = 2 * eps + (k + 2) * EPS + EPS * abs(float(l2)) + 2 * EPS
        return np.array([l1, l2, A], dtype=np.longdouble), np.array([b1, b2, 0.0])
    if kind == EXP:
        r = w - np.min(w)
        x = np.exp(-r)
        S = np.sum(x)
        mu = S / n
        S2 = np.sum((x - mu) ** 2)
        eps_i = 4 * EPS * (r + 1)                              # relative error of each fp64 x_i
        dS = float(np.sum(eps_i * x)) + k * EPS * float(S)
        lse = np.log(S) - np.min(w)
        b0 = dS / float(S) * 1.01 + EPS * abs(float(lse)) + 2 * EPS
        dmu = dS / n * 1.01 + 2 * EPS * float(mu)
        dev = np.abs(x - mu)
        b2 = float(np.sum(2 * dev * (eps_i * x + dmu)) + (k + 3) * EPS * np.sum((dev + eps_i * x + dmu) ** 2)
                   + np.sum((eps_i * x + dmu) ** 2))
        return np.array([lse, S, S2], dtype=np.longdouble), np.array([b0, dS, b2])
    if kind == GAUSS:
        S = np.sum(w)
        mu = S / n
        S2 = np.sum((w - mu) ** 2)
        dS = k * EPS * float(np.sum(np.abs(w)))
        dmu = dS / n * 1.01 + 2 * EPS * abs(float(mu))
        dev = np.abs(w - mu)
        b2 = float(np.sum(2 * dev * dmu) + (k + 3) * EPS * np.sum((dev + dmu) ** 2) + n * dmu ** 2)
        return np.array([S, S2, 0], dtype=np.longdouble), np.array([dS, b2, 0.0])
    raise ValueError(kind)

"""KDE test infrastructure: numpy restatements of the device's log kernel sum (mbar_b200_kde_log_sum) in fp64 and in
long double, the per-query tolerance the device is held to, a numpy stand-in for DeviceKde, and a KDE-capable
FES-shaped stand-in class for the facade.

    l_q = log sum_n w_n k(d_qn / h),   d_qn = sqrt(sum_j (y_qj - x_nj)^2)

Both restatements compute the distance and the kernel's argument with the fp64 operations sklearn uses (rounded
squares summed in dimension order, the correctly rounded sqrt, then d*d/(h*h), d/h or pi/2*d/h), and decide support
by sklearn's d < h.  Near the edge of a compact kernel 1 - u loses every digit u has, so these are the values the
sum is defined on; the long-double version then takes the logs, the kernels and the sum in extended precision.
"""
import math

import numpy as np

from pymbar_b200.fes import KDE_KERNELS

EPS = 2.0 ** -53
HALF_PI = 0.5 * math.pi
BAND = 40.0         # terms further below the largest contribute less than N e^-40 relative


def _as2d(a):
    a = np.asarray(a, np.float64)
    return a.reshape(-1, 1) if a.ndim == 1 else a


def distance_sq(y, x):
    """[Q, N] squared distances as sklearn's euclidean_rdist rounds them: (y_j - x_j)^2 added in dimension order."""
    y, x = _as2d(y), _as2d(x)
    r = np.zeros((len(y), len(x)))
    for j in range(x.shape[1]):
        t = y[:, j:j + 1] - x[None, :, j]
        r = r + t * t
    return r


def log_kernel_terms(kernel, r, h, dtype=np.float64):
    """(log k, inside) for squared distances r: the kernel's argument in sklearn's fp64 arithmetic, log k in `dtype`
    (-inf outside a compact kernel's support)."""
    d = np.sqrt(r)
    inside = d < h
    if kernel == "gaussian":
        lk = -0.5 * r.astype(dtype) / (dtype(h) * dtype(h))
        return lk, np.ones_like(inside)
    if kernel == "exponential":
        return -d.astype(dtype) / dtype(h), np.ones_like(inside)
    with np.errstate(invalid="ignore", divide="ignore"):
        if kernel == "tophat":
            lk = np.zeros(r.shape, dtype)
        elif kernel == "epanechnikov":
            lk = np.log(dtype(1) - ((d * d) / (h * h)).astype(dtype))
        elif kernel == "linear":
            lk = np.log(dtype(1) - (d / h).astype(dtype))
        elif kernel == "cosine":
            lk = np.log(np.cos(((HALF_PI * d) / h).astype(dtype)))
        else:
            raise ValueError(kernel)
    return np.where(inside, lk, dtype(-np.inf)), inside


def log_sum(kernel, h, x, w, y, dtype=np.float64, chunk=64):
    """(l_q [Q] in `dtype`, A_q [Q]): see log_sum_ld."""
    x = _as2d(x)
    y = _as2d(y)
    with np.errstate(divide="ignore"):
        lw = np.log(np.asarray(w, np.float64).astype(dtype))
    out = np.empty(len(y), dtype)
    A = np.zeros(len(y))
    for q0 in range(0, len(y), chunk):
        r = distance_sq(y[q0:q0 + chunk], x)
        lk, _ = log_kernel_terms(kernel, r, h, dtype)
        a = lw[None, :] + lk
        m = a.max(axis=1)
        fin = np.isfinite(m)
        mm = np.where(fin, m, dtype(0))
        with np.errstate(invalid="ignore", divide="ignore"):
            s = np.exp(a - mm[:, None]).sum(axis=1)
            out[q0:q0 + chunk] = np.where(fin, mm + np.log(s), dtype(-np.inf))
            near = np.isfinite(a) & (a >= (mm - BAND)[:, None])
        A[q0:q0 + chunk] = np.where(near, np.abs(a), 0).max(axis=1).astype(np.float64)
    return out, A


def log_sum_ld(kernel, h, x, w, y):
    """(l_q, A_q) in long double: A_q bounds |log w_n + log k_qn| over the terms within BAND of the largest.
    Refuses to run where long double is plain fp64 (it would check the device against itself)."""
    LD = np.longdouble
    if np.finfo(LD).nmant < 63:
        raise RuntimeError(f"needs an 80-bit long double (nmant >= 63), got nmant={np.finfo(LD).nmant}")
    return log_sum(kernel, h, x, w, y, dtype=LD)


def log_sum_f64(kernel, h, x, w, y):
    return log_sum(kernel, h, x, w, y)[0]


# Per-query tolerance of the device against the long-double restatement:  (C1 + C2 sqrt(N)) eps + C3 eps A_q.
#   C1 = 128: the device exp is exp(a (1 + 3.35e-17)) to 1.5 ulp (DESIGN 3.1) and its arguments stay within
#        [-(KDE_RESCALE + BAND), 0] = [-168, 0] for the terms that matter: 0.6 * 168 + 1.5 ulp, plus the exp / log of
#        the chunk combination (1 ulp each) and the cosine kernel's 2 ulp, with margin;
#   C2 = 2: the per-thread sums of positive terms in fixed order, whose rounding errors add like a random walk;
#   C3 = 8: the roundings that scale with the size of a term's logarithm: log w_n, the kernel constant 0.5/h^2 or
#        1/h, the fma forming a_n, a_n - m, and m + log S, each at most one ulp of a value no larger than A_q.
C1, C2, C3 = 128.0, 2.0, 8.0


def tolerance(N, A):
    return (C1 + C2 * math.sqrt(N)) * EPS + C3 * EPS * np.asarray(A, np.float64)


def check_against_ld(got, kernel, h, x, w, y):
    """Entry by entry: -inf exactly where the restatement has no nonzero term, finite values within tolerance."""
    ref, A = log_sum_ld(kernel, h, x, w, y)
    got = np.asarray(got, np.float64)
    inf = ~np.isfinite(ref)
    np.testing.assert_array_equal(np.isneginf(got), inf)
    err = np.abs(got[~inf].astype(np.longdouble) - ref[~inf]).astype(np.float64)
    tol = tolerance(len(np.asarray(w)), A[~inf])
    assert np.all(err <= tol), (float((err / tol).max()), kernel, h)
    return ref


def mpmath_log_sum(kernel, h, x, w, y, dps=50):
    """One query in mpmath from the same fp64 kernel arguments (the reference for log_sum_ld)."""
    import mpmath

    mpmath.mp.dps = dps
    x = _as2d(x)
    y = _as2d(y).reshape(1, -1)
    r = distance_sq(y, x)[0]
    total = mpmath.mpf(0)
    for n in range(len(x)):
        if w[n] == 0:
            continue
        d = math.sqrt(r[n])
        if kernel == "gaussian":
            lk = -mpmath.mpf(r[n]) / (2 * mpmath.mpf(h) ** 2)
        elif kernel == "exponential":
            lk = -mpmath.mpf(d) / mpmath.mpf(h)
        elif not d < h:
            continue
        elif kernel == "tophat":
            lk = mpmath.mpf(0)
        elif kernel == "epanechnikov":
            lk = mpmath.log(1 - mpmath.mpf((d * d) / (h * h)))
        elif kernel == "linear":
            lk = mpmath.log(1 - mpmath.mpf(d / h))
        else:
            lk = mpmath.log(mpmath.cos(mpmath.mpf((HALF_PI * d) / h)))
        total += mpmath.exp(mpmath.log(mpmath.mpf(w[n])) + lk)
    return mpmath.log(total) if total > 0 else -mpmath.inf


class NumpyKde:
    """DeviceKde's interface, answered by the fp64 restatement, with the C ABI's argument checks (test
    infrastructure: the product has no CPU path).  Counts its instances and calls."""

    created = 0
    calls = 0

    def __init__(self, x_n, w_n, device=0):
        from pymbar_b200._lib import MbarB200Error

        x = _as2d(x_n)
        w = np.asarray(w_n, np.float64)
        if w.shape != (x.shape[0],):
            raise ValueError(f"expected shape ({x.shape[0]},), got {w.shape}")
        if not 1 <= x.shape[1] <= 4:
            raise MbarB200Error(-1, "D outside [1, 4]")
        if not np.all((w >= 0) & np.isfinite(w)) or not np.any(w > 0):
            raise MbarB200Error(-1, "bad weights")
        if not np.all(np.isfinite(x)):
            raise MbarB200Error(-5, "non-finite coordinate")
        self.x, self.w = x, w
        self.N, self.D = x.shape
        type(self).created += 1

    def log_sum(self, kernel, h, y):
        from pymbar_b200._lib import MbarB200Error

        if kernel not in KDE_KERNELS or not (math.isfinite(h) and h > 0):
            raise MbarB200Error(-1, "bad kernel or bandwidth")
        y = _as2d(y)
        if not np.all(np.isfinite(y)):
            raise MbarB200Error(-5, "non-finite query")
        type(self).calls += 1
        return log_sum_f64(kernel, h, self.x, self.w, y)

    def close(self):
        pass


def kde_stand_in():
    """A KDE-capable subclass of tests/_fes.StandInFES: sklearn's KernelDensity set up and fitted as fes.py does it
    (restated for the tests), with a _get_fes_kde that marks every call that reaches it."""
    from tests import _fes

    class StandInKdeFES(_fes.StandInFES):
        fallbacks = 0
        generate_fes = _get_fes_histogram = _fes.StandInFES._replaced

        def _setup_fes_kde(self, kde_parameters):
            from sklearn.neighbors import KernelDensity

            from pymbar_b200.utils import ParameterError

            kde = KernelDensity()
            params = kde.get_params()
            for k in kde_parameters:
                if k not in params:
                    raise ParameterError(f"{k} is not a parameter in KernelDensity")
                params[k] = kde_parameters[k]
            kde.set_params(**params)
            self.kde_parameters = kde_parameters
            self.kdes = None
            self.kde = kde

        def _generate_fes_kde(self, b, x_n, w_n):
            x = x_n.reshape(-1, 1) if np.ndim(x_n) == 1 else x_n
            kde = self.kde
            kde.fit(x, sample_weight=self.w_n)

        def get_kde(self):
            return self.kde

        def get_fes(self, x, reference_point="from-lowest", fes_reference=None, uncertainty_method=None):
            if self.fes_type != "kde":
                return super().get_fes(x, reference_point, fes_reference, uncertainty_method)
            x = np.array(x)
            if len(np.shape(x)) <= 1:
                x = x.reshape(-1, 1)
            return self._get_fes_kde(x, reference_point, fes_reference, uncertainty_method)

        def _get_fes_kde(self, x, reference_point="from-normalization", fes_reference=None, uncertainty_method=None):
            type(self).fallbacks += 1
            f = -self.kde.score_samples(x)
            if reference_point == "from-lowest":
                f = f - f.min()
            elif reference_point == "from-specified":
                f = f + self.kde.score_samples(np.array(fes_reference).reshape(1, -1))
            if uncertainty_method is not None:
                raise AssertionError("reached a method the facade replaces")
            return {"f_i": f, "df_i": None}

    return StandInKdeFES

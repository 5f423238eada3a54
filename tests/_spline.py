"""Spline FES test infrastructure: numpy and long-double restatements of the device's B-spline basis sums
(mbar_b200_bspline_moments), the per-entry tolerance the device is held to, a numpy stand-in for DeviceBSpline, the
cases of the fixture tests/golden/fes_spline_1d.npz (tools/make_fes_spline_golden.py), and a spline-capable FES-shaped
stand-in class for the facade, written for the tests from the algorithm pymbar's FES documents (fes.py:701-1100,
:1611-2456).

    S_ki = sum_{n: s_n = k} B_i(x_n),   A_i = sum_n w_n B_i(x_n)

The basis values follow scipy's BSpline (extrapolate=True): the interval is the last one in [k, nb - 1] whose left
knot is <= x, and the k + 1 nonzero values come from the Cox-de Boor triangle.  The fp64 restatement uses scipy's
operations (numpy never contracts them into an FMA), so it matches scipy bit for bit; the long-double one runs the
same triangle in extended precision.

Tolerance of the device against the long-double restatement, entry by entry:

    |S_dev - S_ld| <= (A_C (k + 1)^2 + B_C sqrt(n)) eps T,    T = sum_n |w_n| Babs_i(x_n)

with n the number of samples in the entry's sum and Babs the triangle run on absolute values (|ratio| times
|x - knot|), which equals B inside the base interval and bounds every intermediate sum outside it (extrapolation,
where the triangle's terms have mixed signs).
  * A_C = 4: each of the k levels of the triangle rounds a division, two differences, a product and a sum: at most
    4k (k + 1) eps relative to Babs, under (k + 1)^2 * 4; the weight product adds one rounding;
  * B_C = 2: the device adds each cell's terms in a fixed order (segmented sums of a warp, then tile after tile in a
    CTA, then the CTAs in order), whose rounding errors add like a random walk over the n terms.
"""
import math

import numpy as np
from scipy.integrate import quad
from scipy.interpolate import BSpline, make_lsq_spline
from scipy.optimize import minimize

EPS = 2.0 ** -53
A_C, B_C = 4.0, 2.0
LD = np.longdouble


# ---- restatements -----------------------------------------------------------------------------------------------

def interval(t, k, x):
    """scipy's interval index l in [k, nb - 1] for every x."""
    t = np.asarray(t, np.float64)
    nb = len(t) - k - 1
    return np.clip(np.searchsorted(t, np.asarray(x, np.float64), side="right") - 1, k, nb - 1)


def basis_values(t, k, x, dtype=np.float64, absolute=False):
    """(first [N], h [k + 1, N]): h[a] = B_{first + a}(x), from scipy's Cox-de Boor triangle in `dtype` (absolute:
    every ratio and difference replaced by its magnitude, the bound Babs of the module docstring)."""
    x64 = np.asarray(x, np.float64)
    ell = interval(t, k, x64)
    t = np.asarray(t, np.float64).astype(dtype)
    x = x64.astype(dtype)
    h = np.zeros((k + 1, len(x)), dtype)
    h[0] = 1
    with np.errstate(divide="ignore", invalid="ignore"):
        for j in range(1, k + 1):
            hh = h[:j].copy()
            h[0] = 0
            for n in range(1, j + 1):
                xb, xa = t[ell + n], t[ell + n - j]
                same = xb == xa
                w = hh[n - 1] / (xb - xa)
                db, da = xb - x, x - xa
                if absolute:
                    w, db, da = np.abs(w), np.abs(db), np.abs(da)
                h[n - 1] = np.where(same, h[n - 1], h[n - 1] + w * db)
                h[n] = np.where(same, dtype(0), w * da)
    return ell - k, h


def moments(t, k, x, w=None, s=None, K=None, dtype=np.float64):
    """(S [K, nb], A [nb]) in `dtype`; S is None without labels, A None without weights."""
    nb = len(t) - k - 1
    first, h = basis_values(t, k, x, dtype)
    cols = first[None, :] + np.arange(k + 1)[:, None]
    S = A = None
    if s is not None:
        s = np.asarray(s)
        S = np.zeros((K, nb), dtype)
        np.add.at(S, (np.broadcast_to(s, cols.shape), cols), h)
    if w is not None:
        wv = np.asarray(w, np.float64).astype(dtype)
        A = np.zeros(nb, dtype)
        np.add.at(A, cols, h * wv[None, :])
    return S, A


def moments_ld(t, k, x, w=None, s=None, K=None):
    if np.finfo(LD).nmant < 63:
        raise RuntimeError(f"needs an 80-bit long double (nmant >= 63), got nmant={np.finfo(LD).nmant}")
    return moments(t, k, x, w, s, K, dtype=LD)


def bounds(t, k, x, w=None, s=None, K=None):
    """(T_S [K, nb], n_S [K, nb], T_A [nb], n_A [nb]): the sums of |w_n| Babs_i(x_n) and the term counts."""
    nb = len(t) - k - 1
    first, habs = basis_values(t, k, x, np.float64, absolute=True)
    cols = first[None, :] + np.arange(k + 1)[:, None]
    ones = np.ones_like(habs)
    TS = nS = TA = nA = None
    if s is not None:
        idx = (np.broadcast_to(np.asarray(s), cols.shape), cols)
        TS, nS = np.zeros((K, nb)), np.zeros((K, nb))
        np.add.at(TS, idx, habs)
        np.add.at(nS, idx, ones)
    if w is not None:
        TA, nA = np.zeros(nb), np.zeros(nb)
        np.add.at(TA, cols, habs * np.abs(np.asarray(w, np.float64))[None, :])
        np.add.at(nA, cols, ones)
    return TS, nS, TA, nA


def tolerance(k, T, n):
    return (A_C * (k + 1) ** 2 + B_C * np.sqrt(n)) * EPS * T


def check_against_ld(S, A, t, k, x, w=None, s=None, K=None):
    """Entry by entry within tolerance(); exact zeros where no term enters (an empty state)."""
    S_ld, A_ld = moments_ld(t, k, x, w, s, K)
    TS, nS, TA, nA = bounds(t, k, x, w, s, K)
    worst = 0.0
    for got, ref, T, n in ((S, S_ld, TS, nS), (A, A_ld, TA, nA)):
        if ref is None:
            continue
        got = np.asarray(got, np.float64)
        assert got.shape == ref.shape
        np.testing.assert_array_equal(got[n == 0], 0.0)
        err = np.abs(got.astype(LD) - ref).astype(np.float64)
        tol = tolerance(k, T, n)
        nz = n > 0
        assert np.all(err[nz] <= tol[nz]), (float(np.max(err[nz] / np.maximum(tol[nz], 1e-300))), k)
        if nz.any():
            worst = max(worst, float(np.max(err[nz] / np.maximum(tol[nz], 1e-300))))
    return worst


def knots(kind, k, nb, lo=-1.0, hi=1.0, seed=0):
    """Knot vectors of nb basis functions of degree k: clamped uniform (pymbar's), non-uniform clamped, and with
    repeated interior knots."""
    rng = np.random.RandomState(seed)
    n_inner = nb - k + 1
    if kind == "clamped":
        inner = np.linspace(lo, hi, n_inner)
    elif kind == "nonuniform":
        inner = np.sort(np.concatenate([[lo, hi], rng.uniform(lo, hi, n_inner - 2)]))
    elif kind == "repeated":
        inner = np.sort(np.concatenate([[lo, hi], rng.uniform(lo, hi, n_inner - 2)]))
        if n_inner > 4:
            inner[2] = inner[3]
            if k >= 2 and n_inner > 6:
                inner[5] = inner[4] = inner[3]
    else:
        raise ValueError(kind)
    return np.concatenate([[lo] * k, inner, [hi] * k])


def samples_with_edges(t, N, seed=0, spread=0.25):
    """N samples over [t_0 - spread, t_end + spread]: uniform ones plus every knot and its neighbouring doubles."""
    rng = np.random.RandomState(seed)
    t = np.asarray(t, np.float64)
    span = t[-1] - t[0]
    edge = np.unique(np.concatenate([t, np.nextafter(t, -np.inf), np.nextafter(t, np.inf)]))
    x = rng.uniform(t[0] - spread * span, t[-1] + spread * span, size=max(N - len(edge), 0))
    return np.concatenate([edge, x])[:N] if N >= len(edge) else rng.permutation(edge)[:N]


class NumpyBSpline:
    """DeviceBSpline's interface, answered by the fp64 restatement, with the C ABI's argument checks (test
    infrastructure: the product has no CPU path).  Counts its instances and calls."""

    created = 0
    calls = 0

    def __init__(self, x_n, w_n=None, state_n=None, K=None, device=0):
        from pymbar_b200._lib import MbarB200Error

        x = np.asarray(x_n, np.float64)
        if x.ndim != 1:
            raise ValueError("x_n must be one-dimensional")
        self.x, self.N = x, len(x)
        self.w = None if w_n is None else np.asarray(w_n, np.float64)
        self.s = None if state_n is None else np.asarray(state_n)
        self.K = 0 if state_n is None else (int(self.s.max()) + 1 if K is None else int(K))
        if self.w is not None and not np.all((self.w >= 0) & np.isfinite(self.w)):
            raise MbarB200Error(-1, "bad weights")
        if self.s is not None and not np.all((self.s >= 0) & (self.s < self.K)):
            raise MbarB200Error(-1, "label outside [0, K)")
        if not np.all(np.isfinite(x)):
            raise MbarB200Error(-5, "non-finite coordinate")
        type(self).created += 1

    def moments(self, t, k, want_S=True, want_A=True):
        from pymbar_b200._lib import MbarB200Error

        t = np.asarray(t, np.float64)
        nb = len(t) - k - 1
        if not (0 <= k <= 7 and len(t) >= 2 * (k + 1) and np.all(np.isfinite(t)) and np.all(np.diff(t) >= 0)
                and t[k] < t[nb]):
            raise MbarB200Error(-1, "bad knots or degree")
        type(self).calls += 1
        S, A = moments(t, k, self.x, self.w if want_A else None, self.s if want_S else None, self.K)
        return S, A

    def close(self):
        pass


# ---- the fixture's cases --------------------------------------------------------------------------------------

NSPLINE = 8
XRANGE = (-2.3, 2.5)
XI_FIXED = (np.zeros(NSPLINE - 1), np.linspace(-1.0, 1.0, NSPLINE - 1), 2.0 * np.cos(np.arange(NSPLINE - 1)))
QUERIES = np.linspace(-2.2, 2.4, 24)
FES_REF = 0.0
MC_SEED = 11
MC_STEPS = 300
MAP_A = 0.05           # quadratic prior log p(c) = -MAP_A/2 |c|^2

SPLINE_CASES = [
    {"name": "unbiased_ncg", "weights": "unbiasedstate", "algorithm": "Newton-CG", "init": "zeros"},
    {"name": "biased_ncg", "weights": "biasedstates", "algorithm": "Newton-CG", "init": "zeros"},
    {"name": "simplesum_ncg", "weights": "simplesum", "algorithm": "Newton-CG", "init": "zeros"},
    {"name": "unbiased_lbfgsb", "weights": "unbiasedstate", "algorithm": "L-BFGS-B", "init": "zeros"},
    {"name": "unbiased_map", "weights": "unbiasedstate", "algorithm": "Newton-CG", "init": "zeros", "map": True},
    {"name": "biased_explicit", "weights": "biasedstates", "algorithm": "Newton-CG", "init": "explicit"},
    {"name": "simplesum_bfe", "weights": "simplesum", "algorithm": "Newton-CG", "init": "bias_free_energies"},
]
for _c in SPLINE_CASES:
    _c.setdefault("nspline", NSPLINE)
MC_CASES = ("unbiased_ncg", "biased_ncg", "simplesum_ncg")


def _bias(Ku, c):
    return lambda x: 0.5 * Ku * (x - c) ** 2


def spline_parameters(case, z):
    """The spline_parameters dict of a case, for the fixture's samples z (tests/_fes.load)."""
    centres = np.asarray(z["centres"], np.float64)[:, 0]
    Ku = float(z["Ku"])
    p = {"spline_weights": case["weights"], "nspline": case["nspline"], "kdegree": 3, "xrange": list(XRANGE),
         "fkbias": [_bias(Ku, c) for c in centres], "optimization_algorithm": case["algorithm"],
         "spline_initialize": case["init"]}
    p["optimize_options"] = {"disp": False, "tol": 1e-7}
    if case["init"] == "explicit":
        p["xinit"] = np.linspace(XRANGE[0], XRANGE[1], 12)
        p["yinit"] = 2.0 * p["xinit"] ** 2
    if case["init"] == "bias_free_energies":
        p["bias_centers"] = centres
    if case.get("map"):
        a = MAP_A
        p["objective"] = "map"
        p["map_data"] = {"logprior": lambda c: -0.5 * a * np.dot(c, c), "dlogprior": lambda c: -a * c[1:],
                         "ddlogprior": lambda c: -a * np.eye(len(c) - 1)}
    else:
        p["objective"] = "ml"
    return p


def mc_parameters():
    return {"niterations": MC_STEPS, "sample_every": 1, "print_every": 10 ** 9, "fraction_change": 0.01}


def metropolis_margin(lls, draws):
    """The smallest distance, in log-posterior units, of a Metropolis decision of the chain from flipping.  lls are the
    log-likelihoods in call order: two per step, the current spline's (the reference recomputes it every step, its
    first_step flag is never cleared, fes.py:2046-2056) and the proposal's; no prior.  draws are the uniforms
    compared with exp(-dlogp), in order.  |dlogp| when dlogp <= 0 (accepted without a draw), else |-log u - dlogp|."""
    it = iter(draws)
    margin = math.inf
    for n in range(0, len(lls), 2):
        d = lls[n + 1] - lls[n]
        if d <= 0:
            margin = min(margin, -d)
        else:
            margin = min(margin, abs(-math.log(next(it)) - d))
    return margin


# ---- a spline-capable FES stand-in ----------------------------------------------------------------------------

def spline_stand_in():
    """A spline-capable subclass of tests/_fes.StandInFES: the set-up, fit, objective, gradient, Hessian, information
    criteria, queries and MC chain of a spline FES as fes.py documents them, restated for the tests.  The objective,
    gradient and MC likelihood evaluate the spline on the samples (the O(N) path the facade replaces) and count
    their calls."""
    from tests import _fes

    class StandInSplineFES(_fes.StandInFES):
        generate_fes = _get_fes_histogram = _fes.StandInFES._replaced
        original_calls = 0

        def _setup_fes_spline(self, spline_parameters):
            p = spline_parameters
            if p.get("objective", "ml") == "ml":
                p["objective"] = "ml"
                p["map_data"] = {"logprior": None, "dlogprior": None, "ddlogprior": None}
            p.setdefault("optimize_options", {"disp": True, "ftol": 1e-7, "xtol": 1e-7})
            p["scipy_tol"] = p["optimize_options"].pop("tol", None)
            self.spline_parameters = p
            xinit, yinit = self._initial_points()
            self.spline_data = self._initial_spline(xinit, yinit)
            self.fes_functions = None

        def _initial_points(self):
            p = self.spline_parameters
            ns, k, xr = p["nspline"], p["kdegree"], p["xrange"]
            how = p["spline_initialize"]
            if how == "zeros":
                x = np.linspace(xr[0], xr[1], ns + k)
                return x, np.zeros(len(x))
            if how == "explicit":
                return p["xinit"], p["yinit"]
            # bias_free_energies with bias centres and K < 2 nspline: a least-squares spline through the centres
            fk = self.mbar.f_k
            bc = np.asarray(p["bias_centers"])
            order = np.argsort(bc)
            K = self.mbar.K
            assert K < 2 * ns
            nover = int(np.round(K / 2))
            tinit = np.concatenate([[xr[0]] * k, np.linspace(xr[0], xr[1], nover + 1 - k), [xr[1]] * k])
            b = make_lsq_spline(bc[order], fk[order], tinit, k=k)
            x = np.linspace(xr[0], xr[1], 2 * ns)
            return x, b(x)

        def _initial_spline(self, xinit, yinit):
            p = self.spline_parameters
            ns, k, xr = p["nspline"], p["kdegree"], p["xrange"]
            t = np.concatenate([[xr[0]] * k, np.linspace(xr[0], xr[1], ns + 1 - k), [xr[1]] * k])
            order = np.argsort(xinit)
            b = make_lsq_spline(np.asarray(xinit)[order], np.asarray(yinit)[order], t, k=k)
            b.c = b.c - b.c[0]
            db_c = [BSpline(b.t, np.eye(ns)[i], b.k) for i in range(ns)]
            xri = np.stack([t[:ns], t[k + 1:k + 1 + ns]], axis=1)
            xrij = np.zeros([ns, ns, 2])
            for i in range(ns):
                for j in range(ns):
                    xrij[i, j] = [max(xri[i, 0], xri[j, 0]), min(xri[i, 1], xri[j, 1])]
            return {"initial_coefficients": b.c[1:], "bspline_derivatives": db_c, "bspline": b, "xrangei": xri,
                    "xrangeij": xrij}

        @staticmethod
        def _integrate(func, xlow, xhigh, args=(), method="quad"):
            return quad(func, xlow, xhigh, args)[0]

        def _val_to_spline(self, x, form=None):
            tb = self.spline_data["bspline"]
            return BSpline(tb.t, np.concatenate([[tb.c[0]], x]), tb.k)

        def _scaling(self):
            K, N = self.mbar.K, self.N
            return (N / K) * np.ones(K) if self.spline_parameters["spline_weights"] == "simplesum" else self.mbar.N_k

        def _sample_sum(self, fn, x_n, w_n):
            """The sample term of fn (a spline or basis function) under the fit's weighting, over every sample."""
            mbar, K, N = self.mbar, self.mbar.K, self.N
            how = self.spline_parameters["spline_weights"]
            if how == "unbiasedstate":
                return N * np.dot(w_n, fn(x_n))
            if how == "biasedstates":
                return np.sum(fn(x_n))
            total = 0
            for k in range(K):
                total += (N / K) * np.mean(fn(x_n[mbar.x_kindices == k]))
            return total

        def _bspline_calculate_f(self, xi, x_n, w_n):
            type(self).original_calls += 1
            p = self.spline_parameters
            bloc = self._val_to_spline(xi)
            xr, fkbias = p["xrange"], p["fkbias"]
            f = self._sample_sum(bloc, x_n, w_n)
            if p["spline_weights"] == "unbiasedstate":
                def expf(x):
                    return np.exp(-bloc(x))

                pF = self._integrate(expf, xr[0], xr[1])
                f += self.N * np.log(pF)
            else:
                pF = np.zeros(self.mbar.K)
                expf = []
                for k in range(self.mbar.K):
                    def fk(x, kf=k):
                        return np.exp(-bloc(x) - fkbias[kf](x))

                    pF[k] = self._integrate(fk, xr[0], xr[1], args=(k,))
                    expf.append(fk)
                f += np.dot(self._scaling(), np.log(pF))
            self.spline_data["bspline_expf"] = expf
            self.spline_data["bspline_pF"] = pF
            if p["map_data"]["logprior"] is not None:
                f -= p["map_data"]["logprior"](np.concatenate([[0], xi]))
            return f

        def _bspline_calculate_g(self, xi, x_n, w_n):
            type(self).original_calls += 1
            p = self.spline_parameters
            bloc = self._val_to_spline(xi)
            xr, fkbias, ns = p["xrange"], p["fkbias"], p["nspline"]
            db_c, xri = self.spline_data["bspline_derivatives"], self.spline_data["xrangei"]
            g = np.array([self._sample_sum(db_c[i], x_n, w_n) for i in range(1, ns)], dtype=np.float64)
            if p["spline_weights"] == "unbiasedstate":
                gkquad = 0

                def expf(x):
                    return np.exp(-bloc(x))

                pF = self._integrate(expf, xr[0], xr[1])
                pE = np.zeros(ns - 1)

                def dexpf(x, index):
                    return db_c[index + 1](x) * expf(x)

                for i in range(ns - 1):
                    pE[i] = self._integrate(dexpf, xri[i + 1, 0], xri[i + 1, 1], args=(i,))
                    pE[i] /= pF
                g -= self.N * pE
            else:
                K = self.mbar.K
                gkquad = np.zeros([ns - 1, K])

                def expf(x, k):
                    return np.exp(-bloc(x) - fkbias[k](x))

                for k in range(K):
                    pFk = self._integrate(expf, xr[0], xr[1], args=(k,))
                    for i in range(ns - 1):
                        def dexpf(x, k, i=i):
                            return db_c[i + 1](x) * expf(x, k)

                        pE = self._integrate(dexpf, xri[i + 1, 0], xri[i + 1, 1], args=(k,))
                        gkquad[i, k] = pE / pFk
                g -= np.dot(gkquad, self._scaling())
            if p["map_data"]["dlogprior"] is not None:
                g -= p["map_data"]["dlogprior"](np.concatenate([[0], xi]))
            self.spline_data["bspline_gkquad"] = gkquad
            self.spline_data["bspline_pE"] = pE
            return g

        def _bspline_calculate_h(self, xi, x_n, w_n):
            p = self.spline_parameters
            ns, k = p["nspline"], p["kdegree"]
            db_c, xrij = self.spline_data["bspline_derivatives"], self.spline_data["xrangeij"]
            expf, gkquad = self.spline_data["bspline_expf"], self.spline_data["bspline_gkquad"]
            pF, pE = self.spline_data["bspline_pF"], self.spline_data["bspline_pE"]
            unbiased = p["spline_weights"] == "unbiasedstate"
            if unbiased:
                h = -self.N * np.outer(pE, pE)
            else:
                sc = self._scaling()
                h = np.zeros([ns - 1, ns - 1])
                for kk in range(self.mbar.K):
                    h += -sc[kk] * np.outer(gkquad[:, kk], gkquad[:, kk])
            for i in range(ns - 1):
                for j in range(i + 1):
                    if abs(i - j) > k:
                        continue
                    lo, hi = xrij[i + 1, j + 1]
                    if unbiased:
                        def dd(x, a, b):
                            return db_c[a + 1](x) * db_c[b + 1](x) * expf(x)

                        h[i, j] += self.N * self._integrate(dd, lo, hi, args=(i, j)) / pF
                    else:
                        def dd(x, kk, i=i, j=j):
                            return db_c[i + 1](x) * db_c[j + 1](x) * expf[kk](x)

                        for kk in range(self.mbar.K):
                            h[i, j] += sc[kk] * self._integrate(dd, lo, hi, args=(kk,)) / pF[kk]
            for i in range(ns - 1):
                for j in range(i + 1, ns - 1):
                    h[i, j] = h[j, i]
            if p["map_data"]["ddlogprior"] is not None:
                h -= p["map_data"]["ddlogprior"](np.concatenate([[0], xi]))
            return h

        def _generate_fes_spline(self, b, x_n, w_n):
            p = self.spline_parameters
            xi = self.spline_data["initial_coefficients"].copy()
            f, g, h = self._bspline_calculate_f, self._bspline_calculate_g, self._bspline_calculate_h
            args = (x_n, w_n)
            # optimization_algorithm="Custom-NR" raises UnboundLocalError in the reference (fes.py:1040 reads
            # spline_args, which only the scipy branch defines), so the stand-in has the scipy branch only
            r = minimize(f, xi, args=args, method=p["optimization_algorithm"], jac=g, tol=p["scipy_tol"], hess=h,
                         options=p["optimize_options"])
            xi = r["x"]
            mll = f(xi, *args)
            self.spline_data["first_coefficients"] = xi
            self.spline_data["aic"] = 2 * len(xi) + 2 * mll
            self.spline_data["bic"] = 2 * np.log(self.N) * len(xi) + 2 * mll
            self.fes_function = self._val_to_spline(xi)

        def get_information_criteria(self, type="akaike"):
            return self.spline_data["aic" if type == "akaike" else "bic"]

        def get_fes(self, x, reference_point="from-lowest", fes_reference=None, uncertainty_method=None):
            if self.fes_type != "spline":
                return super().get_fes(x, reference_point, fes_reference, uncertainty_method)
            x = np.array(x)
            if x.ndim <= 1:
                x = x.reshape(-1, 1)
            f = self.fes_function(x[:, 0])
            if reference_point == "from-lowest":
                f = f - np.min(f)
            else:
                f = f + self.fes_function(np.array(fes_reference).reshape(1, -1))
            return {"f_i": f, "df_i": None}

        def _get_MC_loglikelihood(self, x_n, w_n, spline_weights, spline, xrange):
            type(self).original_calls += 1
            N, K = self.N, self.K
            if spline_weights == "unbiasedstate":
                return N * np.dot(w_n, spline(x_n))
            fkbias = self.spline_parameters["fkbias"]
            ll = 0
            for k in range(K):
                xk = x_n[self.mbar.x_kindices == k]

                def ek(x, kf):
                    return np.exp(-(spline(x) + fkbias[kf](x)))

                norm = np.log(self._integrate(ek, xrange[0], xrange[1], args=(k,)))
                vals = spline(xk) + fkbias[k](xk)
                if spline_weights == "simplesum":
                    ll += (N / K) * np.mean(vals)
                    ll += (N / K) * norm
                else:
                    ll += np.sum(vals)
                    ll += self.N_k[k] * norm
            return ll

        def sample_parameter_distribution(self, x_n, mc_parameters=None, decorrelate=False, verbose=False):
            """The Metropolis chain of fes.py:1696-1857 with sample_every = 1 and without decorrelation."""
            p = self.spline_parameters
            mp = mc_parameters
            xr, weights = p["xrange"], p["spline_weights"]
            bspline = self.fes_function
            bspline.c = bspline.c + np.log(self._integrate(lambda x: np.exp(-bspline(x)), xr[0], xr[1]))
            dc = mp["fraction_change"] * (np.max(bspline.c) - np.min(bspline.c))
            new = BSpline(bspline.t, bspline.c, bspline.k)
            naccept = 0
            samples = np.zeros([len(bspline.c), mp["niterations"]])
            logpost = np.zeros(mp["niterations"])
            for n in range(mp["niterations"]):
                # the current spline's likelihood, recomputed at every step as the reference does
                prev = self._get_MC_loglikelihood(x_n, self.w_n, weights, bspline, xr)
                cold = bspline.c
                r = dc * np.random.normal()
                cnew = cold.copy()
                cnew[np.random.randint(len(cold))] += r
                new.c = cnew
                cnew = cnew + np.log(self._integrate(lambda x: np.exp(-new(x)), xr[0], xr[1]))
                new.c = cnew
                lp = self._get_MC_loglikelihood(x_n, self.w_n, weights, new, xr)
                d = lp - prev
                if d <= 0 or np.random.random() < np.exp(-d):
                    bspline.c = new.c
                    prev = lp
                    naccept += 1
                samples[:, n] = bspline.c
                logpost[n] = prev
            self.mc_data = {"samples": samples, "logposteriors": logpost, "naccept": naccept}

    return StandInSplineFES

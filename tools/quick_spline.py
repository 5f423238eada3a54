#!/usr/bin/env python
"""B-spline basis sums at the C3 sample count (N = 1e7, K = 256, cubic, nspline = 20): kernel time, GB/s and
samples/s of mbar_b200_bspline_moments, the upload time of DeviceBSpline, and the wall time of a spline FES fit
through the facade next to one host scipy BSpline evaluation on the same samples; the card and its power limit,
read in the same run.  Not run by bench.py.

    python tools/quick_spline.py [--n 10000000] [--out quick_spline.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pymbar_b200 import DeviceBSpline  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def knots(k, nspline, lo, hi):
    return np.concatenate([[lo] * k, np.linspace(lo, hi, nspline + 1 - k), [hi] * k])


def fit_through_facade(x, s, w, K, k, nspline, lo, hi, centres, Ku):
    """A facade fit ("unbiasedstate", Newton-CG) on a minimal FES-shaped object: the device pass, then the optimiser
    on the moments (the quadratures do not depend on N)."""
    from scipy.interpolate import BSpline, make_lsq_spline
    from scipy.optimize import minimize

    from pymbar_b200 import fes as hist
    from pymbar_b200.facade import SplineMoments

    class Fit:
        pass

    fes = Fit()
    fes.N, fes.K = len(x), K
    fes.mbar = Fit()
    fes.mbar.K, fes.mbar.N_k = K, np.bincount(s, minlength=K)
    fes.spline_parameters = {"spline_weights": "unbiasedstate", "nspline": nspline, "xrange": (lo, hi),
                             "fkbias": [lambda y, c=c: 0.5 * Ku * (y - c) ** 2 for c in centres],
                             "map_data": {"logprior": None, "dlogprior": None, "ddlogprior": None}}
    t = knots(k, nspline, lo, hi)
    xi0 = np.linspace(lo, hi, nspline + k)
    b = make_lsq_spline(xi0, np.zeros(len(xi0)), t, k=k)
    from scipy.integrate import quad

    fes._integrate = lambda f, a, c, args=(): quad(f, a, c, args)[0]
    fes._val_to_spline = lambda xi: BSpline(b.t, np.concatenate([[b.c[0]], xi]), b.k)
    fes.spline_data = {"bspline": b, "bspline_derivatives": [BSpline(t, np.eye(nspline)[i], k) for i in range(nspline)],
                       "xrangei": np.stack([t[:nspline], t[k + 1:k + 1 + nspline]], axis=1)}
    t0 = time.perf_counter()
    with DeviceBSpline(x, w) as d:
        _, A = d.moments(t, k, want_S=False)
    m = SplineMoments(x, w, None, t, k, "unbiasedstate", None, A, len(x))
    r = minimize(lambda xi: hist.spline_objective(fes, xi, m.v), b.c[1:], method="BFGS",
                 jac=lambda xi: hist.spline_gradient(fes, xi, m.v), tol=1e-7)
    return time.perf_counter() - t0, int(r.nit)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    N, K, k, nspline = a.n, 256, 3, 20
    rng = np.random.RandomState(0)
    centres = np.linspace(-2, 2, K)
    s = np.repeat(np.arange(K), N // K + 1)[:N]
    x = centres[s] + 0.15 * rng.standard_normal(N)
    w = np.exp(-2.0 * x ** 2)
    w /= w.sum()
    t = knots(k, nspline, -2.5, 2.5)
    t0 = time.perf_counter()
    d = DeviceBSpline(x, w, s, K=K)
    upload_ms = 1e3 * (time.perf_counter() - t0)
    d.moments(t, k)                                  # warm-up (module load, first launch)
    ms = []
    for _ in range(5):
        d.moments(t, k)
        ms.append(d.last_stats()["ms"])
    chunks = d.last_stats()["chunks"]
    d.close()
    kern = float(np.median(ms))
    from scipy.interpolate import BSpline

    bs = BSpline(t, rng.standard_normal(nspline), k)
    t0 = time.perf_counter()
    bs(x)
    host_eval_s = time.perf_counter() - t0
    fit_s, nit = fit_through_facade(x, s, w, K, k, nspline, -2.5, 2.5, centres, 2.0)
    res = dict(card=card(), N=N, K=K, degree=k, nspline=nspline, kernel_ms=kern, kernel_ms_all=ms, chunks=chunks,
               GBps=20.0 * N / (kern * 1e-3) / 1e9, samples_per_s=N / (kern * 1e-3), upload_ms=upload_ms,
               facade_fit_s=fit_s, facade_fit_iterations=nit, host_bspline_eval_s=host_eval_s)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

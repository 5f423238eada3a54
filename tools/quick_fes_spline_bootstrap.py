#!/usr/bin/env python
"""Spline FES bootstrap replicates at a user-sized shape (default K = 64 umbrella windows, N = 1e6 samples, B = 50
replicates, cubic, nspline = 20) for each spline_weights: the wall time of a bootstrap generate_fes through the
facade (on the FES-shaped stand-in class of the tests, with the device backend), split into b = 0 (the same call
without replicates), drawing the stream with the replicate weights, the replicate solves ("unbiasedstate" only), the
upload and replicate_sums call (with its CUDA-event kernel time) and the replicate fits; then the kernel time of one
replicate_sums call against B single-replicate moments(want_S=False) calls on the same weights; and the card and its
power limit, read in the same run.  The fits' quadratures are host work whose cost does not depend on N; with
"biasedstates" and "simplesum" every objective evaluation integrates over all K states, so --fit-B can cap the number
of replicates fitted for those weightings, and --weightings "" runs the kernel comparison alone.  Not run by
bench.py.

    python tools/quick_fes_spline_bootstrap.py [--K 64] [--N 1000000] [--B 50] [--fit-B 50]
        [--weightings unbiasedstate,biasedstates,simplesum] [--out quick_fes_spline_bootstrap.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pymbar_b200 import DeviceBSpline, facade  # noqa: E402
from pymbar_b200 import fes_bootstrap as fb  # noqa: E402
from pymbar_b200 import mbar_solvers as ms  # noqa: E402
from tests.test_driver_logic_cpu import StandInMBAR  # noqa: E402
from tests.test_fes_spline_bootstrap_cpu import boot_stand_in  # noqa: E402
from tools.quick_fes_bootstrap import card, umbrellas  # noqa: E402

K0, KU = 4.0, 40.0


def parameters(weights, centres, nspline):
    fkbias = [(lambda x, c=c: 0.5 * KU * (x - c) ** 2) for c in centres]
    return {"spline_weights": weights, "nspline": nspline, "kdegree": 3, "xrange": [-2.2, 2.2], "fkbias": fkbias,
            "optimization_algorithm": "Newton-CG", "spline_initialize": "zeros", "objective": "ml",
            "optimize_options": {"disp": False, "tol": 1e-7}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, default=64)
    ap.add_argument("--N", type=int, default=1_000_000)
    ap.add_argument("--B", type=int, default=50)
    ap.add_argument("--fit-B", type=int, default=None, help="replicates fitted for biasedstates / simplesum")
    ap.add_argument("--nspline", type=int, default=20)
    ap.add_argument("--weightings", default="unbiasedstate,biasedstates,simplesum")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    x, u_kn, u_n, N_k = umbrellas(a.K, a.N)
    centres = np.linspace(-2.0, 2.0, a.K)
    StandInMBAR.solvers = ms
    cls = boot_stand_in()
    cls.mbar_class = StandInMBAR
    facade.install_on(StandInMBAR)
    facade.install_fes_on(cls)
    res = dict(card=card(), K=a.K, N=a.N, B=a.B, nspline=a.nspline, degree=3)
    try:
        fes = cls(u_kn, N_k)
        for weights in filter(None, a.weightings.split(",")):
            B = a.B if weights == "unbiasedstate" or a.fit_B is None else a.fit_B
            for _ in range(2):                  # warm-up, then the cost of b = 0 alone
                t0 = time.perf_counter()
                fes.generate_fes(u_n, x, fes_type="spline", spline_parameters=parameters(weights, centres, a.nspline))
                b0 = time.perf_counter() - t0
            s0 = dict(facade.STATS)
            t0 = time.perf_counter()
            fes.generate_fes(u_n, x, fes_type="spline", spline_parameters=parameters(weights, centres, a.nspline),
                             n_bootstraps=B, seed=1)
            total = time.perf_counter() - t0
            split = dict(fes.__dict__.get("_b200_spline_boot_times", {}))
            split["b0_s"] = b0
            split["fits_per_replicate_s"] = split.get("fits", float("nan")) / B
            res[weights] = dict(B=B, generate_s=total, split=split,
                                stats={k: facade.STATS[k] - s0[k] for k in facade.STATS if facade.STATS[k] != s0[k]})
            print(json.dumps({weights: res[weights]}), flush=True)
        # kernel time: one replicate_sums call against B single-replicate moments on the same weights
        # the fit's knots (fes.py:913-918)
        t = np.concatenate([[-2.2] * 3, np.linspace(-2.2, 2.2, a.nspline - 2), [2.2] * 3])
        np.random.seed(1)
        _, V = fb.spline_replicates(N_k, a.B, "biasedstates")
        with DeviceBSpline(x) as d:
            t0 = time.perf_counter()
            d.set_replicates(V)
            upload = time.perf_counter() - t0
            d.replicate_sums(t, 3)
            rep_ms = []
            for _ in range(a.reps):
                d.replicate_sums(t, 3)
                rep_ms.append(d.last_stats()["ms"])
            passes = d.last_stats()["chunks"]
        single_ms = 0.0
        for b in range(a.B):
            with DeviceBSpline(x, V[b]) as one:
                one.moments(t, 3, want_S=False)
                one.moments(t, 3, want_S=False)
                single_ms += one.last_stats()["ms"]
        med = float(np.median(rep_ms))
        res["kernel"] = dict(replicate_sums_ms=med, passes=passes, B_moments_ms=single_ms, speedup=single_ms / med,
                             set_replicates_s=upload, V_bytes=int(V.nbytes))
        print(json.dumps({k: res[k] for k in ("card", "kernel")}), flush=True)
    finally:
        facade.uninstall_from(cls)
        facade.uninstall_from(StandInMBAR)
        ms.clear_cache()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

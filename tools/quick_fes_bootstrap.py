#!/usr/bin/env python
"""FES bootstrap replicates at a user-sized shape (default K = 64 umbrella windows, N = 1e6 samples, B = 50
replicates, a 100-point grid): the wall time of a bootstrap generate_fes + get_fes for a histogram and for a KDE
surface through the facade (on the FES-shaped stand-in classes of the tests, with the device backend), the kernel
time of one log_sum_replicates call against B log_sum calls with the replicates' weights (mbar_b200_last_kde_stats),
where a bootstrap generate_fes spends its time (the same call without replicates, drawing the stream with the
replicate weights, their upload), and the card and its power limit, read in the same run.  The reference's side is counted from the shapes, not timed:
its loop builds K MBAR objects per replicate (fes.py:396-406), K B solves and K B gathers of 8 K N bytes.  Not run
by bench.py.

    python tools/quick_fes_bootstrap.py [--K 64] [--N 1000000] [--B 50] [--out quick_fes_bootstrap.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pymbar_b200 import DeviceKde, facade  # noqa: E402
from pymbar_b200 import mbar_solvers as ms  # noqa: E402
from tests import _fes, _kde  # noqa: E402
from tests.test_driver_logic_cpu import StandInMBAR  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def umbrellas(K, N, seed=0):
    rng = np.random.RandomState(seed)
    centres = np.linspace(-2.0, 2.0, K).reshape(-1, 1)
    K0, Ku = 4.0, 40.0
    n_k = np.full(K, N // K)
    n_k[: N - n_k.sum()] += 1
    x = np.concatenate([rng.normal(Ku * centres[k, 0] / (K0 + Ku), 1.0 / np.sqrt(K0 + Ku), size=n_k[k])
                        for k in range(K)])
    u_kn, u_n = _fes.umbrella_energies(x, centres, K0, Ku)
    return x, u_kn, u_n, n_k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, default=64)
    ap.add_argument("--N", type=int, default=1_000_000)
    ap.add_argument("--B", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    x, u_kn, u_n, N_k = umbrellas(a.K, a.N)
    grid = np.linspace(-1.5, 1.5, 100)
    StandInMBAR.solvers = ms
    cls = _kde.kde_stand_in()
    cls.mbar_class = StandInMBAR
    facade.install_on(StandInMBAR)
    facade.install_fes_on(cls)
    res = dict(card=card(), K=a.K, N=a.N, B=a.B, Q=len(grid))
    try:
        fes = cls(u_kn, N_k)
        kinds = (("histogram", dict(histogram_parameters={"bin_edges": np.linspace(-1.5, 1.5, 101)})),
                 ("kde", dict(kde_parameters={"bandwidth": 0.05})))
        # warm-up, and the cost of b = 0 alone: the first KDE call imports sklearn (several seconds on a fresh host)
        split = {}
        for fes_type, kw in kinds:
            for _ in range(2):
                t0 = time.perf_counter()
                fes.generate_fes(u_n, x, fes_type=fes_type, n_bootstraps=0, seed=1, **kw)
                split[f"{fes_type}_without_replicates_s"] = time.perf_counter() - t0
        for fes_type, kw in kinds:
            s0 = dict(facade.STATS)
            t0 = time.perf_counter()
            fes.generate_fes(u_n, x, fes_type=fes_type, n_bootstraps=a.B, seed=1, **kw)
            t1 = time.perf_counter()
            r = fes.get_fes(grid, reference_point="from-lowest", uncertainty_method="bootstrap")
            t2 = time.perf_counter()
            res[fes_type] = dict(generate_s=t1 - t0, get_fes_s=t2 - t1, finite_df=int(np.isfinite(r["df_i"]).sum()),
                                 stats={k: facade.STATS[k] - s0[k] for k in facade.STATS if facade.STATS[k] != s0[k]})
            print(json.dumps({fes_type: res[fes_type]}), flush=True)
        # kernel time: one replicate pass against B single-weight passes
        dev, settings, _ = fes.__dict__["_b200_kde_dev"]
        y = grid.reshape(-1, 1)
        dev.log_sum_replicates("gaussian", settings["h"], y)
        rep_ms = []
        for _ in range(a.reps):
            dev.log_sum_replicates("gaussian", settings["h"], y)
            rep_ms.append(dev.last_stats()["ms"])
        w = np.asarray(fes.w_n)
        from pymbar_b200 import fes_bootstrap as fb

        V = np.empty((a.B, a.N))
        np.random.seed(1)
        t0 = time.perf_counter()
        fb.draw_replicates(N_k, a.B, lambda b, idx: V.__setitem__(b, np.bincount(idx, weights=w, minlength=a.N)))
        t1 = time.perf_counter()
        dev.set_replicates(V)
        t2 = time.perf_counter()
        # where a KDE bootstrap generate_fes goes besides b = 0: the stream with the replicate weights, their upload
        split.update(draw_and_weights_s=t1 - t0, set_replicates_s=t2 - t1)
        res["generate_split"] = split
        print(json.dumps({"split": split}), flush=True)
        single_ms = 0.0
        for b in range(a.B):
            with DeviceKde(x, V[b]) as one:
                one.log_sum("gaussian", settings["h"], y)
                one.log_sum("gaussian", settings["h"], y)
                single_ms += one.last_stats()["ms"]
        res["kernel"] = dict(log_sum_replicates_ms=float(np.median(rep_ms)), B_log_sum_ms=single_ms,
                             speedup=single_ms / float(np.median(rep_ms)))
        res["reference_counted"] = dict(mbar_solves=a.K * a.B, gathers=a.K * a.B,
                                        gather_bytes=8 * a.K * a.N * a.K * a.B)
        print(json.dumps({k: res[k] for k in ("card", "kernel", "reference_counted")}), flush=True)
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

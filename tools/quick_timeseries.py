#!/usr/bin/env python
"""Lag sums of pymbar.timeseries on the GPU: detect_equilibration at T = 1e5 and 1e6 (nskip = 1, fast) and
statistical_inefficiency(fast=False) at T = 1e8 with tau = 1e3, each as kernel time (CUDA events of the
mbar_b200_acf call), wall time of the pymbar_b200.timeseries call, lag rounds, the lag terms evaluated and their
waste, terms/s and fp64 operations/s (3 per auto-correlation term: the centring of A[n + t], the product and the
sum; the centring of A[n] is shared by a thread's 4 lags) against the DFMA ceiling measured in the same process; the reference's CPU time for
detect_equilibration at T = 8000 when `--reference` points at a pymbar checkout; the card and its power limit.
Not run by bench.py.

    python tools/quick_timeseries.py [--big 100000000] [--reference /path/to/pymbar] [--out quick_timeseries.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pymbar_b200 import DeviceAcf  # noqa: E402
from pymbar_b200 import timeseries as ts  # noqa: E402
from pymbar_b200.problem import measure_fp64_peak  # noqa: E402

FLOPS_PER_TERM = 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def ar1(seed, T, tau):
    from scipy.signal import lfilter

    rng = np.random.RandomState(seed)
    a = np.exp(-1.0 / tau)
    return lfilter([1.0], [1.0, -a], rng.standard_normal(T) * np.sqrt(1 - a * a))


def measure(name, A, starts, fast, wall_fn, dfma):
    with DeviceAcf(A) as dev:
        dev.inefficiency(starts[:2], fast=fast)              # warm-up (module load, first launches)
        t0 = time.perf_counter()
        dev.inefficiency(starts, fast=fast)
        call_s = time.perf_counter() - t0
        st = dev.last_stats()
    t0 = time.perf_counter()
    wall_fn()
    wall = time.perf_counter() - t0
    terms_s = st["terms"] / (st["ms"] * 1e-3)
    r = dict(case=name, kernel_ms=st["ms"], device_call_s=call_s, wall_s=wall, rounds=st["rounds"],
             terms=st["terms"], useful_terms=st["useful_terms"], waste=st["waste"], terms_per_s=terms_s,
             fp64_tflops=FLOPS_PER_TERM * terms_s / 1e12, share_of_dfma=FLOPS_PER_TERM * terms_s / 1e12 / dfma)
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--big", type=int, default=100_000_000)
    ap.add_argument("--reference", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    _, dfma = measure_fp64_peak()
    res = dict(card=card(), dfma_tflops=dfma, cases=[])
    for T in (100_000, 1_000_000):
        A = ar1(T, T, 20.0) + 10.0 * np.exp(-np.arange(T) / (T / 200.0))
        res["cases"].append(measure(f"detect_equilibration T={T}", A, np.arange(T - 1), True,
                                    lambda: ts.detect_equilibration(A, fast=True, nskip=1), dfma))
    A = ar1(7, a.big, 1000.0)
    res["cases"].append(measure(f"statistical_inefficiency fast=False T={a.big}", A, np.array([0]), False,
                                lambda: ts.statistical_inefficiency(A, fast=False), dfma))
    if a.reference:
        sys.path.insert(0, os.path.abspath(a.reference))
        from pymbar import timeseries as ref

        A = ar1(1, 8000, 20.0) + 10.0 * np.exp(-np.arange(8000) / 40.0)
        t0 = time.perf_counter()
        ref.detect_equilibration(A, fast=True, nskip=1)
        res["reference_cpu_s_T8000"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        ts.detect_equilibration(A, fast=True, nskip=1)
        res["device_wall_s_T8000"] = time.perf_counter() - t0
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

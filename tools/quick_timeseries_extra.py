#!/usr/bin/env python
"""The multiple-series correlation function and the FFT rule of pymbar.timeseries on the GPU, per case the kernel
time (CUDA events of the mbar_b200_acf call, after a warm-up call of the same shape), the wall time of the
pymbar_b200.timeseries call, truncate / lag rounds, the lag terms evaluated and their rate, and the card with its
power limit read in the same run:

* normalized_fluctuation_correlation_function_multiple, 10 series x 1e5, 10 x 1e6 and 1000 x 2000 (many short
  series: a few chunks each), with and without truncate;
* statistical_inefficiency_fft at T = 1e8 with tau = 1e3, and at T = 1e6 for a linear drift (crossing near T / 2);
* detect_equilibration_binary_search at T = 1e6.
Not run by bench.py.

    python tools/quick_timeseries_extra.py [--big 100000000] [--out quick_timeseries_extra.json]
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def ar1(seed, T, tau):
    from scipy.signal import lfilter

    rng = np.random.RandomState(seed)
    a = np.exp(-1.0 / tau)
    return lfilter([1.0], [1.0, -a], rng.standard_normal(T) * np.sqrt(1 - a * a))


def report(name, st, wall, **extra):
    r = dict(case=name, kernel_ms=st["ms"], wall_s=wall, rounds=st["rounds"], terms=st["terms"],
             useful_terms=st["useful_terms"], terms_per_s=st["terms"] / (st["ms"] * 1e-3) if st["ms"] else 0.0,
             **extra)
    print(json.dumps(r), flush=True)
    return r


def correlation_multiple(K, n, truncate):
    A_kn = [ar1(100 + k, n, 20.0) for k in range(K)]
    a = np.concatenate(A_kn)
    with DeviceAcf(a, lengths=[n] * K) as dev:
        dev.correlation_multiple(n - 1, truncate)                 # warm-up of the same shape
        C, *_ = dev.correlation_multiple(n - 1, truncate)
        st = dev.last_stats()
    t0 = time.perf_counter()
    ts.normalized_fluctuation_correlation_function_multiple(A_kn, truncate=truncate)
    wall = time.perf_counter() - t0
    return report(f"correlation_multiple {K}x{n} truncate={truncate}", st, wall, returned=int(C.size))


def fft(name, A):
    with DeviceAcf(A) as dev:
        dev.inefficiency([0], rule="fft")
        r = dev.inefficiency([0], rule="fft")
        st = dev.last_stats()
    t0 = time.perf_counter()
    ts.statistical_inefficiency_fft(A)
    wall = time.perf_counter() - t0
    return report(name, st, wall, g=float(r["g"][0]), last_lag=int(r["last_lag"][0]))


def binary_search(T):
    A = ar1(9, T, 20.0) + 10.0 * np.exp(-np.arange(T) / (T / 200.0))
    ts.detect_equilibration_binary_search(A[:1000])               # warm-up
    t0 = time.perf_counter()
    t, g, Neff = ts.detect_equilibration_binary_search(A)
    wall = time.perf_counter() - t0
    r = dict(case=f"detect_equilibration_binary_search T={T}", wall_s=wall, t=int(t), g=float(g), Neff=float(Neff))
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--big", type=int, default=100_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card(), cases=[])
    for K, n in ((10, 100_000), (10, 1_000_000), (1000, 2000)):
        for truncate in (False, True):
            res["cases"].append(correlation_multiple(K, n, truncate))
    res["cases"].append(fft(f"statistical_inefficiency_fft T={a.big} tau=1e3", ar1(7, a.big, 1000.0)))
    T = 1_000_000
    drift = np.linspace(0.0, 1.0, T) + 1e-3 * np.random.RandomState(8).standard_normal(T)
    res["cases"].append(fft(f"statistical_inefficiency_fft T={T} linear drift", drift))
    res["cases"].append(binary_search(T))
    res["card_after"] = card()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

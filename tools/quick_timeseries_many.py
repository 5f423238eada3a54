#!/usr/bin/env python
"""The lockstep many-series functions of pymbar_b200.timeseries on one GPU, against the loop of single-series device
calls on the same inputs, with the card, its power limit and max SM clock read in the same run:

1. detect_equilibration_many(fast=True, nskip=1) on 8000 AR(1) series of T = 5000 with a decaying transient (a
   500-edge x 16-window campaign);
2. the same on 200 series of T = 1e5 (long series, where batching gains least);
3. statistical_inefficiency_many(fast=False) on the 8000 x 5000 set.

Per case: the host wall time of the call (after a warm-up of the same shape; every call ends in a synchronise),
the kernel time (CUDA events of each inefficiency_series call, summed over waves), rounds, waves, kernel launches
(counted by torch.profiler on one more call), lag terms and their rate, and the loop of single-series calls on a stated
prefix of the series with identical outputs asserted.  Not run by bench.py.

    python tools/quick_timeseries_many.py [--prefix 400] [--out quick_timeseries_many.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pymbar_b200 import timeseries as ts  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def campaign(P, T, seed):
    from scipy.signal import lfilter

    rng = np.random.RandomState(seed)
    out = []
    for k in range(P):
        tau = 2.0 + 18.0 * rng.random_sample()
        a = np.exp(-1.0 / tau)
        x = lfilter([1.0], [1.0, -a], rng.standard_normal(T) * np.sqrt(1 - a * a))
        out.append(x + rng.uniform(1.0, 6.0) * np.exp(-np.arange(T) / (T * rng.uniform(0.01, 0.1))))
    return out


def launches(fn):
    """kernel launches of one call, from torch.profiler (None where it cannot run)"""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile

        if not torch.cuda.is_available():
            return None
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
        return sum(e.count for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA and
                   "acf_" in e.key)
    except Exception:          # noqa: BLE001
        return None


def case(name, many, single, A, prefix):
    many(A)                                                          # warm-up of the same shape
    t0 = time.perf_counter()
    out = many(A)
    wall = time.perf_counter() - t0
    st = dict(ts.LAST_MANY_STATS)
    n = min(prefix, len(A))
    single(A[:2])                                                    # warm-up
    t0 = time.perf_counter()
    loop = [single([a])[0] for a in A[:n]]
    loop_wall = time.perf_counter() - t0
    same = all(np.array_equal(np.asarray(x, np.float64), np.asarray(y, np.float64)) and
               [type(v) for v in np.atleast_1d(x)] == [type(v) for v in np.atleast_1d(y)]
               for x, y in zip(out[:n], loop))
    assert same, name
    r = dict(case=name, series=len(A), T=int(A[0].size), wall_s=wall, kernel_ms=st["ms"], rounds=st["rounds"],
             waves=st["waves"], requests=st["requests"], terms=st["terms"],
             terms_per_s=st["terms"] / (st["ms"] * 1e-3) if st["ms"] else 0.0,
             launches=launches(lambda: many(A)), loop_prefix=n, loop_prefix_wall_s=loop_wall,
             loop_wall_s_extrapolated=loop_wall * len(A) / n, identical_on_prefix=same)
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--prefix", type=int, default=400)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card(), cases=[])
    camp = campaign(8000, 5000, 1)

    def eq_many(A):
        return ts.detect_equilibration_many(A, fast=True, nskip=1)

    def eq_single(A):
        return [ts.detect_equilibration(x, fast=True, nskip=1) for x in A]

    def si_many(A):
        return ts.statistical_inefficiency_many(A, fast=False)

    def si_single(A):
        return [ts.statistical_inefficiency(x, fast=False) for x in A]

    res["cases"].append(case("detect_equilibration_many fast nskip=1 8000x5000", eq_many, eq_single, camp, a.prefix))
    res["cases"].append(case("detect_equilibration_many fast nskip=1 200x1e5", eq_many, eq_single,
                             campaign(200, 100_000, 2), max(1, a.prefix // 20)))
    res["cases"].append(case("statistical_inefficiency_many fast=False 8000x5000", si_many, si_single, camp,
                             8000))
    res["card_after"] = card()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

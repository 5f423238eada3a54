#!/usr/bin/env python
"""Time MbarMany.compute_entropy_and_enthalpy against the single-problem loop on the same inputs.

    python tools/quick_mbar_many_expectations.py [P ...] [K=k ...]    (default: 100 1000, K=16 K=32)

Workload: P harmonic ladders (spring constants 1 to 3) with K = 16 and K = 32 states and N_k = 5000 samples each.  For
each (K, P) it reports the wall time of the construction (upload and solve) and of compute_entropy_and_enthalpy, each
ending in a synchronisation; the kernel time and launches of the estimator's device calls (DeviceMbarBatch.last_stats,
summed in MbarMany.device_stats); and the host time of the entropy/enthalpy algebra (one 3K x 3K eigendecomposition
per problem, timed alone on the batched results).  The single-problem path (DeviceProblem upload, then
expectations_inner with the entropy/enthalpy state map and the same algebra) runs on the first SINGLE problems and is
extrapolated to P, labelled as such; the largest difference between the two paths' Delta_s is reported.  The card name
and power limit come from nvidia-smi in the same run.  Results go to stdout as JSON lines.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pymbar_b200 import DeviceProblem  # noqa: E402
from pymbar_b200 import expectations as ex  # noqa: E402
from pymbar_b200.mbar_many import MbarMany  # noqa: E402

NPER, SINGLE = 5000, 30


def ladder(K, seed):
    rng = np.random.RandomState(seed)
    centres = 0.4 * np.arange(K)
    spring = np.linspace(1.0, 3.0, K)
    N_k = np.full(K, NPER, np.float64)
    x = np.repeat(centres, NPER) + rng.normal(size=K * NPER) / np.repeat(np.sqrt(spring), NPER)
    return 0.5 * spring[:, None] * (x[None, :] - centres[:, None]) ** 2, N_k


def single(u, N_k, f):
    K = len(N_k)
    with DeviceProblem(u, N_k) as q:
        inner = ex.expectations_inner(u, N_k, f, u, u, np.array([np.arange(K), np.arange(K)]), return_theta=True,
                                      problem=q)
    return ex.entropy_enthalpy_result(inner, K)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main(Ps, Ks=(16, 32)):
    print(json.dumps(dict(card=card())), flush=True)
    for K in Ks:
        for P in Ps:
            probs = [ladder(K, s) for s in range(P)]
            us, nks = [p[0] for p in probs], [p[1] for p in probs]
            t0 = time.perf_counter()
            m = MbarMany(us, nks, compute_uncertainty=False)
            t_solve = time.perf_counter() - t0
            with m:
                m.compute_entropy_and_enthalpy([us[0]] + [None] * (P - 1))        # warm-up
                m.device_stats.update(ms=0.0, launches=0, calls=0)
                t0 = time.perf_counter()
                res = m.compute_entropy_and_enthalpy()
                t_ent = time.perf_counter() - t0
                stats = dict(m.device_stats)
                f = [r["f_k"] for r in m.results]
            paths = sorted(set(r["path"] for r in res))
            # host algebra alone: the 3K x 3K Theta assembly and its differences, from a saved inner result
            with DeviceProblem(us[0], nks[0]) as q:
                inner = ex.expectations_inner(us[0], nks[0], f[0], us[0], us[0],
                                              np.array([np.arange(K), np.arange(K)]), return_theta=True, problem=q)
            t0 = time.perf_counter()
            for _ in range(20):
                ex.entropy_enthalpy_result(inner, K)
            t_alg = (time.perf_counter() - t0) / 20
            n = min(SINGLE, P)
            single(us[0], nks[0], f[0])                                         # warm-up
            t0 = time.perf_counter()
            ref = [single(us[p], nks[p], f[p]) for p in range(n)]
            t_single = time.perf_counter() - t0
            gap = max(float(np.max(np.abs(a["Delta_s"] - r["Delta_s"]))) for a, r in zip(res, ref))
            print(json.dumps(dict(K=K, P=P, N=K * NPER, construct_s=round(t_solve, 4),
                                  entropy_enthalpy_s=round(t_ent, 4), kernel_ms=round(stats["ms"], 3),
                                  launches=stats["launches"], device_calls=stats["calls"], paths=paths,
                                  theta_host_ms_per_problem=round(1e3 * t_alg, 3),
                                  theta_host_s_all=round(P * t_alg, 4),
                                  single_s_first=round(t_single, 4), single_n=n,
                                  single_s_extrapolated_to_P=round(t_single * P / n, 3),
                                  max_gap_Delta_s=gap)), flush=True)


if __name__ == "__main__":
    Ps = [int(a) for a in sys.argv[1:] if not a.startswith("K=")] or [100, 1000]
    Ks = [int(a[2:]) for a in sys.argv[1:] if a.startswith("K=")] or [16, 32]
    main(Ps, Ks)

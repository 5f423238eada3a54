#!/usr/bin/env python
"""Time MbarMany.compute_entropy_and_enthalpy(uncertainty_method="bootstrap") against the single-problem loop.

    python tools/quick_mbar_many_boot_expectations.py [K:P:B ...]    (default: 16:100:100 32:100:100)

Workload: P harmonic ladders (tools/quick_mbar_many_expectations.py, N_k = 5000 per state) with K states, each with B
bootstrap replicates drawn at construction.  For each case it reports the wall time of compute_entropy_and_enthalpy
under bootstrap after a warm-up, taken with the host clock around the call (every device call in it ends in a
synchronisation); the kernel time, launches, device calls and bytes read of its device calls (MbarMany.device_stats,
summed from DeviceMbarBatch.last_stats); the host time spent regenerating replicate counts (MbarMany.host_stats); and
the single-problem loop (a DeviceProblem upload, then expectations_inner(..., replicates=) with the same counts and the
bootstrap algebra) on the first SINGLE problems, extrapolated to P and labelled as such, with the largest difference
of the two paths' dDelta_s.  The card name and power limit come from nvidia-smi in the same run.  JSON lines on
stdout.
"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from quick_mbar_many_expectations import card, ladder  # noqa: E402

from pymbar_b200 import DeviceProblem  # noqa: E402
from pymbar_b200 import expectations as ex  # noqa: E402
from pymbar_b200.mbar_many import MbarMany  # noqa: E402

SINGLE = 10


def single(m, p, u, N_k):
    K = len(N_k)
    B = m.results[p]["f_k_boots"].shape[0]
    counts = np.array([m._draws[p].counts(b) for b in range(B)])
    with DeviceProblem(u, N_k) as q:
        inner = ex.expectations_inner(u, N_k, m.results[p]["f_k"], u, u, np.array([np.arange(K), np.arange(K)]),
                                      problem=q, replicates=(m.results[p]["f_k_boots"], counts))
    return ex.entropy_enthalpy_result(inner, K, f_k_boots=m.results[p]["f_k_boots"])


def main(cases):
    print(json.dumps(dict(card=card())), flush=True)
    for K, P, B in cases:
        probs = [ladder(K, s) for s in range(P)]
        us, nks = [p[0] for p in probs], [p[1] for p in probs]
        t0 = time.perf_counter()
        m = MbarMany(us, nks, compute_uncertainty=False, n_bootstraps=B, rseed=list(range(P)))
        t_construct = time.perf_counter() - t0
        with m:
            m.compute_entropy_and_enthalpy([us[0]] + [None] * (P - 1), uncertainty_method="bootstrap")   # warm-up
            m.device_stats.update(ms=0.0, launches=0, calls=0, bytes_read=0)
            m.host_stats.update(counts_s=0.0)
            t0 = time.perf_counter()
            res = m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap")
            t_ent = time.perf_counter() - t0
            stats, host = dict(m.device_stats), dict(m.host_stats)
            n = min(SINGLE, P)
            single(m, 0, us[0], nks[0])                                                           # warm-up
            t0 = time.perf_counter()
            ref = [single(m, p, us[p], nks[p]) for p in range(n)]
            t_single = time.perf_counter() - t0
        gap = max(float(np.max(np.abs(a["dDelta_s"] - r["dDelta_s"]))) for a, r in zip(res, ref))
        print(json.dumps(dict(K=K, P=P, B=B, N=K * int(nks[0][0]), construct_s=round(t_construct, 3),
                              boot_entropy_enthalpy_s=round(t_ent, 3), kernel_ms=round(stats["ms"], 3),
                              launches=stats["launches"], device_calls=stats["calls"],
                              bytes_read=stats["bytes_read"], counts_regeneration_s=round(host["counts_s"], 3),
                              paths=sorted(set(r["path"] for r in res)), single_s_first=round(t_single, 3),
                              single_n=n, single_s_extrapolated_to_P=round(t_single * P / n, 2),
                              max_gap_dDelta_s=gap)), flush=True)


if __name__ == "__main__":
    args = sys.argv[1:] or ["16:100:100", "32:100:100"]
    main([tuple(int(x) for x in a.split(":")) for a in args])

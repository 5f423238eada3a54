#!/usr/bin/env python
"""Time mbar_many against a loop of the single-problem path on the same inputs.

    python tools/quick_mbar_many.py [P ...]          (default: 100 1000)

Workload: P harmonic ladders (spring constants 1 to 3) with K = 16 states and N_k = 5000 samples each (N = 80 000 per problem).  For each P it
reports the wall time of mbar_many (upload, solve, all-state update, uncertainties), the kernel time of its solve
(CUDA events, DeviceMbarBatch.last_stats), its launches and iterations; then the wall time of the single-problem path
on every problem (DeviceProblem upload, solve_adaptive with min_sc_iter=0, self_consistent_update, weight_moments),
and the largest |Delta_f| difference between the two.  The card name and power limit come from nvidia-smi in the same
run.  Results go to stdout as JSON lines.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pymbar_b200 import DeviceMbarBatch, DeviceProblem, estimators  # noqa: E402
from pymbar_b200.mbar_many import mbar_many  # noqa: E402

K, NPER = 16, 5000


def ladder(seed):
    rng = np.random.RandomState(seed)
    centres = 0.4 * np.arange(K)
    spring = np.linspace(1.0, 3.0, K)         # f_k spread over about 0.55 kT (see DESIGN.md 3.5g on f_k near 0)
    N_k = np.full(K, NPER, np.float64)
    x = np.repeat(centres, NPER) + rng.normal(size=K * NPER) / np.repeat(np.sqrt(spring), NPER)
    return 0.5 * spring[:, None] * (x[None, :] - centres[:, None]) ** 2, N_k


def single(u, N_k):
    with DeviceProblem(u, N_k) as p:
        f, _ = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=0)
        f = p.self_consistent_update(f)
        f -= f[0]
        _, G = p.weight_moments(f)
    return estimators.free_energy_differences(f, G, N_k)


def main(Ps):
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(card=card)))
    probs = [ladder(s) for s in range(max(Ps))]
    mbar_many([probs[0][0]], [probs[0][1]])          # warm-up: library load, kernel attributes
    single(*probs[0])
    for P in Ps:
        us, ns = [u for u, _ in probs[:P]], [n for _, n in probs[:P]]
        t0 = time.perf_counter()
        res = mbar_many(us, ns)
        t_many = time.perf_counter() - t0
        with DeviceMbarBatch(us, ns) as b:
            t0 = time.perf_counter()
            _, status, iters = b.solve(tol=1e-12)
            t_solve = time.perf_counter() - t0
            st = b.last_stats()
        t0 = time.perf_counter()
        ref = [single(u, n) for u, n in zip(us, ns)]
        t_single = time.perf_counter() - t0
        dmax = max(float(np.max(np.abs(r["Delta_f"] - q["Delta_f"]))) for r, q in zip(res, ref))
        ddmax = max(float(np.max(np.abs(r["dDelta_f"] - q["dDelta_f"]))) for r, q in zip(res, ref))
        print(json.dumps(dict(P=P, K=K, N=K * NPER, mbar_many_s=round(t_many, 3), batch_solve_s=round(t_solve, 3),
                              batch_solve_kernel_ms=round(st["ms"], 2), launches=st["launches"],
                              iterations=st["iterations"], max_problem_iterations=int(iters.max()),
                              paths=sorted(set(r["path"] for r in res)), single_loop_s=round(t_single, 3),
                              speedup=round(t_single / t_many, 2), max_abs_dDelta_f_vs_single=dmax,
                              max_abs_ddDelta_f_vs_single=ddmax)), flush=True)


if __name__ == "__main__":
    main([int(a) for a in sys.argv[1:]] or [100, 1000])

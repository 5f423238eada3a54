#!/usr/bin/env python
"""Time mbar_many(n_bootstraps=B) part by part, and the per-problem bootstrap_f_k loop on the same draws.

    python tools/quick_mbar_many_bootstrap.py [--single-problems M] [P:B ...]     (default: 100:200 1000:50)

Workload: the ladders of tools/quick_mbar_many.py (K = 16, N_k = 5000, N = 80 000 per problem), rseed = 0 .. P - 1.
For each P:B it reports the wall time of mbar_many with uncertainty_method="bootstrap" and of its parts: the main
batched solve (DeviceMbarBatch.solve), the host draws (numpy generators and bincounts), slot uploads
(set_replicates), the waves' solve_replicates calls (wall, CUDA-event kernel time, launches, iterations) and the
all-state updates (weighted moments), with the draws' share of the total.  At the first P it then runs
bootstrap.bootstrap_f_k on one DeviceProblem per problem, over the same draws, for the first M problems (default
all), and reports its time and the largest |f_k_boots| difference between the two paths.  The card name and power
limit come from nvidia-smi in the same run.  Results go to stdout as JSON lines.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pymbar_b200 import DeviceMbarBatch, DeviceProblem, bootstrap  # noqa: E402
from pymbar_b200 import mbar_many as mm  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from quick_mbar_many import K, NPER, ladder  # noqa: E402


class Timer:
    """Wall time and call count of a wrapped method, plus the batch stats of solve_replicates calls."""

    def __init__(self):
        self.t = {}
        self.n = {}
        self.kernel_ms = 0.0
        self.launches = 0
        self.iterations = 0

    def wrap(self, owner, name, key, after=None):
        orig = getattr(owner, name)

        def run(*a, **kw):
            t0 = time.perf_counter()
            out = orig(*a, **kw)
            k = key(a, kw) if callable(key) else key
            self.t[k] = self.t.get(k, 0.0) + time.perf_counter() - t0
            self.n[k] = self.n.get(k, 0) + 1
            if after is not None:
                after(a[0])
            return out

        setattr(owner, name, run)
        return orig

    def stats(self, batch):
        st = batch.last_stats()
        self.kernel_ms += st["ms"]
        self.launches += st["launches"]
        self.iterations += st["iterations"]


def main(argv):
    m_single = None
    if "--single-problems" in argv:
        i = argv.index("--single-problems")
        m_single = int(argv[i + 1])
        argv = argv[:i] + argv[i + 2:]
    runs = [tuple(int(x) for x in a.split(":")) for a in argv] or [(100, 200), (1000, 50)]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(card=card)), flush=True)
    probs = [ladder(s) for s in range(max(P for P, _ in runs))]
    mm.mbar_many([probs[0][0]], [probs[0][1]], n_bootstraps=2, rseed=[0])      # warm-up
    T = Timer()
    T.wrap(DeviceMbarBatch, "solve", "main_solve")
    T.wrap(DeviceMbarBatch, "set_replicates", "slot_upload")
    T.wrap(DeviceMbarBatch, "solve_replicates", "waves", after=T.stats)
    T.wrap(DeviceMbarBatch, "moments", lambda a, kw: "all_state_updates" if kw.get("slots") is not None
           else "main_moments")
    T.wrap(mm._Draws, "next", "host_draws")
    T.wrap(mm._Draws, "__init__", "host_draws")
    for j, (P, B) in enumerate(runs):
        us, ns = [u for u, _ in probs[:P]], [n for _, n in probs[:P]]
        T.t.clear()
        T.n.clear()
        T.kernel_ms = 0.0
        T.launches = T.iterations = 0
        t0 = time.perf_counter()
        res = mm.mbar_many(us, ns, uncertainty_method="bootstrap", n_bootstraps=B, rseed=list(range(P)))
        total = time.perf_counter() - t0
        row = dict(P=P, B=B, K=K, N=K * NPER, total_s=round(total, 3),
                   **{k + "_s": round(v, 3) for k, v in sorted(T.t.items())},
                   host_draws_share=round(T.t.get("host_draws", 0.0) / total, 3), n_waves=T.n.get("waves", 0),
                   waves_kernel_ms=round(T.kernel_ms, 1), waves_launches=T.launches,
                   waves_iterations=T.iterations, boot_single=int(sum(r["boot_single"] for r in res)))
        print(json.dumps(row), flush=True)
        if j == 0:
            M = P if m_single is None else min(P, m_single)
            proto = (dict(method="adaptive", tol=1e-12, options=dict(min_sc_iter=0, gamma=1.0, maxiter=10000)),)
            draws = [bootstrap.bootstrap_indices(ns[p].astype(np.int64), B, p) for p in range(M)]
            t0 = time.perf_counter()
            worst = 0.0
            for p in range(M):
                with DeviceProblem(us[p], ns[p]) as d:
                    fb = bootstrap.bootstrap_f_k(d, res[p]["f_k"], ns[p].astype(np.int64), rints=draws[p],
                                                 solver_protocol=proto)
                worst = max(worst, float(np.max(np.abs(fb - res[p]["f_k_boots"]))))
            t_single = time.perf_counter() - t0
            print(json.dumps(dict(P=P, B=B, single_loop_problems=M, single_loop_s=round(t_single, 3),
                                  single_loop_s_per_problem=round(t_single / M, 4),
                                  batch_waves_plus_updates_s_per_problem=round(
                                      (T.t.get("waves", 0) + T.t.get("all_state_updates", 0)
                                       + T.t.get("slot_upload", 0)) / P, 4),
                                  max_abs_f_k_boots_vs_single=worst)), flush=True)


if __name__ == "__main__":
    main(sys.argv[1:])

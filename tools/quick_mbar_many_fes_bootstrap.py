#!/usr/bin/env python
"""Time MbarMany's bootstrap histogram FES (generate_fes with n_bootstraps = B, then get_fes with "bootstrap")
against the single-problem loop.

    python tools/quick_mbar_many_fes_bootstrap.py [P:N_k:B ...]    (default: 100:500:50 100:5000:50)

Workload: P umbrella problems of K = 32 windows on u0(x) = 2 x^2 with springs of 60 (tests/_fes.umbrella_energies),
N_k samples per window, and a 1-D surface of the unbiased state over x with 100 bins.  For each (P, N_k, B) it
reports the wall time of generate_fes (after a warm-up on one problem), of which the host time spent drawing the
reference's resampling stream (MbarMany.host_stats["fes_draws_s"]: the draws, the coverage check and the counts) is
given separately; the kernel time, launches and bytes read of its device calls (MbarMany.device_stats); the wall
time of get_fes(uncertainty_method="bootstrap"); and the single-problem path (a DeviceProblem upload, then
fes_bootstrap.histogram_replicates from the same generator states, as the FES facade runs it) on the first SINGLE
problems, extrapolated to P and labelled as such, with the largest f_i and df_i differences between the two.  The card
name, power limit and max SM clock come from nvidia-smi in the same run.  Results go to stdout as JSON lines.
"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from quick_mbar_many_fes import card, problem  # noqa: E402

from pymbar_b200 import DeviceProblem  # noqa: E402
from pymbar_b200 import fes as hist  # noqa: E402
from pymbar_b200 import fes_bootstrap as fb  # noqa: E402
from pymbar_b200 import mbar_solvers as ms  # noqa: E402
from pymbar_b200.mbar_many import MbarMany  # noqa: E402

SINGLE, QUERIES = 10, 400
EDGES = np.linspace(-1.5, 1.5, 101)


def single(u_kn, N_k, f, u_n, x, q, seed, B):
    """The single-problem path of one problem: its b = 0 surface, its B replicates and the bootstrap query."""
    protocol = fb.solver_protocol(ms.DEFAULT_SOLVER_PROTOCOL)
    np.random.seed(seed)
    states = fb.draw_replicates(N_k.astype(np.int64), B)
    with DeviceProblem(u_kn, N_k) as p:
        hd = hist.histogram_fes(p, f, u_n, x, EDGES)
        reps = fb.histogram_replicates(p, f, N_k.astype(np.int64), u_n, hd, states, protocol)
    return hist.query(hd, q, "from-lowest", None, lambda j: fb.bootstrap_df(reps, j, len(hd["f"])))


def main(runs):
    print(json.dumps(dict(card=card())), flush=True)
    for P, nper, B in runs:
        probs = [problem(nper, s) for s in range(P)]
        seeds = list(range(1, P + 1))
        with MbarMany([p[0] for p in probs], [p[1] for p in probs], compute_uncertainty=False) as m:
            f = [r["f_k"] for r in m.results]
            qs = [p[3][:QUERIES] for p in probs]
            hp = {"bin_edges": EDGES}
            none = [None] * (P - 1)
            m.generate_fes([probs[0][2]] + none, [probs[0][3]] + none, histogram_parameters=hp, n_bootstraps=B,
                           seed=[0] + none)                                    # warm-up
            m.device_stats.update(ms=0.0, launches=0, calls=0, bytes_read=0)
            m.host_stats.update(fes_draws_s=0.0)
            t0 = time.perf_counter()
            m.generate_fes([p[2] for p in probs], [p[3] for p in probs], histogram_parameters=hp, n_bootstraps=B,
                           seed=seeds)
            t_gen = time.perf_counter() - t0
            gen, draws = dict(m.device_stats), m.host_stats["fes_draws_s"]
            t0 = time.perf_counter()
            out = m.get_fes(qs, uncertainty_method="bootstrap")
            t_get = time.perf_counter() - t0
            n = min(SINGLE, P)
            single(*probs[0][:2], f[0], probs[0][2], probs[0][3], qs[0], seeds[0], 2)      # warm-up
            t0 = time.perf_counter()
            ref = [single(*probs[p][:2], f[p], probs[p][2], probs[p][3], qs[p], seeds[p], B) for p in range(n)]
            t_single = time.perf_counter() - t0
            gap_f = max(float(np.nanmax(np.abs(a["f_i"] - r["f_i"]))) for a, r in zip(out, ref))
            gap_df = max(float(np.nanmax(np.abs(a["df_i"] - r["df_i"]))) for a, r in zip(out, ref))
            print(json.dumps(dict(P=P, K=len(f[0]), N_k=nper, B=B, nbins=len(EDGES) - 1,
                                  boot_single=sum(m.fes_boot_single), generate_fes_s=round(t_gen, 3),
                                  host_draws_s=round(draws, 3), kernel_ms=round(gen["ms"], 3),
                                  launches=gen["launches"], calls=gen["calls"], bytes_read=gen["bytes_read"],
                                  get_fes_bootstrap_s=round(t_get, 4), single_s_first=round(t_single, 3),
                                  single_n=n, single_s_extrapolated_to_P=round(t_single * P / n, 2),
                                  max_gap_f_i=gap_f, max_gap_df_i=gap_df)), flush=True)


if __name__ == "__main__":
    runs = [tuple(int(v) for v in a.split(":")) for a in sys.argv[1:]] or [(100, 500, 50), (100, 5000, 50)]
    main(runs)

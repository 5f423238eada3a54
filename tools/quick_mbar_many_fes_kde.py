#!/usr/bin/env python
"""Time MbarMany's KDE surfaces with bootstrap (generate_fes(fes_type="kde", n_bootstraps=B), then get_fes with
"bootstrap") against the single-problem device loop.

    python tools/quick_mbar_many_fes_kde.py [P:N_k:B ...]    (default: 100:500:50 100:5000:50)

Workload: P umbrella problems of K = 32 windows (tools/quick_mbar_many_fes.problem), N_k samples per window, a
gaussian KDE of the unbiased state with h = 0.1, and two surfaces: 1-D over x with 100 queries, and 2-D over (x, a
normal second coordinate) on a 50 x 50 grid.  For each (P, N_k, B, surface) it reports the wall time of generate_fes
(after a warm-up on one problem), of which the host time spent drawing the reference's resampling stream and the
bincounts of the replicate weights (MbarMany.host_stats["fes_draws_s"]) is given separately, and the bytes of
coordinates uploaded; the wall time of get_fes(uncertainty_method="bootstrap") with the kernel time, launches, calls
and (query, sample) pairs of its DeviceKdeMany calls (MbarMany.kde_stats); and the single-problem device loop
(DeviceProblem log weights, a DeviceKde upload, set_replicates and log_sum_replicates, as the FES facade runs it) on
the first SINGLE problems, extrapolated to P and labelled as such, with the largest f_i and df_i differences between
the two.  The card name, power limit and max SM clock come from nvidia-smi in the same run.  Results go to stdout as
JSON lines.
"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from quick_mbar_many_fes import card, problem  # noqa: E402

from pymbar_b200 import DeviceKde, DeviceProblem  # noqa: E402
from pymbar_b200 import fes as hist  # noqa: E402
from pymbar_b200 import fes_bootstrap as fb  # noqa: E402
from pymbar_b200.mbar_many import MbarMany  # noqa: E402

SINGLE = 10
H = 0.1
PARAMS = {"bandwidth": H, "kernel": "gaussian"}
Q1 = np.linspace(-1.5, 1.5, 100).reshape(-1, 1)
_g = np.linspace(-1.5, 1.5, 50)
Q2 = np.array([[a, b] for a in _g for b in _g])


def single(u_kn, N_k, f, u_n, x, q, seed, B):
    """The single-problem device path of one problem: its weights, its B replicates' weights and the bootstrap query."""
    with DeviceProblem(u_kn, N_k) as p:
        lw = -u_n - p.log_denominator(f)
    w = np.exp(lw - np.max(lw))
    w = w / np.sum(w)
    V = np.empty((B, len(w)))

    def each(b, idx):
        V[b] = np.bincount(idx, weights=w, minlength=len(w))

    np.random.seed(seed)
    fb.draw_replicates(N_k.astype(np.int64), B, each)
    settings = {"kernel": "gaussian", "h": H, "D": q.shape[1]}
    with DeviceKde(x, w) as k:
        k.set_replicates(V)
        return fb.kde_bootstrap_query(k, settings, q, "from-lowest", None, float(np.log(np.sum(w))))


def main(runs):
    print(json.dumps(dict(card=card())), flush=True)
    for P, nper, B in runs:
        probs = [problem(nper, s) for s in range(P)]
        seeds = list(range(1, P + 1))
        with MbarMany([p[0] for p in probs], [p[1] for p in probs], compute_uncertainty=False) as m:
            f = [r["f_k"] for r in m.results]
            for surface, col, q in (("1d", 3, Q1), ("2d", 4, Q2)):
                none = [None] * (P - 1)
                m.generate_fes([probs[0][2]] + none, [probs[0][col]] + none, fes_type="kde", kde_parameters=PARAMS,
                               n_bootstraps=B, seed=[0] + none)                  # warm-up
                m.get_fes([q] + none, uncertainty_method="bootstrap")
                m.host_stats.update(fes_draws_s=0.0)
                m.kde_stats.update(ms=0.0, launches=0, calls=0, pairs=0, upload_bytes=0)
                t0 = time.perf_counter()
                m.generate_fes([p[2] for p in probs], [p[col] for p in probs], fes_type="kde", kde_parameters=PARAMS,
                               n_bootstraps=B, seed=seeds)
                t_gen = time.perf_counter() - t0
                draws, upload = m.host_stats["fes_draws_s"], m.kde_stats["upload_bytes"]
                t0 = time.perf_counter()
                out = m.get_fes([q] * P, uncertainty_method="bootstrap")
                t_get = time.perf_counter() - t0
                st = dict(m.kde_stats)
                n = min(SINGLE, P)
                single(*probs[0][:2], f[0], probs[0][2], probs[0][col], q, seeds[0], 2)      # warm-up
                t0 = time.perf_counter()
                ref = [single(*probs[p][:2], f[p], probs[p][2], probs[p][col], q, seeds[p], B) for p in range(n)]
                t_single = time.perf_counter() - t0
                gap_f = max(float(np.nanmax(np.abs(a["f_i"] - r["f_i"]))) for a, r in zip(out, ref))
                gap_df = max(float(np.nanmax(np.abs(a["df_i"] - r["df_i"]))) for a, r in zip(out, ref))
                print(json.dumps(dict(P=P, K=len(f[0]), N_k=nper, B=B, surface=surface, queries=len(q),
                                      generate_fes_s=round(t_gen, 3), host_draws_bincount_s=round(draws, 3),
                                      upload_bytes=upload, get_fes_bootstrap_s=round(t_get, 3),
                                      kernel_ms=round(st["ms"], 3), launches=st["launches"], calls=st["calls"],
                                      pairs=st["pairs"], single_s_first=round(t_single, 3), single_n=n,
                                      single_s_extrapolated_to_P=round(t_single * P / n, 2),
                                      max_gap_f_i=gap_f, max_gap_df_i=gap_df)), flush=True)


if __name__ == "__main__":
    runs = [tuple(int(v) for v in a.split(":")) for a in sys.argv[1:]] or [(100, 500, 50), (100, 5000, 50)]
    main(runs)

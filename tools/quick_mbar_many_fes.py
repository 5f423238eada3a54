#!/usr/bin/env python
"""Time MbarMany's histogram FES (generate_fes, then an analytical get_fes) against the single-problem loop.

    python tools/quick_mbar_many_fes.py [P:N_k[:1d|2d] ...]    (default: 100:5000 1000:500, both surfaces)

Workload: P umbrella problems of K = 32 windows on u0(x) = 2 x^2 with springs of 60 (tests/_fes.umbrella_energies),
N_k samples per window, and an unbiased second coordinate y ~ N(0, 1).  Each problem gets two surfaces of the unbiased
state: 1-D over x with 100 bins and 2-D over (x, y) with 50 x 50 = 2500 bins.  For each (P, N_k, surface) it reports
the wall time of generate_fes and of get_fes(uncertainty_method="analytical") at the problem's first QUERIES samples
(a bin without samples has no entry to query, in the reference as here), each ending in a
synchronisation, after a warm-up on one problem; the kernel time, launches and bytes read of their device calls
(DeviceMbarBatch.last_stats summed in MbarMany.device_stats); and the single-problem path (a DeviceProblem upload, then
fes.histogram_fes, fes.histogram_theta and fes.query, as the FES facade runs them) on the first SINGLE problems,
extrapolated to P and labelled as such, with the largest f_i and df_i differences between the two.  The card name,
power limit and max SM clock come from nvidia-smi in the same run.  Results go to stdout as JSON lines.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pymbar_b200 import DeviceProblem  # noqa: E402
from pymbar_b200 import fes as hist  # noqa: E402
from pymbar_b200.mbar_many import MbarMany  # noqa: E402
from tests._fes import umbrella_energies  # noqa: E402

K, K0, KU, SINGLE, QUERIES = 32, 4.0, 60.0, 10, 400
EDGES_1D = np.linspace(-1.5, 1.5, 101)
EDGES_2D = [np.linspace(-1.5, 1.5, 51), np.linspace(-2.5, 2.5, 51)]


def problem(nper, seed):
    rng = np.random.RandomState(seed)
    centres = np.linspace(-1.5, 1.5, K)
    x = np.concatenate([rng.normal(KU * c / (K0 + KU), 1.0 / np.sqrt(K0 + KU), size=nper) for c in centres])
    u_kn, u_n = umbrella_energies(x, centres, K0, KU)
    return u_kn, np.full(K, nper, np.float64), u_n, x, np.stack([x, rng.normal(size=x.size)], axis=1)


def single(u_kn, N_k, f, u_n, x, edges, q):
    with DeviceProblem(u_kn, N_k) as p:
        hd = hist.histogram_fes(p, f, u_n, x, edges)
        Theta = hist.histogram_theta(p, f, N_k, u_n, hd)
    return hist.query(hd, q, "from-lowest", None, lambda j: hist.bin_uncertainties(Theta, K, j, len(hd["f"])))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main(runs):
    print(json.dumps(dict(card=card())), flush=True)
    for P, nper, which in runs:
        probs = [problem(nper, s) for s in range(P)]
        t0 = time.perf_counter()
        m = MbarMany([p[0] for p in probs], [p[1] for p in probs], compute_uncertainty=False)
        t_construct = time.perf_counter() - t0
        with m:
            f = [r["f_k"] for r in m.results]
            for surface, edges, col in (("1d_100", EDGES_1D, 3), ("2d_2500", EDGES_2D, 4)):
                if which and not surface.startswith(which):
                    continue
                qs = [p[col][:QUERIES] for p in probs]
                hp = {"bin_edges": edges}
                m.generate_fes([probs[0][2]] + [None] * (P - 1), [probs[0][col]] + [None] * (P - 1),
                               histogram_parameters=hp)                           # warm-up
                m.get_fes([qs[0]] + [None] * (P - 1), uncertainty_method="analytical")
                m.device_stats.update(ms=0.0, launches=0, calls=0, bytes_read=0)
                t0 = time.perf_counter()
                m.generate_fes([p[2] for p in probs], [p[col] for p in probs], histogram_parameters=hp)
                t_gen = time.perf_counter() - t0
                gen = dict(m.device_stats)
                m.device_stats.update(ms=0.0, launches=0, calls=0, bytes_read=0)
                t0 = time.perf_counter()
                out = m.get_fes(qs, uncertainty_method="analytical")
                t_get = time.perf_counter() - t0
                get = dict(m.device_stats)
                n = min(SINGLE, P)
                single(*probs[0][:2], f[0], probs[0][2], probs[0][col], edges, qs[0])  # warm-up
                t0 = time.perf_counter()
                ref = [single(*probs[p][:2], f[p], probs[p][2], probs[p][col], edges, qs[p]) for p in range(n)]
                t_single = time.perf_counter() - t0
                gap_f = max(float(np.nanmax(np.abs(a["f_i"] - r["f_i"]))) for a, r in zip(out, ref))
                gap_df = max(float(np.nanmax(np.abs(a["df_i"] - r["df_i"]))) for a, r in zip(out, ref))
                print(json.dumps(dict(P=P, K=K, N_k=nper, N=K * nper, surface=surface,
                                      construct_s=round(t_construct, 3),
                                      paths=sorted(set(o["path"] for o in out)),
                                      generate_fes_s=round(t_gen, 4), generate_kernel_ms=round(gen["ms"], 3),
                                      generate_launches=gen["launches"], generate_calls=gen["calls"],
                                      generate_bytes_read=gen["bytes_read"],
                                      get_fes_analytical_s=round(t_get, 4), get_kernel_ms=round(get["ms"], 3),
                                      get_launches=get["launches"], get_calls=get["calls"],
                                      get_bytes_read=get["bytes_read"],
                                      single_s_first=round(t_single, 4), single_n=n,
                                      single_s_extrapolated_to_P=round(t_single * P / n, 3),
                                      max_gap_f_i=gap_f, max_gap_df_i=gap_df)), flush=True)


if __name__ == "__main__":
    runs = [(int(a.split(":")[0]), int(a.split(":")[1]), (a.split(":") + [""])[2]) for a in sys.argv[1:]] or \
        [(100, 5000, ""), (1000, 500, "")]
    main(runs)

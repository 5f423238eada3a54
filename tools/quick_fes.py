"""Cost of the histogram-FES kernels (mbar_b200_bin_moments) at C3 (K = 256, N = 1e7, synthesized on the device),
next to a plain fused pass in the same process.  Prints the card name and power limit read in the same run.

    python tools/quick_fes.py [--nbins 100 1000 2500] [--reps 3]

Bytes per call are counted as 8 K N chunks + 20 N (u_kn once per bin chunk; u_n, L'_n and the bin index); the
bin-sum step that precedes the moments reads only the O(N) vectors and is included in the time.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from pymbar_b200 import DeviceProblem  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception as err:  # noqa: BLE001
        return f"unknown ({err})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nbins", type=int, nargs="+", default=[100, 1000, 2500])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--K", type=int, default=256)
    ap.add_argument("--N", type=int, default=10 ** 7)
    a = ap.parse_args()
    K, N = a.K, a.N
    name, power = card()
    N_k = np.full(K, N // K, float)
    N_k[-1] += N - N_k.sum()
    rows = []
    with DeviceProblem(None, N_k, N_local=N) as p:
        p.synthesize(np.linspace(1, 5, K), np.linspace(1, 3, K), seed=0)
        f, _ = p.solve_adaptive(np.zeros(K), tol=1e-12)
        pass_ms = []
        for _ in range(a.reps + 1):
            p.streaming_pass(f)
            pass_ms.append(p.last_pass_ms())
        pass_ms = float(np.median(pass_ms[1:]))
        rng = np.random.RandomState(0)
        u_n = rng.uniform(0.0, 5.0, size=N)
        for nbins in a.nbins:
            # contiguous runs of samples share a bin, as consecutive frames of a trajectory do
            bins = ((np.arange(N) // 64) * 7919 % nbins).astype(np.int32)
            ms = []
            for _ in range(a.reps + 1):
                p.bin_moments(f, u_n, bins, nbins)
                st = p.last_bin_stats()
                ms.append(st["ms"])
            t = float(np.median(ms[1:]))
            nbytes = 8.0 * K * N * st["chunks"] + 20.0 * N
            rows.append(dict(nbins=nbins, chunks=st["chunks"], bin_ms=round(t, 3), pass_ms=round(pass_ms, 3),
                             ratio=round(t / pass_ms, 2), GBps=round(nbytes / t / 1e6, 1)))
            print(json.dumps(rows[-1]), flush=True)
    print(json.dumps(dict(card=name, power_limit=power, K=K, N=N, results=rows)))


if __name__ == "__main__":
    main()

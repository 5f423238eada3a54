#!/usr/bin/env python
"""Kernel-density log sums at the C3 sample count (N = 1e7): kernel time, pairs/s and upload time for D = 1, 2,
Q = 1, 100, 1e4 and the gaussian, epanechnikov and exponential kernels; fp64 instructions per pair counted in the
SASS of the inner loop; the share of the in-process DFMA ceiling (mbar_b200_measure_fp64_peak); the card and its
power limit, read in the same run.  Not run by bench.py.

    python tools/quick_kde.py [--n 10000000] [--out quick_kde.json]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pymbar_b200 import DeviceKde, _lib  # noqa: E402
from pymbar_b200.problem import KDE_KERNELS, measure_fp64_peak  # noqa: E402

FP64 = re.compile(r"\b(DADD|DMUL|DFMA|DSETP|DMNMX)\b")
UNROLL = 4          # kde_partial_kernel's inner loop: #pragma unroll 4


def sass_per_pair(D, kernel):
    """fp64-pipe instructions per pair on the common path of kde_partial_kernel<D, kernel>: those of its innermost
    loop over the unroll factor, without the rescale of the running maximum (the code a branch on d > KDE_RESCALE
    skips, rarely taken)."""
    name = f"_ZN4mbar18kde_partial_kernelILi{D}ELi{KDE_KERNELS.index(kernel)}EEEvNS_9KdeParamsE"
    out = subprocess.run(["cuobjdump", "-sass", "-fun", name, _lib.LIB_PATH], capture_output=True, text=True).stdout
    ins = []
    for line in out.splitlines():
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if m:
            ins.append((int(m.group(1), 16), m.group(2)))
    best = None
    for addr, text in ins:
        b = re.search(r"BRA\s+(?:`\(\.L_x_\d+\)\s*)?0x([0-9a-f]+)", text) or re.search(r"BRA .*?0x([0-9a-f]+)", text)
        if not b:
            continue
        tgt = int(b.group(1), 16)
        if tgt >= addr:
            continue
        body = [(a, t) for a, t in ins if tgt <= a <= addr]
        skipped, rescale = set(), set()
        for a2, t2 in body:
            c = re.match(r"DSETP\.GT\.AND (P\d), PT, R\d+, 128,", t2)      # d > KDE_RESCALE
            if c:
                rescale.add(c.group(1))
            f = re.match(r"@!(P\d)\s+BRA\s.*?0x([0-9a-f]+)", t2)
            if f and f.group(1) in rescale and a2 < int(f.group(2), 16) <= addr:
                skipped.update(a3 for a3, _ in body if a2 < a3 < int(f.group(2), 16))
                rescale.discard(f.group(1))
        n = sum(1 for a2, t in body if a2 not in skipped and FP64.search(t))
        if best is None or (n > 0 and len(body) < best[1] and n >= best[0] // 2) or n > 2 * best[0]:
            best = (n, len(body))
    return None if best is None else best[0] / UNROLL


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    _, dfma = measure_fp64_peak(0)
    dfma_rate = dfma * 1e12 / 2.0                  # DFMA instructions per second (2 flops each)
    rows = []
    rng = np.random.RandomState(0)
    for D in (1, 2):
        x = rng.normal(size=(a.n, D))
        w = rng.uniform(size=a.n)
        t0 = time.perf_counter()
        kde = DeviceKde(x, w)
        upload_ms = 1e3 * (time.perf_counter() - t0)
        for Q in (1, 100, 10_000):
            if D == 2 and Q == 10_000:
                g = np.linspace(-3, 3, 100)
                y = np.array([[p, q] for p in g for q in g])          # a 100 x 100 grid
            else:
                y = rng.normal(size=(Q, D))
            for kernel in ("gaussian", "epanechnikov", "exponential"):
                kde.log_sum(kernel, 0.05, y)                          # warm-up
                ms = []
                for _ in range(a.reps):
                    kde.log_sum(kernel, 0.05, y)
                    ms.append(kde.last_stats()["ms"])
                ms = float(np.median(ms))
                pairs = float(a.n) * Q / (ms * 1e-3)
                ipp = sass_per_pair(D, kernel)
                share = None if ipp is None else pairs * ipp / dfma_rate
                row = dict(D=D, Q=Q, kernel=kernel, kernel_ms=ms, pairs_per_s=pairs, upload_ms=upload_ms,
                           fp64_per_pair=ipp, dfma_share=share, chunks=kde.last_stats()["chunks"])
                rows.append(row)
                print(json.dumps(row), flush=True)
        kde.close()
    res = dict(card=card(), dfma_tflops=dfma, N=a.n, rows=rows)
    print(json.dumps({k: v for k, v in res.items() if k != "rows"}))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

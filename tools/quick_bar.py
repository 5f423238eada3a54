#!/usr/bin/env python
"""BAR / EXP sums of pymbar.other_estimators on the GPU: per bar_zero evaluation at 1e3, 1e5 and 1e7 values per side
the kernel time (CUDA events of one mbar_b200_work call), the bytes it read and their share of the HBM roofline
(3.35 TB/s, H100 SXM), the device calls per `bar`, the wall time of one `bar`; and the wall time of `bar_many` on 100
pairs of 1e5 values per side.  The card and its power limit come first.  Not run by bench.py.

    python tools/quick_bar.py [--out quick_bar.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pymbar_b200 import DeviceWork  # noqa: E402
from pymbar_b200 import other_estimators as oe  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def pair(n, seed):
    rng = np.random.RandomState(seed)
    return rng.normal(2.0, 1.0, n), rng.normal(-0.5, 1.0, n)


def one_size(n):
    w_F, w_R = pair(n, n % 97)
    M = np.log(1.0)
    with DeviceWork([w_F, w_R]) as dev:
        reqs = list(zip(*oe._zero_requests(M, 1.2)))
        dev.evaluate(*reqs)                                  # warm-up
        ms = []
        for _ in range(5):
            dev.evaluate(*reqs)
            ms.append(dev.last_stats()["ms"])
        st = dev.last_stats()
    oe.bar(w_F, w_R)                                         # warm-up of the driver
    n0 = oe.EVALUATIONS[0]
    t0 = time.perf_counter()
    oe.bar(w_F, w_R)
    wall = time.perf_counter() - t0
    k = float(np.median(ms))
    r = dict(n_per_side=n, kernel_ms=k, launches=st["launches"], bytes_read=st["bytes_read"],
             hbm_share=st["bytes_read"] / (k * 1e-3) / HBM_BYTES_PER_S, device_calls_per_bar=oe.EVALUATIONS[0] - n0,
             bar_wall_s=wall)
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card(), sizes=[one_size(n) for n in (1_000, 100_000, 10_000_000)])
    wF, wR = zip(*[pair(100_000, s) for s in range(100)])
    oe.bar_many(wF[:2], wR[:2])
    n0 = oe.EVALUATIONS[0]
    t0 = time.perf_counter()
    oe.bar_many(list(wF), list(wR))
    res["bar_many_100x1e5_wall_s"] = time.perf_counter() - t0
    res["bar_many_100x1e5_device_calls"] = oe.EVALUATIONS[0] - n0
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

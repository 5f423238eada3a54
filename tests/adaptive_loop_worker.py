"""Worker for tests/test_gpu_adaptive_loop.py: runs the device-resident adaptive solves of `solves()` in a process whose
environment switches off the CUDA graph (MBAR_B200_NO_GRAPH) or the candidate-batched pass (MBAR_B200_NO_M2), which
the library reads once per process, and writes each solve's f and counters to the npz named on the command line."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def solves(DeviceProblem):
    """{name: (f, result)} of the same solves in every process: three shapes, batch 4, two solves per context (the
    second runs every batch from the captured graph when graphs are on)."""
    from tests import _moments as M

    out = {}
    for K, unsampled in ((9, (0,)), (100, (50,)), (300, (0, 299))):
        case = M.ladder(K, 20, gaps=(1.5,), unsampled=unsampled, seed=K, f_noise=0.5)
        with DeviceProblem(case["u"], case["N"]) as p:
            p.set_loop_mode("device", 4)
            for rep in range(2):
                f, r = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=1, gamma=0.5 if rep else 1.0)
                out[f"K{K}|{rep}"] = (f, r)
    return out


def main(path):
    from pymbar_b200 import DeviceProblem

    arrays, meta = {}, {}
    for name, (f, r) in solves(DeviceProblem).items():
        arrays[name] = f
        meta[name] = {k: (float(v) if isinstance(v, float) else int(v)) for k, v in r.items()}
    arrays["meta"] = np.array(json.dumps(meta))
    np.savez(path, **arrays)
    print("ADAPTIVE_WORKER_OK")


if __name__ == "__main__":
    main(sys.argv[1])

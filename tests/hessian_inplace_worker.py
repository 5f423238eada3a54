"""Worker for tests/test_gpu_hessian_paths.py: runs with MBAR_B200_HESSIAN_INPLACE=1, which the library reads once
per process, so every Hessian of this process (K <= 64 included) goes to hessian_inplace_kernel.  Runs the four
paths on every ladder case and the device-resident and stepped solvers on two well-overlapping ladders, and writes
the raw results to the npz named on the command line; the parent process checks them."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SOLVE_K = (17, 65)


def main(out):
    assert os.environ.get("MBAR_B200_HESSIAN_INPLACE") == "1"
    from pymbar_b200 import DeviceProblem
    from tests import _moments as M

    arrays, names = {}, {}
    for name in M.cases():
        case = M.build(name)
        for path in M.PATHS:
            with DeviceProblem(case["u"], case["N"]) as p:
                d = M.device_moments(p, case, path)
            for key, v in d.items():
                if isinstance(v, str):
                    names[f"{name}|{path}|{key}"] = v
                else:
                    arrays[f"{name}|{path}|{key}"] = v
    for K in SOLVE_K:
        case = M.solve_ladder(K, seed=K)
        with DeviceProblem(case["u"], case["N"]) as p:
            for batch in (2, 16):
                p.set_loop_mode("device", batch)
                for rep in range(2):       # the second solve of a context runs from a captured graph
                    f, r = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=0)
                    arrays[f"solve{K}|b{batch}|{rep}"] = f
                    names[f"solve{K}|b{batch}|{rep}|ok"] = bool(r["success"])
            names[f"solve{K}|graph_launches"] = p.loop_stats()["graph_launches"]
            names[f"solve{K}|hname"] = p.last_kernels()["hessian_kernel"]
            p.set_loop_mode("stepped")
            f, r = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=0)
            arrays[f"solve{K}|stepped"] = f
            names[f"solve{K}|stepped|ok"] = bool(r["success"])
    arrays["names"] = np.array(json.dumps(names))
    np.savez(out, **arrays)
    print("INPLACE_OK")


if __name__ == "__main__":
    main(sys.argv[1])

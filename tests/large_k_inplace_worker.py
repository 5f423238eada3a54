"""Worker for tests/test_gpu_large_k.py: runs with MBAR_B200_HESSIAN_INPLACE=1, which the library reads once per
process, so every Hessian of this process goes to hessian_inplace_kernel.  Runs the moments and Hessian calls of the
K = 4100 case and writes the raw results to the npz named on the command line; the parent process checks them."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main(out):
    assert os.environ.get("MBAR_B200_HESSIAN_INPLACE") == "1"
    from pymbar_b200 import DeviceProblem
    from tests import test_gpu_large_k as T

    c = T.moments_case(4100)
    with DeviceProblem(c["u"], c["N"]) as p:
        d = T.device_moments(p, c)
    np.savez(out, **{k: np.asarray(v) for k, v in d.items()})
    print("INPLACE_OK")


if __name__ == "__main__":
    main(sys.argv[1])

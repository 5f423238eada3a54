#!/usr/bin/env python
"""Generate tests/golden/mbar_many_bootstrap.npz by running the UNMODIFIED reference
pymbar.MBAR(u_kn, N_k, n_bootstraps=20, rseed=1000 + i, initial_f_k=golden_f_init) on each problem i of
tests/_mbar_many.golden_problems().

    python tools/make_mbar_many_bootstrap_golden.py /path/to/pymbar-checkout

Imports pymbar from the given checkout through the numexpr stub in oracle/ref_shim, as oracle/make_golden.py does.
The inputs are rebuilt from their seeds, not stored.  For problem i the file holds the reference's p<i>_f_k_boots
[20, K] and p<i>_dDelta_f (compute_free_energy_differences(uncertainty_method="bootstrap")); "names" lists the
problems in order, "n_bootstraps" and "seed0" the draw parameters.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "mbar_many_bootstrap.npz")
B = 20
SEED0 = 1000


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    import pymbar

    from tests import _mbar_many

    data = {}
    names = []
    for i, (name, (u, N_k)) in enumerate(_mbar_many.golden_problems()):
        m = pymbar.MBAR(u, N_k, n_bootstraps=B, rseed=SEED0 + i, initial_f_k=_mbar_many.golden_f_init(name, len(N_k)))
        r = m.compute_free_energy_differences(uncertainty_method="bootstrap")
        p = f"p{i}_"
        data[p + "f_k_boots"] = np.array(m.f_k_boots)
        data[p + "dDelta_f"] = r["dDelta_f"]
        names.append(name)
        print(f"{name}: K={len(N_k)} N={u.shape[1]} max dDelta_f {np.max(r['dDelta_f']):.3g}")
    data["names"] = np.array(names)
    data["n_bootstraps"] = np.array(B)
    data["seed0"] = np.array(SEED0)
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

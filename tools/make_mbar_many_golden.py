#!/usr/bin/env python
"""Generate tests/golden/mbar_many.npz by running the UNMODIFIED reference pymbar.MBAR(u_kn, N_k) with its default
protocol on each problem of tests/_mbar_many.golden_problems(), from golden_f_init.

    python tools/make_mbar_many_golden.py /path/to/pymbar-checkout

Imports pymbar from the given checkout through the numexpr stub in oracle/ref_shim, as oracle/make_golden.py does.
The inputs are rebuilt from their seeds, not stored.  For problem i the file holds the reference's p<i>_f_k, p<i>_Delta_f, p<i>_dDelta_f and
p<i>_Theta (compute_free_energy_differences(return_theta=True)); "names" lists the problems in order.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "mbar_many.npz")


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
        m = pymbar.MBAR(u, N_k, initial_f_k=_mbar_many.golden_f_init(name, len(N_k)))
        r = m.compute_free_energy_differences(return_theta=True)
        p = f"p{i}_"
        data[p + "f_k"] = np.array(m.f_k)
        data[p + "Delta_f"] = r["Delta_f"]
        data[p + "dDelta_f"] = r["dDelta_f"]
        data[p + "Theta"] = r["Theta"]
        names.append(name)
        print(f"{name}: K={len(N_k)} N={u.shape[1]} f span {np.ptp(m.f_k):.1f}")
    data["names"] = np.array(names)
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

#!/usr/bin/env python
"""Generate tests/golden/mbar_many_expectations.npz by running the UNMODIFIED reference pymbar.MBAR(u_kn, N_k) with
its default protocol on each problem of tests/_mbar_many_expectations.expectation_problems().

    python tools/make_mbar_many_expectations_golden.py /path/to/pymbar-checkout

Imports pymbar from the given checkout through the numexpr stub in oracle/ref_shim, as oracle/make_golden.py does.
The inputs are rebuilt from their seeds, not stored.  For problem i, with (A, A_k, u_ln) = requests(u_kn), the file
holds p<i>_avg_* (compute_expectations(A): mu, sigma), p<i>_diff_* (compute_expectations(A_k, output="differences",
state_dependent=True)), p<i>_pert_* (compute_perturbed_free_energies(u_ln)), p<i>_ent_* (compute_entropy_and_enthalpy()),
p<i>_ovl_* (compute_overlap(), for K > 1) and p<i>_neff_N_eff (compute_effective_sample_number()); "names" lists the problems.
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "mbar_many_expectations.npz")


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    import pymbar

    from tests import _mbar_many_expectations as E

    data = {}
    names = []
    for i, (name, (u, N_k)) in enumerate(E.expectation_problems()):
        A, A_k, u_ln = E.requests(u)
        m = pymbar.MBAR(u, N_k)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            res = dict(avg=m.compute_expectations(A),
                       diff=m.compute_expectations(A_k, output="differences", state_dependent=True),
                       pert=m.compute_perturbed_free_energies(u_ln),
                       ent=m.compute_entropy_and_enthalpy(),
                       ovl=m.compute_overlap() if len(N_k) > 1 else {},   # one state: no second eigenvalue
                       neff=dict(N_eff=m.compute_effective_sample_number()))
        for what, keys in E.KEYS.items():
            for k in keys:
                if k not in res[what]:
                    continue
                data[f"p{i}_{what}_{k}"] = np.asarray(res[what][k])
        names.append(name)
        print(f"{name}: K={len(N_k)} N={u.shape[1]}")
    data["names"] = np.array(names)
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

#!/usr/bin/env python
"""Generate tests/golden/mbar_many_boot_expectations.npz by running the UNMODIFIED reference
pymbar.MBAR(u_kn, N_k, n_bootstraps=16, rseed=2000 + i) on each problem i of
tests/_mbar_many_boot_expectations.boot_problems() and asking its estimators for bootstrap uncertainties.

    python tools/make_mbar_many_boot_expectations_golden.py /path/to/pymbar-checkout

Imports pymbar from the given checkout through the numexpr stub in oracle/ref_shim, as oracle/make_golden.py does.
The inputs are rebuilt from their seeds, not stored.  For problem i, with (A, A_k, u_ln) = requests(u_kn) of
tests/_mbar_many_expectations.py and uncertainty_method="bootstrap" throughout, the file holds p<i>_avg_sigma
(compute_expectations(A)), p<i>_diff_sigma (compute_expectations(A_k, output="differences", state_dependent=True)),
p<i>_pert_dDelta_f (compute_perturbed_free_energies(u_ln)), p<i>_ent_dDelta_{f,u,s} (compute_entropy_and_enthalpy()),
p<i>_inner_bootstrapped_{observables,f} (compute_expectations_inner of the averages request) and p<i>_f_k_boots;
"names" lists the problems, "n_bootstraps" and "seed0" the draw parameters.  The keys that do not depend on the
replicates (mu, Delta_f, ...) are those of tests/golden/mbar_many_expectations.npz.
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "mbar_many_boot_expectations.npz")
B = 16
SEED0 = 2000


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    import pymbar

    from tests import _mbar_many_boot_expectations as BE
    from tests import _mbar_many_expectations as E

    data = {}
    names = []
    for i, (name, (u, N_k)) in enumerate(BE.boot_problems()):
        A, A_k, u_ln = E.requests(u)
        K = len(N_k)
        m = pymbar.MBAR(u, N_k, n_bootstraps=B, rseed=SEED0 + i)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            avg = m.compute_expectations(A.copy(), uncertainty_method="bootstrap")
            diff = m.compute_expectations(A_k.copy(), output="differences", state_dependent=True,
                                          uncertainty_method="bootstrap")
            pert = m.compute_perturbed_free_energies(u_ln, uncertainty_method="bootstrap")
            ent = m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap")
            state_map = np.array([np.arange(K), np.zeros(K, int)])
            inner = m.compute_expectations_inner(A.copy().reshape(1, -1), m.u_kn, state_map,
                                                 uncertainty_method="bootstrap")
        p = f"p{i}_"
        data[p + "avg_sigma"] = np.asarray(avg["sigma"])
        data[p + "diff_sigma"] = np.asarray(diff["sigma"])
        data[p + "pert_dDelta_f"] = np.asarray(pert["dDelta_f"])
        for k in ("dDelta_f", "dDelta_u", "dDelta_s"):
            data[p + "ent_" + k] = np.asarray(ent[k])
        data[p + "inner_bootstrapped_observables"] = np.asarray(inner["bootstrapped_observables"])
        data[p + "inner_bootstrapped_f"] = np.asarray(inner["bootstrapped_f"])
        data[p + "f_k_boots"] = np.array(m.f_k_boots)
        names.append(name)
        print(f"{name}: K={K} N={u.shape[1]} max avg sigma {np.max(avg['sigma']):.3g}")
    data["names"] = np.array(names)
    data["n_bootstraps"] = np.array(B)
    data["seed0"] = np.array(SEED0)
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

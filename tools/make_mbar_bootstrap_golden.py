#!/usr/bin/env python
"""Generate tests/golden/mbar_bootstrap.npz by running the UNMODIFIED reference pymbar.MBAR with n_bootstraps > 0.

    python tools/make_mbar_bootstrap_golden.py /path/to/pymbar-checkout

The inputs are the fixtures of tests/_cases (SMALL, with its empty-state cases, and REF_SUITE), loaded through
_cases.load, so no new sample data is stored.  For each case and seed (n_bootstraps = NB, rseed = seed) the file
holds, with keys prefixed "<case>_s<seed>_":
  * f_k_boots [NB, K], bootstrap_rints [NB, N] and after: one mbar.rng.random() drawn after construction;
  * fed_dDelta_f: compute_free_energy_differences(uncertainty_method="bootstrap"); fed_theta_dDelta_f and fed_Theta
    with return_theta=True;
  * avg_mu / avg_sigma, diff_mu / diff_sigma, sd_mu / sd_sigma: compute_expectations(bootstrap) of x_n (averages,
    differences) and of u_kn with state_dependent=True;
  * mult_mu / mult_sigma / mult_cov: compute_multiple_expectations(bootstrap) of [x_n, x_n^2] at state 0's energies,
    with compute_covariance=True;
  * pert_Delta_f / pert_dDelta_f: compute_perturbed_free_energies(bootstrap) of the fixture's pert_u_ln;
  * ee_<key>: compute_entropy_and_enthalpy(bootstrap), every key;
  * inner_obs / inner_f: "bootstrapped_observables" and "bootstrapped_f" of compute_expectations_inner(bootstrap)
    with x_n at every state.
For each case and the first seed, "<case>_bar_f_k_boots" is f_k_boots of an initialize="BAR" run, and
"<case>_perm" with "<case>_il_*" (f_k_boots, bootstrap_rints, after) a run with the samples interleaved (u_kn[:, perm],
x_kindices = the state of each permuted sample).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden")
NB = 20
SEEDS = (11, 2024)
EE_KEYS = ("Delta_f", "dDelta_f", "Delta_u", "dDelta_u", "Delta_s", "dDelta_s")


def interleaving(N_k):
    """Sample order that takes one sample of each state in turn (states with samples left), as a permutation."""
    blocks = np.split(np.arange(int(np.sum(N_k))), np.cumsum(N_k)[:-1])
    out, i = [], 0
    while any(i < len(b) for b in blocks):
        out.extend(int(b[i]) for b in blocks if i < len(b))
        i += 1
    return np.array(out, dtype=np.int64)


def run(name, seed, data, first):
    import pymbar

    from tests import _cases

    z = _cases.load(name)
    u, N_k, x = z["u_kn"], z["N_k"], z["x_n"]
    K = len(N_k)
    p = f"{name}_s{seed}_"
    m = pymbar.MBAR(u, N_k, n_bootstraps=NB, rseed=seed)
    data[p + "after"] = np.float64(m.rng.random())
    data[p + "f_k_boots"] = np.array(m.f_k_boots)
    data[p + "bootstrap_rints"] = np.array(m.bootstrap_rints, dtype=np.int64)
    data[p + "fed_dDelta_f"] = m.compute_free_energy_differences(uncertainty_method="bootstrap")["dDelta_f"]
    r = m.compute_free_energy_differences(uncertainty_method="bootstrap", return_theta=True)
    data[p + "fed_theta_dDelta_f"], data[p + "fed_Theta"] = r["dDelta_f"], r["Theta"]
    r = m.compute_expectations(x.copy(), uncertainty_method="bootstrap")
    data[p + "avg_mu"], data[p + "avg_sigma"] = r["mu"], r["sigma"]
    r = m.compute_expectations(x.copy(), output="differences", uncertainty_method="bootstrap")
    data[p + "diff_mu"], data[p + "diff_sigma"] = r["mu"], r["sigma"]
    r = m.compute_expectations(u.copy(), state_dependent=True, uncertainty_method="bootstrap")
    data[p + "sd_mu"], data[p + "sd_sigma"] = r["mu"], r["sigma"]
    r = m.compute_multiple_expectations(np.array([x, x ** 2]), u[0].copy(), compute_covariance=True,
                                        uncertainty_method="bootstrap")
    data[p + "mult_mu"], data[p + "mult_sigma"], data[p + "mult_cov"] = r["mu"], r["sigma"], r["covariances"]
    r = m.compute_perturbed_free_energies(z["pert_u_ln"].copy(), uncertainty_method="bootstrap")
    data[p + "pert_Delta_f"], data[p + "pert_dDelta_f"] = r["Delta_f"], r["dDelta_f"]
    r = m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap")
    for key in EE_KEYS:
        data[p + "ee_" + key] = np.asarray(r[key])
    state_map = np.array([np.arange(K), np.zeros(K, int)])
    r = m.compute_expectations_inner(x.copy()[None], u.copy(), state_map, uncertainty_method="bootstrap")
    data[p + "inner_obs"], data[p + "inner_f"] = r["bootstrapped_observables"], r["bootstrapped_f"]
    if first:
        m = pymbar.MBAR(u, N_k, n_bootstraps=NB, rseed=seed, initialize="BAR")
        data[f"{name}_bar_f_k_boots"] = np.array(m.f_k_boots)
        perm = interleaving(N_k)
        labels = np.repeat(np.arange(K), N_k)[perm]
        m = pymbar.MBAR(u[:, perm], N_k, n_bootstraps=NB, rseed=seed, x_kindices=labels)
        data[f"{name}_perm"] = perm
        data[f"{name}_il_after"] = np.float64(m.rng.random())
        data[f"{name}_il_f_k_boots"] = np.array(m.f_k_boots)
        data[f"{name}_il_bootstrap_rints"] = np.array(m.bootstrap_rints, dtype=np.int64)
    print(f"{p}: f_k_boots[0]={data[p + 'f_k_boots'][0]} avg_sigma={data[p + 'avg_sigma']}")


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    from tests import _cases

    cases = _cases.SMALL + _cases.REF_SUITE
    data = {"cases": np.array(cases), "seeds": np.array(SEEDS), "n_bootstraps": np.int64(NB)}
    for name in cases:
        for i, seed in enumerate(SEEDS):
            run(name, seed, data, i == 0)
    np.savez_compressed(os.path.join(OUT, "mbar_bootstrap.npz"), **data)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

#!/usr/bin/env python
"""Generate tests/golden/fes_spline_bootstrap.npz by running the UNMODIFIED reference pymbar.FES with
fes_type="spline" and n_bootstraps > 0.

    python tools/make_fes_spline_bootstrap_golden.py /path/to/pymbar-checkout

The samples are those of the histogram fixture fes_hist_1d and the spline parameters those of tests/_spline (the
cases in CASES: each spline_weights with Newton-CG, L-BFGS-B and the MAP objective), so no new sample data is stored.
For each case and seed (n_bootstraps = NB) the file holds, with keys prefixed "<case>_s<seed>_":
  * c [NB, nspline]: fes_functions[b].c; c0 [nspline]: fes_function.c;
  * obj / gnorm [NB]: the reference's _bspline_calculate_f and the norm of _bspline_calculate_g at replicate b's final
    coefficients, on that replicate's own x_nb and w_nb (evaluated after the run, so the fit is not disturbed);
  * V [NB, N] (unbiasedstate only): the replicate's weight on each resident sample, sum of w_nb[m] over the
    positions m with bootstrap_indices[m] = n;
  * f_<ref> / df_<ref> [Q]: get_fes(uncertainty_method="bootstrap") for from-lowest and from-specified;
  * after: one np.random.random() drawn right after generate_fes returns.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden")
CASES = ("unbiased_ncg", "biased_ncg", "simplesum_ncg", "unbiased_lbfgsb", "unbiased_map")
NB = 5
SEEDS = (7, 2024)
REFS = ("from-lowest", "from-specified")


def run(name, seed, data):
    import pymbar

    from tests import _fes, _spline

    z = _fes.load("fes_hist_1d")
    case = next(c for c in _spline.SPLINE_CASES if c["name"] == name)
    p = f"{name}_s{seed}_"
    fes = pymbar.FES(z["u_kn"], z["N_k"])
    seen = []
    orig_fit = fes._generate_fes_spline

    def recording_fit(b, x_n, w_n):
        if b > 0:
            seen.append((np.array(x_n), np.array(w_n)))
        return orig_fit(b, x_n, w_n)

    fes._generate_fes_spline = recording_fit
    fes.generate_fes(z["u_n"], z["x_n"], fes_type="spline", spline_parameters=_spline.spline_parameters(case, z),
                     n_bootstraps=NB, seed=seed)
    data[p + "after"] = np.float64(np.random.random())
    assert len(fes.fes_functions) == NB == len(seen)
    data[p + "c"] = np.array([s.c for s in fes.fes_functions])
    data[p + "c0"] = np.array(fes.fes_function.c)
    for ref in REFS:
        r = fes.get_fes(_spline.QUERIES, reference_point=ref, fes_reference=_spline.FES_REF,
                        uncertainty_method="bootstrap")
        tag = ref.split("-")[1]
        data[p + "f_" + tag], data[p + "df_" + tag] = np.ravel(r["f_i"]), np.ravel(r["df_i"])
    obj, gnorm = np.zeros(NB), np.zeros(NB)
    for b, (x_nb, w_nb) in enumerate(seen):
        xi = fes.fes_functions[b].c[1:]
        obj[b] = fes._bspline_calculate_f(xi, x_nb, w_nb)
        gnorm[b] = np.linalg.norm(fes._bspline_calculate_g(xi, x_nb, w_nb))
    data[p + "obj"], data[p + "gnorm"] = obj, gnorm
    if case["weights"] == "unbiasedstate":
        # the positions' weights summed onto the samples they repeat (x_nb identifies them: x_n has no ties)
        order = np.argsort(z["x_n"])
        assert np.all(np.diff(z["x_n"][order]) > 0)
        V = np.zeros((NB, len(z["x_n"])))
        for b, (x_nb, w_nb) in enumerate(seen):
            n = order[np.searchsorted(z["x_n"][order], x_nb)]
            assert np.array_equal(z["x_n"][n], x_nb)
            V[b] = np.bincount(n, weights=w_nb, minlength=len(z["x_n"]))
        data[p + "V"] = V
    print(f"{p}: gnorm={gnorm} df_lowest[:3]={data[p + 'df_lowest'][:3]}", flush=True)


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    from tests import _spline

    data = {"cases": np.array(CASES), "seeds": np.array(SEEDS), "n_bootstraps": np.int64(NB),
            "source": np.array("fes_hist_1d"), "queries": _spline.QUERIES, "fes_reference": np.array(_spline.FES_REF)}
    for name in CASES:
        for seed in SEEDS:
            run(name, seed, data)
    np.savez_compressed(os.path.join(OUT, "fes_spline_bootstrap.npz"), **data)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

#!/usr/bin/env python
"""Generate tests/golden/fes_spline_1d.npz by running the UNMODIFIED reference pymbar.FES with fes_type="spline".

    python tools/make_fes_spline_golden.py /path/to/pymbar-checkout

The samples are those of the histogram fixture fes_hist_1d, loaded through tests/_fes.load, so no new sample data is
stored.  The biases are Ku/2 (x - c_k)^2 with the fixture's centres.  For each case (tests/_spline.SPLINE_CASES: each
spline_weights with Newton-CG, L-BFGS-B, a MAP objective with a quadratic prior, and the "zeros",
"explicit" and "bias_free_energies" initialisations; optimization_algorithm="Custom-NR" raises UnboundLocalError in
the reference, fes.py:1040) the file holds:
  * f, g, h [case, 3, ...], pF and pE: _bspline_calculate_f, _g and _h at three fixed coefficient vectors (XI_FIXED),
    called in that order, and spline_data["bspline_pF"] / ["bspline_pE"] after them;
  * c, aic, bic: the final fes_function.c and the information criteria;
  * f_lowest / f_specified [case, Q]: get_fes on the query grid;
  * for the cases in MC_CASES, a seeded sample_parameter_distribution (MC_STEPS steps, sample_every = 1,
    decorrelate=False, no prior): mc_samples, mc_logpost, mc_naccept, and mc_margin, the smallest distance of a
    Metropolis decision from flipping (tests/_spline.metropolis_margin, from the log-likelihoods of every step and
    the uniforms drawn).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden")


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    import pymbar

    from tests import _fes, _spline

    z = _fes.load("fes_hist_1d")
    cases = _spline.SPLINE_CASES
    nxi = len(_spline.XI_FIXED)
    data = {"source": np.array("fes_hist_1d"), "queries": _spline.QUERIES, "fes_reference": np.array(_spline.FES_REF)}
    nsp = [c["nspline"] for c in cases]
    assert len(set(nsp)) == 1
    ns = nsp[0]
    C = len(cases)
    for key, shape in (("f", (C, nxi)), ("g", (C, nxi, ns - 1)), ("h", (C, nxi, ns - 1, ns - 1)),
                       ("pF", (C, nxi, len(z["N_k"]))), ("pE", (C, nxi, ns - 1)), ("c", (C, ns)), ("aic", (C,)),
                       ("bic", (C,)), ("f_lowest", (C, len(_spline.QUERIES))),
                       ("f_specified", (C, len(_spline.QUERIES)))):
        data[key] = np.full(shape, np.nan)
    M = len(_spline.MC_CASES)
    data["mc_samples"] = np.zeros((M, ns, _spline.MC_STEPS))
    data["mc_logpost"] = np.zeros((M, _spline.MC_STEPS))
    data["mc_naccept"] = np.zeros(M, np.int64)
    data["mc_margin"] = np.zeros(M)
    for i, case in enumerate(cases):
        fes = pymbar.FES(z["u_kn"], z["N_k"])
        params = _spline.spline_parameters(case, z)
        fes.generate_fes(z["u_n"], z["x_n"], fes_type="spline", spline_parameters=params)
        for j, xi in enumerate(_spline.XI_FIXED):
            data["f"][i, j] = fes._bspline_calculate_f(xi, z["x_n"], fes.w_n)
            data["g"][i, j] = fes._bspline_calculate_g(xi, z["x_n"], fes.w_n)
            data["h"][i, j] = fes._bspline_calculate_h(xi, z["x_n"], fes.w_n)
            pF = np.atleast_1d(fes.spline_data["bspline_pF"])
            data["pF"][i, j, :len(pF)] = pF
            pE = np.atleast_1d(fes.spline_data["bspline_pE"])
            data["pE"][i, j, :len(pE)] = pE
        data["c"][i] = fes.fes_function.c
        data["aic"][i] = fes.get_information_criteria("akaike")
        data["bic"][i] = fes.get_information_criteria("bayesian")
        data["f_lowest"][i] = fes.get_fes(_spline.QUERIES, reference_point="from-lowest")["f_i"]
        data["f_specified"][i] = fes.get_fes(_spline.QUERIES, reference_point="from-specified",
                                             fes_reference=_spline.FES_REF)["f_i"]
        if case["name"] in _spline.MC_CASES:
            m = _spline.MC_CASES.index(case["name"])
            draws, lls = [], []
            orig_random = np.random.random
            orig_ll = fes._get_MC_loglikelihood

            def recording_ll(*a, **k):
                v = orig_ll(*a, **k)
                lls.append(v)
                return v

            fes._get_MC_loglikelihood = recording_ll

            def recording_random(*a, **k):
                u = orig_random(*a, **k)
                draws.append(u)
                return u

            np.random.random = recording_random
            try:
                np.random.seed(_spline.MC_SEED)
                try:
                    fes.sample_parameter_distribution(z["x_n"], mc_parameters=_spline.mc_parameters(),
                                                      decorrelate=False, verbose=False)
                except UnboundLocalError:
                    pass                    # fes.py:1855-1857 read names only decorrelate=True defines
            finally:
                np.random.random = orig_random
            mc = fes.mc_data
            data["mc_samples"][m] = mc["samples"]
            data["mc_logpost"][m] = mc["logposteriors"]
            data["mc_naccept"][m] = mc["naccept"]
            data["mc_margin"][m] = _spline.metropolis_margin(lls, draws)
        print(f"{case['name']:22s} c[:3]={data['c'][i][:3]} aic={data['aic'][i]:.6f}")
    np.savez_compressed(os.path.join(OUT, "fes_spline_1d.npz"), **data)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

#!/usr/bin/env python
"""Generate tests/golden/timeseries_many.npz by running the UNMODIFIED reference pymbar.timeseries.

    python tools/make_timeseries_many_golden.py /path/to/pymbar-checkout

The series are tests/_timeseries_many.series() (seeded); names and digest (tests/_timeseries_many.digest of every
series and partner, in order) identify them.  Per case key, the reference's output for every series, in list order:
  eq__<fast>__<nskip>                  detect_equilibration: [n, 3] of (t, g, Neff_max); eqerr__...: 1 where it raised
  si__<auto|cross>__<fast>__<mintime>  statistical_inefficiency g (NaN where it raised ParameterError)
  sub__<conservative>__<g>             subsample_correlated_data: the index lists concatenated, with subn__...: their
                                       lengths (g "None": computed, "per-series": g_i = 1.5 + 0.25 i)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "timeseries_many.npz")


def per_series_g(n):
    return [1.5 + 0.25 * i for i in range(n)]


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    from pymbar import timeseries as ref
    from pymbar.utils import ParameterError

    from tests import _timeseries_many as cases

    names, A, B = cases.series()
    data = {"names": np.array(names), "digest": np.array(cases.digest(A, B))}
    for fast, nskip in cases.EQ_CASES:
        res, err = [], []
        for a in A:
            try:
                t, g, Neff = ref.detect_equilibration(a, fast=fast, nskip=nskip)
                res.append([float(t), float(g), float(Neff)])
                err.append(0)
            except ParameterError:
                res.append([np.nan] * 3)
                err.append(1)
        data[f"eq__{int(fast)}__{nskip}"] = np.array(res)
        data[f"eqerr__{int(fast)}__{nskip}"] = np.array(err)
        print(f"eq fast={fast} nskip={nskip}: {sum(err)} raised")
    for kind, fast, mintime in cases.SI_CASES:
        gs = []
        for a, b in zip(A, B):
            try:
                gs.append(ref.statistical_inefficiency(a, b if kind == "cross" else None, fast=fast, mintime=mintime))
            except ParameterError:
                gs.append(np.nan)
        data[f"si__{kind}__{int(fast)}__{mintime}"] = np.array(gs, np.float64)
    for conservative, g in cases.SUB_CASES:
        gl = per_series_g(len(A)) if g == "per-series" else [g] * len(A)
        idx = []
        for a, gi in zip(A, gl):
            try:
                idx.append(list(ref.subsample_correlated_data(a, g=gi, conservative=conservative)))
            except ParameterError:
                idx.append([-1])
        key = f"{int(conservative)}__{g}"
        data["sub__" + key] = np.array([v for x in idx for v in x], np.int64)
        data["subn__" + key] = np.array([len(x) for x in idx], np.int64)
    np.savez_compressed(OUT, **data)
    print("wrote", OUT)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

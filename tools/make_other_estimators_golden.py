#!/usr/bin/env python
"""Generate tests/golden/other_estimators.npz by running the UNMODIFIED reference pymbar.other_estimators.

    python tools/make_other_estimators_golden.py /path/to/pymbar-checkout

Stored: the work vectors (w__<name>, seeded) and `cases`, a JSON list with one entry per call:
  {"id", "fn" (bar / bar_zero / exp / exp_gauss / bar_overlap), "args" (vector names), "kwargs",
   "result": {key: [repr of the value, its type name]} or "value": [repr, type] (bar_zero, bar_overlap),
   or "error": [exception class name, message], and "g" where is_timeseries made the reference call
   pymbar.timeseries.statistical_inefficiency (its return value, so that a test without pymbar can stand in for it)}.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "other_estimators.npz")


def _ar1(seed, T, tau, mu=1.0, sigma=1.0):
    rng = np.random.RandomState(seed)
    a = np.exp(-1.0 / tau)
    x = np.zeros(T)
    e = rng.standard_normal(T) * np.sqrt(1 - a * a)
    for t in range(1, T):
        x[t] = a * x[t - 1] + e[t]
    return mu + sigma * x


def vectors(ref_testsystems):
    v = {}
    v["gauss_F"], v["gauss_R"] = ref_testsystems.gaussian_work_example(mu_F=None, DeltaF=1.0, seed=0)
    np.random.seed(0)
    exp_case = ref_testsystems.exponential_distributions.ExponentialTestCase(np.array([1.0, 4.0]))
    v["expo_F"], v["expo_R"], _ = exp_case.sample(np.array([500, 800]), mode="wFwR")
    rng = np.random.RandomState(7)
    v["uneq_F"] = rng.normal(1.5, 1.2, 50)
    v["uneq_R"] = rng.normal(-0.5, 1.2, 5000)
    v["one_F"] = np.array([0.7])
    v["one_R"] = rng.normal(-0.2, 0.8, 300)
    v["int_F"] = rng.randint(-3, 8, 400).astype(np.int64)
    v["int_R"] = rng.randint(-6, 4, 350).astype(np.int64)
    v["big_F"], v["big_R"] = ref_testsystems.gaussian_work_example(N_F=1000, N_R=1200, mu_F=None, DeltaF=300.0,
                                                                   sigma_F=2.0, seed=3)
    v["far_F"] = rng.normal(0.0, 1.0, 200)                   # no overlap at all: the uncertainty overflows
    v["far_R"] = rng.normal(-2000.0, 1.0, 200)
    v["wide_F"] = np.concatenate([rng.normal(0.0, 1.0, 100), [800.0]])   # spread above 745
    v["wide_R"] = rng.normal(-1.0, 1.0, 100)
    v["ar1"] = _ar1(11, 3000, 15.0, mu=2.0, sigma=0.7)
    return v


PAIRS = ["gauss", "expo", "uneq", "one", "int", "big", "far", "wide"]


def cases():
    out = []
    for p in PAIRS:
        for method in ("false-position", "bisection", "self-consistent-iteration"):
            for um in ("BAR", "MBAR"):
                out.append(dict(id=f"bar_{p}_{method}_{um}", fn="bar", args=[p + "_F", p + "_R"],
                                kwargs=dict(method=method, uncertainty_method=um)))
        out.append(dict(id=f"bar_{p}_noiter", fn="bar", args=[p + "_F", p + "_R"],
                        kwargs=dict(iterated_solution=False)))
        out.append(dict(id=f"bar_{p}_nounc", fn="bar", args=[p + "_F", p + "_R"],
                        kwargs=dict(compute_uncertainty=False)))
    for p, d in (("gauss", 0.8), ("expo", -1.0), ("big", 299.0)):
        out.append(dict(id=f"bar_{p}_sci_DF{d}", fn="bar", args=[p + "_F", p + "_R"],
                        kwargs=dict(method="self-consistent-iteration", DeltaF=d)))
        out.append(dict(id=f"bar_{p}_noiter_DF{d}", fn="bar", args=[p + "_F", p + "_R"],
                        kwargs=dict(iterated_solution=False, DeltaF=d, uncertainty_method="MBAR")))
    for method in ("false-position", "bisection", "self-consistent-iteration"):
        out.append(dict(id=f"bar_gauss_maxit2_{method}", fn="bar", args=["gauss_F", "gauss_R"],
                        kwargs=dict(method=method, maximum_iterations=2)))
    out.append(dict(id="bar_gauss_tol1e-6", fn="bar", args=["gauss_F", "gauss_R"],
                    kwargs=dict(relative_tolerance=1e-6)))
    for p in ("gauss", "expo", "int", "far"):
        for d in (-3.0, 0.0, 1.0, 2.5):
            out.append(dict(id=f"zero_{p}_{d}", fn="bar_zero", args=[p + "_F", p + "_R"], kwargs=dict(DeltaF=d)))
    for name in ("gauss_F", "gauss_R", "expo_F", "int_F", "big_F", "ar1", "wide_F"):
        for fn in ("exp", "exp_gauss"):
            out.append(dict(id=f"{fn}_{name}", fn=fn, args=[name], kwargs={}))
            out.append(dict(id=f"{fn}_{name}_nounc", fn=fn, args=[name], kwargs=dict(compute_uncertainty=False)))
    for fn in ("exp", "exp_gauss"):
        out.append(dict(id=f"{fn}_ar1_ts", fn=fn, args=["ar1"], kwargs=dict(is_timeseries=True)))
    out.append(dict(id="overlap_gauss", fn="bar_overlap", args=["gauss_F", "gauss_R"], kwargs={}))
    return out


def _enc(x):
    return [repr(float(x)), type(x).__name__]


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    import pymbar
    from pymbar import other_estimators as ref
    from pymbar import testsystems
    from pymbar import timeseries

    v = vectors(testsystems)
    si = timeseries.statistical_inefficiency
    done = []
    for c in cases():
        args = [v[a] for a in c["args"]]
        seen = []

        def record(*a, **k):
            seen.append(si(*a, **k))
            return seen[-1]

        timeseries.statistical_inefficiency = record
        try:
            fn = pymbar.bar_overlap if c["fn"] == "bar_overlap" else getattr(ref, c["fn"])
            r = fn(*args, **c["kwargs"])
            if isinstance(r, dict):
                c["result"] = {k: _enc(x) for k, x in r.items()}
            else:
                c["value"] = _enc(r)
        except Exception as e:                          # the reference's own errors are part of the fixture
            c["error"] = [type(e).__name__, str(e)]
        finally:
            timeseries.statistical_inefficiency = si
        if seen:
            c["g"] = repr(float(seen[0]))
        np.seterr(over="warn")
        print(c["id"], c.get("result", c.get("value", c.get("error"))))
        done.append(c)
    data = {f"w__{k}": x for k, x in v.items()}
    data["cases"] = np.array(json.dumps(done))
    np.savez_compressed(OUT, **data)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

"""The seeded series and the cases of tests/golden/timeseries.npz (tools/make_timeseries_golden.py)."""
import numpy as np

MULTI_LENGTHS = [300, 700, 1100, 500]

# (series, fast, mintime) for statistical_inefficiency
SI_CASES = [(name, fast, mintime) for name in ("white", "ar5", "ar50", "trans10", "trans1000", "offset", "int",
                                                "cross", "long")
            for fast, mintime in ((False, 3), (True, 3), (False, 0), (False, 20), (True, 20))
            if name != "long" or (fast, mintime) == (False, 3)]
# (series, fast, nskip) for detect_equilibration
EQ_CASES = [("ar5", True, 1), ("trans10", True, 1), ("trans10", False, 1), ("trans1000", True, 7),
            ("offset", True, 1), ("const3", True, 1), ("const01", True, 1), ("int", True, 1), ("ar50", True, 7),
            ("ar50", True, 50), ("white", True, 1)]
# (series, N_max, norm) for normalized_fluctuation_correlation_function
CORR_CASES = [("ar5", None, True), ("ar5", 25, True), ("ar5", 25, False), ("cross", 25, True),
              ("cross", None, False), ("offset", 25, True)]


def ar1(rng, T, tau):
    a = np.exp(-1.0 / tau)
    x = np.empty(T)
    x[0] = rng.standard_normal()
    e = rng.standard_normal(T) * np.sqrt(1 - a * a)
    for n in range(1, T):
        x[n] = a * x[n - 1] + e[n]
    return x


def series():
    rng = np.random.RandomState(20261015)
    s = {}
    s["white"] = rng.standard_normal(1200)
    s["ar5"] = ar1(rng, 1500, 5.0)
    s["ar50"] = ar1(rng, 6000, 50.0)
    x = ar1(rng, 1500, 5.0)
    s["trans10"] = x + 10.0 * np.exp(-np.arange(1500) / 60.0)
    x = ar1(rng, 3000, 5.0)
    s["trans1000"] = x + 1000.0 * np.exp(-np.arange(3000) / 80.0)
    s["offset"] = 1.0e6 + ar1(rng, 1500, 5.0)
    x = ar1(rng, 900, 5.0) + 3.0 * np.exp(-np.arange(900) / 50.0)
    s["const3"] = np.concatenate([x, np.full(100, 3.0)])
    s["const01"] = np.concatenate([x, np.full(100, 0.1)])
    s["int"] = np.round(40.0 * ar1(rng, 1200, 5.0)).astype(np.int64)
    s["cross"] = ar1(rng, 2000, 8.0)
    s["cross_b"] = 0.6 * s["cross"] + 0.8 * ar1(rng, 2000, 3.0)
    s["long"] = ar1(rng, 20000, 50.0)
    s["multi"] = ar1(rng, sum(MULTI_LENGTHS), 5.0)
    return s


def constant_tail(name):
    return name.startswith("const")

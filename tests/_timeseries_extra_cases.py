"""The seeded series and the cases of tests/golden/timeseries_extra.npz (tools/make_timeseries_fft_golden.py)."""
import numpy as np

from tests._timeseries_cases import ar1

# multiple-series sets: name -> lengths (series in list order)
MULTI_SETS = {"auto": [300, 700, 1100, 500], "cross": [300, 700, 1100, 500], "int": [400, 250, 600],
              "offset": [500, 800], "negpart": [200, 2000]}
# (set, N_max, norm, truncate) for normalized_fluctuation_correlation_function_multiple
CORRM_CASES = [(name, n_max, norm, trunc) for name in ("auto", "cross", "int", "offset")
               for n_max in (None, 25, "limit") for norm in (True, False) for trunc in (False, True)
               if name == "auto" or (norm, trunc) != (False, True)] + \
              [("negpart", None, True, True), ("negpart", None, True, False), ("negpart", 40, False, True),
               ("auto", 5000, True, False)]
# (series, mintime) for statistical_inefficiency_fft; the X, X**2 and energy series and the Gaussian and repeated
# Gaussian series have the shapes of the reference's own tests (pymbar/tests/test_timeseries.py:61-104)
FFT_CASES = [(name, mintime) for name in ("ar5", "white", "int", "offset", "drift")
             for mintime in (0, 3, 20)] + \
            [("X", 3), ("X2", 3), ("energy", 3), ("gauss", 3), ("gauss3", 3)]
# (series, bs_nodes) for detect_equilibration_binary_search; "concat" is the reference's comparison series
# (pymbar/tests/test_timeseries.py:119-139), "normal" its binary-search test
BS_CASES = [("normal", 10), ("concat0", 10), ("concat1", 10), ("concat2", 10), ("trans", 10), ("trans", 6),
            ("ar5", 7)]


def n_max_of(name, n_max):
    return max(MULTI_SETS[name]) - 1 if n_max == "limit" else n_max


def case_key(name, n_max, norm, trunc):
    return f"{name}__{n_max}__{int(norm)}__{int(trunc)}"


def series():
    rng = np.random.RandomState(20261016)
    s = {}
    L = MULTI_SETS["auto"]
    s["m_auto"] = ar1(rng, sum(L), 5.0)
    s["m_cross"] = ar1(rng, sum(L), 8.0)
    s["m_cross_b"] = 0.6 * s["m_cross"] + 0.8 * ar1(rng, sum(L), 3.0)
    s["m_int"] = np.round(40.0 * ar1(rng, sum(MULTI_SETS["int"]), 5.0)).astype(np.int64)
    s["m_offset"] = 1.0e6 + ar1(rng, sum(MULTI_SETS["offset"]), 5.0)
    # series 0 alternates in sign (its lag-1 sum is negative), series 1 is slow: the running numerator is negative
    # after series 0 at t = 1 while the total is positive
    alt = np.where(np.arange(200) % 2 == 0, 1.0, -1.0) * (1.0 + 0.1 * rng.standard_normal(200))
    s["m_negpart"] = np.concatenate([alt, ar1(rng, 2000, 30.0)])
    s["ar5"] = ar1(rng, 1500, 5.0)
    s["white"] = rng.standard_normal(1200)
    s["int"] = np.round(40.0 * ar1(rng, 1200, 5.0)).astype(np.int64)
    s["offset"] = 1.0e6 + ar1(rng, 1500, 5.0)
    s["drift"] = np.linspace(0.0, 1.0, 600) + 1e-3 * rng.standard_normal(600)
    X = rng.normal(0.0, 1.0, 10000) / 10.0
    Y = rng.normal(0.0, 1.0, 10000)
    s["X"] = X
    s["X2"] = X ** 2
    s["energy"] = 10 * X ** 2 / 2.0 + Y ** 2 / 2.0
    s["gauss"] = rng.normal(size=100000)
    s["gauss3"] = np.repeat(rng.normal(size=30000), 3)
    s["normal"] = rng.normal(size=10000)
    for k in range(3):
        s[f"concat{k}"] = np.concatenate([ar1(rng, 100, 5.0) + 2.0, ar1(rng, 100, 5.0) + 1.0, ar1(rng, 200, 5.0)])
    s["trans"] = ar1(rng, 3000, 5.0) + 10.0 * np.exp(-np.arange(3000) / 60.0)
    return s


def multi(s, name):
    """(A_kn, B_kn or None) of a multiple-series set."""
    L = MULTI_SETS[name]
    off = np.cumsum([0] + L[:-1])
    A = s["m_" + name]
    B = s.get("m_" + name + "_b")
    return [A[o:o + n] for o, n in zip(off, L)], None if B is None else [B[o:o + n] for o, n in zip(off, L)]

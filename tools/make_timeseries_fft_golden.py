#!/usr/bin/env python
"""Generate tests/golden/timeseries_extra.npz by running the UNMODIFIED reference pymbar.timeseries.

    python tools/make_timeseries_fft_golden.py /path/to/pymbar-checkout

statistical_inefficiency_fft and detect_equilibration_binary_search import statsmodels.  This script installs a
stand-in `statsmodels.api` in sys.modules, for this process only, whose tsa.stattools.acf(x, adjusted=True,
fft=True, nlags) is a restatement of statsmodels' acovf (tests/_timeseries_extra.sm_acf: demean, np.fft on a length
>= 2N + 1, divide by N - t, then by lag 0); the reference's own code then applies its stop rule, sums g_t and runs
its binary-search grid.  normalized_fluctuation_correlation_function_multiple runs as it is.

A sha256 digest of each series (tests/_timeseries_extra_cases.series, seeded) and, per case key:
  cm__<set>__<N_max>__<norm>__<truncate>  normalized_fluctuation_correlation_function_multiple; with truncate
                                          cmmargin__<key>: the smallest |running numerator| / bound of its decisions
  fft__<series>__<mintime>                statistical_inefficiency_fft, with margin__fft__<key> and
                                          fftmargin__fft__<key>: the smallest |C| / bound of the long-double walk
                                          against the device's bound and against the FFT's rounding bound
  bs__<series>__<bs_nodes>                detect_equilibration_binary_search (t, g, Neff_max) and bsgap__<key>: the
                                          smallest relative gap between the two largest Neff of a round
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "timeseries_extra.npz")


def install_statsmodels_stand_in(acf):
    sm = types.ModuleType("statsmodels")
    api = types.ModuleType("statsmodels.api")
    api.tsa = types.SimpleNamespace(stattools=types.SimpleNamespace(acf=acf))
    sm.api = api
    sys.modules["statsmodels"] = sm
    sys.modules["statsmodels.api"] = api


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    from pymbar import timeseries as ref

    from tests import _timeseries_extra as tsx
    from tests import _timeseries_extra_cases as cases

    install_statsmodels_stand_in(tsx.sm_acf)
    series = cases.series()
    # the series come from the seeded generator; a digest of each guards against a change in the generator
    data = {f"digest__{k}": np.array(tsx.digest(v)) for k, v in series.items()}
    for name, L in cases.MULTI_SETS.items():
        data[f"lengths__{name}"] = np.array(L)
    ld = {}
    for name, n_max, norm, trunc in cases.CORRM_CASES:
        A_kn, B_kn = cases.multi(series, name)
        nm = cases.n_max_of(name, n_max)
        key = cases.case_key(name, n_max, norm, trunc)
        C = ref.normalized_fluctuation_correlation_function_multiple(A_kn, B_kn, N_max=nm, norm=norm,
                                                                     truncate=trunc)
        data["cm__" + key] = C
        if trunc:
            if name not in ld:
                ld[name] = tsx.ld_corr_multiple(A_kn, B_kn)
            lim = max(cases.MULTI_SETS[name]) - 1
            stop = tsx.corr_multiple_stop(ld[name], min(lim, nm or lim))
            assert stop == C.size, (key, stop, C.size)
            data["cmmargin__" + key] = tsx.corr_multiple_margin(ld[name], stop)
        print(f"cm {key}: {C.size} entries", f"margin {data.get('cmmargin__' + key)}" if trunc else "")
    for name, mintime in cases.FFT_CASES:
        A = series[name]
        key = f"{name}__{mintime}"
        g = ref.statistical_inefficiency_fft(A, mintime=mintime)
        data["fft__" + key] = np.float64(g)
        res = tsx.ld_walk_fft(A, 0, mintime)
        data["margin__fft__" + key], data["fftmargin__fft__" + key] = tsx.fft_margins(res)
        assert abs(max(1.0, float(res["g"])) - g) <= res["g_bound"], key
        print(f"fft {key}: g={g} last lag {res['last_lag']} margins {data['margin__fft__' + key]:.3g} "
              f"{data['fftmargin__fft__' + key]:.3g}")
    for name, nodes in cases.BS_CASES:
        A = series[name]
        key = f"{name}__{nodes}"
        t, g, Neff = ref.detect_equilibration_binary_search(A, bs_nodes=nodes)
        data["bs__" + key] = np.array([float(t), float(g), float(Neff)])
        data["bsgap__" + key] = np.float64(binary_search_gap(ref, A, nodes))
        print(f"bs {key}: t={t} g={g} Neff={Neff} gap={data['bsgap__' + key]:.3g}")
    np.savez_compressed(OUT, **data)


def binary_search_gap(ref, A_t, bs_nodes):
    """the reference's binary-search loop (timeseries.py:936-968) again, returning the smallest relative gap between
    the two largest Neff of a round"""
    T = A_t.size
    start, end = 1, T - 1
    n_grid = min(bs_nodes, T)
    gap = np.inf
    while True:
        time_grid = np.unique((10 ** np.linspace(np.log10(start), np.log10(end), n_grid)).round().astype("int"))
        Neff_t = np.ones(time_grid.size)
        for k, t in enumerate(time_grid):
            if t < T - 1:
                Neff_t[k] = (T - t + 1) / ref.statistical_inefficiency_fft(A_t[t:])
        top = np.sort(Neff_t)[-2:]
        gap = min(gap, (top[1] - top[0]) / top[1])
        k = Neff_t.argmax()
        if end - start < 4:
            break
        if k == 0:
            start, end = time_grid[0], time_grid[1]
        elif k == time_grid.size - 1:
            start, end = time_grid[-2], time_grid[-1]
        else:
            start, end = time_grid[k - 1], time_grid[k + 1]
    return gap


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

#!/usr/bin/env python
"""Generate tests/golden/timeseries.npz by running the UNMODIFIED reference pymbar.timeseries.

    python tools/make_timeseries_golden.py /path/to/pymbar-checkout

The series (tests/_timeseries_cases.series, seeded) and, per case key, the reference's output are stored:
  si__<series>__<fast>__<mintime>      statistical_inefficiency g
  eq__<series>__<fast>__<nskip>        detect_equilibration (t, g, Neff_max) and eqgap__...: the gap between the two
                                       largest float32 Neff values
  multi__<fast>                        statistical_inefficiency_multiple g and its [(t, C)] as multiCt__<fast> [n, 2]
  corr__<series>__<N_max>__<norm>      normalized_fluctuation_correlation_function
and margin__<key>: the smallest |C| / bound among the stop decisions of the long-double walk (tests/_timeseries.py),
so that a device result within the bound cannot flip a decision.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "timeseries.npz")


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    from pymbar import timeseries as ref

    from tests import _timeseries as tsr
    from tests import _timeseries_cases as cases

    series = cases.series()
    data = {f"series__{k}": v for k, v in series.items()}
    data["multi_lengths"] = np.array(cases.MULTI_LENGTHS)
    for name, fast, mintime in cases.SI_CASES:
        A = series[name]
        B = series[name + "_b"] if name + "_b" in series else None
        key = f"{name}__{int(fast)}__{mintime}"
        data["si__" + key] = np.float64(ref.statistical_inefficiency(A, B, fast=fast, mintime=mintime))
        if not cases.constant_tail(name):
            data["margin__si__" + key] = tsr.stop_margin(tsr.ld_walk(A, B, 0, fast, mintime))
    for name, fast, nskip in cases.EQ_CASES:
        A = series[name]
        t, g, Neff = ref.detect_equilibration(A, fast=fast, nskip=nskip)
        key = f"{name}__{int(fast)}__{nskip}"
        data["eq__" + key] = np.array([float(t), float(g), float(Neff)])
        # the gap between the two largest Neff: recompute the reference's Neff_t
        T = A.size
        g_t = np.ones(T - 1, np.float32)
        Neff_t = np.ones(T - 1, np.float32)
        for s in range(0, T - 1, nskip):
            try:
                g_t[s] = ref.statistical_inefficiency(A[s:T], fast=fast)
            except Exception:
                g_t[s] = T - s + 1
            Neff_t[s] = (T - s + 1) / g_t[s]
        top = np.sort(Neff_t)[-2:]
        data["eqgap__" + key] = np.float64(top[1] - top[0])
        assert Neff_t.argmax() == t and top[1] - top[0] > 0, key
        print(f"eq {key}: t={t} g={g} Neff={Neff} gap={top[1] - top[0]}")
    A_kn = [series["multi"][o:o + n] for o, n in zip(np.cumsum([0] + cases.MULTI_LENGTHS[:-1]), cases.MULTI_LENGTHS)]
    for fast in (False, True):
        g, Ct = ref.statistical_inefficiency_multiple(A_kn, fast=fast, return_correlation_function=True)
        data[f"multi__{int(fast)}"] = np.float64(g)
        data[f"multiCt__{int(fast)}"] = np.array([[t, c] for t, c in Ct])
        navg = np.mean(np.array(cases.MULTI_LENGTHS, np.float64))
        data[f"margin__multi__{int(fast)}"] = tsr.stop_margin(
            tsr.ld_walk(series["multi"], None, 0, fast, 10, lengths=np.array(cases.MULTI_LENGTHS), navg=navg))
    for name, n_max, norm in cases.CORR_CASES:
        A = series[name]
        B = series[name + "_b"] if name + "_b" in series else None
        data[f"corr__{name}__{n_max}__{int(norm)}"] = ref.normalized_fluctuation_correlation_function(
            A, B, N_max=n_max, norm=norm)
    for k, v in sorted(data.items()):
        if k.startswith(("si__", "multi__", "margin__")):
            print(k, float(v))
    np.savez_compressed(OUT, **data)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

"""normalized_fluctuation_correlation_function_multiple, statistical_inefficiency_fft and
detect_equilibration_binary_search of pymbar_b200.timeseries and the facade on the CPU, over the numpy stand-in of
DeviceAcf (tests/_timeseries_extra.py), against tests/golden/timeseries_extra.npz from the unmodified reference
(tools/make_timeseries_fft_golden.py)."""
import os
import sys
import types

import numpy as np
import pytest

from tests import _timeseries_extra as tsx
from tests import _timeseries_extra_cases as cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "timeseries_extra.npz")
OLD = ("statistical_inefficiency", "statistical_inefficiency_multiple", "normalized_fluctuation_correlation_function",
       "detect_equilibration")
NEW = ("normalized_fluctuation_correlation_function_multiple", "statistical_inefficiency_fft",
       "detect_equilibration_binary_search")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def series():
    return cases.series()


def _fake_module(names):
    mod = types.ModuleType("fake_timeseries")
    mod.calls = []
    for name in names:
        def orig(*args, _name=name, **kwargs):
            mod.calls.append(_name)
            return "original"
        setattr(mod, name, orig)
    return mod


@pytest.fixture()
def stand_in(monkeypatch):
    """pymbar_b200.timeseries over NumpyAcfExtra, and the facade on a module with every name whose originals record
    their calls."""
    from pymbar_b200 import facade
    from pymbar_b200 import timeseries as ts

    monkeypatch.setattr(ts, "DeviceAcf", tsx.NumpyAcfExtra)
    mod = _fake_module(OLD + NEW)
    facade.install_timeseries_on(mod)
    try:
        yield mod
    finally:
        facade.uninstall_from(mod)


@pytest.fixture(scope="module")
def ld_multi(series):
    return {name: tsx.ld_corr_multiple(*cases.multi(series, name)) for name in cases.MULTI_SETS}


def test_golden_matches_the_cases(golden, series):
    for k, v in series.items():
        assert str(golden["digest__" + k]) == tsx.digest(v), k


def test_correlation_multiple_within_the_long_double_bound(golden, series, stand_in, ld_multi):
    from pymbar_b200 import facade

    before = facade.STATS["ts_correlation_multiple"]
    for name, n_max, norm, trunc in cases.CORRM_CASES:
        A_kn, B_kn = cases.multi(series, name)
        key = cases.case_key(name, n_max, norm, trunc)
        want = golden["cm__" + key]
        C = stand_in.normalized_fluctuation_correlation_function_multiple(
            A_kn, B_kn, N_max=cases.n_max_of(name, n_max), norm=norm, truncate=trunc)
        assert type(C) is np.ndarray and C.dtype == np.float64 and C.shape == want.shape, key
        if trunc:
            assert golden["cmmargin__" + key] > 100, key
        res = ld_multi[name]
        bound = np.array([float(b) for b in res["C_bound"][:C.size]])
        assert np.all(bound < 1e-6)
        if norm:
            assert C.size == 0 or C[0] == 1.0
            assert np.all(np.abs(C - want) <= 2 * bound), key
        else:
            scale = abs(float(res["sigma2"])) * (1 + 1e-9)
            extra = 4 * tsx.EPS * (np.abs(want) + abs(float(res["mean_a"] * res["mean_b"])))
            assert np.all(np.abs(C - want) <= 2 * bound * scale + extra), key
    assert stand_in.calls == []
    assert facade.STATS["ts_correlation_multiple"] == before + len(cases.CORRM_CASES)


def test_correlation_multiple_checks_and_errors(series, stand_in):
    from pymbar_b200 import facade
    from pymbar_b200 import timeseries as ts
    from pymbar_b200 import utils as u

    A_kn, _ = cases.multi(series, "auto")
    with pytest.raises(u.ParameterError):
        ts.normalized_fluctuation_correlation_function_multiple(tuple(A_kn))
    with pytest.raises(u.ParameterError):
        ts.normalized_fluctuation_correlation_function_multiple(A_kn, A_kn[:2])
    with pytest.raises(u.ParameterError):
        ts.normalized_fluctuation_correlation_function_multiple(A_kn, [x[:-1] for x in A_kn])
    for bad in ([x.astype(np.float32) for x in A_kn], [list(x) for x in A_kn], [np.full(10, 0.1), np.full(5, 0.1)],
                []):
        with pytest.raises(ts.NotOnDevice):
            ts.normalized_fluctuation_correlation_function_multiple(bad)
    # an empty series adds nothing to any sum
    dev = tsx.NumpyAcfExtra(np.concatenate(A_kn), lengths=[x.size for x in A_kn])
    with_empty = ts.normalized_fluctuation_correlation_function_multiple(A_kn[:2] + [np.zeros(0)] + A_kn[2:],
                                                                         N_max=30)
    assert np.array_equal(with_empty, dev.correlation_multiple(30)[0])
    f0 = facade.STATS["ts_fallbacks"]
    assert stand_in.normalized_fluctuation_correlation_function_multiple([x.astype(np.float32) for x in A_kn]) \
        == "original"
    assert stand_in.normalized_fluctuation_correlation_function_multiple([np.full(10, 3.0)]) == "original"
    assert facade.STATS["ts_fallbacks"] == f0 + 2
    with pytest.raises(u.ParameterError):
        stand_in.normalized_fluctuation_correlation_function_multiple(np.stack([A_kn[0], A_kn[0]]))


def test_fft_within_the_long_double_bound(golden, series, stand_in):
    from pymbar_b200 import facade

    before = facade.STATS["ts_fft"]
    for name, mintime in cases.FFT_CASES:
        if name in ("gauss", "gauss3"):
            continue                                   # the stand-in is slow at T = 1e5; checked on the GPU
        key = f"{name}__{mintime}"
        assert golden["margin__fft__" + key] > 1e4 and golden["fftmargin__fft__" + key] > 1e4, key
        g = stand_in.statistical_inefficiency_fft(series[name], mintime=mintime)
        want = float(golden["fft__" + key])
        res = tsx.ld_walk_fft(series[name], 0, mintime)
        assert abs(g - want) <= 2 * res["g_bound"], (key, g, want)
        assert type(g) is (float if want == 1.0 else np.float64), key
    assert stand_in.calls == []
    assert facade.STATS["ts_fft"] == before + len([c for c in cases.FFT_CASES if c[0] not in ("gauss", "gauss3")])


def test_fft_rule_of_the_stand_in_against_long_double(series):
    for name in ("ar5", "drift", "offset"):
        A = series[name].astype(np.float64)
        for start in (0, 1, 511, 512):
            r = tsx.NumpyAcfExtra(A).inefficiency([start], mintime=3, rule="fft", trace_cap=600)
            res = tsx.ld_walk_fft(A, start, 3)
            n = len(res["C"])
            assert r["last_lag"][0] == res["last_lag"]
            cb = np.array([float(b) for b in res["C_bound"]])
            assert np.all(np.abs(r["trace"][0, :n] - np.array(res["C"], dtype=np.float64)) <= cb)
            assert abs(r["g"][0] - float(res["g"])) <= res["g_bound"]


def test_binary_search_reproduces_the_fixture(golden, series, stand_in):
    from pymbar_b200 import facade

    before = facade.STATS["ts_binary_search"]
    for name, nodes in cases.BS_CASES:
        key = f"{name}__{nodes}"
        t, g, Neff = stand_in.detect_equilibration_binary_search(series[name], bs_nodes=nodes)
        want = golden["bs__" + key]
        assert type(t) is np.int64 and type(g) is np.float64 and type(Neff) is np.float64, key
        assert t == int(want[0]), (key, t, want)
        gb = tsx.ld_walk_fft(series[name], int(t), 3)["g_bound"]
        assert golden["bsgap__" + key] > 20 * gb, key
        assert abs(g - want[1]) <= 2 * gb and abs(Neff - want[2]) <= 2 * gb / want[1] * want[2] * 1.01, key
    assert stand_in.calls == []
    assert facade.STATS["ts_binary_search"] == before + len(cases.BS_CASES)


def test_binary_search_edges(stand_in, monkeypatch):
    from pymbar_b200 import timeseries as ts

    assert ts.detect_equilibration_binary_search(np.full(40, 2.5)) == (0, 1, 40)
    with pytest.raises(AssertionError):
        ts.detect_equilibration_binary_search(np.arange(10.0), bs_nodes=4)
    x = np.random.RandomState(2).standard_normal(300)
    for bad in (x.astype(np.float32), x[:1], np.concatenate([x, np.full(1000, 0.1)])):
        with pytest.raises(ts.NotOnDevice):
            ts.detect_equilibration_binary_search(bad)
    # T = 2: no start is evaluated
    t, g, Neff = ts.detect_equilibration_binary_search(np.array([0.0, 1.0]))
    assert (t, g, Neff) == (1, 1.0, 1.0)
    # one device call per round
    calls = []
    orig = tsx.NumpyAcfExtra.inefficiency

    def counting(self, *a, **k):
        calls.append(np.atleast_1d(a[0]).size)
        return orig(self, *a, **k)

    monkeypatch.setattr(tsx.NumpyAcfExtra, "inefficiency", counting)
    ts.detect_equilibration_binary_search(x)
    assert len(calls) >= 2 and all(1 <= c <= 10 for c in calls)


def test_fallbacks_reach_the_original(stand_in):
    from pymbar_b200 import facade

    x = np.random.RandomState(1).standard_normal(300)
    f0 = facade.STATS["ts_fallbacks"]
    assert stand_in.statistical_inefficiency_fft(x.astype(np.float32)) == "original"
    assert stand_in.statistical_inefficiency_fft(np.full(50, 0.1)) == "original"
    assert stand_in.statistical_inefficiency_fft(x[:1]) == "original"
    assert stand_in.statistical_inefficiency_fft(x, mintime=2.5) == "original"
    assert stand_in.detect_equilibration_binary_search(list(x)) == "original"
    assert stand_in.detect_equilibration_binary_search(np.concatenate([x, np.full(1000, 0.1)])) == "original"
    bad = x.copy()
    bad[3] = np.inf
    assert stand_in.statistical_inefficiency_fft(bad) == "original"            # device error
    assert facade.STATS["ts_fallbacks"] == f0 + 7
    assert stand_in.calls == ["statistical_inefficiency_fft"] * 4 + ["detect_equilibration_binary_search"] * 2 + \
        ["statistical_inefficiency_fft"]


def test_statistical_inefficiency_fft_true_reaches_the_device(monkeypatch):
    """The original statistical_inefficiency(fft=True) calls the module's statistical_inefficiency_fft, which the
    facade rebinds: one pinned fall-back, then the device."""
    from pymbar_b200 import facade
    from pymbar_b200 import timeseries as ts

    monkeypatch.setattr(ts, "DeviceAcf", tsx.NumpyAcfExtra)
    mod = types.ModuleType("fake_timeseries")
    exec("def statistical_inefficiency(A_n, B_n=None, fast=False, mintime=3, fft=False):\n"
         "    if fft and B_n is None:\n"
         "        return statistical_inefficiency_fft(A_n, mintime=mintime)\n"
         "    raise AssertionError('original called')\n"
         "def statistical_inefficiency_fft(A_n, mintime=3):\n"
         "    raise ModuleNotFoundError(\"No module named 'statsmodels'\")\n", mod.__dict__)
    facade.install_timeseries_on(mod)
    try:
        x = cases.series()["ar5"]
        f0, d0 = facade.STATS["ts_fallbacks"], facade.STATS["ts_fft"]
        g = mod.statistical_inefficiency(x, fft=True)
        assert facade.STATS["ts_fallbacks"] == f0 + 1 and facade.STATS["ts_fft"] == d0 + 1
        assert g == ts.statistical_inefficiency_fft(x)
        with pytest.raises(ModuleNotFoundError):            # a fall-back still raises as the original does
            mod.statistical_inefficiency_fft(np.full(30, 0.1))
    finally:
        facade.uninstall_from(mod)


def test_rebinding_and_restore():
    from pymbar_b200 import facade

    full = _fake_module(OLD + NEW)
    stub = _fake_module(OLD)
    orig = {n: getattr(full, n) for n in OLD + NEW}
    facade.install_timeseries_on(full)
    facade.install_timeseries_on(stub)
    try:
        for n in OLD + NEW:
            assert getattr(full, n) is not orig[n] and getattr(full, n).__module__ == "pymbar_b200.facade"
        for n in NEW:
            assert not hasattr(stub, n)
    finally:
        facade.uninstall_from(full)
        facade.uninstall_from(stub)
    for n in OLD + NEW:
        assert getattr(full, n) is orig[n]
    for n in NEW:
        assert not hasattr(stub, n)


def test_install_rebinds_the_new_names(tmp_path):
    """install() on a pymbar-shaped package whose timeseries has the new names, and uninstall() restores them."""
    import pymbar_b200

    stub = "def {}(*args, **kwargs):\n    raise AssertionError('stand-in called')\n\n\n"
    pkg = tmp_path / "pymbar"
    pkg.mkdir()
    (pkg / "__init__.py").write_text("from . import mbar, mbar_solvers, utils  # noqa: F401\n")
    (pkg / "utils.py").write_text("class ParameterError(Exception):\n    pass\n\n\n" +
                                  "".join(stub.format(n) for n in ("kln_to_kn", "kn_to_n")))
    (pkg / "mbar_solvers.py").write_text("".join(stub.format(n) for n in pymbar_b200._PATCHED))
    (pkg / "mbar.py").write_text("from .utils import kln_to_kn, kn_to_n  # noqa: F401\n\n\nclass MBAR:\n    pass\n")
    (pkg / "timeseries.py").write_text("".join(stub.format(n) for n in OLD + NEW))
    sys.path.insert(0, str(tmp_path))
    try:
        import pymbar.timeseries as tsm

        orig = {n: getattr(tsm, n) for n in NEW}
        pymbar_b200.install()
        try:
            for n in NEW:
                assert getattr(tsm, n) is not orig[n] and getattr(tsm, n).__module__ == "pymbar_b200.facade"
        finally:
            pymbar_b200.uninstall()
        for n in NEW:
            assert getattr(tsm, n) is orig[n]
    finally:
        sys.path.remove(str(tmp_path))
        for name in [m for m in sys.modules if m == "pymbar" or m.startswith("pymbar.")]:
            del sys.modules[name]


def test_constant_series_with_inexact_mean_reach_the_original(stand_in):
    """np.full(n, 0.1).std() is rounding noise, not 0: the binary search and the FFT function must still call the
    original, as for every constant series."""
    from pymbar_b200 import facade
    from pymbar_b200 import timeseries as ts

    x = np.full(100, 0.1)
    assert x.std() != 0.0
    with pytest.raises(ts.NotOnDevice):
        ts.detect_equilibration_binary_search(x)
    f0 = facade.STATS["ts_fallbacks"]
    assert stand_in.detect_equilibration_binary_search(x) == "original"
    assert stand_in.statistical_inefficiency_fft(x) == "original"
    assert facade.STATS["ts_fallbacks"] == f0 + 2
    assert stand_in.calls == ["detect_equilibration_binary_search", "statistical_inefficiency_fft"]


def test_stand_in_keeps_the_series_chunk_grid_at_every_lag():
    """A (series, lag) sum runs over the chunks of the series' own length, whatever the lag: the terms past the
    window add nothing.  At L = 600000 the chunks are 586 samples while a window of 500000 would have 512."""
    rng = np.random.RandomState(6)
    L = 600_000
    x = rng.standard_normal(L - 100_000)
    assert tsx.chunk_size(L) != tsx.chunk_size(x.size)
    full = np.concatenate([x, np.zeros(L - x.size)])
    assert tsx._series_sum(x, L) == tsx._series_sum(full)
    a = rng.standard_normal(L + 1000)
    dev = tsx.NumpyAcfExtra(a, lengths=[L, 1000])
    mua, mub, _ = dev.multi_moments()
    t = 100_000
    num = dev.multi_numerator(t, mua, mub)[0]
    s0 = tsx._series_sum(np.concatenate([(a[:L - t] - mua) * (a[t:L] - mub), np.zeros(t)]))
    assert num == 0.0 + s0

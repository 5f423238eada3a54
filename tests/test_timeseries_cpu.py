"""pymbar_b200.timeseries and its facade on the CPU, over the numpy stand-in of DeviceAcf (tests/_timeseries.py),
against tests/golden/timeseries.npz from the unmodified reference (tools/make_timeseries_golden.py)."""
import os
import sys
import types

import numpy as np
import pytest

from tests import _timeseries as tsr
from tests import _timeseries_cases as cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "timeseries.npz")
NAMES = ("statistical_inefficiency", "statistical_inefficiency_multiple",
         "normalized_fluctuation_correlation_function", "detect_equilibration")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _series(z, name):
    return z["series__" + name]


@pytest.fixture()
def stand_in(monkeypatch):
    """pymbar_b200.timeseries over NumpyAcf, and the facade installed on a module whose originals record calls."""
    from pymbar_b200 import facade
    from pymbar_b200 import timeseries as ts

    monkeypatch.setattr(ts, "DeviceAcf", tsr.NumpyAcf)
    mod = types.ModuleType("fake_timeseries")
    mod.calls = []
    for name in NAMES:
        def orig(*args, _name=name, **kwargs):
            mod.calls.append(_name)
            return "original"
        setattr(mod, name, orig)
    facade.install_timeseries_on(mod)
    try:
        yield mod
    finally:
        facade.uninstall_from(mod)


def _g_tol(A, B, fast, mintime):
    res = tsr.ld_walk(A, B, 0, fast, mintime)
    b = tsr.g_bound(res)
    assert b < 1e-6
    return 2 * b + 1e-15


def test_facade_reproduces_inefficiency_fixtures(golden, stand_in):
    for name, fast, mintime in cases.SI_CASES:
        if name == "long":
            continue                                   # the stand-in is slow at T = 2e4; checked on the GPU
        A = _series(golden, name)
        B = golden.get("series__" + name + "_b")
        g = stand_in.statistical_inefficiency(A, B, fast=fast, mintime=mintime)
        want = float(golden[f"si__{name}__{int(fast)}__{mintime}"])
        assert abs(g - want) <= _g_tol(A, B, fast, mintime), (name, fast, mintime, g, want)
    assert stand_in.calls == []


def test_facade_reproduces_equilibration_fixtures(golden, stand_in):
    from pymbar_b200 import facade

    before = facade.STATS["ts_equilibration"]
    for name, fast, nskip in cases.EQ_CASES:
        A = _series(golden, name)
        t, g, Neff = stand_in.detect_equilibration(A, fast=fast, nskip=nskip)
        want = golden[f"eq__{name}__{int(fast)}__{nskip}"]
        assert type(t) is np.int64 and type(g) is np.float32 and type(Neff) is np.float32
        assert t == int(want[0]) and g == np.float32(want[1]) and Neff == np.float32(want[2]), (name, t, g, Neff, want)
    assert stand_in.calls == [] and facade.STATS["ts_equilibration"] == before + len(cases.EQ_CASES)


def test_facade_reproduces_multiple_and_correlation_fixtures(golden, stand_in):
    A = _series(golden, "multi")
    L = cases.MULTI_LENGTHS
    A_kn = [A[o:o + n] for o, n in zip(np.cumsum([0] + L[:-1]), L)]
    navg = np.mean(np.array(L, np.float64))
    for fast in (False, True):
        g, Ct = stand_in.statistical_inefficiency_multiple(A_kn, fast=fast, return_correlation_function=True)
        res = tsr.ld_walk(A, None, 0, fast, 10, lengths=np.array(L), navg=navg)
        assert abs(g - float(golden[f"multi__{int(fast)}"])) <= 2 * tsr.g_bound(res) + 1e-15
        want = golden[f"multiCt__{int(fast)}"]
        assert [t for t, _ in Ct] == [int(t) for t in want[:, 0]]
        bound = np.array([float(b) for b in res["C_bound"]])
        assert np.all(np.abs(np.array([c for _, c in Ct]) - want[:, 1]) <= 2 * bound)
        assert stand_in.statistical_inefficiency_multiple(A_kn, fast=fast) == g
    # 2-D input: equal lengths
    two = A[:1200].reshape(3, 400)
    assert isinstance(stand_in.statistical_inefficiency_multiple(two), float)
    for name, n_max, norm in cases.CORR_CASES:
        Aa = _series(golden, name)
        B = golden.get("series__" + name + "_b")
        C = stand_in.normalized_fluctuation_correlation_function(Aa, B, N_max=n_max, norm=norm)
        want = golden[f"corr__{name}__{n_max}__{int(norm)}"]
        assert C.shape == want.shape
        scale = np.max(np.abs(want))
        np.testing.assert_allclose(C, want, rtol=0, atol=1e-9 * scale)
    assert stand_in.calls == []


def test_fp64_restatement_within_long_double_bound(golden):
    """The device's order (NumpyAcf) against the long-double loop: every C, the stop lag and g within the bound, and
    the bound below 1e-6."""
    for name, fast, mintime in [("ar5", False, 3), ("offset", True, 3), ("trans1000", False, 20), ("cross", True, 0),
                                ("int", False, 0)]:
        A = _series(golden, name).astype(np.float64)
        B = golden.get("series__" + name + "_b")
        for start in (0, 1, 511, 512, 777):
            dev = tsr.NumpyAcf(A, B)
            r = dev.inefficiency([start], fast=fast, mintime=mintime, trace_cap=1024)
            res = tsr.ld_walk(A, B, start, fast, mintime)
            n = len(res["C"])
            assert r["last_lag"][0] == res["last_lag"]
            Cb = np.array([float(b) for b in res["C_bound"]])
            assert np.all(Cb < 1e-6)
            assert np.all(np.abs(r["trace"][0, :n] - np.array(res["C"], dtype=np.float64)) <= Cb)
            assert np.all(np.isnan(r["trace"][0, n:]))
            assert abs(r["g"][0] - float(res["g"])) <= tsr.g_bound(res) < 1e-6
            assert abs(r["sigma2"][0] - float(res["sigma2"])) <= float(res["sigma2_bound"])


def test_neff_matches_the_reference_expression():
    rng = np.random.RandomState(3)
    g = (1.0 + 50 * rng.random_sample(2000)).astype(np.float32)
    counts = rng.randint(2, 3_000_000, size=2000)
    from pymbar_b200 import timeseries as ts

    got = ts.neff(counts, g)
    want = np.array([np.float32(int(c) / gg) for c, gg in zip(counts, g)], np.float32)
    assert np.array_equal(got, want)


def test_lag_helpers():
    from pymbar_b200 import timeseries as ts

    assert [int(ts.lag(i, True)) for i in range(5)] == [1, 2, 4, 7, 11]
    for fast in (False, True):
        for n in range(0, 40):
            assert ts.lag_count(int(ts.lag(n, fast)), fast) == n + 1
    assert ts.mean_is_exact(3.0, 10 ** 6) and not ts.mean_is_exact(0.1, 1000) and ts.mean_is_exact(0.0, 5)


def test_fallbacks_reach_the_original(stand_in):
    from pymbar_b200 import facade

    rng = np.random.RandomState(1)
    x = rng.standard_normal(300)
    f0 = facade.STATS["ts_fallbacks"]
    assert stand_in.statistical_inefficiency(x, fft=True) == "original"
    assert stand_in.statistical_inefficiency(x.astype(np.float32)) == "original"
    assert stand_in.statistical_inefficiency(x.reshape(3, 100)) == "original"
    bad = x.copy()
    bad[7] = np.nan
    assert stand_in.statistical_inefficiency(bad) == "original"                  # device error
    assert stand_in.normalized_fluctuation_correlation_function(x.astype(np.float32)) == "original"
    assert stand_in.detect_equilibration(list(x)) == "original"
    assert stand_in.statistical_inefficiency_multiple([np.full(10, 0.1), np.full(20, 0.1)]) == "original"
    assert stand_in.statistical_inefficiency_multiple([x.astype(np.float32)]) == "original"
    assert facade.STATS["ts_fallbacks"] == f0 + 8
    assert stand_in.calls == ["statistical_inefficiency"] * 4 + ["normalized_fluctuation_correlation_function",
                                                                   "detect_equilibration"] + \
        ["statistical_inefficiency_multiple"] * 2
    c = (facade.STATS["ts_inefficiency"], facade.STATS["ts_correlation"])
    stand_in.statistical_inefficiency(x)
    stand_in.normalized_fluctuation_correlation_function(x, N_max=5)
    assert (facade.STATS["ts_inefficiency"], facade.STATS["ts_correlation"]) == (c[0] + 1, c[1] + 1)


def test_constant_series_follow_the_reference(golden, stand_in):
    from pymbar_b200 import utils as u

    with pytest.raises(u.ParameterError):
        stand_in.statistical_inefficiency(np.full(50, 3.0))
    # 0.1's mean is inexact in numpy: the reference runs its loop on the rounding noise; so does the host path
    x = np.full(50, 0.1)
    from pymbar_b200 import timeseries as ts

    assert stand_in.statistical_inefficiency(x) == max(1.0, ts._host_inefficiency(x, None, False, 3))


@pytest.fixture()
def pymbar_with_timeseries(tmp_path):
    """A pymbar-shaped package with (ts=True) or without a timeseries module; every function in it raises."""
    import pymbar_b200

    def make(ts):
        stub = "def {}(*args, **kwargs):\n    raise AssertionError('stand-in called')\n\n\n"
        pkg = tmp_path / ("with_ts" if ts else "without_ts") / "pymbar"
        pkg.mkdir(parents=True)
        (pkg / "__init__.py").write_text("from . import mbar, mbar_solvers, utils  # noqa: F401\n")
        (pkg / "utils.py").write_text("class ParameterError(Exception):\n    pass\n\n\n" +
                                      "".join(stub.format(n) for n in ("kln_to_kn", "kn_to_n")))
        (pkg / "mbar_solvers.py").write_text("".join(stub.format(n) for n in pymbar_b200._PATCHED))
        (pkg / "mbar.py").write_text("from .utils import kln_to_kn, kn_to_n  # noqa: F401\n\n\nclass MBAR:\n    pass\n")
        if ts:
            (pkg / "timeseries.py").write_text("".join(stub.format(n) for n in NAMES + ("subsample_correlated_data",)))
        sys.path.insert(0, str(pkg.parent))
        return str(pkg.parent)

    made = []
    try:
        yield lambda ts: made.append(make(ts)) or made[-1]
    finally:
        for p in made:
            if p in sys.path:
                sys.path.remove(p)
        for name in [m for m in sys.modules if m == "pymbar" or m.startswith("pymbar.")]:
            del sys.modules[name]


def test_install_patches_and_restores_timeseries(pymbar_with_timeseries):
    import pymbar_b200

    pymbar_with_timeseries(True)
    import pymbar.timeseries as tsm

    orig = {n: getattr(tsm, n) for n in NAMES}
    sub = tsm.subsample_correlated_data
    pymbar_b200.install()
    try:
        for n in NAMES:
            assert getattr(tsm, n) is not orig[n] and getattr(tsm, n).__module__ == "pymbar_b200.facade"
        assert tsm.subsample_correlated_data is sub
    finally:
        pymbar_b200.uninstall()
    for n in NAMES:
        assert getattr(tsm, n) is orig[n]


def test_install_without_timeseries_module(pymbar_with_timeseries):
    import pymbar_b200
    from pymbar_b200 import facade

    pymbar_with_timeseries(False)
    pymbar_b200.install()
    try:
        assert not any(isinstance(k, types.ModuleType) for k in facade._SAVED)
    finally:
        pymbar_b200.uninstall()
    assert not facade._SAVED

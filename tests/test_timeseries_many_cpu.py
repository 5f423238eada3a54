"""The _many functions of pymbar_b200.timeseries on the CPU, over a numpy stand-in of the segmented DeviceAcf
(tests/_timeseries_many.SeriesNumpyAcf), against tests/golden/timeseries_many.npz from the unmodified reference
(tools/make_timeseries_many_golden.py) and against the loop of the single-series functions on the same stand-in."""
import os

import numpy as np
import pytest

from tests import _timeseries as tsr
from tests import _timeseries_many as cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "timeseries_many.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.fixture()
def ts(monkeypatch):
    from pymbar_b200 import timeseries

    monkeypatch.setattr(timeseries, "DeviceAcf", cases.SeriesNumpyAcf)
    return timeseries


@pytest.fixture(scope="module")
def data():
    names, A, B = cases.series()
    short = [i for i, a in enumerate(A) if a.size < cases.LONG]        # the stand-in is slow on the long series
    return names, A, B, short


def test_series_match_the_fixture_inputs(golden, data):
    names, A, B, _ = data
    assert list(golden["names"]) == names and str(golden["digest"]) == cases.digest(A, B)


def test_detect_equilibration_many_reproduces_fixture_and_loop(golden, data, ts):
    """On the series of at most cases.SHORT[nskip] samples (lengths 2, 3, 511, 512, 513, a one-sample constant tail
    and the constant series; with nskip = 3 also the exact and inexact constant tails, integer data, white noise and
    a transient): the stand-in costs a numpy pass per (start, lag).  The GPU tests run every series."""
    names, A, _, _ = data
    for fast, nskip in cases.EQ_CASES:
        short = [i for i, a in enumerate(A) if a.size <= cases.SHORT[nskip]]
        assert len(short) >= (7 if nskip == 1 else 12)
        As = [A[i] for i in short]
        out = ts.detect_equilibration_many(As, fast=fast, nskip=nskip)
        loop = [ts.detect_equilibration(a, fast=fast, nskip=nskip) for a in As]
        assert [tuple(map(type, x)) for x in out] == [tuple(map(type, x)) for x in loop]
        assert out == loop
        want = golden[f"eq__{int(fast)}__{nskip}"]
        for (t, g, Neff), i in zip(out, short):
            if np.ptp(A[i]) > 0:
                assert type(t) is np.int64 and type(g) is np.float32 and type(Neff) is np.float32
            assert t == int(want[i, 0]) and g == np.float32(want[i, 1]) and Neff == np.float32(want[i, 2]), \
                (names[i], fast, nskip, (t, g, Neff), want[i])


def test_statistical_inefficiency_many_reproduces_fixture_and_loop(golden, data, ts):
    from pymbar_b200 import utils as u

    names, A, B, _ = data
    ok = [i for i, a in enumerate(A) if a.size <= 1500 and np.ptp(a) > 0]      # the GPU tests run every series
    for kind, fast, mintime in cases.SI_CASES:
        Bl = [B[i] for i in ok] if kind == "cross" else None
        got = ts.statistical_inefficiency_many([A[i] for i in ok], Bl, fast=fast, mintime=mintime)
        loop = [ts.statistical_inefficiency(A[i], None if Bl is None else Bl[j], fast, mintime)
                for j, i in enumerate(ok)]
        assert got.dtype == np.float64 and np.array_equal(got, np.array(loop))
        want = golden[f"si__{kind}__{int(fast)}__{mintime}"]
        for j, i in enumerate(ok):
            b = None if Bl is None else Bl[j]
            res = tsr.ld_walk(A[i], b, 0, fast, mintime)
            assert abs(got[j] - want[i]) <= 2 * tsr.g_bound(res) + 1e-15, (names[i], kind, fast, mintime)
    const = names.index("constant_400")
    assert np.isnan(golden["si__auto__0__3"][const])
    with pytest.raises(u.ParameterError):
        ts.statistical_inefficiency_many([A[const]])


def test_subsample_many_reproduces_fixture(golden, data, ts):
    names, A, _, short = data
    for conservative, g in cases.SUB_CASES:
        key = f"{int(conservative)}__{g}"
        flat, n = golden["sub__" + key], golden["subn__" + key]
        off = np.concatenate([[0], np.cumsum(n)])
        idx = [i for i in short if g is not None or np.ptp(A[i]) > 0]
        gl = [1.5 + 0.25 * i for i in idx] if g == "per-series" else g
        got = ts.subsample_correlated_data_many([A[i] for i in idx], g=gl, conservative=conservative)
        for j, i in enumerate(idx):
            assert type(got[j]) is list and all(type(v) is int for v in got[j])
            assert got[j] == flat[off[i]:off[i + 1]].tolist(), (names[i], key)


def test_lowest_failing_index_is_raised(ts):
    from pymbar_b200 import _lib
    from pymbar_b200 import utils as u

    rng = np.random.RandomState(4)
    good = [rng.standard_normal(300) for _ in range(4)]
    bad_nan = good[1].copy()
    bad_nan[5] = np.nan
    const = np.full(50, 3.0)
    with pytest.raises(u.ParameterError):                          # index 1 (constant) before index 2 (NaN)
        ts.statistical_inefficiency_many([good[0], const, bad_nan, good[2]])
    with pytest.raises(_lib.MbarB200Error):                        # index 1 (NaN) before index 2 (constant)
        ts.statistical_inefficiency_many([good[0], bad_nan, const, good[2]])
    with pytest.raises(u.ParameterError):                          # a shape mismatch at index 2
        ts.statistical_inefficiency_many(good[:3], [good[0], good[1], good[2][:10]])
    with pytest.raises(AttributeError):                            # a list has no .std(): index 0 raises first
        ts.detect_equilibration_many([list(good[0]), bad_nan])
    with pytest.raises(_lib.MbarB200Error):
        ts.detect_equilibration_many([good[0], bad_nan, [1.0, 2.0]])


def test_small_waves_give_the_same_results(data, ts, monkeypatch):
    _, A, B, short = data
    As = [A[i] for i in short[:12]]
    want = ts.detect_equilibration_many(As, fast=True, nskip=5)
    waves = ts.LAST_MANY_STATS["waves"]
    want_si = ts.statistical_inefficiency_many(As, [B[i] for i in short[:12]], fast=True)
    monkeypatch.setattr(ts, "WAVE_BYTES", 3 * ts.REQUEST_BYTES)
    assert ts.detect_equilibration_many(As, fast=True, nskip=5) == want
    assert waves == 1 and ts.LAST_MANY_STATS["waves"] > 50
    assert np.array_equal(ts.statistical_inefficiency_many(As, [B[i] for i in short[:12]], fast=True), want_si)


def test_empty_short_and_g_forms(ts):
    rng = np.random.RandomState(9)
    x = rng.standard_normal(400)
    assert ts.detect_equilibration_many([]) == [] and ts.subsample_correlated_data_many([]) == []
    assert ts.statistical_inefficiency_many([]).shape == (0,)
    short = [np.array([1.5]), np.array([1.0, 2.0]), np.array([2.0, 2.0]), np.array([0.3, 1.0, 0.1])]
    assert ts.detect_equilibration_many(short) == [ts.detect_equilibration(a) for a in short]
    si = [np.array([1.0, 2.0]), np.array([0.3, 1.0, 0.1]), x]
    assert np.array_equal(ts.statistical_inefficiency_many(si), [ts.statistical_inefficiency(a) for a in si])
    with pytest.raises(Exception) as many:
        ts.statistical_inefficiency_many([x, np.array([])])
    with pytest.raises(Exception) as single:
        ts.statistical_inefficiency(np.array([]))
    assert type(many.value) is type(single.value)
    with pytest.raises(Exception) as many:
        ts.detect_equilibration_many([x, np.array([])])
    with pytest.raises(Exception) as single:
        ts.detect_equilibration(np.array([]))
    assert type(many.value) is type(single.value)
    g = ts.statistical_inefficiency(x)
    y = rng.standard_normal(250)
    gy = ts.statistical_inefficiency(y)
    for conservative in (False, True):
        both = ts.subsample_correlated_data_many([x, y], g=None, conservative=conservative)
        assert both == ts.subsample_correlated_data_many([x, y], g=0, conservative=conservative)
        assert both == ts.subsample_correlated_data_many([x, y], g=[g, 0.0], conservative=conservative) == \
            ts.subsample_correlated_data_many([x, y], g=[g, gy], conservative=conservative)
        assert ts.subsample_correlated_data_many([x, y], g=2.5, conservative=conservative) == \
            ts.subsample_correlated_data_many([x, y], g=[2.5, 2.5], conservative=conservative)
    assert ts.subsample_correlated_data_many([x], g=2.5, conservative=True) == [list(range(0, 400, 3))]
    # round half to even, each index once: g = 0.5 keeps every index, g = 2.5 rounds 2.5 -> 2 and 7.5 -> 8
    assert ts.subsample_correlated_data_many([x[:6]], g=0.5) == [[0, 1, 2, 3, 4, 5]]
    assert ts.subsample_correlated_data_many([x[:10]], g=2.5) == [[0, 2, 5, 8]]
    with pytest.raises(ValueError):
        ts.subsample_correlated_data_many([x, y], g=[1.0])

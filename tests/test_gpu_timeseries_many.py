"""mbar_b200_acf_inefficiency_series on the H100: every request the same bits as `inefficiency` on an object holding its
series alone, across permutations, split calls and waves; every new error; and the _many functions of
pymbar_b200.timeseries against tests/golden/timeseries_many.npz and against the loop of the single-series functions,
bit for bit, up to a campaign-sized call."""
import os

import numpy as np
import pytest

from tests import _timeseries as tsr
from tests import _timeseries_many as cases

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "timeseries_many.npz")
KEYS = ("mean_a", "mean_b", "sigma2", "g", "last_lag", "status")
LENGTHS = [2, 3, 511, 512, 513, 1025, 70001, 524289]


def ar1(seed, T, tau):
    from scipy.signal import lfilter

    rng = np.random.RandomState(seed)
    a = np.exp(-1.0 / tau)
    return lfilter([1.0], [1.0, -a], rng.standard_normal(T) * np.sqrt(1 - a * a))


def _series(lengths, seed=0):
    A = [ar1(seed + T, T, 6.0) + 3.0 * np.exp(-np.arange(T) / 50.0) for T in lengths]
    B = [0.5 * a + ar1(seed + a.size + 1, a.size, 2.0) for a in A]
    return A, B


def _starts(T):
    NC = tsr.chunk_size(T)
    return sorted({s for s in (0, NC - 1, NC, NC + 1, T // 2, T - 2) if 0 <= s < T})


def _same(r, want, idx=None):
    for k in KEYS:
        got = r[k] if idx is None else r[k][idx]
        assert np.array_equal(got, want[k]), k


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def test_requests_match_one_series_objects():
    """Every request of one segmented call against `inefficiency` on an unsegmented object of its series alone:
    lengths around the chunk sizes up to 524289 (NC = 513), starts at the chunk edges, auto and cross, fast on and off,
    mintime 0, 3 and 20."""
    from pymbar_b200 import DeviceAcf

    A, B = _series(LENGTHS)
    ser = np.concatenate([np.full(len(_starts(T)), k, np.int32) for k, T in enumerate(LENGTHS)])
    st = np.concatenate([_starts(T) for T in LENGTHS]).astype(np.int64)
    for cross in (False, True):
        with DeviceAcf(np.concatenate(A), np.concatenate(B) if cross else None, lengths=LENGTHS) as dev:
            for fast in (False, True):
                for mintime in (0, 3, 20):
                    r = dev.inefficiency_series(ser, st, fast=fast, mintime=mintime)
                    stats = dev.last_stats()
                    assert stats["rounds"] >= 1 and stats["terms"] >= stats["useful_terms"] > 0
                    for k, T in enumerate(LENGTHS):
                        with DeviceAcf(A[k], B[k] if cross else None) as one:
                            want = one.inefficiency(_starts(T), fast=fast, mintime=mintime)
                        _same(r, want, ser == k)


def test_same_bits_permuted_split_and_repeated():
    from pymbar_b200 import DeviceAcf

    lengths = [700, 3000, 513, 1025, 9000, 2]
    A, _ = _series(lengths, seed=11)
    rng = np.random.RandomState(5)
    ser = np.concatenate([np.full(T - 1 if T > 1 else 1, k, np.int32) for k, T in enumerate(lengths)])
    st = np.concatenate([np.arange(max(T - 1, 1)) for T in lengths]).astype(np.int64)
    with DeviceAcf(np.concatenate(A), lengths=lengths) as dev:
        base = dev.inefficiency_series(ser, st, fast=True, mintime=3)
        perm = rng.permutation(ser.size)
        r = dev.inefficiency_series(ser[perm], st[perm], fast=True, mintime=3)
        _same(r, {k: v[perm] for k, v in base.items()})
        cut = ser.size // 3
        r1 = dev.inefficiency_series(ser[:cut], st[:cut], fast=True, mintime=3)
        r2 = dev.inefficiency_series(ser[cut:], st[cut:], fast=True, mintime=3)
        _same({k: np.concatenate([r1[k], r2[k]]) for k in KEYS}, base)
        _same(dev.inefficiency_series(ser, st, fast=True, mintime=3), base)


def test_errors():
    from pymbar_b200 import DeviceAcf, _lib

    A, _ = _series([600, 900])
    with DeviceAcf(np.concatenate(A), lengths=[600, 900]) as dev:
        for ser, st in (([], []), ([2], [0]), ([-1], [0]), ([0], [600]), ([1], [-1]), ([0, 1], [0, 900])):
            with pytest.raises(_lib.MbarB200Error) as e:
                dev.inefficiency_series(np.array(ser, np.int32), np.array(st, np.int64))
            assert e.value.status == -1
        r = dev.inefficiency_series([1, 0, 1], [898, 598, 899])  # the object is still usable
        assert r["status"].tolist() == [0, 0, 1]                   # one sample left: sigma^2 = 0
    with DeviceAcf(A[0]) as dev:
        with pytest.raises(_lib.MbarB200Error) as e:
            dev.inefficiency_series([0], [0])
        assert e.value.status == -1
    with DeviceAcf(np.concatenate(A), lengths=[600, 900]) as dev:  # and the existing rule-0 refusal stays
        with pytest.raises(_lib.MbarB200Error):
            dev.inefficiency([0])


def _check_golden_eq(out, z, key, skip=()):
    want, err = z["eq__" + key], z["eqerr__" + key]
    assert not err.any()
    for i, (t, g, Neff) in enumerate(out):
        if i in skip:
            continue
        assert type(t) in (np.int64, int) and t == int(want[i, 0]), (key, i, t, want[i])
        assert np.float32(g) == np.float32(want[i, 1]) and np.float32(Neff) == np.float32(want[i, 2]), (key, i)


def _si_tol(a, b, fast, mintime):
    res = tsr.ld_walk(a, b, 0, fast, mintime)
    return 2 * tsr.g_bound(res) + 1e-15


def test_many_functions_match_golden_and_the_single_loop(golden, monkeypatch):
    from pymbar_b200 import timeseries as ts
    from pymbar_b200 import utils as u

    names, A, B = cases.series()
    assert list(golden["names"]) == names and str(golden["digest"]) == cases.digest(A, B)
    for fast, nskip in cases.EQ_CASES:
        out = ts.detect_equilibration_many(A, fast=fast, nskip=nskip)
        assert ts.LAST_MANY_STATS["waves"] == 1
        loop = [ts.detect_equilibration(a, fast=fast, nskip=nskip) for a in A]
        assert [tuple(map(type, x)) for x in out] == [tuple(map(type, x)) for x in loop]
        assert out == loop
        _check_golden_eq(out, golden, f"{int(fast)}__{nskip}")
        monkeypatch.setattr(ts, "WAVE_BYTES", 997 * ts.REQUEST_BYTES)
        assert ts.detect_equilibration_many(A, fast=fast, nskip=nskip) == out
        assert ts.LAST_MANY_STATS["waves"] > 10
        monkeypatch.undo()
    few = ts.detect_equilibration_many(A[:9], fast=True, nskip=7)
    monkeypatch.setattr(ts, "WAVE_BYTES", 3 * ts.REQUEST_BYTES)           # three requests per wave
    assert ts.detect_equilibration_many(A[:9], fast=True, nskip=7) == few
    assert ts.LAST_MANY_STATS["waves"] > 100
    monkeypatch.undo()
    ok = [i for i, a in enumerate(A) if np.ptp(a) > 0 and a.size > 1]
    for kind, fast, mintime in cases.SI_CASES:
        Bl = B if kind == "cross" else None
        want = golden[f"si__{kind}__{int(fast)}__{mintime}"]
        got = ts.statistical_inefficiency_many([A[i] for i in ok], None if Bl is None else [Bl[i] for i in ok],
                                               fast=fast, mintime=mintime)
        loop = [ts.statistical_inefficiency(A[i], None if Bl is None else Bl[i], fast, mintime) for i in ok]
        assert got.dtype == np.float64 and np.array_equal(got, np.array(loop))
        for j, i in enumerate(ok):
            tol = _si_tol(A[i], None if Bl is None else Bl[i], fast, mintime)
            assert abs(got[j] - want[i]) <= tol, (names[i], kind, fast, mintime, got[j], want[i])
        with pytest.raises(u.ParameterError):             # the entirely constant series
            ts.statistical_inefficiency_many(A, Bl, fast=fast, mintime=mintime)
    for conservative, g in cases.SUB_CASES:
        key = f"{int(conservative)}__{g}"
        flat, n = golden["sub__" + key], golden["subn__" + key]
        off = np.concatenate([[0], np.cumsum(n)])
        gl = [1.5 + 0.25 * i for i in range(len(A))] if g == "per-series" else g
        idx = ok if g is None else range(len(A))
        got = ts.subsample_correlated_data_many([A[i] for i in idx], g=gl if g != "per-series" else
                                                [gl[i] for i in idx], conservative=conservative)
        for j, i in enumerate(idx):
            assert got[j] == flat[off[i]:off[i + 1]].tolist(), (names[i], key)


def test_campaign_sized_call():
    """512 series of T = 4000 with a decaying transient, nskip = 1: 2 047 488 requests in one call."""
    from pymbar_b200 import timeseries as ts

    A = [ar1(1000 + k, 4000, 4.0 + (k % 7)) + 4.0 * np.exp(-np.arange(4000) / (100.0 + k)) for k in range(512)]
    out = ts.detect_equilibration_many(A, fast=True, nskip=1)
    st = dict(ts.LAST_MANY_STATS)
    assert st["waves"] == 1 and st["requests"] == 512 * 3999 and st["rounds"] >= 3
    print("campaign stats:", st)
    assert out == [ts.detect_equilibration(a, fast=True, nskip=1) for a in A]

"""mbar_b200_acf on the H100: per start, sigma^2, C at every evaluated lag, g and the stop lag against the long-double
loop within the bound (tests/_timeseries.py), the same bits as the device-order numpy restatement, bit-identity
across calls, starts and batches, every error, the facade against the fixtures, and a full-size detect_equilibration."""
import numpy as np
import pytest

from tests import _timeseries as tsr
from tests import _timeseries_cases as cases

pytestmark = pytest.mark.gpu


def ar1(seed, T, tau):
    rng = np.random.RandomState(seed)
    a = np.exp(-1.0 / tau)
    e = rng.standard_normal(T) * np.sqrt(1 - a * a)
    from scipy.signal import lfilter

    return lfilter([1.0], [1.0, -a], e)


def _check_against_ld(A, B, starts, fast, mintime, r, trace_cap):
    for j, s in enumerate(starts):
        res = tsr.ld_walk(A, B, int(s), fast, mintime)
        if res["sigma2"] == 0:
            assert r["status"][j] == 1
            continue
        n = len(res["C"])
        assert r["status"][j] == 0 and r["last_lag"][j] == res["last_lag"], (s, r["last_lag"][j], res["last_lag"])
        Cb = np.array([float(b) for b in res["C_bound"]])
        m = min(n, trace_cap)
        assert np.all(np.abs(r["trace"][j, :m] - np.array(res["C"][:m], dtype=np.float64)) <= Cb[:m]), s
        assert abs(r["g"][j] - float(res["g"])) <= tsr.g_bound(res), s
        assert abs(r["sigma2"][j] - float(res["sigma2"])) <= float(res["sigma2_bound"])


@pytest.mark.parametrize("T", [2, 3, 4, 511, 512, 513, 1025, 70001])
def test_small_to_medium_series_match_device_order_and_long_double(T):
    from pymbar_b200 import DeviceAcf

    A = ar1(T, T, 6.0) + 3.0 * np.exp(-np.arange(T) / 50.0)
    B = 0.5 * A + ar1(T + 1, T, 2.0)
    NC = tsr.chunk_size(T)
    starts = sorted({s for s in (0, 1, NC - 1, NC, NC + 1, T // 2, T - 3, T - 2, T - 1) if 0 <= s < T})
    for b in (None, B):
        for fast, mintime in ((False, 3), (True, 0), (False, 20), (True, 3)):
            with DeviceAcf(A, b) as dev:
                r = dev.inefficiency(starts, fast=fast, mintime=mintime, trace_cap=256)
            if T <= 1025:
                want = tsr.NumpyAcf(A, b).inefficiency(starts, fast=fast, mintime=mintime, trace_cap=256)
                for k in ("mean_a", "mean_b", "sigma2", "g", "last_lag", "status"):
                    assert np.array_equal(r[k], want[k]), (k, T, fast)
                assert np.array_equal(r["trace"], want["trace"], equal_nan=True)
            _check_against_ld(A, b, starts, fast, mintime, r, 256)


def test_long_series_fast_off_and_offset():
    """T = 2e6, one start and many lags (the n range split over chunks), fast off, and a mean of 1e6 with sigma 1."""
    from pymbar_b200 import DeviceAcf

    T = 2_000_000
    A = 1.0e6 + ar1(5, T, 10.0)
    starts = [0, 2047, 2048, 999_999]
    with DeviceAcf(A) as dev:
        r = dev.inefficiency(starts, fast=False, mintime=3, trace_cap=512)
        st = dev.last_stats()
    _check_against_ld(A, None, starts, False, 3, r, 512)
    assert st["rounds"] <= 12 and st["waste"] <= 2.0, st


def test_segments_match_device_order_and_long_double():
    from pymbar_b200 import DeviceAcf

    L = np.array([300, 700, 1100, 500, 3])
    A = ar1(9, int(L.sum()), 5.0)
    navg = np.mean(L.astype(np.float64))
    for fast in (False, True):
        with DeviceAcf(A, lengths=L) as dev:
            r = dev.inefficiency([0], fast=fast, multiple=True, navg=navg, trace_cap=1200)
        want = tsr.NumpyAcf(A, lengths=L).inefficiency([0], fast=fast, multiple=True, navg=navg, trace_cap=1200)
        for k in ("g", "last_lag", "sigma2"):
            assert np.array_equal(r[k], want[k]), k
        res = tsr.ld_walk(A, None, 0, fast, 10, lengths=L, navg=navg)
        assert r["last_lag"][0] == res["last_lag"] and abs(r["g"][0] - float(res["g"])) <= tsr.g_bound(res)


def test_bit_identity_alone_among_all_and_shuffled():
    from pymbar_b200 import DeviceAcf

    T = 9000
    A = ar1(11, T, 12.0) + 20.0 * np.exp(-np.arange(T) / 300.0)
    every = np.arange(0, T - 1)
    with DeviceAcf(A) as dev:
        full = dev.inefficiency(every, fast=True)
        again = dev.inefficiency(every, fast=True)
        rng = np.random.RandomState(0)
        sub = rng.choice(every, size=300, replace=False)
        part = dev.inefficiency(sub, fast=True)
        alone = [dev.inefficiency([s], fast=True) for s in sub[:20]]
    for k in ("g", "sigma2", "mean_a", "last_lag"):
        assert np.array_equal(full[k], again[k])
        assert np.array_equal(full[k][sub], part[k])
        assert all(np.array_equal(full[k][[s]], a[k]) for s, a in zip(sub[:20], alone))


def test_errors_leave_the_object_usable():
    from pymbar_b200 import DeviceAcf, _lib

    x = ar1(2, 1000, 4.0)
    bad = x.copy()
    bad[5] = np.inf
    with pytest.raises(_lib.MbarB200Error) as e:
        DeviceAcf(bad)
    assert e.value.status == -5
    with pytest.raises(_lib.MbarB200Error) as e:
        DeviceAcf(x, np.where(np.arange(1000) == 3, np.nan, x))
    assert e.value.status == -5
    for lengths in ([500, 400], [0, 1000], [1200, -200]):
        with pytest.raises(_lib.MbarB200Error) as e:
            DeviceAcf(x, lengths=lengths)
        assert e.value.status == -1
    with pytest.raises(_lib.MbarB200Error):
        DeviceAcf(np.zeros(0))
    with DeviceAcf(x) as dev:
        good = dev.inefficiency([0, 10])
        for kwargs in (dict(starts=[1000]), dict(starts=[-1]), dict(starts=[0], multiple=True, navg=10.0)):
            with pytest.raises(_lib.MbarB200Error) as e:
                dev.inefficiency(**kwargs)
            assert e.value.status == -1
            assert np.array_equal(dev.inefficiency([0, 10])["g"], good["g"])
        for n_max in (-1, 1000):
            with pytest.raises(_lib.MbarB200Error):
                dev.correlation(0, n_max)
        C, *_ = dev.correlation(0, 30)
        assert C.shape == (31,)
    with DeviceAcf(np.full(100, 3.0)) as dev:
        r = dev.inefficiency([0, 50])
        assert list(r["status"]) == [1, 1] and list(r["g"]) == [1.0, 1.0]
        with pytest.raises(_lib.MbarB200Error):
            dev.correlation(0, 5)


def test_facade_on_device_reproduces_fixtures():
    import os
    import types

    from pymbar_b200 import facade

    z = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", "timeseries.npz")))
    mod = types.ModuleType("fake_timeseries")
    for name in ("statistical_inefficiency", "statistical_inefficiency_multiple",
                 "normalized_fluctuation_correlation_function", "detect_equilibration"):
        setattr(mod, name, lambda *a, **k: (_ for _ in ()).throw(AssertionError("original called")))
    facade.install_timeseries_on(mod)
    try:
        for name, fast, mintime in cases.SI_CASES:
            A = z["series__" + name]
            B = z.get("series__" + name + "_b")
            g = mod.statistical_inefficiency(A, B, fast=fast, mintime=mintime)
            res = tsr.ld_walk(A, B, 0, fast, mintime)
            assert abs(g - float(z[f"si__{name}__{int(fast)}__{mintime}"])) <= 2 * tsr.g_bound(res) + 1e-15
        for name, fast, nskip in cases.EQ_CASES:
            t, g, Neff = mod.detect_equilibration(z["series__" + name], fast=fast, nskip=nskip)
            want = z[f"eq__{name}__{int(fast)}__{nskip}"]
            assert t == int(want[0]) and g == np.float32(want[1]) and Neff == np.float32(want[2]), name
        A = z["series__multi"]
        L = cases.MULTI_LENGTHS
        A_kn = [A[o:o + n] for o, n in zip(np.cumsum([0] + L[:-1]), L)]
        for fast in (False, True):
            g, Ct = mod.statistical_inefficiency_multiple(A_kn, fast=fast, return_correlation_function=True)
            want = z[f"multiCt__{int(fast)}"]
            assert [t for t, _ in Ct] == [int(t) for t in want[:, 0]]
            assert abs(g - float(z[f"multi__{int(fast)}"])) < 1e-9 * g
        for name, n_max, norm in cases.CORR_CASES:
            C = mod.normalized_fluctuation_correlation_function(z["series__" + name], z.get("series__" + name + "_b"),
                                                                N_max=n_max, norm=norm)
            want = z[f"corr__{name}__{n_max}__{int(norm)}"]
            np.testing.assert_allclose(C, want, rtol=0, atol=1e-9 * np.max(np.abs(want)))
    finally:
        facade.uninstall_from(mod)


def test_full_size_detect_equilibration():
    """T = 1e6, nskip = 1, fast: every start in one call; 32 starts against long double, O(log L) rounds and at most
    twice the lag terms the stop rule needed."""
    from pymbar_b200 import DeviceAcf
    from pymbar_b200 import timeseries as ts

    T = 1_000_000
    A = ar1(21, T, 20.0) + 10.0 * np.exp(-np.arange(T) / 200.0)
    starts = np.arange(0, T - 1)
    with DeviceAcf(A) as dev:
        r = dev.inefficiency(starts, fast=True, mintime=3)
        st = dev.last_stats()
    assert st["rounds"] <= 8 and st["waste"] <= 2.0, st
    pick = np.unique(np.concatenate([[0, 1, 1023, 1024, 4095, 4096, T - 3, T - 2],
                                     np.random.RandomState(4).choice(T - 1, 24, replace=False)]))
    with DeviceAcf(A) as dev:
        rp = dev.inefficiency(pick, fast=True, mintime=3, trace_cap=64)
    for k in ("g", "last_lag", "sigma2"):
        assert np.array_equal(rp[k], r[k][pick])
    _check_against_ld(A, None, pick, True, 3, rp, 64)
    t, g, Neff = ts.detect_equilibration(A, fast=True, nskip=1)
    g_t = np.where(r["g"] < 1.0, 1.0, r["g"]).astype(np.float32)
    Neff_t = ts.neff(T - starts + 1, g_t)
    assert t == Neff_t.argmax() and g == g_t[t] and Neff == Neff_t.max()

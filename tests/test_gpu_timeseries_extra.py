"""mbar_b200_acf_correlation_multiple and the FFT rule of mbar_b200_acf_inefficiency on the H100: the same bits as
the device-order numpy restatement (tests/_timeseries_extra.py) across chunk and series boundaries, bit-identity
across calls, the truncate rounds, every error, the facade against tests/golden/timeseries_extra.npz, and a
10 x 1e5 correlation function."""
import numpy as np
import pytest

from tests import _timeseries_extra as tsx
from tests import _timeseries_extra_cases as cases

pytestmark = pytest.mark.gpu


def ar1(seed, T, tau):
    from scipy.signal import lfilter

    rng = np.random.RandomState(seed)
    a = np.exp(-1.0 / tau)
    return lfilter([1.0], [1.0, -a], rng.standard_normal(T) * np.sqrt(1 - a * a))


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


@pytest.mark.parametrize("lengths", [[511, 512, 513], [1, 1025, 3, 40], [2000, 600, 1], [1300]])
def test_correlation_multiple_matches_device_order(lengths):
    from pymbar_b200 import DeviceAcf

    N = sum(lengths)
    A = ar1(N, N, 6.0) + 2.0
    B = 0.5 * A + ar1(N + 1, N, 2.0)
    Lmax = max(lengths)
    for b in (None, B):
        want_dev = tsx.NumpyAcfExtra(A, b, lengths=lengths)
        for n_max in sorted({0, 1, 7, 8, 9, min(lengths) + 2, 600, Lmax - 1} & set(range(Lmax))):
            for truncate in (False, True):
                with DeviceAcf(A, b, lengths=lengths) as dev:
                    got = dev.correlation_multiple(n_max, truncate)
                want = want_dev.correlation_multiple(n_max, truncate)
                assert got[0].shape == want[0].shape, (lengths, n_max, truncate)
                assert all(_same(x, y) for x, y in zip(got, want)), (lengths, n_max, truncate)
                if got[0].size:
                    assert got[0][0] == 1.0


def test_correlation_multiple_long_series_chunks():
    """a series longer than 512 * 1024 samples (chunks of more than 512) next to short ones"""
    from pymbar_b200 import DeviceAcf

    lengths = [700_001, 5, 1024]
    N = sum(lengths)
    A = 1.0e3 + ar1(3, N, 20.0)
    with DeviceAcf(A, lengths=lengths) as dev:
        got = dev.correlation_multiple(12, False)
    want = tsx.NumpyAcfExtra(A, lengths=lengths).correlation_multiple(12, False)
    assert all(_same(x, y) for x, y in zip(got, want))


@pytest.mark.parametrize("T", [2, 3, 4, 511, 512, 513, 1025, 4000])
def test_fft_rule_matches_device_order_and_long_double(T):
    from pymbar_b200 import DeviceAcf

    A = ar1(T, T, 6.0) + 3.0 * np.exp(-np.arange(T) / 50.0)
    NC = tsx.chunk_size(T)
    starts = sorted({s for s in (0, 1, NC - 1, NC, NC + 1, T // 2, T - 3, T - 2, T - 1) if 0 <= s < T})
    for mintime in (0, 3, 20):
        with DeviceAcf(A) as dev:
            r = dev.inefficiency(starts, mintime=mintime, rule="fft", trace_cap=256)
        want = tsx.NumpyAcfExtra(A).inefficiency(starts, mintime=mintime, rule="fft", trace_cap=256)
        for k in ("mean_a", "mean_b", "sigma2", "g", "last_lag", "status", "trace"):
            assert _same(r[k], want[k]), (k, T, mintime)
        for j, s in enumerate(starts):
            if T - s < 2:
                continue
            res = tsx.ld_walk_fft(A, int(s), mintime)
            assert r["last_lag"][j] == res["last_lag"] and abs(r["g"][j] - float(res["g"])) <= res["g_bound"]


def test_repeat_calls_are_bit_identical_and_rounds_are_counted():
    from pymbar_b200 import DeviceAcf

    s = cases.series()
    A_kn, _ = cases.multi(s, "auto")
    L = [x.size for x in A_kn]
    A = np.concatenate(A_kn)
    with DeviceAcf(A, lengths=L) as dev:
        first = dev.correlation_multiple(max(L) - 1, True)
        st = dev.last_stats()
        again = dev.correlation_multiple(max(L) - 1, True)
        full = dev.correlation_multiple(max(L) - 1, False)
        st_full = dev.last_stats()
    assert all(_same(x, y) for x, y in zip(first, again))
    n = first[0].size                                          # the stop lag
    assert _same(first[0], full[0][:n])
    rounds, cum, B = 0, 0, 8
    while cum <= n:                                            # rounds of 8, 8, 16, 32, ... lags until the stop lag
        cum += B
        rounds += 1
        if rounds > 1:
            B *= 2
    assert st["rounds"] == rounds and st_full["rounds"] == 0, (st, n)
    assert st["terms"] <= 2 * st["useful_terms"] + 8 * sum(L) and st_full["terms"] == st_full["useful_terms"]
    x = s["drift"]
    with DeviceAcf(x) as dev:
        r1 = dev.inefficiency([0, 1, 100], rule="fft")
        st = dev.last_stats()
        r2 = dev.inefficiency([0, 1, 100], rule="fft")
    assert all(_same(r1[k], r2[k]) for k in r1)
    assert st["rounds"] <= 7 and st["waste"] <= 2.0, st


def test_errors_leave_the_object_usable():
    from pymbar_b200 import DeviceAcf, _lib

    x = ar1(2, 1000, 4.0)
    with DeviceAcf(x) as dev:
        with pytest.raises(_lib.MbarB200Error) as e:
            dev.correlation_multiple(5)
        assert e.value.status == -1
        with pytest.raises(_lib.MbarB200Error):
            dev.inefficiency([0], fast=True, rule="fft")
        for kwargs in (dict(rule="fft", multiple=True), dict(rule="direct")):
            with pytest.raises(ValueError):
                dev.inefficiency([0], **kwargs)
        g = dev.inefficiency([0, 5], rule="fft")["g"]
        assert np.array_equal(dev.inefficiency([0, 5], rule="fft")["g"], g)
    with DeviceAcf(x, x[::-1].copy()) as dev:
        with pytest.raises(_lib.MbarB200Error):
            dev.inefficiency([0], rule="fft")
    with DeviceAcf(x, lengths=[400, 600]) as dev:
        for n_max in (-1, 600):
            with pytest.raises(_lib.MbarB200Error):
                dev.correlation_multiple(n_max)
        with pytest.raises(_lib.MbarB200Error):
            dev.inefficiency([0], rule="fft")
        C, *_ = dev.correlation_multiple(599)
        assert C.shape == (599,) and C[0] == 1.0
    with DeviceAcf(np.full(100, 3.0), lengths=[30, 70]) as dev:
        with pytest.raises(_lib.MbarB200Error):
            dev.correlation_multiple(5)


def test_facade_on_device_reproduces_fixtures():
    import os
    import types

    from pymbar_b200 import facade

    z = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", "timeseries_extra.npz")))
    s = cases.series()
    mod = types.ModuleType("fake_timeseries")
    for name in ("normalized_fluctuation_correlation_function_multiple", "statistical_inefficiency_fft",
                 "detect_equilibration_binary_search"):
        setattr(mod, name, lambda *a, **k: (_ for _ in ()).throw(AssertionError("original called")))
    facade.install_timeseries_on(mod)
    try:
        ld = {name: tsx.ld_corr_multiple(*cases.multi(s, name)) for name in cases.MULTI_SETS}
        for name, n_max, norm, trunc in cases.CORRM_CASES:
            A_kn, B_kn = cases.multi(s, name)
            key = cases.case_key(name, n_max, norm, trunc)
            want = z["cm__" + key]
            C = mod.normalized_fluctuation_correlation_function_multiple(A_kn, B_kn, N_max=cases.n_max_of(name, n_max),
                                                                         norm=norm, truncate=trunc)
            assert C.shape == want.shape, key
            bound = np.array([float(b) for b in ld[name]["C_bound"][:C.size]])
            if norm:
                assert C.size == 0 or C[0] == 1.0
                assert np.all(np.abs(C - want) <= 2 * bound), key
            else:
                scale = abs(float(ld[name]["sigma2"])) * (1 + 1e-9)
                extra = 4 * tsx.EPS * (np.abs(want) + abs(float(ld[name]["mean_a"] * ld[name]["mean_b"])))
                assert np.all(np.abs(C - want) <= 2 * bound * scale + extra), key
        for name, mintime in cases.FFT_CASES:
            key = f"{name}__{mintime}"
            g = mod.statistical_inefficiency_fft(s[name], mintime=mintime)
            res = tsx.ld_walk_fft(s[name], 0, mintime)
            assert abs(g - float(z["fft__" + key])) <= 2 * res["g_bound"], key
        for name, nodes in cases.BS_CASES:
            key = f"{name}__{nodes}"
            t, g, Neff = mod.detect_equilibration_binary_search(s[name], bs_nodes=nodes)
            want = z["bs__" + key]
            gb = tsx.ld_walk_fft(s[name], int(t), 3)["g_bound"]
            assert t == int(want[0]) and abs(g - want[1]) <= 2 * gb, key
            assert abs(Neff - want[2]) <= 2 * gb / want[1] * want[2] * 1.01, key
    finally:
        facade.uninstall_from(mod)


def test_ten_series_of_1e5():
    """10 x 1e5 samples, every lag to 1e5 - 1: C(0) == 1.0 and C at sampled lags, the means and sigma^2 are the
    device-order restatement's bits."""
    from pymbar_b200 import DeviceAcf

    L = [100_000] * 10
    A_kn = [ar1(40 + k, n, 10.0) for k, n in enumerate(L)]
    A = np.concatenate(A_kn)
    with DeviceAcf(A, lengths=L) as dev:
        C, mua, mub, s2 = dev.correlation_multiple(L[0] - 1)
    assert C.shape == (L[0] - 1,) and C[0] == 1.0
    ref = tsx.NumpyAcfExtra(A, lengths=L)
    assert (mua, mub, s2) == ref.multi_moments()
    for t in np.unique(np.concatenate([[0, 1, 2, 511, 512, 513, 1023, L[0] - 2],
                                       np.random.RandomState(5).randint(0, L[0] - 1, 16)])):
        num, den, _ = ref.multi_numerator(int(t), mua, mub)
        assert C[t] == num / den / s2, t


def test_long_series_at_large_lags_match_device_order():
    """a series of 600000 samples (chunks of 586) at lags up to 1e5, where the window L - t alone would give chunks
    of 512: C, the means and sigma^2 at sampled lags are the restatement's bits"""
    from pymbar_b200 import DeviceAcf

    L = [600_000, 1000]
    A = ar1(12, sum(L), 30.0)
    n_max = 100_100
    with DeviceAcf(A, lengths=L) as dev:
        C, mua, mub, s2 = dev.correlation_multiple(n_max)
    assert C.shape == (n_max,) and C[0] == 1.0
    ref = tsx.NumpyAcfExtra(A, lengths=L)
    assert (mua, mub, s2) == ref.multi_moments()
    for t in (1, 513, 999, 1000, 50_000, 99_999, 100_000, n_max - 1):
        num, den, _ = ref.multi_numerator(t, mua, mub)
        assert C[t] == num / den / s2, t

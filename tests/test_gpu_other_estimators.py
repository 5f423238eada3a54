"""mbar_b200_work on the H100: every request kind against long double within the bound (tests/_other_estimators.py)
from 1 value to 1e7 and at the chunk edges, bit-identity across calls and request sets, every error with the object
usable after it, the facade against the reference's fixtures, bar_many against single-pair calls, and a full-size
pair."""
import json
import os
import sys
import types

import numpy as np
import pytest

from tests import _other_estimators as oer

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "other_estimators.npz")
KINDS = ((oer.FERMI, 0.4, -1.3), (oer.FERMI, -3.0, 2.0), (oer.FERMI_MOMENTS, -0.7, 0.0), (oer.FERMI_MOMENTS, 2.5, 0.0),
         (oer.EXP, 0.0, 0.0), (oer.GAUSS, 0.0, 0.0))


def _work(n, seed):
    return np.random.RandomState(seed).normal(1.0, 2.0, n)


@pytest.mark.parametrize("n", [1, 2, 4095, 4096, 4097, 8192, 8193, 4096 * 2048, 4096 * 2048 + 1, 10_000_000])
def test_every_kind_within_the_long_double_bound(n):
    from pymbar_b200 import DeviceWork

    w = _work(n, n % 1000)
    with DeviceWork([w]) as dev:
        out = dev.evaluate([0] * len(KINDS), [k for k, _, _ in KINDS], [a for _, a, _ in KINDS],
                           [b for _, _, b in KINDS])
        st = dev.last_stats()
    assert st["launches"] == 4 and st["values_read"] == 2 * n * len(KINDS)
    for (kind, c1, c2), got in zip(KINDS, out):
        want, b = oer.ld_request(w, kind, c1, c2, A=got[2] if kind == oer.FERMI_MOMENTS else None)
        if kind == oer.FERMI_MOMENTS:
            assert got[2] == np.max(w + c1)                      # max(w + c) = fl(max w + c)
        for j in range(3):
            err = abs(float(np.longdouble(got[j]) - want[j]))
            assert err <= b[j], (n, kind, j, err, b[j])


def test_bit_identity_across_calls_and_request_sets():
    from pymbar_b200 import DeviceWork

    vs = [_work(n, s) for s, n in enumerate((1, 300, 4097, 50_000, 1_000_003))]
    reqs = [(v, k, c1 + 0.1 * v, c2) for v in range(len(vs)) for k, c1, c2 in KINDS]
    with DeviceWork(vs) as dev:
        cols = list(zip(*reqs))
        full = dev.evaluate(*cols)
        again = dev.evaluate(*cols)
        assert np.array_equal(full, again, equal_nan=True)
        rng = np.random.RandomState(1)
        sub = rng.permutation(len(reqs))[:11]
        part = dev.evaluate(*zip(*[reqs[i] for i in sub]))
        assert np.array_equal(part, full[sub], equal_nan=True)
        for i in sub[:5]:
            assert np.array_equal(dev.evaluate(*zip(reqs[i])), full[i:i + 1], equal_nan=True)
    # the same vector in another object, at another offset
    with DeviceWork([_work(77, 9), vs[3]]) as dev:
        r = [x for x in reqs if x[0] == 3]
        got = dev.evaluate([1] * len(r), *list(zip(*r))[1:])
    assert np.array_equal(got, full[[i for i, x in enumerate(reqs) if x[0] == 3]], equal_nan=True)


def test_overflow_follows_the_reference():
    """Where the reference's formulas overflow the device gives the same inf or NaN as numpy."""
    from pymbar_b200 import DeviceWork

    w = np.concatenate([_work(100, 3), [800.0]])
    with DeviceWork([w, _work(50, 4) - 2000.0]) as dev:
        out = dev.evaluate([0, 1, 0, 1], [1, 1, 0, 2], [0.0, 1200.0, -1000.0, 0.0], [0.0, 0.0, 0.0, 0.0])
    ws = [w, _work(50, 4) - 2000.0]
    want = np.array([oer.request(ws[v], k, a, 0.0) for v, k, a in ((0, 1, 0.0), (1, 1, 1200.0), (0, 0, -1000.0),
                                                                   (1, 2, 0.0))])
    assert np.array_equal(np.isnan(out), np.isnan(want)) and np.array_equal(np.isinf(out), np.isinf(want))
    assert np.array_equal(out[np.isinf(out)], want[np.isinf(want)])
    assert not np.all(np.isfinite(want[:2]))


def test_errors_leave_the_object_usable():
    from pymbar_b200 import DeviceWork, _lib

    w = _work(1000, 2)
    for bad in (np.inf, -np.inf, np.nan):
        x = w.copy()
        x[17] = bad
        with pytest.raises(_lib.MbarB200Error) as e:
            DeviceWork([w, x])
        assert e.value.status == -5
    for vs in ([w, w[:0]], [w[:0]]):
        with pytest.raises(_lib.MbarB200Error) as e:
            DeviceWork(vs)
        assert e.value.status == -1
    with DeviceWork([w, w[:10]]) as dev:
        good = dev.evaluate([0, 1], [0, 3], [0.5, 0.0], [0.1, 0.0])
        for args in (([2], [0], [0.0], [0.0]), ([-1], [0], [0.0], [0.0]), ([0], [4], [0.0], [0.0]),
                     ([0, 1], [0, -1], [0.0, 0.0], [0.0, 0.0]), ([0], ["softplus"], [0.0], [0.0])):
            with pytest.raises(_lib.MbarB200Error) as e:
                dev.evaluate(*args)
            assert e.value.status == -1
            assert np.array_equal(dev.evaluate([0, 1], [0, 3], [0.5, 0.0], [0.1, 0.0]), good)


class _Errors:
    class ParameterError(Exception):
        pass

    class ConvergenceError(Exception):
        pass

    class BoundsError(Exception):
        pass


def _close(got, want, rel):
    if np.isnan(want) or np.isinf(want):
        return (np.isnan(want) and np.isnan(got)) or got == want
    return abs(got - want) <= rel * max(1.0, abs(want))


def test_facade_on_device_reproduces_fixtures(monkeypatch):
    from pymbar_b200 import facade
    from pymbar_b200 import timeseries as dts

    z = np.load(GOLDEN)
    vec = {k: z[k] for k in z.files if k.startswith("w__")}
    cases = json.loads(str(z["cases"]))
    mod = types.ModuleType("fake_other_estimators")
    for name in ("bar", "bar_zero", "exp", "exp_gauss"):
        setattr(mod, name, lambda *a, **k: (_ for _ in ()).throw(AssertionError("original called")))
    for cls in ("ParameterError", "ConvergenceError", "BoundsError"):
        setattr(mod, cls, getattr(_Errors, cls))
    # is_timeseries reaches pymbar.timeseries.statistical_inefficiency: here the device's
    ts = types.ModuleType("pymbar.timeseries")
    ts.statistical_inefficiency = lambda A, B=None, fast=False, mintime=3, fft=False: dts.statistical_inefficiency(
        A, B, fast=fast, mintime=mintime)
    pkg = types.ModuleType("pymbar")
    pkg.timeseries = ts
    monkeypatch.setitem(sys.modules, "pymbar", pkg)
    monkeypatch.setitem(sys.modules, "pymbar.timeseries", ts)
    facade.install_other_estimators_on(mod)
    try:
        checked = 0
        for case in cases:
            if case["fn"] == "bar_overlap":
                continue
            args = [vec["w__" + a] for a in case["args"]]
            fn = getattr(mod, case["fn"])
            if "error" in case:
                with pytest.raises(Exception) as e:
                    fn(*args, **case["kwargs"])
                assert type(e.value) is getattr(_Errors, case["error"][0]), case["id"]
                assert str(e.value).split(" max_delta")[0] == case["error"][1].split(" max_delta")[0]
            elif "value" in case:
                got = fn(*args, **case["kwargs"])
                assert _close(got, float(case["value"][0]), 1e-10), (case["id"], got)
            else:
                got = fn(*args, **case["kwargs"])
                assert sorted(got) == sorted(case["result"]), case["id"]
                for k, (text, tname) in case["result"].items():
                    assert type(got[k]).__name__ == tname, (case["id"], k)
                    assert _close(got[k], float(text), 1e-10 if k == "Delta_f" else 1e-9), (case["id"], k, got[k],
                                                                                           text)
            checked += 1
        assert checked == len(cases) - 1
    finally:
        facade.uninstall_from(mod)


def test_bar_many_200_pairs_bit_identical_to_single_pair_calls():
    from pymbar_b200 import other_estimators as oe

    rng = np.random.RandomState(5)
    wF = [rng.normal(1.0 + 0.01 * p, 1.0, 200 + 37 * p) for p in range(200)]
    wR = [rng.normal(-1.0 - 0.01 * p, 1.0, 150 + 53 * p) for p in range(200)]
    n0 = oe.EVALUATIONS[0]
    many = oe.bar_many(wF, wR)
    batch_calls = oe.EVALUATIONS[0] - n0
    singles = []
    for p in range(200):
        n0 = oe.EVALUATIONS[0]
        one = oe.bar(wF[p], wR[p])
        singles.append(oe.EVALUATIONS[0] - n0)
        for k in one:
            assert np.float64(one[k]).tobytes() == np.float64(many[p][k]).tobytes(), (p, k)
    assert batch_calls == max(singles)


def test_full_size_pair():
    """1e7 values per side: the device driver against the reference's arithmetic in numpy (NumpyWork)."""
    from pymbar_b200 import other_estimators as oe

    rng = np.random.RandomState(8)
    n = 10_000_000
    w_F = rng.normal(2.0, 1.5, n)
    w_R = rng.normal(-0.5, 1.5, n)
    got = oe.bar(w_F, w_R)
    saved = oe.DeviceWork
    try:
        oe.DeviceWork = oer.NumpyWork
        want = oe.bar(w_F, w_R)
    finally:
        oe.DeviceWork = saved
    assert _close(got["Delta_f"], want["Delta_f"], 1e-10) and _close(got["dDelta_f"], want["dDelta_f"], 1e-9), (got,
                                                                                                                 want)

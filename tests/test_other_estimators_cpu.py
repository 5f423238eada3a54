"""pymbar_b200.other_estimators and its facade on the CPU, over the numpy stand-in of DeviceWork
(tests/_other_estimators.py), against tests/golden/other_estimators.npz from the unmodified reference
(tools/make_other_estimators_golden.py)."""
import json
import os
import sys
import types

import numpy as np
import pytest

from tests import _other_estimators as oer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "other_estimators.npz")
NAMES = ("bar", "bar_zero", "exp", "exp_gauss")


@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLDEN)
    return {k: z[k] for k in z.files if k.startswith("w__")}, json.loads(str(z["cases"]))


class _Errors:
    class ParameterError(Exception):
        pass

    class ConvergenceError(Exception):
        pass

    class BoundsError(Exception):
        pass


def _fake_timeseries(monkeypatch, g_values):
    """pymbar.timeseries whose statistical_inefficiency hands back the reference's recorded g."""
    ts = types.ModuleType("pymbar.timeseries")
    ts.calls = []

    def statistical_inefficiency(A, B=None, *args, **kwargs):
        ts.calls.append((A, B))
        return g_values.pop(0)

    ts.statistical_inefficiency = statistical_inefficiency
    pkg = types.ModuleType("pymbar")
    pkg.timeseries = ts
    monkeypatch.setitem(sys.modules, "pymbar", pkg)
    monkeypatch.setitem(sys.modules, "pymbar.timeseries", ts)
    return ts


@pytest.fixture()
def stand_in(monkeypatch):
    """pymbar_b200.other_estimators over NumpyWork, and the facade installed on a module whose originals record calls
    and which carries its own exception classes."""
    from pymbar_b200 import facade
    from pymbar_b200 import other_estimators as oe

    monkeypatch.setattr(oe, "DeviceWork", oer.NumpyWork)
    mod = types.ModuleType("fake_other_estimators")
    mod.calls = []
    for name in NAMES:
        def orig(*args, _name=name, **kwargs):
            mod.calls.append(_name)
            return "original"
        setattr(mod, name, orig)
    for cls in ("ParameterError", "ConvergenceError", "BoundsError"):
        setattr(mod, cls, getattr(_Errors, cls))
    facade.install_other_estimators_on(mod)
    try:
        yield mod
    finally:
        facade.uninstall_from(mod)


def _check_result(got, case):
    want = case["result"]
    assert isinstance(got, dict) and sorted(got) == sorted(want), (case["id"], got)
    for k, (text, tname) in want.items():
        assert type(got[k]).__name__ == tname, (case["id"], k, type(got[k]))
        w = float(text)
        assert (np.isnan(w) and np.isnan(got[k])) or got[k] == w, (case["id"], k, repr(got[k]), text)
        if not np.isnan(w):
            assert np.float64(got[k]).tobytes() == np.float64(w).tobytes(), (case["id"], k)


def test_facade_reproduces_every_fixture_bit_for_bit(golden, stand_in, monkeypatch):
    from pymbar_b200 import facade

    vec, cases = golden
    before = dict(facade.STATS)
    n = {name: 0 for name in NAMES}
    for case in cases:
        if case["fn"] == "bar_overlap":
            continue
        args = [vec["w__" + a] for a in case["args"]]
        fn = getattr(stand_in, case["fn"])
        ts = _fake_timeseries(monkeypatch, [float(case["g"])]) if "g" in case else None
        np.seterr(over="raise")
        if "error" in case:
            with pytest.raises(Exception) as e:
                fn(*args, **case["kwargs"])
            assert type(e.value) is getattr(_Errors, case["error"][0]) and str(e.value) == case["error"][1], case["id"]
        elif "value" in case:
            got = fn(*args, **case["kwargs"])
            assert type(got).__name__ == case["value"][1] and got == float(case["value"][0]), (case["id"], got)
        else:
            _check_result(fn(*args, **case["kwargs"]), case)
        if case["fn"] in ("bar", "bar_zero"):
            assert np.geterr()["over"] == "warn", case["id"]          # bar_zero's side effect
        if ts is not None:
            x, y = ts.calls[0]
            assert x is y or np.array_equal(x, y)
            if case["fn"] == "exp":
                w = args[0]
                assert np.array_equal(x, np.exp(-w - np.max(-w)))
            monkeypatch.delitem(sys.modules, "pymbar")
            monkeypatch.delitem(sys.modules, "pymbar.timeseries")
        n[case["fn"]] += "error" not in case
    np.seterr(over="warn")
    assert stand_in.calls == []
    for name in NAMES:
        assert facade.STATS["oe_" + name] - before["oe_" + name] == n[name], name
    assert facade.STATS["oe_evaluations"] > before["oe_evaluations"]
    assert facade.STATS["oe_fallbacks"] == before["oe_fallbacks"]


def test_bar_overlap_reaches_the_patched_bar(golden, stand_in):
    """bar_overlap stays the reference's: it calls `bar` through its module's globals, which now hold the patched one,
    and asserts MBAR's answer against that bar result (the fixture's bar case on the same pair)."""
    vec, cases = golden
    case = next(c for c in cases if c["id"] == "bar_gauss_false-position_BAR")
    ns = {"bar": stand_in.bar}
    exec("def bar_overlap(w_F, w_R):\n    return bar(w_F, w_R)\n", ns)
    _check_result(ns["bar_overlap"](vec["w__gauss_F"], vec["w__gauss_R"]), case)
    assert any(c["fn"] == "bar_overlap" and "value" in c for c in cases)


def test_bar_many_equals_per_pair_bar(golden, monkeypatch):
    from pymbar_b200 import other_estimators as oe

    monkeypatch.setattr(oe, "DeviceWork", oer.NumpyWork)
    vec, _ = golden
    pairs = ["gauss", "expo", "uneq", "one", "int", "big", "wide"]
    wF = [vec[f"w__{p}_F"] for p in pairs]
    wR = [vec[f"w__{p}_R"] for p in pairs]
    for kwargs in (dict(), dict(method="bisection", uncertainty_method="MBAR"), dict(iterated_solution=False),
                   dict(method="self-consistent-iteration", DeltaF=0.5)):
        many = oe.bar_many(wF, wR, **kwargs)
        for p in range(len(pairs)):
            one = oe.bar(wF[p], wR[p], **kwargs)
            assert sorted(one) == sorted(many[p])
            for k in one:
                assert np.float64(one[k]).tobytes() == np.float64(many[p][k]).tobytes(), (pairs[p], k)
    # the lowest-index failing pair's exception wins; pairs in lockstep share device calls
    far = (vec["w__far_F"], vec["w__far_R"])
    with pytest.raises(oe._u.BoundsError):
        oe.bar_many([wF[0], far[0], wF[1]], [wR[0], far[1], wR[1]], method="bisection")
    with pytest.raises(oe._u.ConvergenceError):
        oe.bar_many([wF[0], wF[1]], [wR[0], wR[1]], maximum_iterations=2)
    calls = []
    orig = oer.NumpyWork.evaluate
    monkeypatch.setattr(oer.NumpyWork, "evaluate", lambda self, *a: calls.append(len(a[0])) or orig(self, *a))
    oe.bar_many(wF, wR)
    single = []
    for p in range(len(pairs)):
        n0 = len(calls)
        oe.bar(wF[p], wR[p])
        single.append(len(calls) - n0)
    assert len(calls) - sum(single) == max(single)      # the batch took as many calls as its slowest pair


def test_numpy_work_within_long_double_bound(golden):
    """The reference's fp64 sums (NumpyWork) against long double: the bound holds, and it stays far below the
    tolerances of the GPU tests."""
    vec, _ = golden
    for name in ("gauss_F", "expo_R", "uneq_R", "int_F", "big_F", "ar1"):
        w = vec["w__" + name].astype(np.float64)
        for kind, c1, c2 in ((oer.FERMI, 0.3, -1.1), (oer.FERMI, -2.0, 4.0), (oer.FERMI_MOMENTS, -1.2, 0.0),
                             (oer.EXP, 0.0, 0.0), (oer.GAUSS, 0.0, 0.0)):
            got = oer.request(w, kind, c1, c2)
            want, b = oer.ld_request(w, kind, c1, c2, A=got[2] if kind == oer.FERMI_MOMENTS else None)
            for j in range(3):
                err = abs(float(np.longdouble(got[j]) - want[j]))
                assert err <= b[j], (name, kind, j, err, b[j])
            scale = np.abs(np.array(want, dtype=np.float64)) + 1.0
            assert np.all(b <= 1e-9 * scale), (name, kind, b)


def test_fallbacks_reach_the_original(golden, stand_in):
    from pymbar_b200 import facade

    vec, _ = golden
    wF, wR = vec["w__gauss_F"], vec["w__gauss_R"]
    f0 = facade.STATS["oe_fallbacks"]
    bad = wF.copy()
    bad[3] = np.nan
    calls = [
        ("bar", lambda: stand_in.bar(list(wF), wR)),                                   # not an ndarray
        ("bar", lambda: stand_in.bar(wF.astype(np.float32), wR)),                      # float32
        ("bar", lambda: stand_in.bar(wF.reshape(20, 10), wR)),                         # 2-D
        ("bar", lambda: stand_in.bar(wF[:0], wR)),                                     # empty
        ("bar", lambda: stand_in.bar(bad, wR)),                                        # non-finite: device error
        ("bar", lambda: stand_in.bar(wF, wR, verbose=True)),
        ("bar", lambda: stand_in.bar(wF, wR, method="newton")),
        ("bar", lambda: stand_in.bar(wF, wR, uncertainty_method="svd")),
        ("bar_zero", lambda: stand_in.bar_zero(wF.astype(np.float32), wR, 0.0)),
        ("bar_zero", lambda: stand_in.bar_zero(wF, np.array([np.inf]), 0.0)),
        ("exp", lambda: stand_in.exp(list(wF))),
        ("exp", lambda: stand_in.exp(np.array([2 ** 60], np.int64))),                 # integers inexact in fp64
        ("exp", lambda: stand_in.exp(np.array([1, 2], np.uint32))),
        ("exp_gauss", lambda: stand_in.exp_gauss(bad)),
    ]
    for name, call in calls:
        assert call() == "original", name
    assert stand_in.calls == [name for name, _ in calls]
    assert facade.STATS["oe_fallbacks"] == f0 + len(calls)
    # an unknown method is fine when iterated_solution=False forces self-consistent iteration, as in the reference
    assert isinstance(stand_in.bar(wF, wR, method="newton", iterated_solution=False), dict)
    assert facade.STATS["oe_fallbacks"] == f0 + len(calls)


def test_reference_value_error_on_unknown_uncertainty_method_is_the_originals():
    """The reference formats the unknown uncertainty_method with {:d} and so raises ValueError; the restated driver
    (called directly, without the facade's fallback) does the same."""
    from pymbar_b200 import other_estimators as oe

    with pytest.raises(ValueError):
        next(oe._bar_steps(10, 10, uncertainty_method="svd"))
    with pytest.raises(oe._u.ParameterError):
        next(oe._bar_steps(10, 10, method="newton"))


@pytest.fixture()
def pymbar_with_oe(tmp_path):
    """A pymbar-shaped package with (oe=True) or without an other_estimators module; every function in it raises."""
    import pymbar_b200

    def make(oe):
        stub = "def {}(*args, **kwargs):\n    raise AssertionError('stand-in called')\n\n\n"
        pkg = tmp_path / ("with_oe" if oe else "without_oe") / "pymbar"
        pkg.mkdir(parents=True)
        init = "from . import mbar, mbar_solvers, utils  # noqa: F401\n"
        if oe:
            init += "from .other_estimators import bar, bar_overlap, bar_zero, exp, exp_gauss  # noqa: F401\n"
        (pkg / "__init__.py").write_text(init)
        (pkg / "utils.py").write_text("class ParameterError(Exception):\n    pass\n\n\n" +
                                      "".join(stub.format(n) for n in ("kln_to_kn", "kn_to_n")))
        (pkg / "mbar_solvers.py").write_text("".join(stub.format(n) for n in pymbar_b200._PATCHED))
        (pkg / "mbar.py").write_text("from .utils import kln_to_kn, kn_to_n  # noqa: F401\n\n\nclass MBAR:\n    pass\n")
        if oe:
            (pkg / "other_estimators.py").write_text("".join(stub.format(n) for n in NAMES + ("bar_overlap",)))
        sys.path.insert(0, str(pkg.parent))
        return str(pkg.parent)

    made = []
    try:
        yield lambda oe: made.append(make(oe)) or made[-1]
    finally:
        for p in made:
            if p in sys.path:
                sys.path.remove(p)
        for name in [m for m in sys.modules if m == "pymbar" or m.startswith("pymbar.")]:
            del sys.modules[name]


def test_install_patches_and_restores_module_and_package(pymbar_with_oe):
    import pymbar_b200

    pymbar_with_oe(True)
    import pymbar
    import pymbar.other_estimators as oem

    orig = {n: getattr(oem, n) for n in NAMES}
    overlap = oem.bar_overlap
    pymbar_b200.install()
    try:
        for n in NAMES:
            assert getattr(oem, n) is not orig[n] and getattr(oem, n).__module__ == "pymbar_b200.facade"
            assert getattr(pymbar, n) is getattr(oem, n)
        assert oem.bar_overlap is overlap and pymbar.bar_overlap is overlap
    finally:
        pymbar_b200.uninstall()
    for n in NAMES:
        assert getattr(oem, n) is orig[n] and getattr(pymbar, n) is orig[n]


def test_install_without_other_estimators_module(pymbar_with_oe):
    import pymbar_b200
    from pymbar_b200 import facade

    pymbar_with_oe(False)
    import pymbar

    pymbar_b200.install()
    try:
        assert not any(isinstance(k, types.ModuleType) for k in facade._SAVED)
        assert not hasattr(pymbar, "bar")
    finally:
        pymbar_b200.uninstall()
    assert not facade._SAVED

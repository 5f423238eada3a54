"""KDE free-energy surfaces on the CPU: the restatement of the device's log kernel sum and the host normalisation
against sklearn's score_samples, the support boundary, far queries, the long-double restatement against mpmath, and
the facade over the CPU mirror with a numpy stand-in for DeviceKde, against the outputs of the unmodified reference
FES (tests/golden/fes_kde_*.npz, tools/make_fes_kde_golden.py)."""
import math
import os

import numpy as np
import pytest

from pymbar_b200 import fes as hist
from tests import _kde
from tests.test_driver_logic_cpu import StandInMBAR, mirror  # noqa: F401  (fixture)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LD_OK = np.finfo(np.longdouble).nmant >= 63


def _score(kernel, bw, x, w, y):
    """score_samples from the restatement and the host algebra of pymbar_b200.fes."""
    x2 = x.reshape(len(x), -1)
    s = hist.kde_settings({"kernel": kernel, "bandwidth": bw, "metric": "euclidean", "metric_params": None,
                           "atol": 0, "rtol": 0, "algorithm": "auto", "leaf_size": 40, "breadth_first": True},
                          *x2.shape)
    ell = _kde.log_sum_f64(kernel, s["h"], x2, w, y)
    return ell + hist.kde_log_norm(kernel, x2.shape[1], s["h"]) - np.log(np.sum(w)), s["h"]


def _data(D, N=300, seed=0):
    rng = np.random.RandomState(seed + D)
    x = rng.normal(size=(N, D))
    w = rng.uniform(0, 1, size=N) * np.exp(rng.uniform(-5, 5, size=N))
    w[rng.choice(N, 10, replace=False)] = 0.0
    y = np.vstack([rng.normal(scale=1.5, size=(30, D)), x[:3] + 1e-3])
    return x, w, y


@pytest.mark.parametrize("kernel", hist.KDE_KERNELS)
@pytest.mark.parametrize("D", [1, 2, 3, 4])
@pytest.mark.parametrize("bw", [0.3, "scott", "silverman"])
def test_restatement_and_normalisation_match_sklearn(kernel, D, bw):
    KernelDensity = pytest.importorskip("sklearn.neighbors").KernelDensity
    x, w, y = _data(D)
    # one leaf holding every sample: sklearn then sums every pair.  With its default leaf size the traversal stops
    # short of the exact sum even at atol = rtol = 0 (up to 2e-9 depth first and 2e-7 breadth first on these data,
    # and a finite remnant for a query that no sample reaches under a compact kernel)
    kde = KernelDensity(kernel=kernel, bandwidth=bw, leaf_size=len(x) + 1).fit(x, sample_weight=w)
    want = kde.score_samples(y)
    got, h = _score(kernel, bw, x, w, y)
    assert h == kde.bandwidth_
    if kernel == "cosine" and D == 4:
        # sklearn's cosine normalisation in 4-D takes the log of a negative number: NaN, reproduced
        assert np.all(np.isnan(want)) and np.all(np.isnan(got))
        return
    np.testing.assert_array_equal(np.isneginf(got), np.isneginf(want))
    fin = np.isfinite(want)
    assert fin.sum() >= 3
    assert np.all(np.abs(got[fin] - want[fin]) <= 1e-11 * np.maximum(1.0, np.abs(want[fin])))


@pytest.mark.parametrize("D", [1, 2])
@pytest.mark.parametrize("kernel", ["tophat", "epanechnikov", "linear", "cosine"])
def test_support_boundary_is_decided_as_sklearn_does(kernel, D):
    """One sample at distance exactly h from the query, and at the neighbouring doubles: in or out of the support as
    sklearn decides it (a correctly rounded sqrt of the rounded squares, then d < h), with sklearn's kernel value."""
    KernelDensity = pytest.importorskip("sklearn.neighbors").KernelDensity
    rng = np.random.RandomState(5)
    h = 0.37
    for trial in range(40):
        y = rng.uniform(-1, 1, size=D)
        if D == 1:
            base = y[0] + h
            xs = [[base], [np.nextafter(base, -np.inf)], [np.nextafter(base, np.inf)]]
        else:
            phi = rng.uniform(0, 2 * np.pi)
            p = y + h * np.array([np.cos(phi), np.sin(phi)])
            xs = [p, [np.nextafter(p[0], -np.inf), p[1]], [np.nextafter(p[0], np.inf), p[1]],
                  [p[0], np.nextafter(p[1], y[1])]]
        for xv in xs:
            x = np.array([xv, y + 5.0])          # a second sample far away: sklearn's tree needs no special case
            w = np.array([1.0, 1e-300])
            want = KernelDensity(kernel=kernel, bandwidth=h).fit(x, sample_weight=w).score_samples(y[None])
            got, _ = _score(kernel, h, x, w, y[None])
            assert np.isneginf(got[0]) == np.isneginf(want[0]), (trial, xv)
            if np.isfinite(want[0]):
                assert abs(got[0] - want[0]) <= 1e-11 * max(1.0, abs(want[0]))
            if LD_OK:
                ld, _ = _kde.log_sum_ld(kernel, h, x, w, y[None])
                assert np.isneginf(ld[0]) == np.isneginf(got[0])


def test_far_queries_have_finite_answers():
    """Every gaussian term underflows in the linear domain; sklearn still answers (about -1.5e5 and -2.0e8)."""
    KernelDensity = pytest.importorskip("sklearn.neighbors").KernelDensity
    rng = np.random.RandomState(1)
    x = rng.normal(size=(200, 1))
    w = rng.uniform(size=200)
    y = np.array([[x.max() + 30.0], [x.min() - 1000.0]])
    want = KernelDensity(bandwidth=0.05).fit(x, sample_weight=w).score_samples(y)
    got, _ = _score("gaussian", 0.05, x, w, y)
    assert np.all(np.isfinite(got)) and want[0] < -1e5 and want[1] < -1e8
    assert np.all(np.abs(got - want) <= 1e-11 * np.abs(want))
    # exponential: far too, compact kernels: nothing in reach -> -inf
    got, _ = _score("exponential", 0.05, x, w, y)
    assert np.all(np.isfinite(got))
    got, _ = _score("epanechnikov", 0.05, x, w, y)
    assert np.all(np.isneginf(got))


@pytest.mark.skipif(not LD_OK, reason="long double is plain fp64 here")
@pytest.mark.parametrize("kernel", hist.KDE_KERNELS)
def test_long_double_restatement_against_mpmath(kernel):
    mpmath = pytest.importorskip("mpmath")
    rng = np.random.RandomState(11)
    x = rng.normal(size=(60, 2))
    w = np.exp(rng.uniform(-300, 300, size=60))
    w[3] = 0.0
    y = np.array([[0.1, -0.2], [1.5, 0.3], [40.0, 0.0]])
    ld, _ = _kde.log_sum_ld(kernel, 0.8, x, w, y)
    for q in range(len(y)):
        ref = _kde.mpmath_log_sum(kernel, 0.8, x, w, y[q])
        if ref == -mpmath.inf:
            assert np.isneginf(ld[q])
        else:
            assert abs(float(ld[q] - np.longdouble(str(ref)))) <= 1e-15 * max(1.0, abs(float(ref)))


def test_tolerance_is_stated_in_eps():
    assert _kde.tolerance(1e6, 0.0) == pytest.approx((128 + 2 * 1e3) * 2.0 ** -53)
    assert _kde.tolerance(1, 1e8) > 8 * 2.0 ** -53 * 1e8


def test_settings_resolve_or_refuse():
    base = {"kernel": "gaussian", "bandwidth": 1.0, "metric": "euclidean", "metric_params": None, "atol": 0,
            "rtol": 0, "algorithm": "auto", "leaf_size": 40, "breadth_first": True}
    assert hist.kde_settings(base, 100, 2) == {"kernel": "gaussian", "h": 1.0, "D": 2}
    assert hist.kde_settings(dict(base, bandwidth="scott"), 1000, 1)["h"] == 1000 ** (-1 / 5)
    assert hist.kde_settings(dict(base, bandwidth="silverman"), 1000, 3)["h"] == (1000 * 5 / 4) ** (-1 / 7)
    for bad in ({"metric": "manhattan"}, {"metric_params": {"p": 2}}, {"kernel": "box"}, {"bandwidth": -1.0},
                {"bandwidth": float("nan")}, {"bandwidth": "wide"}, {"atol": -1}, {"algorithm": "brute"},
                {"leaf_size": 0}):
        assert hist.kde_settings(dict(base, **bad), 100, 2) is None, bad
    assert hist.kde_settings(base, 100, 5) is None
    # atol, rtol, algorithm, leaf_size, breadth_first are accepted and ignored
    assert hist.kde_settings(dict(base, atol=1e-3, rtol=1e-2, algorithm="ball_tree", leaf_size=3,
                                  breadth_first=False), 100, 2)["h"] == 1.0


def test_kernel_norm_matches_sklearn():
    kernel_norm = pytest.importorskip("sklearn.neighbors._kd_tree").kernel_norm
    for kernel in hist.KDE_KERNELS:
        for D in range(1, 5):
            for h in (0.05, 1.0, 3.7):
                np.testing.assert_allclose(hist.kde_log_norm(kernel, D, h), kernel_norm(h, D, kernel, return_log=True),
                                           rtol=1e-15, atol=1e-15, equal_nan=True)


def test_dimension_check_draws_as_sklearn_sample_does():
    """_get_fes_kde asks KernelDensity.sample() for the dimension: the device path leaves numpy's global generator
    where the reference leaves it, and raises NotImplementedError for the kernels sklearn cannot sample from."""
    KernelDensity = pytest.importorskip("sklearn.neighbors").KernelDensity
    x, w, _ = _data(2)
    for kernel in ("gaussian", "tophat"):
        kde = KernelDensity(kernel=kernel, bandwidth=0.3).fit(x, sample_weight=w)
        np.random.seed(3)
        kde.sample()
        want = np.random.uniform()
        np.random.seed(3)
        hist._draw_as_sample(kernel, 2)
        assert np.random.uniform() == want
    with pytest.raises(NotImplementedError):
        hist._draw_as_sample("cosine", 2)


# ---- the facade over the mirror ---------------------------------------------------------------------------------

def _golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False))


def _params(g, i):
    bw = str(g["bandwidths"][i])
    return {"kernel": str(g["kernels"][i]), "bandwidth": bw if bw in ("scott", "silverman") else float(bw)}


def _ref(g):
    r = g["fes_reference"]
    return r.tolist() if r.ndim else float(r)


@pytest.fixture()
def kde_facade(mirror, monkeypatch):  # noqa: F811
    pytest.importorskip("sklearn")
    from pymbar_b200 import facade
    from tests import _fes

    monkeypatch.setattr(mirror, "DeviceKde", _kde.NumpyKde)
    mirror.DeviceProblem = _fes.OracleFESProblem
    StandInMBAR.solvers = mirror
    cls = _kde.kde_stand_in()
    cls.mbar_class = StandInMBAR
    facade.install_on(StandInMBAR)
    facade.install_fes_on(cls)
    yield cls
    facade.uninstall_from(cls)
    facade.uninstall_from(StandInMBAR)


def check_kde_facade(cls, name, atol=1e-8):
    """generate_fes / get_fes through the facade against the reference's outputs: no sklearn fit and no Log_W_nk
    download until something reads FES.kde."""
    from pymbar_b200 import facade
    from tests import _fes

    g = _golden(name)
    z = _fes.load(str(g["source"]))
    for i in range(len(g["kernels"])):
        s0 = dict(facade.STATS)
        fes = cls(z["u_kn"], z["N_k"])
        fes.generate_fes(z["u_n"], z["x_n"], fes_type="kde", kde_parameters=_params(g, i))
        assert not hasattr(fes.__dict__["_b200_kde"], "tree_")              # not fitted
        for tag, ref in (("lowest", "from-lowest"), ("specified", "from-specified"),
                         ("normalization", "from-normalization")):
            if g["get_fes_raises"][i]:
                with pytest.raises(NotImplementedError):
                    fes.get_fes(g["queries"], reference_point=ref, fes_reference=_ref(g))
                continue
            r = fes.get_fes(g["queries"], reference_point=ref, fes_reference=_ref(g))
            want = g["f_" + tag][i]
            assert r["df_i"] is None
            _same_support(r["f_i"], want)
            fin = np.isfinite(want) & np.isfinite(r["f_i"])
            np.testing.assert_allclose(r["f_i"][fin], want[fin], rtol=1e-12, atol=atol)
        assert facade.STATS["fes_kde_fits"] == s0["fes_kde_fits"]
        assert facade.STATS["redeemed"] == s0["redeemed"] and facade.STATS["fes_w_kn"] == s0["fes_w_kn"]
        assert facade.STATS["fes_kde_queries"] == s0["fes_kde_queries"] + (0 if g["get_fes_raises"][i] else 3)
        # the first read of FES.kde fits sklearn's tree as the reference does
        kde = fes.get_kde()
        assert facade.STATS["fes_kde_fits"] == s0["fes_kde_fits"] + 1
        score = kde.score_samples(g["queries"].reshape(len(g["queries"]), -1))
        fin = np.isfinite(g["score"][i]) & np.isfinite(score)
        assert fin.sum() >= len(fin) // 2
        dev = -fes.__dict__["_b200_kde_dev"][0].log_sum(str(g["kernels"][i]), kde.bandwidth_, g["queries"])
        _same_support(dev, -g["score"][i])
        np.testing.assert_allclose(score[fin], g["score"][i][fin], rtol=1e-12, atol=atol)
        fes.get_kde()
        assert facade.STATS["fes_kde_fits"] == s0["fes_kde_fits"] + 1
    return fes


def _same_support(f, want):
    """+inf where the reference has +inf; where the device finds no sample in reach of a compact kernel, the
    reference's tree may still report a finite remnant of an unresolved node bound (see
    test_restatement_and_normalisation_match_sklearn), at least e^20 below the surface's largest density."""
    f, want = np.asarray(f), np.asarray(want)
    assert np.all(np.isinf(f[np.isinf(want)]))
    remnant = np.isinf(f) & np.isfinite(want)
    assert np.all(want[remnant] > np.min(want[np.isfinite(want)]) + 20), want[remnant]


@pytest.mark.parametrize("name", ["fes_kde_1d", "fes_kde_2d"])
def test_facade_against_the_reference(kde_facade, name):
    check_kde_facade(kde_facade, name)


def test_facade_falls_through_and_uninstalls(kde_facade):
    from pymbar_b200 import facade
    from tests import _fes

    z = _fes.load("fes_hist_1d")
    cls = kde_facade
    fes = cls(z["u_kn"], z["N_k"])
    q = np.linspace(-1, 1, 5)
    # bootstraps are the original's
    with pytest.raises(AssertionError, match="facade replaces"):
        fes.generate_fes(z["u_n"], z["x_n"], fes_type="kde", kde_parameters={}, n_bootstraps=2)
    # a device surface: bootstrap uncertainties go to the original method, which fits first
    fes.generate_fes(z["u_n"], z["x_n"], fes_type="kde", kde_parameters={"bandwidth": 0.2})
    f0 = cls.fallbacks
    fits = facade.STATS["fes_kde_fits"]
    with pytest.raises(AssertionError, match="facade replaces"):
        fes.get_fes(q, uncertainty_method="bootstrap")
    assert cls.fallbacks == f0 + 1 and facade.STATS["fes_kde_fits"] == fits + 1
    # a NaN query is a device error: the original answers (sklearn raises)
    with pytest.raises(ValueError):
        fes.get_fes(np.array([0.0, np.nan]))
    assert cls.fallbacks == f0 + 2
    # parameters the device does not serve: sklearn fits at generate_fes, get_fes is the original's
    created = _kde.NumpyKde.created
    fes.generate_fes(z["u_n"], z["x_n"], fes_type="kde", kde_parameters={"metric": "manhattan", "bandwidth": 0.2})
    assert _kde.NumpyKde.created == created and hasattr(fes.kde, "tree_")
    r = fes.get_fes(q)
    assert cls.fallbacks == f0 + 3 and np.all(np.isfinite(r["f_i"]))
    # a device error at creation (a NaN sample): the original fit, and sklearn's error
    x_bad = np.array(z["x_n"], float)
    x_bad[3] = np.nan
    with pytest.raises(ValueError):
        fes.generate_fes(z["u_n"], x_bad, fes_type="kde", kde_parameters={"bandwidth": 0.2})
    # a histogram after a device KDE does not keep the KDE's device object
    fes.generate_fes(z["u_n"], z["x_n"], fes_type="kde", kde_parameters={"bandwidth": 0.2})
    assert "_b200_kde_dev" in fes.__dict__
    fes.generate_fes(z["u_n"], z["x_n"], histogram_parameters={"bin_edges": z["bin_edges"][0]})
    assert "_b200_kde_dev" not in fes.__dict__
    facade.uninstall_from(cls)
    assert "kde" not in cls.__dict__ and cls.__dict__["_get_fes_kde"].__qualname__.endswith("StandInKdeFES._get_fes_kde")
    facade.install_fes_on(cls)                          # (the fixture uninstalls again)


def test_query_errors_follow_the_reference(kde_facade):
    from pymbar_b200.utils import ParameterError
    from tests import _fes

    z = _fes.load("fes_hist_2d")
    fes = kde_facade(z["u_kn"], z["N_k"])
    fes.generate_fes(z["u_n"], z["x_n"], fes_type="kde", kde_parameters={"bandwidth": 0.2})
    q = np.zeros((3, 2))
    with pytest.raises(ParameterError):
        fes.get_fes(q, reference_point="all-differences")
    with pytest.raises(ParameterError):                 # DataError is a ParameterError where pymbar is absent
        fes.get_fes(np.zeros((3, 3)))
    with pytest.raises(ValueError):
        fes.get_fes(q, reference_point="from-specified", fes_reference=[0.0, 0.0, 0.0])
    r = fes.get_fes(q, reference_point="from-specified", fes_reference=[0.0, 0.0])
    np.testing.assert_array_equal(r["f_i"], 0.0)
    assert math.isfinite(fes.get_fes(q, reference_point="from-normalization")["f_i"][0])

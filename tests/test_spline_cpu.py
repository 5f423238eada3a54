"""Spline free-energy surfaces on the CPU: the restatement of the device's B-spline basis sums against scipy's basis
evaluation and against long double, the spline-capable FES stand-in against the outputs of the unmodified reference
FES (tests/golden/fes_spline_1d.npz, tools/make_fes_spline_golden.py), and the facade over the CPU mirror with a
numpy stand-in for DeviceBSpline."""
import os

import numpy as np
import pytest
from scipy.interpolate import BSpline

from pymbar_b200 import fes as hist
from tests import _spline
from tests.test_driver_logic_cpu import StandInMBAR, mirror  # noqa: F401  (fixture)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LD_OK = np.finfo(np.longdouble).nmant >= 63
KINDS = ("clamped", "nonuniform", "repeated")


@pytest.mark.parametrize("k", range(8))
@pytest.mark.parametrize("kind", KINDS)
def test_basis_restatement_is_scipys_bit_for_bit(k, kind):
    """Every basis value, on knots, next to them, inside and outside [t_k, t_nb], equals BSpline(t, e_i, k)(x)."""
    nb = k + 9
    t = _spline.knots(kind, k, nb, seed=k)
    x = _spline.samples_with_edges(t, 400, seed=k)
    first, h = _spline.basis_values(t, k, x)
    for i in range(nb):
        want = BSpline(t, np.eye(nb)[i], k)(x)
        a = i - first
        got = np.where((a >= 0) & (a <= k), h[np.clip(a, 0, k), np.arange(len(x))], 0.0)
        np.testing.assert_array_equal(got, want, err_msg=f"basis {i}")


@pytest.mark.parametrize("k", range(8))
def test_moments_restatement_matches_scipy_sums(k):
    nb = k + 6
    t = _spline.knots("nonuniform", k, nb, seed=3)
    x = _spline.samples_with_edges(t, 300, seed=4)
    rng = np.random.RandomState(k)
    w = rng.uniform(0, 2, size=len(x))
    s = rng.randint(0, 3, size=len(x))
    S, A = _spline.moments(t, k, x, w, s, 3)
    for i in range(nb):
        B = BSpline(t, np.eye(nb)[i], k)(x)
        np.testing.assert_allclose(A[i], np.dot(w, B), rtol=1e-13, atol=1e-13)
        for st in range(3):
            np.testing.assert_allclose(S[st, i], B[s == st].sum(), rtol=1e-13, atol=1e-13)


@pytest.mark.skipif(not LD_OK, reason="long double is plain fp64 here")
@pytest.mark.parametrize("k", range(8))
@pytest.mark.parametrize("kind", KINDS)
def test_fp64_restatement_within_tolerance_of_long_double(k, kind):
    """The fp64 restatement (scipy's basis values, summed in another order) meets the bound the device is held to."""
    nb = k + 12
    t = _spline.knots(kind, k, nb, seed=k + 7)
    x = _spline.samples_with_edges(t, 3000, seed=k)
    rng = np.random.RandomState(k)
    w = rng.uniform(0, 1, size=len(x)) * np.exp(rng.uniform(-3, 3, size=len(x)))
    s = rng.randint(0, 4, size=len(x))
    S, A = _spline.moments(t, k, x, w, s, 5)          # state 4 is empty
    _spline.check_against_ld(S, A, t, k, x, w, s, 5)


def test_tolerance_form():
    assert _spline.tolerance(3, 1.0, 1e6) == pytest.approx((4 * 16 + 2 * 1e3) * 2.0 ** -53)


def test_sample_terms_restate_the_reference_weightings():
    rng = np.random.RandomState(0)
    S = rng.uniform(size=(3, 5))
    A = rng.uniform(size=5)
    N_k = np.array([4, 7, 0])
    S[2] = 0.0                                           # the empty state has no terms
    np.testing.assert_array_equal(hist.spline_sample_terms(S, A, "unbiasedstate", 11, N_k), 11 * A)
    np.testing.assert_array_equal(hist.spline_sample_terms(S, A, "biasedstates", 11, N_k), S.sum(axis=0))
    v = hist.spline_sample_terms(S, A, "simplesum", 11, N_k)
    assert np.all(np.isnan(v))                           # an empty state: np.mean of nothing in the reference
    v = hist.spline_sample_terms(S[:2], A, "simplesum", 11, N_k[:2])
    np.testing.assert_allclose(v, (11 / 2) * (S[0] / 4 + S[1] / 7), rtol=1e-15)
    with pytest.raises(ValueError):
        hist.spline_sample_terms(S, A, "other", 11, N_k)


# ---- the stand-in and the facade over the mirror ------------------------------------------------------------------

def golden():
    return dict(np.load(os.path.join(GOLDEN, "fes_spline_1d.npz"), allow_pickle=False))


@pytest.fixture()
def spline_facade(mirror, monkeypatch):  # noqa: F811
    from pymbar_b200 import facade
    from tests import _fes

    monkeypatch.setattr(mirror, "DeviceBSpline", _spline.NumpyBSpline)
    mirror.DeviceProblem = _fes.OracleFESProblem
    StandInMBAR.solvers = mirror
    cls = _spline.spline_stand_in()
    cls.mbar_class = StandInMBAR
    facade.install_on(StandInMBAR)
    facade.install_fes_on(cls)
    yield cls
    facade.uninstall_from(cls)
    facade.uninstall_from(StandInMBAR)


def _fit(cls, case, z):
    fes = cls(z["u_kn"], z["N_k"])
    x = np.array(z["x_n"])
    fes.generate_fes(z["u_n"], x, fes_type="spline", spline_parameters=_spline.spline_parameters(case, z))
    return fes, x


def _sum_abs_terms(fes, x, xi):
    """Sum of |terms| of the objective's sample part: the scale its rounding differences are relative to."""
    b = fes._val_to_spline(xi)
    how = fes.spline_parameters["spline_weights"]
    first, h = _spline.basis_values(b.t, b.k, x)       # (not BSpline.__call__, which the facade test watches)
    vals = np.abs(sum(b.c[first + a] * h[a] for a in range(b.k + 1)))
    if how == "unbiasedstate":
        return fes.N * np.dot(fes.w_n, vals) + fes.N * 50
    return vals.sum() * (fes.N / fes.mbar.K / 300 if how == "simplesum" else 1) + fes.N * 50


def check_case(cls, i, g, z, served):
    """One fixture case through the facade (served: from moments; else: the stand-in's O(N) path)."""
    from pymbar_b200 import facade

    case = _spline.SPLINE_CASES[i]
    s0 = dict(facade.STATS)
    o0 = cls.original_calls
    fes, x = _fit(cls, case, z)
    assert facade.STATS["fes_spline_moments"] == s0["fes_spline_moments"] + (1 if served else 0)
    for j, xi in enumerate(_spline.XI_FIXED):
        f = fes._bspline_calculate_f(xi, x, fes.w_n)
        gr = fes._bspline_calculate_g(xi, x, fes.w_n)
        h = fes._bspline_calculate_h(xi, x, fes.w_n)
        # f and g: the sample terms move by rounding only (the weights are recomputed, c . v instead of a sum over
        # samples); 1e-13 of the sum of |terms|, which the reference's own fp64 sums also carry
        scale = _sum_abs_terms(fes, x, xi)
        assert abs(f - g["f"][i, j]) <= 1e-13 * scale, (case["name"], j, f - g["f"][i, j], scale)
        assert np.all(np.abs(gr - g["g"][i, j]) <= 1e-13 * scale)
        # the quadratures are the reference's, on the same integrands: bit-identical, and so is the Hessian
        pF = np.atleast_1d(fes.spline_data["bspline_pF"])
        np.testing.assert_array_equal(pF, g["pF"][i, j, :len(pF)])
        pE = np.atleast_1d(fes.spline_data["bspline_pE"])
        np.testing.assert_array_equal(pE, g["pE"][i, j, :len(pE)])
        np.testing.assert_array_equal(h, g["h"][i, j])
    # the optimiser sees f and g perturbed at the rounding level: its stopping point moves within its tolerance
    # (tol 1e-7 on the objective's scale, about 1e3-1e4 here), so the coefficients agree to 1e-5 and the surface
    # to 1e-5 kT
    np.testing.assert_allclose(fes.fes_function.c, g["c"][i], rtol=0, atol=1e-5)
    assert abs(fes.get_information_criteria("akaike") - g["aic"][i]) <= 1e-9 * abs(g["aic"][i])
    assert abs(fes.get_information_criteria("bayesian") - g["bic"][i]) <= 1e-9 * abs(g["bic"][i])
    r = fes.get_fes(_spline.QUERIES, reference_point="from-lowest")
    np.testing.assert_allclose(r["f_i"], g["f_lowest"][i], rtol=0, atol=1e-5)
    r = fes.get_fes(_spline.QUERIES, reference_point="from-specified", fes_reference=_spline.FES_REF)
    np.testing.assert_allclose(np.ravel(r["f_i"]), g["f_specified"][i], rtol=0, atol=1e-5)
    if served:
        assert cls.original_calls == o0
        assert facade.STATS["fes_spline_calls"] > s0["fes_spline_calls"]
    else:
        assert cls.original_calls > o0
    return fes, x


@pytest.mark.parametrize("i", range(len(_spline.SPLINE_CASES)), ids=[c["name"] for c in _spline.SPLINE_CASES])
def test_stand_in_reproduces_the_reference(spline_facade, mirror, monkeypatch, i):  # noqa: F811
    """With the device refusing (a stand-in that raises), every call reaches the stand-in's own O(N) methods, which
    reproduce the reference: this pins the stand-in to pymbar's FES."""
    from pymbar_b200._lib import MbarB200Error

    def refuse(*a, **k):
        raise MbarB200Error(-5, "refused")

    monkeypatch.setattr(mirror, "DeviceBSpline", refuse)
    check_case(spline_facade, i, golden(), _load(), served=False)


def _load():
    from tests import _fes

    return _fes.load("fes_hist_1d")


@pytest.mark.parametrize("i", range(len(_spline.SPLINE_CASES)), ids=[c["name"] for c in _spline.SPLINE_CASES])
def test_facade_against_the_reference(spline_facade, monkeypatch, i):
    """Through the facade: one moments pass, no BSpline evaluation on a state's worth of samples."""
    z = _load()
    smallest = int(np.min(z["N_k"]))
    calls = []
    orig_call = BSpline.__call__

    def watch(self, x, *a, **k):
        calls.append(np.size(x))
        return orig_call(self, x, *a, **k)

    monkeypatch.setattr(BSpline, "__call__", watch)
    check_case(spline_facade, i, golden(), z, served=True)
    assert max(calls) < smallest, max(calls)


@pytest.mark.parametrize("m", range(len(_spline.MC_CASES)), ids=list(_spline.MC_CASES))
@pytest.mark.parametrize("through", ["facade", "stand_in"])
def test_mc_chain_makes_the_reference_decisions(spline_facade, mirror, monkeypatch, m, through):  # noqa: F811
    """The seeded chain accepts and rejects as the reference does: every log-likelihood differs from the
    reference's by far less than the recorded margin of its closest Metropolis decision, so the chain follows the
    same path, and its samples and log posteriors agree to rounding."""
    from pymbar_b200 import facade
    from pymbar_b200._lib import MbarB200Error

    if through == "stand_in":
        def refuse(*a, **k):
            raise MbarB200Error(-5, "refused")

        monkeypatch.setattr(mirror, "DeviceBSpline", refuse)
    g, z = golden(), _load()
    name = _spline.MC_CASES[m]
    i = [c["name"] for c in _spline.SPLINE_CASES].index(name)
    fes, x = _fit(spline_facade, _spline.SPLINE_CASES[i], z)
    calls0 = facade.STATS["fes_spline_calls"]
    np.random.seed(_spline.MC_SEED)
    fes.sample_parameter_distribution(x, mc_parameters=_spline.mc_parameters(), decorrelate=False, verbose=False)
    mc = fes.mc_data
    assert mc["naccept"] == g["mc_naccept"][m]
    # the log posteriors differ from the reference's because the fit stopped at coefficients 1e-5 away (see
    # check_case) and by rounding; every difference is under a quarter of the recorded margin of the reference's
    # closest Metropolis decision, so no decision could have gone the other way
    diff = np.max(np.abs(mc["logposteriors"] - g["mc_logpost"][m]))
    assert diff < g["mc_margin"][m] / 4, (diff, g["mc_margin"][m])
    np.testing.assert_allclose(mc["samples"], g["mc_samples"][m], rtol=0, atol=1e-5)
    served = facade.STATS["fes_spline_calls"] - calls0
    assert served == (2 * _spline.MC_STEPS if through == "facade" else 0)


def test_fallbacks_and_uninstall(spline_facade):
    from pymbar_b200 import facade

    cls = spline_facade
    g, z = golden(), _load()
    case = _spline.SPLINE_CASES[0]
    fes, x = _fit(cls, case, z)
    xi = _spline.XI_FIXED[1]
    o0, c0 = cls.original_calls, facade.STATS["fes_spline_calls"]
    # the moments' own arrays: served
    fes._bspline_calculate_f(xi, x, fes.w_n)
    assert cls.original_calls == o0 and facade.STATS["fes_spline_calls"] == c0 + 1
    # another x_n (equal values, another array), another w_n: the original
    fes._bspline_calculate_f(xi, x.copy(), fes.w_n)
    fes._bspline_calculate_g(xi, x, fes.w_n.copy())
    assert cls.original_calls == o0 + 2
    # other knots: the original
    b = fes.spline_data["bspline"]
    fes.spline_data["bspline"] = BSpline(b.t + 1e-3, b.c, b.k)
    fes._bspline_calculate_f(xi, x, fes.w_n)
    assert cls.original_calls == o0 + 3
    fes.spline_data["bspline"] = b
    # an MC likelihood of another spline, or with other weights: the original
    other = BSpline(b.t * 1.01, b.c, b.k)
    fes._get_MC_loglikelihood(x, fes.w_n, "unbiasedstate", other, _spline.XRANGE)
    fes._get_MC_loglikelihood(x, fes.w_n, "biasedstates", b, _spline.XRANGE)
    assert cls.original_calls == o0 + 5
    # a NaN sample is a device error: the fit runs the original methods
    x_bad = np.array(z["x_n"], float)
    x_bad[3] = np.nan
    m0 = facade.STATS["fes_spline_moments"]
    fes2 = cls(z["u_kn"], z["N_k"])
    o1 = cls.original_calls
    with np.errstate(invalid="ignore"):
        try:
            fes2.generate_fes(z["u_n"], x_bad, fes_type="spline", spline_parameters=_spline.spline_parameters(case, z))
        except Exception:
            pass
    assert facade.STATS["fes_spline_moments"] == m0 and cls.original_calls > o1
    assert "_b200_spline" not in fes2.__dict__
    # 2-D samples: no moments
    fes3 = cls(z["u_kn"], z["N_k"])
    try:
        fes3.generate_fes(z["u_n"], x.reshape(-1, 1), fes_type="spline",
                          spline_parameters=_spline.spline_parameters(case, z))
    except Exception:
        pass
    assert facade.STATS["fes_spline_moments"] == m0 and "_b200_spline" not in fes3.__dict__
    # a histogram after a spline drops the moments
    fes.generate_fes(z["u_n"], z["x_n"], histogram_parameters={"bin_edges": z["bin_edges"][0]})
    assert "_b200_spline" not in fes.__dict__
    facade.uninstall_from(cls)
    for name in ("_bspline_calculate_f", "_bspline_calculate_g", "_get_MC_loglikelihood"):
        assert cls.__dict__[name].__qualname__.endswith("StandInSplineFES." + name)
    facade.install_fes_on(cls)                          # (the fixture uninstalls again)


def test_numpy_stand_in_checks_like_the_library():
    from pymbar_b200._lib import MbarB200Error

    x = np.linspace(0, 1, 10)
    for bad in (dict(w_n=-np.ones(10)), dict(w_n=np.full(10, np.nan)), dict(state_n=np.arange(10), K=3)):
        with pytest.raises(MbarB200Error):
            _spline.NumpyBSpline(x, **bad)
    with pytest.raises(MbarB200Error):
        _spline.NumpyBSpline(np.array([0.0, np.inf]))
    d = _spline.NumpyBSpline(x, np.ones(10), np.zeros(10, int), K=1)
    t = _spline.knots("clamped", 3, 6)
    for bad_t, k in ((t, 8), (t[::-1], 3), (t[:7], 3), (np.where(t > 0, t, np.nan), 3), (np.zeros(10), 3)):
        with pytest.raises(MbarB200Error):
            d.moments(bad_t, k)

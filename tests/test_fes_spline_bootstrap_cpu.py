"""Spline FES bootstrap replicates on the CPU: the facade's spline bootstrap path over the CPU mirror, with numpy
stand-ins for the device (a weighted-solve problem and a DeviceBSpline with replicate sums), against the unmodified
reference's replicates, uncertainties and generator state (tests/golden/fes_spline_bootstrap.npz,
tools/make_fes_spline_bootstrap_golden.py); every fall-back rule; the counters; and b = 0 still matching
tests/golden/fes_spline_1d.npz."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
from scipy.interpolate import BSpline
from scipy.optimize import minimize

from pymbar_b200 import fes_bootstrap as fb
from pymbar_b200._lib import MbarB200Error
from tests import _fes, _spline
from tests.test_driver_logic_cpu import StandInMBAR, mirror  # noqa: F401  (fixture)
from tests.test_fes_bootstrap_cpu import WeightedOracleProblem, _falls_back, _same_state

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = dict(np.load(os.path.join(_fes.GOLDEN, "fes_spline_bootstrap.npz"), allow_pickle=False))
S1 = dict(np.load(os.path.join(_fes.GOLDEN, "fes_spline_1d.npz"), allow_pickle=False))
NB = int(G["n_bootstraps"])
CASES = [(str(c), int(s)) for c in G["cases"] for s in G["seeds"]]
NAMES = [c["name"] for c in _spline.SPLINE_CASES]


def boot_stand_in():
    """tests/_spline's stand-in with what a bootstrap spline surface adds (fes.py:804-807, :998-1001, :1095-1098,
    :1675-1687): fes_functions in the set-up, the replicate fits from b = 0's coefficients, and the bootstrap std of
    get_fes."""

    class StandInSplineBootFES(_spline.spline_stand_in()):
        generate_fes = _get_fes_histogram = _fes.StandInFES._replaced

        def _setup_fes_spline(self, spline_parameters):
            super()._setup_fes_spline(spline_parameters)
            self.fes_functions = list() if self.n_bootstraps > 0 else None

        def _generate_fes_spline(self, b, x_n, w_n):
            if b == 0:
                return super()._generate_fes_spline(b, x_n, w_n)
            p = self.spline_parameters
            xi = self.spline_data["first_coefficients"].copy()
            r = minimize(self._bspline_calculate_f, xi, args=(x_n, w_n), method=p["optimization_algorithm"],
                         jac=self._bspline_calculate_g, tol=p["scipy_tol"], hess=self._bspline_calculate_h,
                         options=p["optimize_options"])
            self.fes_functions.append(self._val_to_spline(r["x"]))

        def get_fes(self, x, reference_point="from-lowest", fes_reference=None, uncertainty_method=None):
            out = super().get_fes(x, reference_point, fes_reference)
            if uncertainty_method == "bootstrap":
                q = np.array(x).reshape(-1, 1)[:, 0]
                if reference_point == "from-lowest":
                    fmin = np.min(self.fes_function(q))
                else:
                    fmin = -self.fes_function(np.array(fes_reference).reshape(1, -1))
                fall = np.zeros([len(q), len(self.fes_functions)])
                for b, f in enumerate(self.fes_functions):
                    fall[:, b] = f(q) - fmin
                out["df_i"] = np.std(fall, axis=-1)
            return out

    return StandInSplineBootFES


class ReplicateNumpyBSpline(_spline.NumpyBSpline):
    """NumpyBSpline with the replicate entry points, answered row by row by the fp64 restatement, with the C ABI's
    checks.  Counts its replicate-sum calls and keeps the last uploaded weights."""

    replicate_calls = 0
    last_V = None

    def set_replicates(self, V):
        V = np.array(V, np.float64)
        if V.ndim != 2 or V.shape[1] != self.N:
            raise ValueError("replicate weights must be [B, N]")
        self.B = 0
        if len(V) < 1 or not np.all((V >= 0) & np.isfinite(V)):
            raise MbarB200Error(-1, "bad replicate weights")
        self.V, self.B = V, len(V)
        type(self).last_V = V

    def replicate_sums(self, t, k):
        t = np.asarray(t, np.float64)
        nb = len(t) - k - 1
        if not (0 <= k <= 7 and len(t) >= 2 * (k + 1) and np.all(np.isfinite(t)) and np.all(np.diff(t) >= 0)
                and t[k] < t[nb]):
            raise MbarB200Error(-1, "bad knots or degree")
        if self.B < 1:
            raise MbarB200Error(-4, "no replicates uploaded")
        type(self).replicate_calls += 1
        return np.array([_spline.moments(t, k, self.x, v)[1] for v in self.V])


@pytest.fixture()
def boot_spline(mirror, monkeypatch):  # noqa: F811
    from pymbar_b200 import facade

    monkeypatch.setattr(mirror, "DeviceBSpline", ReplicateNumpyBSpline)
    monkeypatch.setattr(mirror, "DeviceProblem", WeightedOracleProblem)
    StandInMBAR.solvers = mirror
    cls = boot_stand_in()
    cls.mbar_class = StandInMBAR
    facade.install_on(StandInMBAR)
    facade.install_fes_on(cls)
    yield cls
    facade.uninstall_from(cls)
    facade.uninstall_from(StandInMBAR)


def _case(name):
    return _spline.SPLINE_CASES[NAMES.index(name)]


def check_spline_bootstrap(cls, name, seed, watch=None):
    """generate_fes / get_fes of a bootstrap spline surface against the reference.

    Replicate coefficients are held to b = 0's tolerance, atol 1e-5: the objective and gradient move by rounding only,
    so the optimiser stops within its own tolerance of the reference's point.  Where a Newton-CG "unbiasedstate"
    replicate's objective is flat along some coefficient (a replicate with few samples at an edge of the range), the
    stopping point is not defined to 1e-5 and its coefficients spread by up to about 1 kT; there the replicate is
    held instead to the reference's objective at its own final coefficients (1e-9 relative), which is what the
    optimiser minimises, and df_i is compared where every replicate's coefficients agree."""
    from pymbar_b200 import facade

    z = _fes.load("fes_hist_1d")
    case = _case(name)
    p = f"{name}_s{seed}_"
    s0 = dict(facade.STATS)
    o0, r0 = cls.original_calls, ReplicateNumpyBSpline.replicate_calls
    fes = cls(z["u_kn"], z["N_k"])
    x = np.array(z["x_n"])
    fes.generate_fes(z["u_n"], x, fes_type="spline", spline_parameters=_spline.spline_parameters(case, z),
                     n_bootstraps=NB, seed=seed)
    assert np.random.random() == G[p + "after"]
    # b = 0 is the fit of the surface without bootstraps
    i = NAMES.index(name)
    np.testing.assert_allclose(fes.fes_function.c, S1["c"][i], rtol=0, atol=1e-5)
    np.testing.assert_allclose(fes.fes_function.c, G[p + "c0"], rtol=0, atol=1e-5)
    assert abs(fes.get_information_criteria("akaike") - S1["aic"][i]) <= 1e-9 * abs(S1["aic"][i])
    assert abs(fes.get_information_criteria("bayesian") - S1["bic"][i]) <= 1e-9 * abs(S1["bic"][i])
    assert isinstance(fes.__dict__["_b200_spline"], facade.SplineMoments)
    assert "_b200_spline_replicate" not in fes.__dict__
    # the replicates
    assert len(fes.fes_functions) == NB and all(isinstance(f, BSpline) for f in fes.fes_functions)
    c = np.array([f.c for f in fes.fes_functions])
    close = np.all(np.abs(c - G[p + "c"]) <= 1e-5, axis=1)
    for tag, rp in (("lowest", "from-lowest"), ("specified", "from-specified")):
        r = fes.get_fes(_spline.QUERIES, reference_point=rp, fes_reference=_spline.FES_REF,
                        uncertainty_method="bootstrap")
        np.testing.assert_allclose(np.ravel(r["f_i"]), G[p + "f_" + tag], rtol=0, atol=1e-5)
        if np.all(close):
            np.testing.assert_allclose(r["df_i"], G[p + "df_" + tag], rtol=0, atol=1e-5)
    # the work: one solve per replicate for "unbiasedstate" only, one replicate-sum call, no O(N) objective, no
    # download of the weight matrices, no fall-back
    solves = NB if case["weights"] == "unbiasedstate" else 0
    assert facade.STATS["fes_boot_spline_solves"] == s0["fes_boot_spline_solves"] + solves
    assert facade.STATS["fes_boot_spline_sums"] == s0["fes_boot_spline_sums"] + 1
    assert ReplicateNumpyBSpline.replicate_calls == r0 + 1
    assert facade.STATS["fes_boot_fallbacks"] == s0["fes_boot_fallbacks"]
    assert facade.STATS["redeemed"] == s0["redeemed"] and facade.STATS["fes_w_kn"] == s0["fes_w_kn"]
    assert cls.original_calls == o0
    if case["weights"] == "unbiasedstate":
        # the replicate weights are the reference's w_nb summed onto the samples
        np.testing.assert_allclose(ReplicateNumpyBSpline.last_V, G[p + "V"], rtol=1e-9, atol=1e-15)
    for b in np.flatnonzero(~close):
        assert case["weights"] == "unbiasedstate" and case["algorithm"] == "Newton-CG", (name, seed, b)
        obj = replicate_objective(fes, x, z, seed, b)
        assert abs(obj - G[p + "obj"][b]) <= 1e-9 * abs(G[p + "obj"][b]), (b, obj, G[p + "obj"][b])
    return fes


def replicate_objective(fes, x, z, seed, b):
    """The reference's objective of replicate b at its final coefficients, on the replicate's own x_nb and w_nb (the
    stand-in's own O(N) method, as the golden file's obj was computed)."""
    state = np.random.get_state()
    np.random.seed(seed)
    states = fb.draw_replicates(z["N_k"], NB)
    np.random.set_state(state)
    idx = fb.replicate_indices(states[b], z["N_k"])
    V = ReplicateNumpyBSpline.last_V
    w = V[b][idx] / np.bincount(idx, minlength=len(x))[idx]
    own = next(c for c in type(fes).__mro__ if "_bspline_calculate_f" in c.__dict__ and c is not type(fes))
    return own._bspline_calculate_f(fes, fes.fes_functions[b].c[1:], x[idx], w)


@pytest.mark.parametrize("name,seed", CASES)
def test_spline_replicates_on_the_mirror(boot_spline, monkeypatch, name, seed):
    """No spline is evaluated on a state's worth of samples: the replicates' objectives come from their sums."""
    z = _fes.load("fes_hist_1d")
    calls = []
    orig_call = BSpline.__call__

    def watch(self, x, *a, **k):
        calls.append(np.size(x))
        return orig_call(self, x, *a, **k)

    monkeypatch.setattr(BSpline, "__call__", watch)
    fes = check_spline_bootstrap(boot_spline, name, seed)
    assert max(calls) < int(np.min(z["N_k"])) and len(fes.fes_functions) == NB


def test_replicate_weights_of_every_weighting():
    """spline_replicates: V is c_b, c_b N / (K N_s) or the normalised weights, and the stream is draw_replicates'."""
    N_k = np.array([3, 5, 2])
    N, K = 10, 3
    rng = np.random.RandomState(0)
    lw = rng.normal(size=N)
    for how in ("biasedstates", "simplesum", "unbiasedstate"):
        np.random.seed(4)
        states, V = fb.spline_replicates(N_k, 3, how, lambda idx: lw)
        after = np.random.random()
        np.random.seed(4)
        assert all(_same_state(a, b) for a, b in zip(states, fb.draw_replicates(N_k, 3)))
        assert np.random.random() == after
        for b, st in enumerate(states):
            c = np.bincount(fb.replicate_indices(st, N_k), minlength=N).astype(float)
            if how == "biasedstates":
                np.testing.assert_array_equal(V[b], c)
            elif how == "simplesum":
                np.testing.assert_allclose(V[b], c * N / (K * np.repeat(N_k, N_k)), rtol=1e-15)
            else:
                want = c * np.exp(lw) / np.sum(c * np.exp(lw))
                np.testing.assert_allclose(V[b], want, rtol=1e-14)
                assert np.all(V[b][c == 0] == 0)
    with pytest.raises(ValueError):
        fb.spline_replicates(N_k, 2, "other")
    assert fb.in_block_order(np.repeat([0, 1, 2], N_k), N_k)
    assert not fb.in_block_order(np.roll(np.repeat([0, 1, 2], N_k), 1), N_k)


def test_entry_points_are_declared():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mbar_b200.h")).read(), flags=re.S)
    from pymbar_b200 import _lib

    for name in ("mbar_b200_bspline_set_replicates", "mbar_b200_bspline_replicate_sums"):
        assert re.search(rf"\b{name}\s*\(", src) and name in _lib.SIGNATURES


def test_replicate_kernels_build_for_sm90a_without_spills():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    out = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v",
                          "-c", os.path.join(ROOT, "pymbar_b200", "csrc", "bspline.cu"), "-o", os.devnull],
                         capture_output=True, text=True, check=True).stderr
    blocks = [b for b in out.split("Compiling entry function")[1:] if "bsp_replicate_kernel" in b.split("\n")[0]]
    assert len(blocks) == 8                            # degrees 0..7
    for b in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in b, b


def test_fallbacks(boot_spline, mirror, monkeypatch):  # noqa: F811
    from pymbar_b200 import facade

    cls = boot_spline
    z = _fes.load("fes_hist_1d")
    case = _case("biased_ncg")

    def call(fes, x=None, params=None):
        return lambda: fes.generate_fes(z["u_n"], z["x_n"] if x is None else x, fes_type="spline",
                                        spline_parameters=_spline.spline_parameters(case, z) if params is None
                                        else params, n_bootstraps=2)

    # samples out of block order: the reference labels replicate positions with b = 0's labels
    f = cls(z["u_kn"], z["N_k"])
    f.mbar.x_kindices = np.roll(np.asarray(f.mbar.x_kindices), 1)
    _falls_back(cls, call(f))
    # 2-D samples
    f = cls(z["u_kn"], z["N_k"])
    _falls_back(cls, call(f, x=np.asarray(z["x_n"]).reshape(-1, 1)))
    # an unknown spline_weights
    params = _spline.spline_parameters(case, z)
    params["spline_weights"] = "other"
    _falls_back(cls, call(f, params=params))
    # a state without samples
    ze = _fes.load("fes_hist_empty")
    fe = cls(ze["u_kn"], ze["N_k"])
    _falls_back(cls, lambda: fe.generate_fes(ze["u_n"], ze["x_n"], fes_type="spline",
                                             spline_parameters=_spline.spline_parameters(case, ze), n_bootstraps=2))
    # device errors, after b = 0 is fitted: the original gets the spline_parameters as they were given
    for where in ("set_replicates", "replicate_sums"):
        def refuse(self, *a, **k):
            raise MbarB200Error(-2, "refused")

        with monkeypatch.context() as m:
            m.setattr(ReplicateNumpyBSpline, where, refuse)
            params = _spline.spline_parameters(case, z)
            given = {key: (dict(v) if isinstance(v, dict) else v) for key, v in params.items()}
            f = cls(z["u_kn"], z["N_k"])
            n0 = facade.STATS["fes_boot_fallbacks"]
            np.random.seed(99)
            entry = np.random.get_state()
            with pytest.raises(AssertionError, match="facade replaces"):
                f.generate_fes(z["u_n"], z["x_n"], fes_type="spline", spline_parameters=params, n_bootstraps=2)
            assert _same_state(entry, np.random.get_state())
            assert facade.STATS["fes_boot_fallbacks"] == n0 + 1
            assert "_b200_spline" not in f.__dict__ and "_b200_spline_replicate" not in f.__dict__
            # the set-up had popped optimize_options["tol"] and filled in map_data
            assert set(params) == set(given) and params["optimize_options"] == given["optimize_options"]
            assert all(params[key] is given[key] for key in given if not isinstance(given[key], dict))
    # a DeviceBSpline without replicate entry points, and a problem without multiplicities for "unbiasedstate"
    monkeypatch.setattr(mirror, "DeviceBSpline", _spline.NumpyBSpline)
    _falls_back(cls, call(cls(z["u_kn"], z["N_k"])))
    monkeypatch.setattr(mirror, "DeviceBSpline", ReplicateNumpyBSpline)
    monkeypatch.setattr(mirror, "DeviceProblem", _fes.OracleFESProblem)
    case = _case("unbiased_ncg")
    _falls_back(cls, call(cls(z["u_kn"], z["N_k"])))

"""GPU parity at the edges of the fp64 exponent range (inputs and bands: tests/_edges.py).

Every comparison is made in the log domain against the oracle (or the analytic answer of an offset copy) to
1e-8 absolute where finite; where the reference weight is exactly 0 the device must return 0 too.  Each check
also asserts which kernel answered (`last_kernels()`), as predicted by `_edges.bands`, so that a case cannot
pass through a path it was not built for."""
import numpy as np
import pytest
from scipy.special import logsumexp

from oracle import mbar_oracle as orc
from tests import _edges as E

pytestmark = pytest.mark.gpu

TOL = 1e-8


@pytest.fixture(scope="module")
def lib():
    import pymbar_b200
    from pymbar_b200 import _lib

    _lib.load()
    if _lib.device_count() == 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return pymbar_b200


@pytest.fixture
def mode(request, monkeypatch):
    if request.param is not None:
        monkeypatch.setenv("MBAR_B200_FUSED_MODE", request.param)
    return request.param


def ref_log_S(u, N, f):
    """log S_k = logsumexp_n(f_k - u_kn - L_n) for every state, L_n over the sampled states."""
    s = N > 0
    L = orc.log_denominator_n(u[s], N[s], f[s])
    return logsumexp(f[:, None] - u - L[None, :], axis=1)


def assert_answered(p, b, CL=None):
    """The kernel that produced the last result is the one `bands` predicts (skipped within a hair of a
    threshold, where rounding may legitimately decide either way)."""
    k = p.last_kernels()["pass_kernel"]
    if b["answer"] == "fused" and b["margin"] > 1.0:
        assert k.startswith("pass_fused_kernel") and f"MODE={b['mode']}" in k, (k, b["reason"])
        if CL is not None:
            assert f"CL={CL}>" in k or f"CL={CL}," in k, k
    elif b["answer"] == "generic" and b.get("margin", -np.inf) < -1.0:
        assert k.startswith("pass_generic_kernel"), (k, b["reason"])


def check_sampled_primitives(p, u, N, f, b, CL=None):
    s = N > 0
    np.testing.assert_allclose(p.self_consistent_update(f), orc.self_consistent_update(u, N, f), rtol=0, atol=TOL)
    assert_answered(p, b, CL)
    S, sumL, _ = p.streaming_pass(f)
    assert_log_S(S[s], ref_log_S(u, N, f)[s])
    np.testing.assert_allclose(sumL, orc.log_denominator_n(u[s], N[s], f[s]).sum(), rtol=1e-13, atol=TOL)
    assert_answered(p, b, CL)
    np.testing.assert_allclose(p.gradient(f)[s], orc.mbar_gradient(u[s], N[s], f[s]), rtol=0, atol=TOL * N.max())
    np.testing.assert_allclose(p.objective(f), orc.mbar_objective(u[s], N[s], f[s]), rtol=1e-13, atol=TOL)


def assert_log_S(S, lS):
    """S = sum_n W_nk against the reference's log S: 1e-8 in the log domain where the reference's S is a normal
    double; where it is not, the device may return at most the smallest normal double."""
    tiny = np.finfo(np.float64).tiny
    normal = lS > np.log(tiny) + 1e-3
    with np.errstate(divide="ignore"):
        np.testing.assert_allclose(np.log(S[normal]), lS[normal], rtol=0, atol=TOL)
    assert np.all((S[~normal] >= 0.0) & (S[~normal] <= tiny * 1.001)), S[~normal]


def host_iterates(u, N, f0, iters):
    s = N > 0
    f = f0.copy()
    for _ in range(iters):
        nxt = orc.self_consistent_update(u[s], N[s], f[s])
        f[s] = nxt - nxt[0]
    return f


# ---------------------------------------------------------------- A. floor band (sampled states)
@pytest.mark.parametrize("mode", [None, "1"], indirect=True)
@pytest.mark.parametrize("start", E.A_STARTS)
@pytest.mark.parametrize("delta", E.A_DELTAS)
def test_floor_band_pair(lib, delta, start, mode):
    case = E.offset_pair(delta)
    u, N = case["u"], case["N"]
    f = np.array([0.0, start])
    b = E.bands(u, N, f, all_states=False, mode_env=mode)
    with lib.DeviceProblem(u, N) as p:
        check_sampled_primitives(p, u, N, f, b, CL=1)
        np.testing.assert_allclose(p.log_W_nk(f), orc.mbar_log_W_nk(u, N, f), rtol=0, atol=TOL)
        # two candidates in one call: this start and the answer
        S2, L2 = p.pass_multi(np.stack([f, case["f_true"]]))
        for m, fm in enumerate((f, case["f_true"])):
            assert_log_S(S2[m], ref_log_S(u, N, fm))
            np.testing.assert_allclose(L2[m], orc.log_denominator_n(u, N, fm).sum(), rtol=1e-13, atol=TOL)
        for it in (1, 2, 3):
            np.testing.assert_allclose(p.sci_iterate(f, it), host_iterates(u, N, f, it), rtol=0, atol=TOL)
        f_sci, r = p.solve_sci(f, tol=1e-13, maxiter=100)
        assert r["success"]
        np.testing.assert_allclose(f_sci, case["f_true"], rtol=0, atol=TOL)
        f_ad, r = p.solve_adaptive(f, tol=1e-12, min_sc_iter=0)
        np.testing.assert_allclose(f_ad, case["f_true"], rtol=0, atol=TOL)


@pytest.mark.parametrize("start", [70.0, 300.0])
def test_floor_band_noisy(lib, start):
    case = E.offset_pair(800.0, noisy=True)
    u, N = case["u"], case["N"]
    f = np.array([0.0, start])
    with lib.DeviceProblem(u, N) as p:
        check_sampled_primitives(p, u, N, f, E.bands(u, N, f, all_states=False))
        np.testing.assert_allclose(p.sci_iterate(f, 2), host_iterates(u, N, f, 2), rtol=0, atol=TOL)


@pytest.mark.parametrize("mode", [None, "1"], indirect=True)
@pytest.mark.parametrize("delta", [712.0, 800.0])
@pytest.mark.parametrize("K,CL", [(64, 1), (96, 1), (300, 2), (1100, 8)])
def test_floor_band_shapes(lib, K, CL, delta, mode, monkeypatch):
    case = E.offset_copies(K, delta)
    u, N = case["u"], case["N"]
    odd = np.arange(K) % 2 == 1
    with lib.DeviceProblem(u, N) as p:
        for start in (100.0, 300.0, delta):
            f = np.where(odd, start, 0.0)
            check_sampled_primitives(p, u, N, f, E.bands(u, N, f, all_states=False, mode_env=mode), CL=CL)
            np.testing.assert_allclose(p.sci_iterate(f, 2), host_iterates(u, N, f, 2), rtol=0, atol=TOL)
        if K == 300:
            monkeypatch.setenv("MBAR_B200_M2_CLUSTERS", "1")
            fs = np.stack([np.where(odd, 300.0, 0.0), case["f_true"]])
            S2, _ = p.pass_multi(fs)
            for m in range(2):
                assert_log_S(S2[m], ref_log_S(u, N, fs[m]))


# ---------------------------------------------------------------- B. unsampled rows far below / above
def check_all_state_paths(lib, case, delta_true):
    u, N = case["u"], case["N"]
    f0 = np.zeros(3)
    b = E.bands(u, N, f0, all_states=True)
    want = orc.self_consistent_update(u, N, f0)
    with lib.DeviceProblem(u, N) as p:
        np.testing.assert_allclose(p.self_consistent_update(f0), want, rtol=0, atol=TOL)
        assert_answered(p, b)
        if case["f_true"] is not None:
            ft = case["f_true"]
            # at the answer the all-state pass is well inside the fused kernel's range up to delta ~ 1000
            np.testing.assert_allclose(p.self_consistent_update(ft), orc.self_consistent_update(u, N, ft),
                                       rtol=0, atol=TOL)
            assert_answered(p, E.bands(u, N, ft, all_states=True))
            S, G = p.weight_moments(ft)
            W = orc.mbar_W_nk(u, N, ft)
            np.testing.assert_allclose(S, W.sum(0), rtol=1e-10)
            np.testing.assert_allclose(G, W.T @ W, rtol=1e-9, atol=1e-300)
        with lib.DeviceProblem(u[:2], N[:2]) as base, base.augmented(u[2:]) as q:
            np.testing.assert_allclose(q.self_consistent_update(f0), want, rtol=0, atol=TOL)
            assert_answered(q, b)
    if case["f_true"] is None:
        return
    ms = lib.mbar_solvers
    proto = tuple(dict(st) for st in ms.DEFAULT_SOLVER_PROTOCOL)
    got = ms.solve_mbar_for_all_states(u, N.astype(np.int64), np.zeros(3), np.array([0, 1]), proto)
    np.testing.assert_allclose(got, case["f_true"], rtol=0, atol=TOL)
    from pymbar_b200 import expectations as ex

    from pymbar_b200 import estimators as est

    u0, fs, Ns = u[0], case["f_true"][:2], N[:2]
    r = ex.compute_perturbed_free_energies(u[:2], Ns.astype(np.int64), fs, np.stack([u0, u[2]]),
                                           compute_uncertainty=False)
    np.testing.assert_allclose(r["Delta_f"][0, 1], delta_true, rtol=0, atol=TOL)
    # uncertainties against a state that is not a copy of state 0 (between copies dDelta_f is 0 up to rounding):
    # the estimators fed with the oracle's W^T W of the augmented problem
    u_ln = np.stack([1.1 * u0, u[2]])
    r = ex.compute_perturbed_free_energies(u[:2], Ns.astype(np.int64), fs, u_ln)
    u_aug = np.vstack([u[:2], u_ln])
    N_aug = np.concatenate([Ns, np.zeros(2)])
    f_aug = orc.self_consistent_update(u_aug, N_aug, np.concatenate([fs, np.zeros(2)]))
    f_aug[:2] = fs
    W = orc.mbar_W_nk(u_aug, N_aug, f_aug)
    Theta = est.asymptotic_covariance(W.T @ W, N_aug, method=None)[np.ix_([2, 3], [2, 3])]
    np.testing.assert_allclose(r["Delta_f"], f_aug[2:][None, :] - f_aug[2:][:, None], rtol=0, atol=TOL)
    np.testing.assert_allclose(r["dDelta_f"], est.error_of_differences(Theta), rtol=1e-7, atol=1e-10)
    # an observable under the appended state, against the oracle's weights of that state
    A = np.cos(u0)
    L = orc.log_denominator_n(u[:2], Ns, fs)
    w = np.exp(-u[2] - L - logsumexp(-u[2] - L))
    mu = ex.compute_expectations(u[:2], Ns.astype(np.int64), fs, A, u_ln=u[2], compute_uncertainty=False)["mu"][0]
    np.testing.assert_allclose(mu, w @ A, rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize("delta", E.B_BELOW)
def test_wrap_band_unsampled_below(lib, delta):
    check_all_state_paths(lib, E.with_unsampled(delta, -1.0), -delta)


@pytest.mark.parametrize("delta", E.B_ABOVE)
def test_unsampled_above(lib, delta):
    check_all_state_paths(lib, E.with_unsampled(delta, +1.0), delta)


@pytest.mark.parametrize("delta", [2500.0, 9.9e4])
def test_wrap_band_noisy(lib, delta):
    check_all_state_paths(lib, E.with_unsampled(delta, -1.0, noisy=True), None)


# ---------------------------------------------------------------- C. mode and range boundaries
@pytest.mark.parametrize("spread", E.C_SPREADS)
def test_mode_boundaries(lib, spread):
    case = E.spread_pair(spread)
    u, N, f = case["u"], case["N"], case["f"]
    b = E.bands(u, N, f, all_states=False)
    assert b["kernel"] == ("fused" if spread < E.FUSED_SPREAD else "generic")
    with lib.DeviceProblem(u, N) as p:
        check_sampled_primitives(p, u, N, f, b, CL=1)
        np.testing.assert_allclose(p.log_W_nk(f), orc.mbar_log_W_nk(u, N, f), rtol=0, atol=TOL)
        np.testing.assert_allclose(p.hessian(f), orc.mbar_hessian(u, N, f), rtol=1e-9, atol=1e-10)
        np.testing.assert_allclose(p.sci_iterate(f, 2), host_iterates(u, N, f, 2), rtol=0, atol=TOL)


@pytest.mark.parametrize("spread,answer", [(1149.0, "fused"), (1150.0, "fused"), (1155.0, "generic"),
                                           (1157.0, "generic")])
def test_denominator_near_range_flag(lib, spread, answer):
    """The pass centres c on mid, so at f = (0, spread) every sample of this pair has D_n = 2 e^(-spread/2):
    6.3e-250 / 3.8e-250 (fused MODE=1 answers) and 3.2e-251 / 1.2e-251 (the 1e-250 flag sends the pass to the
    log-domain kernel), within a factor 10 of the flag on either side."""
    case = E.spread_pair(spread)
    u, N, f = case["u"], case["N"], case["f"]
    b = E.bands(u, N, f, all_states=False)
    assert b["kernel"] == "fused" and b["mode"] == 1 and b["answer"] == answer
    assert abs(b["logD_min"] - np.log(1e-250)) < np.log(10.0)
    with lib.DeviceProblem(u, N) as p:
        check_sampled_primitives(p, u, N, f, b, CL=1)


@pytest.mark.parametrize("spread", [1199.9, 1200.1])
def test_fused_answers_next_to_spread_limit(lib, spread):
    """u_1 = u_0 + 1144.9 at f = (0, spread): D_n ~ e^-545 keeps clear of the range flag and of the underflow
    test, so the fused MODE=1 kernel answers at spread 1199.9; at 1200.1 the host does not launch it."""
    case = E.offset_pair(1144.9)
    u, N = case["u"], case["N"]
    f = np.array([0.0, spread])
    b = E.bands(u, N, f, all_states=False)
    assert b["answer"] == ("fused" if spread < E.FUSED_SPREAD else "generic")
    with lib.DeviceProblem(u, N) as p:
        check_sampled_primitives(p, u, N, f, b, CL=1)
        np.testing.assert_allclose(p.log_W_nk(f), orc.mbar_log_W_nk(u, N, f), rtol=0, atol=TOL)


@pytest.mark.parametrize("K", [64, 300])
def test_pass_multi_batched(lib, K, monkeypatch):
    """pass_multi with two MODE=3 candidates runs the batched M=2 kernel (clusters above K = 128 when enabled);
    when the shared e0 = exp(-u') of the odd states is floored, both candidates are poisoned and the call falls
    back to the log-domain kernel."""
    monkeypatch.setenv("MBAR_B200_M2_CLUSTERS", "1")
    odd = np.arange(K) % 2 == 1
    for delta, starts, answer in ((500.0, (300.0, 500.0), "fused"), (800.0, (300.0, 100.0), "generic")):
        case = E.offset_copies(K, delta)
        u, N = case["u"], case["N"]
        fs = np.stack([np.where(odd, st, 0.0) for st in starts])
        bs = [E.bands(u, N, fm, all_states=False) for fm in fs]
        assert all(b["mode"] == 3 and b["answer"] == answer for b in bs)
        with lib.DeviceProblem(u, N) as p:
            S2, L2 = p.pass_multi(fs)
            k = p.last_kernels()["pass_kernel"]
            if answer == "fused":
                assert "M=2" in k and f"CL={1 if K <= 128 else 4}," in k, k      # 16 states per thread
            else:
                assert k.startswith("pass_generic_kernel"), k
        for m in range(2):
            assert_log_S(S2[m], ref_log_S(u, N, fs[m]))
            np.testing.assert_allclose(L2[m], orc.log_denominator_n(u, N, fs[m]).sum(), rtol=1e-13, atol=TOL)


# ---------------------------------------------------------------- D. the device exp
def _mp_exp(a):
    import mpmath

    with mpmath.workprec(120):
        return [mpmath.exp(mpmath.mpf(float(x))) for x in a]


def _exp_args():
    rng = np.random.RandomState(2024)
    a = list(rng.uniform(-800.0, 800.0, 100000))
    for x in (708.39, 709.78, 745.13, 707.7, 708.4):
        a += [x, -x, np.nextafter(x, 0), -np.nextafter(x, 0)]
    ln2_32 = np.log(2.0) / 32
    for j in range(-32768, 32768, 97):           # table-index boundaries and the magic-constant rounding ties
        for x in (j * ln2_32, (j + 0.5) * ln2_32):
            a += [x, np.nextafter(x, np.inf), np.nextafter(x, -np.inf)]
    a += [0.0, -0.0, 5e-324, -5e-324, 1e-300]
    return np.array([x for x in a if -800.0 <= x <= 709.7])


@pytest.mark.parametrize("which", [0, 1, 2])
def test_device_exp(lib, which):
    from pymbar_b200.problem import probe_exp

    a = _exp_args()
    got = probe_exp(a, which)
    ref = _mp_exp(a)
    normal = a >= -707.7
    import mpmath

    with mpmath.workprec(120):
        rel = np.array([float(abs(mpmath.mpf(float(g)) - r) / r) for g, r, ok in zip(got, ref, normal) if ok])
    ulp = rel / 2.0 ** -52          # in units of the largest ulp of [1, 2) relative to the value
    small = np.abs(a[normal]) < 1.0
    assert ulp[small].max() <= 2.0, ulp[small].max()
    # Deliberately not 2 ulp beyond |a| = 1: the reduction subtracts n ln2/32 as one double, so the device computes
    # exp(a (1 + d)), d = MBAR_EXP_LN2N_LO / MBAR_EXP_LN2N = 3.35e-17 (up to 108 ulp at |a| = 708).  Applying the
    # remainder costs one more fp64 instruction per entry in the fused pass (DESIGN.md 3.1); beyond that term the
    # error must stay within 2 ulp.
    red = np.abs(a[normal]) * (7.247021293269686e-19 / 0.0216608493924982909)
    assert np.all(rel <= 2 * 2.0 ** -52 + red), (ulp.max(), a[normal][np.argmax(rel - red)])
    # below the normal range: never denormal, never above 2^-1020 (the floor-aware underflow threshold's premise)
    low = got[~normal]
    assert np.all((low >= 0.0) & (low <= 2.0 ** -1020)), low.max()
    assert np.all(got[(a == 0.0)] == 1.0)

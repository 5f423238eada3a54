"""Round-2 kernels through the C ABI: device-resident solver loops (mbar_solvers.py:510-667 adaptive,
self-consistent iteration), the on-device Newton step (Cholesky of H[1:,1:]), the candidate-batched pass and the
three Hessian kernel paths (mbar_solvers.py:395-411), against the oracle / the reference-generated fixtures and
against the host-stepped loops of round 1."""
import numpy as np
import pytest

from oracle import mbar_oracle as orc
from oracle import testsystems as ots
from tests import _cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    import pymbar_b200
    from pymbar_b200 import _lib

    _lib.load()
    if _lib.device_count() == 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return pymbar_b200


@pytest.mark.parametrize("batch", [1, 4])
@pytest.mark.parametrize("name", _cases.ALL)
def test_adaptive_device_resident_vs_reference_and_stepped(lib, name, batch):
    z = _cases.load(name)
    u, N = z["u_kn"], z["N_k"].astype(float)
    s = N > 0
    K = len(N)
    ref = np.zeros(K)
    ref[s] = z["adaptive_x"]
    with lib.DeviceProblem(u, N) as p:
        p.set_loop_mode("device", batch)
        polls0 = p.loop_stats()["polls"]
        f_dev, r = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=0)
        polls = p.loop_stats()["polls"] - polls0
        assert r["success"], r
        assert np.max(np.abs(f_dev[s] - ref[s])) < 1e-8                    # reference adaptive() solution
        assert r["iterations"] == r["nr_iterations"] + r["sci_iterations"]
        # no per-iteration host round trip: one poll per batch of iterations
        assert polls <= -(-r["iterations"] // batch) + 1, (polls, r)
        p.set_loop_mode("stepped")
        f_st, r2 = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=0)
        assert r2["success"]
        assert np.max(np.abs(f_dev[s] - f_st[s])) < 1e-9
        # gradient norm reported by the device loop is the real one at the returned point
        g = p.gradient(f_dev)
        assert abs(np.linalg.norm(g) - r["gnorm"]) < 1e-7 * N.max()


@pytest.mark.parametrize("name", ["small_osc_8x40", "small_empty_state", "osc_50x100"])
def test_sci_device_resident(lib, name):
    z = _cases.load(name)
    u, N = z["u_kn"], z["N_k"].astype(float)
    s = N > 0
    K = len(N)
    ref = np.zeros(K)
    ref[s] = z["adaptive_x"]
    with lib.DeviceProblem(u, N) as p:
        p.set_loop_mode("device", 8)
        polls0 = p.loop_stats()["polls"]
        f_dev, r = p.solve_sci(np.zeros(K), tol=1e-12, maxiter=50000)
        polls = p.loop_stats()["polls"] - polls0
        assert r["success"] and np.max(np.abs(f_dev[s] - ref[s])) < 1e-7, r
        assert polls <= -(-r["iterations"] // 8) + 1
        p.set_loop_mode("stepped")
        f_st, r2 = p.solve_sci(np.zeros(K), tol=1e-12, maxiter=50000)
        assert r2["success"] and abs(r2["iterations"] - r["iterations"]) <= 2
        assert np.max(np.abs(f_dev[s] - f_st[s])) < 1e-10
        # maxiter is honoured exactly by the device loop
        p.set_loop_mode("device", 4)
        f7, r7 = p.solve_sci(np.zeros(K), tol=1e-30, maxiter=7)
        assert r7["iterations"] == 7 and not r7["success"]
        f_host = np.zeros(K)
        for _ in range(7):
            nxt = orc.self_consistent_update(u[s], N[s], f_host[s])
            f_host[s] = nxt - nxt[0]
        np.testing.assert_allclose(f7[s], f_host[s], atol=1e-11)


@pytest.mark.parametrize("name", ["small_osc_8x40", "small_empty_state"])
def test_sci_epilogue_kernel_path_matches_in_kernel_epilogue(lib, name, monkeypatch):
    """MBAR_B200_NO_FUSED_EPILOGUE=1 takes the path of sharded problems without peer memory (pass, all-reduce,
    sci_loop_epilogue_kernel) on one GPU: the same f, bit for bit, as the pass kernel's own epilogue."""
    z = _cases.load(name)
    u, N = z["u_kn"], z["N_k"].astype(float)
    K = len(N)
    f0 = np.zeros(K)
    with lib.DeviceProblem(u, N) as p:
        p.set_loop_mode("device", 4)
        out = {}
        for epilogue in ("in-kernel", "kernel"):
            if epilogue == "kernel":
                monkeypatch.setenv("MBAR_B200_NO_FUSED_EPILOGUE", "1")
            launches0 = p.counters()["launches"]
            f_it = p.sci_iterate(f0, 5)
            launches = p.counters()["launches"] - launches0
            f_sol, r = p.solve_sci(f0, tol=1e-12, maxiter=5000)
            out[epilogue] = (f_it, launches, f_sol, r)
    (f_it, launches, f_sol, r), (g_it, g_launches, g_sol, g_r) = out["in-kernel"], out["kernel"]
    assert (launches, g_launches) == (5, 10)      # one launch per iteration | pass + epilogue kernel
    assert g_it.tobytes() == f_it.tobytes()
    assert r["success"] and g_r["success"] and g_r["iterations"] == r["iterations"]
    assert g_sol.tobytes() == f_sol.tobytes()


def _random_problem(K, N, seed, empty=()):
    u, N_k = ots.oscillators(K, max(1, N // K), seed=seed)
    N_k = N_k.astype(float)
    for e in empty:
        N_k[e] = 0.0
    rng = np.random.RandomState(seed)
    f = rng.normal(scale=0.5, size=K)
    f -= f[0]
    return u, N_k, f


@pytest.mark.parametrize("K", [2, 5, 16, 17, 32, 33, 48, 64, 65, 96, 128, 129, 200, 256, 300, 384])
def test_hessian_kernel_paths_vs_oracle(lib, K):
    """K <= 64: warp-per-tile kernel (KT = 2, 4, 8); K > 64: materialised weights + 128 x 128 block pairs with
    partial last blocks; unsampled states anywhere."""
    empty = () if K < 5 else (1, K - 2)
    u, N_k, f = _random_problem(K, 37 * K if K < 100 else 12 * K, seed=K, empty=empty)
    s = N_k > 0
    with lib.DeviceProblem(u, N_k) as p:
        H = p.hessian(f)
        H_ref = orc.mbar_hessian(u[s], N_k[s], f[s])
        scale = np.max(np.abs(H_ref))
        np.testing.assert_allclose(H[np.ix_(s, s)], H_ref, rtol=1e-10, atol=1e-11 * scale)
        assert np.all(H[~s] == 0) and np.all(H[:, ~s] == 0)
        np.testing.assert_allclose(H, H.T, rtol=0, atol=0)
        names = p.last_kernels()
        assert ("hessian_small_kernel" in names["hessian_kernel"]) == (K <= 64), names
        # the fused pass at this f stored the weights itself (no separate sweep, no exp in the Hessian kernels)
        assert "WST" in names["pass_kernel"] and "weights stored by the fused pass" in names["hessian_kernel"], names
        # all states (weight moments): unsampled rows switched on
        S, G = p.weight_moments(f)
        W = orc.mbar_W_nk(u, N_k, f)
        np.testing.assert_allclose(G, W.T @ W, rtol=1e-9, atol=1e-13 * np.max(W.T @ W))


def test_hessian_weighted_samples(lib):
    """bootstrap multiplicities enter the second moments as sqrt(w_n) on both factors"""
    for K in (24, 130):
        u, N_k, f = _random_problem(K, 40 * K, seed=3 + K)
        rng = np.random.RandomState(5)
        w = rng.poisson(1.0, size=u.shape[1]).astype(float)
        with lib.DeviceProblem(u, N_k) as p:
            p.set_sample_weights(w)
            _, _, G = p.streaming_pass(f, want_G=True)
            W = orc.mbar_W_nk(u, N_k, f)
            np.testing.assert_allclose(G, (W * w[:, None]).T @ W, rtol=1e-9, atol=1e-16)


@pytest.mark.parametrize("K", [3, 40, 161, 200, 320])
def test_device_newton_step_sizes(lib, K):
    """Cholesky + triangular solves on the device: shared-memory variant (n <= 160) and the L2-resident one;
    one adaptive iteration from f = 0 must reproduce the oracle's first iterate."""
    u, N_k, _ = _random_problem(K, 30 * K, seed=100 + K)
    with lib.DeviceProblem(u, N_k) as p:
        p.set_loop_mode("device", 1)
        f1, r = p.solve_adaptive(np.zeros(K), tol=1e-12, maxiter=1, min_sc_iter=0)
        assert r["iterations"] == 1
        ref = orc.adaptive(u, N_k, np.zeros(K), tol=1e-12, options=dict(maxiter=1, min_sc_iter=0))["x"]
        np.testing.assert_allclose(f1, ref, atol=5e-9)
        f_dev, r = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=0)
        assert r["success"] and r["nr_iterations"] >= 1
        g = orc.mbar_gradient(u, N_k, f_dev)
        assert np.max(np.abs(g)) < 1e-7 * N_k.max()


def test_pass_multi(lib):
    z = _cases.load("osc_50x100")
    u, N = z["u_kn"], z["N_k"].astype(float)
    K = len(N)
    rng = np.random.RandomState(1)
    f2 = np.stack([z["f_rand"], z["f_rand"] + rng.normal(scale=0.1, size=K)])
    with lib.DeviceProblem(u, N) as p:
        S, sumL = p.pass_multi(f2)
        for m in range(2):
            S1, sumL1, _ = p.streaming_pass(f2[m])
            np.testing.assert_allclose(S[m], S1, rtol=1e-13)
            np.testing.assert_allclose(sumL[m], sumL1, rtol=1e-14)
            S_ref, L_ref = orc.single_pass_sums(u, N, f2[m])
            np.testing.assert_allclose(S[m], S_ref, rtol=1e-11)
        # wildly different candidates (fused range flag -> robust path) still answer correctly
        f_far = np.stack([z["f_rand"], np.linspace(0, 900, K)])
        S, sumL = p.pass_multi(f_far)
        S_ref, L_ref = orc.single_pass_sums(u, N, f_far[1])
        np.testing.assert_allclose(sumL[1], L_ref.sum(), rtol=1e-12)


def test_device_loop_falls_back_on_extreme_start(lib):
    """A start hundreds of kT from self-consistency underflows the linear-domain sums of the fused kernel: the
    device loop must hand over to the robust stepped path and still converge to the reference solution."""
    z = _cases.load("small_osc_8x40")
    u, N = z["u_kn"], z["N_k"].astype(float)
    K = len(N)
    f0 = np.linspace(0.0, 700.0, K)
    with lib.DeviceProblem(u, N) as p:
        f, r = p.solve_adaptive(f0, tol=1e-12, min_sc_iter=0)
        assert r["success"] and np.max(np.abs(f - z["adaptive_x"])) < 1e-8
        f, r = p.solve_sci(f0, tol=1e-13, maxiter=100000)
        assert r["success"] and np.max(np.abs(f - z["adaptive_x"])) < 1e-7


def test_fp64_peak_probe_and_kernel_names(lib):
    from pymbar_b200.problem import measure_fp64_peak

    dmma, dfma = measure_fp64_peak(0)
    assert 15.0 < dmma < 80.0 and 15.0 < dfma < 80.0, (dmma, dfma)
    z = _cases.load("osc_50x100")
    with lib.DeviceProblem(z["u_kn"], z["N_k"].astype(float)) as p:
        p.gradient(z["f_rand"])
        assert "pass_fused_kernel<" in p.last_kernels()["pass_kernel"]
        p.set_kernel("generic")
        p.gradient(z["f_rand"])
        assert "pass_generic_kernel<" in p.last_kernels()["pass_kernel"]


def test_precondition_u_kn_and_c1_on_gpu(lib):
    """Row a6 (precondition_u_kn, mbar_solvers.py:710-735) through the mirror on the GPU vs probes of the
    reference's output, on BASELINE config C1 (HarmonicOscillatorsTestCase defaults, K=5, N=5000)."""
    z = _cases.load("c1_harmonic_5x1000")
    u, N = z["u_kn"], z["N_k"]
    ms = lib.mbar_solvers
    for tag, f in (("zero", np.zeros(5)), ("rand", z["f_rand"])):
        pc = ms.precondition_u_kn(u, N, f)
        assert pc.shape == u.shape and pc.flags.writeable
        np.testing.assert_allclose(pc[:, :64], z[f"{tag}_precond_head"], rtol=0, atol=1e-11)
        np.testing.assert_allclose(pc.sum(1), z[f"{tag}_precond_rowsum"], rtol=1e-12)
        # the preconditioned objective is ~0 at f (what the shift is for, mbar_solvers.py:726-734)
        np.testing.assert_allclose(ms.mbar_objective(pc, N, f), z[f"{tag}_precond_obj"], atol=1e-7)
    ms.clear_cache()


@pytest.mark.parametrize("method", ["lm", "BFGS", "Newton-CG", "trust-ncg", "dogleg", "CG"])
def test_scipy_methods_against_the_device(lib, method):
    """solve_mbar_once (mbar_solvers.py:738-883) hands device closures (gradient / Hessian / objective) to
    scipy.optimize.root / minimize for every method family of mbar_solvers.py:120-139."""
    z = _cases.load("small_osc_8x40")
    ms = lib.mbar_solvers
    u, N = z["u_kn"], z["N_k"].astype(float)
    f, results = ms.solve_mbar_once(u, N, np.zeros(len(N)), method=method, tol=1e-12)
    f_ref, _ = orc.solve_mbar_once(u, N, np.zeros(len(N)), method=method, tol=1e-12)
    # (CG stops on its own loose criterion: both sides sit ~1e-7 from the optimum)
    assert np.max(np.abs(f - f_ref)) < (1e-6 if method == "CG" else 1e-7)
    assert np.max(np.abs(f - z["fk_default"])) < 1e-6
    ms.clear_cache()


def test_hessian_beyond_2048_states(lib):
    """K > 2048: generic pass + the block-pair Hessian in several launches (153 pairs at K = 2100); ADVICE r1:
    mbar_hessian must not refuse what mbar_b200_create accepts."""
    K = 2100
    u, N_k, f = _random_problem(K, 2 * K, seed=77)
    with lib.DeviceProblem(u, N_k) as p:
        H = p.hessian(f)
        H_ref = orc.mbar_hessian(u, N_k, f)
        np.testing.assert_allclose(H, H_ref, rtol=1e-9, atol=1e-11 * np.max(np.abs(H_ref)))


@pytest.mark.parametrize("K", [2, 5, 16, 31, 64, 100, 128, 200, 256, 300, 512, 700, 1024])
def test_candidate_batched_pass_kernel(lib, K):
    """pass_fused_kernel<..., M = 2>: two candidate vectors on the same staged tile (single CTA up to K = 128,
    clusters of 2 / 4 / 8 CTAs above), against two single-candidate launches and the oracle."""
    import os

    empty = () if K < 5 else (2,)
    u, N_k, f = _random_problem(K, (40 if K < 300 else 6) * K, seed=500 + K, empty=empty)
    s = N_k > 0
    rng = np.random.RandomState(K)
    f2 = np.stack([f, f + rng.normal(scale=0.3, size=K)])
    f2[:, ~s] = 0.0
    # (above 128 states the batched kernel needs clusters and is not the default: switch it on for the test)
    os.environ["MBAR_B200_M2_CLUSTERS"] = "1"
    try:
        _run_m2_case(lib, u, N_k, f2, s, rng)
    finally:
        del os.environ["MBAR_B200_M2_CLUSTERS"]


def _run_m2_case(lib, u, N_k, f2, s, rng):
    with lib.DeviceProblem(u, N_k) as p:
        S, sumL = p.pass_multi(f2)
        assert "M=2" in p.last_kernels()["pass_kernel"], p.last_kernels()
        for m in range(2):
            S1, sumL1, _ = p.streaming_pass(f2[m])
            np.testing.assert_allclose(S[m], S1, rtol=1e-12, atol=1e-300)
            np.testing.assert_allclose(sumL[m], sumL1, rtol=1e-13)
            S_ref, L_ref = orc.single_pass_sums(u[s], N_k[s], f2[m][s])
            np.testing.assert_allclose(S[m][s], S_ref, rtol=1e-11)
            np.testing.assert_allclose(sumL[m], L_ref.sum(), rtol=1e-12)
        # bootstrap multiplicities ride through the batched kernel too (masked family)
        w = rng.poisson(1.0, size=u.shape[1]).astype(float)
        p.set_sample_weights(w)
        Sw, sumLw = p.pass_multi(f2)
        S1, sumL1, _ = p.streaming_pass(f2[1])
        np.testing.assert_allclose(Sw[1], S1, rtol=1e-12, atol=1e-300)
        np.testing.assert_allclose(sumLw[1], sumL1, rtol=1e-13)


@pytest.mark.parametrize("K", [24, 48, 96, 192, 384, 768])
def test_24_row_kernel_family(lib, K):
    """K = 8 warps x 24 states (x CTAs of a cluster): the R = 24 family of the fused pass, unmasked when every
    state is sampled, masked otherwise; pass, weights for the Hessian and device loop against the oracle."""
    for empty in ((), (3,)):
        per = 30 if K < 300 else 8
        u, N_k, f = _random_problem(K, per * K, seed=900 + K, empty=empty)
        for e in empty:      # an unsampled state has no samples in the data set (sum N_k = N, as pymbar requires)
            u = np.delete(u, np.s_[e * per:(e + 1) * per], axis=1)
        s = N_k > 0
        with lib.DeviceProblem(u, N_k) as p:
            S, sumL, _ = p.streaming_pass(f)
            assert "R=24" in p.last_kernels()["pass_kernel"], p.last_kernels()
            assert ("FULL" in p.last_kernels()["pass_kernel"]) == (len(empty) == 0)
            S_ref, L_ref = orc.single_pass_sums(u[s], N_k[s], f[s])
            np.testing.assert_allclose(S[s], S_ref, rtol=1e-11)
            np.testing.assert_allclose(sumL, L_ref.sum(), rtol=1e-12)
            H = p.hessian(f)
            np.testing.assert_allclose(H[np.ix_(s, s)], orc.mbar_hessian(u[s], N_k[s], f[s]), rtol=1e-9,
                                       atol=1e-11 * N_k.max())
            if K <= 192:
                fk, r = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=0)
                assert r["success"]
                g = orc.mbar_gradient(u[s], N_k[s], fk[s])
                assert np.max(np.abs(g)) < 1e-7 * N_k.max()


@pytest.mark.parametrize("name", ["small_osc_8x40", "osc_50x100", "osc_200x50"])
def test_adaptive_iteration_as_cuda_graph(lib, name):
    """After the first batch a context runs, one adaptive iteration is captured into a CUDA graph and relaunched;
    the graph is reused across batches and solves (quantised centring).  Same answers as the kernel-by-kernel
    path, and the counters show the graph actually carried the iterations."""
    z = _cases.load(name)
    u, N = z["u_kn"], z["N_k"].astype(float)
    K = len(N)
    with lib.DeviceProblem(u, N) as p:
        p.set_loop_mode("device", 2)
        f1, r1 = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=0)      # batch 1 plain, later batches graph
        st1 = p.loop_stats()
        f2, r2 = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=0)      # graph from the first batch on
        st2 = p.loop_stats()
        assert r1["success"] and r2["success"]
        assert np.max(np.abs(f1 - z["adaptive_x"])) < 1e-8 and np.max(np.abs(f2 - f1)) < 1e-12
        assert r2["iterations"] == r1["iterations"]
        assert st2["graph_launches"] - st1["graph_launches"] >= r2["iterations"], (st1, st2, r2)
        assert st2["graph_captures"] == st1["graph_captures"] == 1, (st1, st2)   # one capture serves both solves
        # a different start changes nothing about the launch parameters either
        f3, r3 = p.solve_adaptive(z["f_rand"], tol=1e-12, min_sc_iter=0)
        assert r3["success"] and np.max(np.abs(f3 - f1)) < 1e-8

"""The device-resident adaptive loop (loops.cu: adapt_pre_kernel, newton_build_kernel, newton_kernel<SMEM>, the
ridge retry, the Newton range check, adapt_post_kernel, poll_batches and the fallback of solve_adaptive_device),
step by step against the long-double restatement of tests/_adaptive.py, and its loop mechanics against itself and
the host-stepped loop.

One step at a time: solve_adaptive(f, maxiter=1) chained from the device's own output, each step compared with the
restatement from the same f: the chosen candidate (self-consistent: within its propagated bound; Newton: the
backward error of the step it took, which holds at any condition of A, and the forward error that implies), the
reported gradient norm, max_delta, and the choice wherever the two candidates' norms differ by more than their
bounds.  Newton sizes n = 1 ... 2047 put the system on both sides of the shared-memory limit (n <= 158), of the
256 / 512 / 1024-thread bands, and of K = 128 (one candidate-batched pass above it two launches)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import mbar_oracle as orc
from tests import _adaptive as AD
from tests import _large_k as LK
from tests import _moments as M

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = (1, 2, 31, 32, 95, 96, 157, 158, 159, 160, 255, 511, 1023, 1024, 2047)
TOL = 1e-12
WORST = {}     # n -> worst backward-error ratio of a device Newton step


@pytest.fixture(scope="module")
def lib():
    import pymbar_b200
    from pymbar_b200 import _lib

    _lib.load()
    if _lib.device_count() == 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return pymbar_b200


def shape_case(n):
    """A permuted, well-overlapping ladder with n + 1 sampled states; unsampled states first, in the middle and last
    (where K stays within 2048), bootstrap multiplicities on every third shape (each state's samples redrawn N_k times
    with replacement: about Poisson(1) each, and the MBAR equations keep a root), gamma = 0.5 on every other."""
    i = SHAPES.index(n)
    extra = 2048 - (n + 1)
    where = [(0,), (1,), (0, 1, 2)][i % 3]
    n_un = min(len(where), extra)
    K = n + 1 + n_un
    unsampled = tuple(sorted({(0, K // 2, K - 1)[w] for w in where[:n_un]}))
    case = LK.permuted_ladder(K, 10 if n < 100 else 3, seed=700 + n, unsampled=unsampled, gaps=(1.5,), f_noise=0.5)
    s = case["N"] > 0
    f = case["f"].copy()
    f -= f[np.flatnonzero(s)[0]]
    f[~s] = 0.0
    mult = None
    if i % 3 == 2:
        rng = np.random.RandomState(n)
        owner = np.repeat(np.arange(K), case["N"].astype(int))
        mult = np.zeros(owner.size)
        for k in np.flatnonzero(s):
            idx = np.flatnonzero(owner == k)
            mult[idx] = rng.multinomial(idx.size, np.full(idx.size, 1.0 / idx.size))
    case.update(f=f, mult=mult, gamma=0.5 if i % 2 else 1.0)
    return case


def check_step(p, case, f, min_sc_iter, label):
    """One device step from f against the restatement; returns (f_next, result, restated iteration)."""
    u, N, gamma = case["u"], case["N"], case["gamma"]
    s = N > 0
    it = AD.iteration(u, N, f, gamma=gamma, tol=TOL, min_sc_iter=min_sc_iter, mult=case["mult"])
    f1, r = p.solve_adaptive(f, tol=TOL, maxiter=1, min_sc_iter=min_sc_iter, gamma=gamma)
    assert r["iterations"] == 1 and r["iterations"] == r["nr_iterations"] + r["sci_iterations"], (label, r)
    st = p.adaptive_stats()
    assert st["device_iterations"] == 1 and not st["fell_back"], (label, st)
    assert np.all(f1[~s] == f[~s]), label                       # unsampled states carried through untouched
    choice = "nr" if r["nr_iterations"] else "sci"
    if min_sc_iter:
        assert choice == "sci", label
    free = it["active"][1:]
    g0 = it["active"][0]
    assert f1[g0] == 0.0, label
    if choice == "sci":
        d = np.abs(f1 - it["f_sci"].astype(np.float64))
        worst = float((d[s] / it["tol_fsci"][s]).max())
        assert worst <= 1.0, (label, "f_sci", worst)
        S_c, tolS_c, df = it["S_sci"], it["tolS_sci"], float(d[s].max())
    else:
        assert it["f_nr"] is not None, label
        ratio, res, bound = AD.newton_backward(it, f, f1, gamma)
        WORST[it["n"]] = max(WORST.get(it["n"], 0.0), ratio)
        assert ratio <= 1.0, (label, "backward", ratio, res, bound)
        d = np.abs(f1 - it["f_nr"].astype(np.float64))
        fwd = gamma * AD.forward_bound(it, f, f1, gamma) + AD.EPS * np.abs(f1).max()
        assert float(d[free].max()) <= fwd, (label, "forward", float(d[free].max()), fwd)
        S_c, tolS_c, df = it["S_nr"], it["tolS_nr"], float(d[free].max())
    # the reported gradient norm: that of the chosen candidate
    gn = float(it[f"gn_{choice}"])
    tol_gn = AD.gn_tolerance(N, S_c, tolS_c, gn, df, it["S"].astype(np.float64))
    assert abs(r["gnorm"] ** 2 - gn) <= tol_gn, (label, "gnorm", r["gnorm"] ** 2, gn, tol_gn)
    # the choice, where the candidates' norms are further apart than their bounds
    if not min_sc_iter and it["f_nr"] is not None:
        bnd = {}
        for c in ("sci", "nr"):
            dfc = float(np.max(it["tol_fsci"][s])) if c == "sci" else \
                gamma * AD.forward_bound(it, f, it["f_nr"].astype(np.float64), gamma)
            bnd[c] = AD.gn_tolerance(N, it[f"S_{c}"], it[f"tolS_{c}"], float(it[f"gn_{c}"]), dfc,
                                     it["S"].astype(np.float64))
        if abs(float(it["gn_sci"]) - float(it["gn_nr"])) > bnd["sci"] + bnd["nr"]:
            assert choice == it["choice"], (label, "choice", it["gn_sci"], it["gn_nr"], bnd)
    # max_delta: the relative change of the device's own step
    md = float(AD.rel_change(f1[free], f[free], min(1e-8, TOL)).max()) if free.size else 0.0
    assert abs(r["max_delta"] - md) <= 8 * AD.EPS * md + 1e-300, (label, r["max_delta"], md)
    return f1, r, it


@pytest.mark.parametrize("min_sc_iter", [0, 1])
@pytest.mark.parametrize("n", SHAPES)
def test_step_by_step_against_extended_precision(lib, n, min_sc_iter):
    case = shape_case(n)
    K = len(case["N"])
    # the restatement costs about 15 s per step at n = 2047 (a device step well under one): a few forced
    # self-consistent steps, and up to twelve free ones.  Full Newton steps converge in those; gamma = 0.5 only
    # halves the error per step, so there the gradient norm must have dropped instead
    steps = (3 if n < 1000 else 2) if min_sc_iter else 12
    converges = case["gamma"] == 1.0
    with lib.DeviceProblem(case["u"], case["N"]) as p:
        if case["mult"] is not None:
            p.set_sample_weights(case["mult"])
        p.set_loop_mode("device", 4)
        f = case["f"]
        done = False
        gnorms = []
        for step in range(steps):
            f, r, _ = check_step(p, case, f, min_sc_iter, f"n={n} K={K} msc={min_sc_iter} step {step}")
            gnorms.append(r["gnorm"])
            if r["success"]:
                done = True
                break
        st = p.adaptive_stats()
        assert st["newton_smem"] == (n <= 158) and st["newton_threads"] == (1024 if n >= 96 else 512 if n >= 32
                                                                              else 256), st
    if not min_sc_iter:
        if converges:
            assert done, (n, "did not converge in", steps, gnorms)
        else:
            assert gnorms[-1] < 1e-3 * gnorms[0], (n, gnorms)
        assert n in WORST, (n, "no Newton step was taken")
        print(f"n={n}: worst backward-error ratio {WORST[n]:.3g} over {len(gnorms)} steps")


def clusters(sizes, gap, seed, n_per=20):
    """Harmonic ladders (gaps of 1.5) of the given sizes, one after another with `gap` between them: cross-cluster
    weights about exp(-gap^2 / 2).  gap = inf: every cross-cluster energy is +inf.  State order permuted, one
    unsampled state in the middle."""
    rng = np.random.RandomState(seed)
    centres, owner_cluster = [], []
    x0 = 0.0
    for c, m in enumerate(sizes):
        centres += list(x0 + 1.5 * np.arange(m))
        owner_cluster += [c] * m
        x0 = centres[-1] + (gap if np.isfinite(gap) else 100.0)
    K = len(centres) + 1
    perm = rng.permutation(K)
    centres = np.concatenate([centres, [0.0]])[perm]
    cl = np.concatenate([owner_cluster, [-1]])[perm]
    N = np.where(cl >= 0, float(n_per), 0.0)
    owner = np.repeat(np.arange(K), N.astype(int))
    x = centres[owner] + rng.normal(size=owner.size)
    u = 0.5 * (x[None, :] - centres[:, None]) ** 2
    if not np.isfinite(gap):
        u[(cl[:, None] != cl[owner][None, :]) & (cl[:, None] >= 0)] = np.inf
    return u, N, cl


def per_cluster_reference(u, N, cl):
    f = np.zeros(len(N))
    for c in range(cl.max() + 1):
        rows = np.flatnonzero(cl == c)
        cols = np.flatnonzero(np.isin(np.repeat(np.arange(len(N)), N.astype(int)), rows))
        fc = orc.adaptive(u[np.ix_(rows, cols)], N[rows], np.zeros(rows.size), tol=1e-12,
                          options=dict(min_sc_iter=0))["x"]
        f[rows] = fc - fc[0]
    return f


@pytest.mark.parametrize("gap", [34.0, np.inf])
def test_clusters_weak_and_decoupled(lib, gap):
    """Four clusters coupled at about e^-578 (1e-251), or not at all (+inf cross energies).  The offset between
    clusters is then not (or barely) identified: A is singular to working precision, so the device factorisation
    meets a non-positive pivot and takes the ridge retry (or, had the pivot come out positive, a candidate far out of
    range would be rejected).  What can be identified: no fault, finite f, and every within-cluster difference
    against each cluster solved on its own.  The host-stepped loop (additive ridge) is held to the same answer; its
    iteration count differs (DESIGN.md)."""
    u, N, cl = clusters((5, 7, 4, 6), gap, seed=11)
    ref = per_cluster_reference(u, N, cl)
    for mode in ("device", "stepped"):
        with lib.DeviceProblem(u, N) as p:
            p.set_loop_mode(mode, 4)
            f, r = p.solve_adaptive(np.zeros(len(N)), tol=1e-12, maxiter=300, min_sc_iter=0)
            st = p.adaptive_stats()
        print(f"gap={gap} {mode}: {r} {st}")
        assert r["iterations"] == r["nr_iterations"] + r["sci_iterations"]
        s = N > 0
        assert np.all(np.isfinite(f[s]))
        for c in range(cl.max() + 1):
            rows = np.flatnonzero(cl == c)
            d = (f[rows] - f[rows[0]]) - ref[rows]
            assert np.max(np.abs(d)) < 1e-7, (mode, gap, c, d)
        if mode == "device":
            assert st["ridge_retries"] + st["newton_rejected"] + st["newton_failed"] >= 1, st
            assert st["newton_failed"] <= st["ridge_retries"], st


def solve_ladder(K=40, seed=3):
    case = M.ladder(K, 20, gaps=(1.5,), unsampled=(K // 2,), seed=seed, f_noise=0.5)
    return case["u"], case["N"]


@pytest.mark.parametrize("maxiter", [6, 8, 9])
def test_maxiter_inside_and_on_batch_edge(lib, maxiter):
    """Batch 4: maxiter 6 ends inside the second batch, 8 on its edge, 9 one into the third; the count is exact and
    the iterate is the host-stepped loop's after as many steps."""
    u, N = solve_ladder()
    K = len(N)
    with lib.DeviceProblem(u, N) as p:
        p.set_loop_mode("device", 4)
        f, r = p.solve_adaptive(np.zeros(K), tol=1e-30, maxiter=maxiter, min_sc_iter=100)
        assert r["iterations"] == maxiter == r["sci_iterations"] and not r["success"], r
        p.set_loop_mode("stepped")
        f2, r2 = p.solve_adaptive(np.zeros(K), tol=1e-30, maxiter=maxiter, min_sc_iter=100)
        assert r2["iterations"] == maxiter
        np.testing.assert_allclose(f, f2, rtol=0, atol=1e-11)


@pytest.mark.parametrize("min_sc_iter", [0, 1, 3, 5])
def test_first_steps_are_self_consistent(lib, min_sc_iter):
    u, N = solve_ladder(seed=4)
    K = len(N)
    with lib.DeviceProblem(u, N) as p:
        p.set_loop_mode("device", 2)
        f, r = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=min_sc_iter)
        assert r["success"] and r["sci_iterations"] >= min(min_sc_iter, r["iterations"]), r
        f3, r3 = p.solve_adaptive(np.zeros(K), tol=1e-12, maxiter=min_sc_iter, min_sc_iter=min_sc_iter) \
            if min_sc_iter else (None, dict(nr_iterations=0))
        assert r3["nr_iterations"] == 0, r3
        p.set_loop_mode("stepped")
        f2, r2 = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=min_sc_iter)
        # (the last steps' choice sits at rounding level, so only the count is compared with the stepped loop)
        assert r2["sci_iterations"] >= min(min_sc_iter, r2["iterations"]), r2
        assert abs(r2["iterations"] - r["iterations"]) <= 1, (r, r2)
        np.testing.assert_allclose(f, f2, rtol=0, atol=1e-10)


def test_batch_sizes_agree(lib):
    """Batch 1, 4 and 64: the same choices and iteration count, f to 1e-11 (the quantised centring of the fused pass
    is recomputed at every poll, so the bits may differ)."""
    u, N = solve_ladder(K=120, seed=5)
    K = len(N)
    res = {}
    with lib.DeviceProblem(u, N) as p:
        for batch in (1, 4, 64):
            p.set_loop_mode("device", batch)
            res[batch] = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=2, gamma=0.5)
    f1, r1 = res[1]
    assert r1["success"]
    for batch in (4, 64):
        f, r = res[batch]
        assert (r["iterations"], r["nr_iterations"], r["sci_iterations"]) == \
               (r1["iterations"], r1["nr_iterations"], r1["sci_iterations"]), (batch, r, r1)
        np.testing.assert_allclose(f, f1, rtol=0, atol=1e-11)


def run_worker(tmp_path, **env):
    out = str(tmp_path / ("_".join(env) + ".npz"))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "adaptive_loop_worker.py"), out],
                       capture_output=True, text=True, timeout=1800, cwd=ROOT, env=dict(os.environ, **env))
    assert r.returncode == 0 and "ADAPTIVE_WORKER_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    z = np.load(out)
    return {k: z[k] for k in z.files if k != "meta"}, json.loads(str(z["meta"]))


def test_graph_replay_matches_plain_launches(lib, tmp_path):
    """The captured iteration relaunched as a CUDA graph gives the bits of the kernel-by-kernel launches at the
    same batch size; the two-launch candidate passes (no M = 2) the same choices and f to 1e-12."""
    sys.path.insert(0, ROOT)
    from tests.adaptive_loop_worker import solves

    here = solves(lib.DeviceProblem)
    plain, meta = run_worker(tmp_path, MBAR_B200_NO_GRAPH="1")
    nom2, meta2 = run_worker(tmp_path, MBAR_B200_NO_M2="1")
    for name, (f, r) in here.items():
        assert plain[name].tobytes() == f.tobytes(), name
        assert meta[name]["iterations"] == r["iterations"] and meta[name]["nr_iterations"] == r["nr_iterations"]
        assert (meta2[name]["iterations"], meta2[name]["nr_iterations"]) == (r["iterations"], r["nr_iterations"])
        np.testing.assert_allclose(nom2[name], f, rtol=0, atol=1e-12)


def spread_ladder(K=16, spread=1203.0, seed=8, n_per=51):
    """A well-overlapping ladder with state offsets b_k: f_k moves by exactly b_k, so the exact c = f + log N spreads
    just over the fused pass's limit of 1200."""
    rng = np.random.RandomState(seed)
    x = 1.5 * np.arange(K)
    N = np.full(K, float(n_per))
    owner = np.repeat(np.arange(K), n_per)
    u = 0.5 * ((x[owner] + rng.normal(size=owner.size))[None, :] - x[:, None]) ** 2
    f_base = orc.adaptive(u, N, np.zeros(K), tol=1e-13, options=dict(min_sc_iter=0))["x"]
    b = (spread - (f_base[-1] - f_base[0])) * np.linspace(0.0, 1.0, K)
    return u + b[:, None], N, f_base + b


@pytest.mark.parametrize("min_sc_iter", [0, 2])
def test_fallback_after_first_poll_keeps_the_accounting(lib, min_sc_iter):
    """Started at 0.95 f, the fused pass accepts the first batch; once f spreads past 1200 it refuses, and the
    host-stepped loop finishes from the last polled f.  The counts of both parts add up, the first min_sc_iter
    steps are self-consistent, and the whole solve takes the steps of the host-stepped loop from the same start."""
    u, N, f_exact = spread_ladder()
    K = len(N)
    f0 = 0.95 * f_exact
    assert np.ptp(f_exact + np.log(N)) > 1200.0 > np.ptp(f0 + np.log(N))
    with lib.DeviceProblem(u, N) as p:
        p.set_loop_mode("device", 1)
        f, r = p.solve_adaptive(f0, tol=1e-12, min_sc_iter=min_sc_iter)
        st = p.adaptive_stats()
        assert st["fell_back"] and st["device_iterations"] >= 1, (st, r)
        assert r["success"] and r["iterations"] == r["nr_iterations"] + r["sci_iterations"], (r, st)
        assert r["sci_iterations"] >= min(min_sc_iter, r["iterations"]), r
        p.set_loop_mode("stepped")
        f2, r2 = p.solve_adaptive(f0, tol=1e-12, min_sc_iter=min_sc_iter)
        assert (r["iterations"], r["nr_iterations"], r["sci_iterations"]) == \
               (r2["iterations"], r2["nr_iterations"], r2["sci_iterations"]), (r, r2, st)
        np.testing.assert_allclose(f, f2, rtol=0, atol=1e-8)
        np.testing.assert_allclose(f, f_exact - f_exact[0], rtol=0, atol=1e-6)

"""Every entry point from 2049 to 8192 states, and the generic pass at every warps-per-CTA configuration, against the
sparse long-double reference of tests/_large_k.py.

The generic pass sizes itself from K: 8 warps per CTA up to K = 1070, one warp per CTA from K = 5865 (DESIGN 3.2).
Each case takes K on both sides of every change, three sample counts (fewer tiles than warps, about one tile per
warp, three tiles per warp), with and without unsampled (log-domain) rows and with multiplicities, and asserts the
launched configuration against `generic_plan`.  The Hessian cases run 561 and 2080 block pairs (5 and 17 launches of
at most 128) on ladders whose state order is permuted, so neighbouring states couple across arbitrary block pairs.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import _large_k as LK
from tests import _moments as M

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADROOM = {}          # check -> largest |error| / tolerance seen
EPS = M.EPS


@pytest.fixture(scope="module")
def lib():
    import pymbar_b200
    from pymbar_b200 import _lib

    _lib.load()
    if _lib.device_count() == 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    yield pymbar_b200
    for label in sorted(HEADROOM):
        print(f"\n[large K] {label}: max |error|/tol = {HEADROOM[label]:.3g}", end="")
    print()


@pytest.fixture(scope="module")
def sm_count(lib):
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def within(label, err, tol):
    """max |err| / tol (<= 1 passes), recorded for the headroom table."""
    err = np.abs(np.asarray(err, np.float64))
    tol = np.asarray(tol, np.float64)
    r = float(np.max(err / tol)) if err.size else 0.0
    HEADROOM[label] = max(HEADROOM.get(label, 0.0), r)
    worst = int(np.argmax(err / tol)) if err.size else -1
    assert r <= 1.0, (label, r, worst)


def expect_pass_kernel(p, plan, log_rows):
    name = p.last_kernels()["pass_kernel"]
    rows = "log-domain rows" if log_rows else "linear rows"
    assert name == f"pass_generic_kernel<{rows}> grid={plan['grid']} warps={plan['W']}", (name, plan)


# ---- 1. the generic pass at every W -----------------------------------------------------------------------------
VARIANTS = ("linear", "log", "mult")


def generic_matrix(sm_count=132):
    """(K, regime, variant) for every K of generic_ks and every regime.  Each K runs all three variants: 'linear'
    (every state sampled, pass_generic_kernel<linear rows>) goes to a regime with at least K samples, rotating
    over those; the other two regimes take 'log' (unsampled rows) and 'mult' (multiplicities and an unsampled row)."""
    out = []
    for i, K in enumerate(LK.generic_ks()):
        full = [r for r in LK.REGIMES if LK.regime_n(K, r, sm_count) >= K]
        lin = full[i % len(full)]
        rest = [r for r in LK.REGIMES if r != lin]
        other = ("log", "mult") if i % 2 == 0 else ("mult", "log")
        var = {lin: "linear", rest[0]: other[0], rest[1]: other[1]}
        out += [(K, r, var[r]) for r in LK.REGIMES]
    return out


GEN = generic_matrix()


def generic_case(K, regime, variant, sm):
    N = LK.regime_n(K, regime, sm)
    seed = K * 3 + LK.REGIMES.index(regime)
    if variant == "linear":
        assert N >= K, (K, regime)
        c = LK.permuted_ladder(K, N / K, seed, n_inf=7)
    elif N < K:
        # few samples: most states unsampled; a compressed ladder keeps every unsampled row within the stored range
        uns = LK.few_sampled(K, N, seed)
        n_s = K - len(uns)
        c = LK.permuted_ladder(K, N / n_s, seed, unsampled=uns, gaps=(min(39.0, 1200.0 / K),))
    else:
        uns = {"linear": (), "log": (0, K // 2, K - 1), "mult": (K // 3,)}[variant]
        c = LK.permuted_ladder(K, N / (K - len(uns)), seed, unsampled=uns, n_inf=7)
    return c


@pytest.mark.parametrize("K,regime,variant", GEN, ids=[f"K{K}-{r}-{v}" for K, r, v in GEN])
def test_generic_pass(lib, sm_count, K, regime, variant):
    c = generic_case(K, regime, variant, sm_count)
    u, N_k, f = c["u"], c["N"], c["f"]
    N = u.shape[1]
    s = N_k > 0
    mult = c["mult"] if variant == "mult" else None
    plan = LK.generic_plan(K, N, sm_count)
    if regime == "few":
        assert plan["n_tiles"] < plan["W"] or (plan["W"] <= 2 and N < 32), plan
    else:
        assert plan["tiles_per_warp"] == (1 if regime == "one" else 3) and plan["grid"] == plan["max_grid"], plan
    ref = LK.sparse_moments_ld(u, N_k, f, mult=mult, all_rows=True)
    tol = LK.pass_tolerances(ref, N_k, plan, mult)
    log_rows = variant != "linear"
    assert log_rows == bool((~s).any()), (variant, int((~s).sum()))       # the case is what its id says
    tag = f"W={plan['W']} {regime}"
    with lib.DeviceProblem(u, N_k) as p:
        if K <= LK.FUSED_K_MAX:
            p.set_kernel("generic")
        if mult is not None:
            p.set_sample_weights(mult)
        S0, sL0, _ = p.streaming_pass(f)
        expect_pass_kernel(p, plan, log_rows)
        S1, sL1, _ = p.streaming_pass(f)
        g = p.gradient(f)
        obj = p.objective(f)
        L = p.log_denominator(f)
        fn0 = p.self_consistent_update(f)
        expect_pass_kernel(p, plan, log_rows)
        fn1 = p.self_consistent_update(f)
    assert np.array_equal(S0, S1) and sL0 == sL1 and np.array_equal(fn0, fn1)
    S_ref = ref["S"].astype(np.float64)
    within(f"S {tag}", (S0 - S_ref)[s], tol["S"][s])
    assert np.all(S0[~s] == 0)
    sumL_ref = float(ref["sumL"])
    within(f"sumL {tag}", sL0 - sumL_ref, LK.sumL_tolerance(ref, plan, mult))
    g_ref = N_k * (S_ref - 1.0)
    within(f"gradient {tag}", (g - g_ref)[s], (N_k * tol["S"] + 2 * EPS * (np.abs(g_ref) + N_k))[s])
    nf = np.sum(N_k * f)
    obj_ref = sumL_ref - nf
    tol_obj = LK.sumL_tolerance(ref, plan, mult) + (K + 2) * EPS * np.sum(np.abs(N_k * f)) + 2 * EPS * abs(obj_ref)
    within(f"objective {tag}", obj - obj_ref, tol_obj)
    within(f"log_denominator {tag}", L - ref["L"].astype(np.float64), tol["L"])
    check_update(fn0, f, ref, tol, s, f"update {tag}")


def check_update(fn, f, ref, tol, s, label, log_all=False):
    """f - log S_k: sampled rows through the relative error of S, unsampled rows through that of log S (every row
    when the pass ran all rows in the log domain)."""
    logS = ref["logS"].astype(np.float64)
    S = ref["S"].astype(np.float64)
    exp_f = f - logS
    zero = np.isneginf(logS)                           # S_k = 0 (all its weights have multiplicity 0): f = +inf
    assert np.all(fn[zero] == np.inf), label
    with np.errstate(divide="ignore", invalid="ignore"):
        lin = np.log1p(np.minimum(tol["S"] / np.where(s & ~zero, S, 1.0), 0.5)) * 1.01
        t = np.where(s & (not log_all), lin, tol["logS"])
    t = t + 2 * EPS * (np.abs(f) + np.abs(exp_f))
    within(label, (fn - exp_f)[~zero], t[~zero])


# ---- 2. the all-log-domain retry --------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [3000, 8192])
@pytest.mark.parametrize("offset", [700.0, 750.0])
def test_log_domain_retry(lib, sm_count, K, offset):
    """A sampled state's f raised by 700 or 750 leaves its neighbours' S_k below 1e-280: the pass is repeated with
    every row in the log domain (run_pass attempt 2), which the kernel name shows for a problem without unsampled
    states."""
    c = LK.permuted_ladder(K, 1, seed=K + int(offset), gaps=(1.5,))
    u, N_k, f = c["u"], c["N"], c["f"].copy()
    assert np.all(N_k > 0)
    f[K // 2] += offset
    ref = LK.sparse_moments_ld(u, N_k, f, all_rows=True)
    assert np.min(ref["S"]) < 1e-280
    plan = LK.generic_plan(K, u.shape[1], sm_count)
    tol = LK.pass_tolerances(ref, N_k, plan)
    with lib.DeviceProblem(u, N_k) as p:
        fn = p.self_consistent_update(f)
        expect_pass_kernel(p, plan, True)
        S, _, _ = p.streaming_pass(f)
        expect_pass_kernel(p, plan, True)
    s = N_k > 0
    # every row came from the log-domain sums: hold it to their tolerance, not to the linear sum's absolute floor
    check_update(fn, f, ref, tol, s, f"update (log-domain retry) K={K}", log_all=True)
    S_ref = ref["S"].astype(np.float64)
    within(f"S (log-domain retry) K={K}", S - S_ref, S_ref * np.expm1(tol["logS"]) * 1.01 + 2 * EPS * S_ref)


# ---- 3. moments and Hessian above 2048 --------------------------------------------------------------------------
def check_sparse_G(label, G, ref, N_k, all_rows, S, N):
    """G (the API's scaling) against the support of Ghat entry by entry (_moments.entry_tol's tolerance), every entry
    off the support under its floor, symmetry, and row sums tied to the same call's S."""
    K = len(N_k)
    s = N_k > 0
    sc = np.where(s, N_k, 1.0 if all_rows else 0.0)
    assert np.array_equal(G, G.T)
    i, j, v = ref["Gi"], ref["Gj"], ref["Gv"]
    diag = i == j
    wmax = float(np.sqrt(np.max(v[diag].astype(np.float64)))) if diag.any() else 1.0
    A = ref["A"]
    rho = 8 * EPS * (A[i] + A[j]) + 8 * EPS * np.sqrt(float(N)) + 64 * EPS      # _moments.entry_tol
    alpha = 4.0 * N * M.FLOOR * max(1.0, wmax) + float(ref["drop"])
    tol = rho * v + alpha
    Gd_sup = G[i, j] * sc[i] * sc[j]
    r = M.excess(Gd_sup, v, tol)
    HEADROOM[f"Ghat {label}"] = max(HEADROOM.get(f"Ghat {label}", 0.0), r)
    assert r <= 1.0, (label, r)
    off = G.copy()
    off[i, j] = 0.0
    off[j, i] = 0.0
    off *= sc[:, None]
    off *= sc[None, :]
    within(f"Ghat off support {label}", np.max(np.abs(off)), alpha)
    del off
    if not all_rows:
        assert np.all(G[~s] == 0) and np.all(G[:, ~s] == 0)
    # row sums over sampled columns = s_i S_i
    tol_full = np.zeros(K)
    np.add.at(tol_full, i, np.where(s[j], tol.astype(np.float64), 0.0))
    np.add.at(tol_full, j, np.where(s[i] & ~diag, tol.astype(np.float64), 0.0))
    lhs = (G[:, s] * sc[s][None, :]).sum(axis=1) * sc
    rows = np.ones(K, bool) if all_rows else s
    bound = 2 * tol_full + K * EPS * np.abs(lhs) + K * alpha
    within(f"row sums {label}", (lhs - sc * S)[rows], bound[rows])


def moments_case(K):
    return LK.permuted_ladder(K, 2 if K < 8192 else 1, seed=K, unsampled=(0, K // 2, K - 1))


def device_moments(p, c):
    """streaming_pass(want_G) with the multiplicities, weight_moments and hessian on DeviceProblem `p`, each twice
    (the repeat is compared here and only its equality kept, to hold one K x K copy per call at K = 8192)."""
    f = c["f"]
    d = {}
    p.set_sample_weights(c["mult"])
    try:
        d["S"], _, d["G"] = p.streaming_pass(f, want_G=True)
        d["G_name"] = p.last_kernels()["hessian_kernel"]
        S1, _, G1 = p.streaming_pass(f, want_G=True)
        d["G_same"] = bool(np.array_equal(d["S"], S1) and np.array_equal(d["G"], G1))
        del G1
    finally:
        p.set_sample_weights(None)
    d["Sw"], d["Gw"] = p.weight_moments(f)
    d["Gw_name"] = p.last_kernels()["hessian_kernel"]
    S1, G1 = p.weight_moments(f)
    d["Gw_same"] = bool(np.array_equal(d["Sw"], S1) and np.array_equal(d["Gw"], G1))
    del G1
    d["H"] = p.hessian(f)
    d["H_name"] = p.last_kernels()["hessian_kernel"]
    d["H_same"] = bool(np.array_equal(d["H"], p.hessian(f)))
    return d


def check_moments(K, c, d, expect, label):
    u, N_k, f, mult = c["u"], c["N"], c["f"], c["mult"]
    N = u.shape[1]
    s = N_k > 0
    for key in ("G_name", "Gw_name", "H_name"):
        assert expect in str(d[key]), (key, d[key], expect)
    assert d["G_same"] and d["Gw_same"] and d["H_same"]
    ref = LK.sparse_moments_ld(u, N_k, f, mult=mult, all_rows=False, want_G=True)
    check_sparse_G(f"{label} streaming_pass(want_G, mult) K={K}", d["G"], ref, N_k, False, d["S"], N)
    ref = LK.sparse_moments_ld(u, N_k, f, all_rows=True, want_G=True)
    check_sparse_G(f"{label} weight_moments K={K}", d["Gw"], ref, N_k, True, d["Sw"], N)
    # hessian: sampled rows, -H off the diagonal is the same Ghat
    off = np.outer(s, s)
    np.fill_diagonal(off, False)
    sc = np.where(s, N_k, 1.0)
    Gs = d["Gw"] * sc[:, None] * sc[None, :]
    np.testing.assert_allclose(-d["H"][off], Gs[off], rtol=4 * EPS, atol=1e-300)
    assert np.all(d["H"][~s] == 0) and np.all(d["H"][:, ~s] == 0)


def block_pairs(K):
    nB = -(-K // 128)
    return nB * (nB + 1) // 2


@pytest.mark.parametrize("K", [4100, 8192])
def test_moments_and_hessian(lib, K):
    c = moments_case(K)
    with lib.DeviceProblem(c["u"], c["N"]) as p:
        d = device_moments(p, c)
    check_moments(K, c, d, f"weights_kernel + hessian_big_kernel (128x128 block pairs: {block_pairs(K)},", "big")


def test_inplace_hessian_4100(lib, tmp_path):
    """hessian_inplace_kernel, which the library takes when the 8 K N weight buffer cannot be allocated, at K = 4100
    (561 block pairs in five launches, four of them starting at a nonzero pair index), forced in a subprocess: the
    switch is read once per process."""
    out = str(tmp_path / "inplace.npz")
    env = dict(os.environ, MBAR_B200_HESSIAN_INPLACE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "large_k_inplace_worker.py"), out],
                       capture_output=True, text=True, timeout=1200, cwd=ROOT, env=env)
    assert r.returncode == 0 and "INPLACE_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    z = np.load(out)
    d = {k: (z[k].item() if z[k].ndim == 0 else z[k]) for k in z.files}
    check_moments(4100, moments_case(4100), d, "hessian_inplace_kernel", "inplace")


# ---- 4. log W at 8192 -------------------------------------------------------------------------------------------
def test_log_w_8192(lib, sm_count):
    K = 8192
    c = LK.permuted_ladder(K, 0.5, seed=81)
    u, N_k, f = c["u"], c["N"], c["f"]
    N = u.shape[1]
    ref = LK.sparse_moments_ld(u, N_k, f)
    L = ref["L"].astype(np.float64)
    x = ref["x"]
    rows_per_chunk = (64 << 20) // (K * 32 * 8) * 32
    n0 = 32 * 37
    n = N - n0 - 5
    assert n > 2 * rows_per_chunk and n0 % rows_per_chunk != 0

    def check(lw, a, label):
        worst = 0.0
        for b in range(0, lw.shape[0], 256):
            rr = np.arange(a + b, min(a + lw.shape[0], a + b + 256))
            uu = u[:, rr].T
            up = uu - x[rr, None]
            clamped = ~(up < 1e6)
            got = lw[b:b + len(rr)]
            assert np.all(np.isneginf(got[clamped])), label
            exp = f[None, :] - uu - L[rr, None]
            t = ref["dL"][rr, None] + 3 * EPS * (np.abs(f)[None, :] + np.abs(up) + np.abs(L[rr] + x[rr])[:, None])
            e = np.where(clamped, 0.0, np.abs(got - exp) / t)
            worst = max(worst, float(e.max()))
        HEADROOM[f"log W {label}"] = worst
        assert worst <= 1.0, (label, worst)

    plan = LK.generic_plan(K, N, sm_count)
    with lib.DeviceProblem(u, N_k) as p:
        full = p.log_W_nk(f)
        expect_pass_kernel(p, plan, True)
        check(full, 0, "all rows, pageable")
        del full
        page = p.log_W_nk(f, rows=n, row0=n0)
        check(page, n0, "rows, pageable")
        holder = lib.PinnedArray((n, K))
        try:
            p.log_W_nk(f, rows=n, row0=n0, out=holder.array)
            assert np.array_equal(holder.array, page)
        finally:
            holder.free()


# ---- 5. the self-consistent iteration at W = 3 ------------------------------------------------------------------
def test_sci_iterate_w3(lib, sm_count):
    K = 2700
    c = LK.permuted_ladder(K, 2, seed=27, gaps=(1.5,))
    u, N_k, f = c["u"], c["N"], c["f"]
    plan = LK.generic_plan(K, u.shape[1], sm_count)
    assert plan["W"] == 3
    fh = f.copy()
    tol = 0.0
    refs = []
    for _ in range(3):
        ref = LK.sparse_moments_ld(u, N_k, fh, all_rows=True)
        t = LK.pass_tolerances(ref, N_k, plan)
        nxt = fh - ref["logS"].astype(np.float64)
        step = np.max(t["S"] / ref["S"].astype(np.float64)) * 1.01 + 4 * EPS * np.max(np.abs(nxt))
        tol = 2 * tol + 2 * step          # the step's own error, and what the map does to the one before (Lipschitz 2)
        fh = nxt - nxt[0]
        refs.append((fh.copy(), tol))
    with lib.DeviceProblem(u, N_k) as p:
        for it in (1, 3):
            fd = p.sci_iterate(f, it)
            expect_pass_kernel(p, plan, False)
            within(f"sci_iterate x{it} W=3", fd - refs[it - 1][0], np.full(K, refs[it - 1][1]))


def ld_fixed_point_residual(u, N_k, f, plan):
    """max_k |f'_k - f_k| of the long-double self-consistent update f' = f - log S (gauge f'_0 = 0 taken from f),
    and the device-rounding part of it that a converged f may still show."""
    ref = LK.sparse_moments_ld(u, N_k, f, all_rows=True)
    t = LK.pass_tolerances(ref, N_k, plan)
    nxt = f - ref["logS"].astype(np.float64)
    nxt -= nxt[0] - f[0]
    step = 2 * float(np.max(t["S"] / ref["S"].astype(np.float64))) + 4 * EPS * float(np.max(np.abs(nxt)))
    return float(np.max(np.abs(nxt - f))), step


def test_solve_sci_w3(lib, sm_count):
    """solve_sci above 2048 states (the host-stepped loop over the generic pass, W = 3) converges to a fixed point of
    the long-double update.  The states span 13.5 standard deviations, so the self-consistent iteration converges in
    a few hundred steps."""
    K, tol = 2700, 1e-12
    c = LK.permuted_ladder(K, 2, seed=2700, gaps=(0.005,))
    u, N_k = c["u"], c["N"]
    plan = LK.generic_plan(K, u.shape[1], sm_count)
    assert plan["W"] == 3
    with lib.DeviceProblem(u, N_k) as p:
        f, r = p.solve_sci(np.zeros(K), tol=tol, maxiter=20000)
        assert r["success"], r
        expect_pass_kernel(p, plan, False)
    resid, step = ld_fixed_point_residual(u, N_k, f, plan)
    # the stopping rule: relative change below tol (absolute below tol max|f|); what is left of the contraction
    # after that is a small multiple of the last change
    bound = 20 * tol * max(1.0, float(np.max(np.abs(f)))) + step
    HEADROOM["solve_sci fixed point W=3"] = resid / bound
    assert resid <= bound, (resid, bound, r)


# ---- 6. augmented contexts at the cap, and the facade past it ---------------------------------------------------
def test_augmented_at_the_cap(lib, sm_count):
    from pymbar_b200 import _lib

    K0 = 4096
    c = LK.permuted_ladder(K0, 1, seed=4096)
    u, N_k, f = c["u"], c["N"], c["f"]
    E = _lib.MAX_STATES - K0
    rng = np.random.RandomState(1)
    extra = u[rng.randint(0, K0, size=E)] + rng.uniform(0.0, 3.0, size=(E, 1))
    with lib.DeviceProblem(u, N_k) as p:
        with p.augmented(extra) as q:
            assert q.K == _lib.MAX_STATES
            fa = np.concatenate([f, np.zeros(E)])
            fn = q.self_consistent_update(fa)
            expect_pass_kernel(q, LK.generic_plan(q.K, u.shape[1], sm_count), True)
        with pytest.raises(_lib.MbarB200Error) as e:
            p.augmented(np.vstack([extra, extra[:1]]))
        assert e.value.status == -1
    Na = np.concatenate([N_k, np.zeros(E)])
    ua = np.vstack([u, extra])
    ref = LK.sparse_moments_ld(ua, Na, fa, all_rows=True)
    plan = LK.generic_plan(_lib.MAX_STATES, u.shape[1], sm_count)
    tol = LK.pass_tolerances(ref, Na, plan)
    check_update(fn, fa, ref, tol, Na > 0, "augmented to the cap: update")


def test_facade_expectations_both_sides_of_the_cap(lib, sm_count, monkeypatch):
    """compute_expectations_inner of an MBAR object with K states appends 2K rows for state-dependent observables:
    at 3K = 2100 the device answers (checked against the long-double restatement of the augmented problem); at
    3K > 8192 the original method does."""
    from pymbar_b200 import _lib, facade
    from tests.test_large_k_cpu import OriginalInnerMBAR

    from pymbar_b200 import problem

    # the pass kernel of every self-consistent update the facade runs
    seen = []
    orig_update = problem.DeviceProblem.self_consistent_update

    def recording_update(self, f_k):
        out = orig_update(self, f_k)
        seen.append((self.K, self.N, self.last_kernels()["pass_kernel"]))
        return out

    monkeypatch.setattr(problem.DeviceProblem, "self_consistent_update", recording_update)
    OriginalInnerMBAR.calls = []
    facade.install_on(OriginalInnerMBAR)
    try:
        for K, served in ((700, True), (_lib.MAX_STATES // 3 + 1, False)):
            c = LK.permuted_ladder(K, 3, seed=K, gaps=(1.5,))
            m = OriginalInnerMBAR.__new__(OriginalInnerMBAR)
            m.u_kn, m.N_k, m.f_k, m.K = c["u"], c["N"].astype(np.int64), c["f"], K
            N = c["u"].shape[1]
            A = np.random.RandomState(K).uniform(0.5, 2.0, size=(K, N))
            table = np.array([np.arange(K), np.arange(K)])
            s0 = dict(facade.STATS)
            seen.clear()
            r = m.compute_expectations_inner(A, c["u"], table)
            if not served:
                assert r == {"original": True} and not seen
                assert facade.STATS["expectations_fallbacks"] == s0["expectations_fallbacks"] + 1
                continue
            assert facade.STATS["expectations"] == s0["expectations"] + 1
            plan = LK.generic_plan(3 * K, N, sm_count)
            assert seen == [(3 * K, N, f"pass_generic_kernel<log-domain rows> grid={plan['grid']} warps={plan['W']}")]
            guard = 4.0 * np.finfo(np.float64).eps
            lo = A.min(axis=1)
            floor = lo - np.abs(guard * lo)
            extra = np.vstack([c["u"], c["u"] - np.log(A - floor[:, None])])
            ua = np.vstack([c["u"], extra])
            Na = np.concatenate([c["N"], np.zeros(2 * K)])
            fa = np.concatenate([c["f"], np.zeros(2 * K)])
            ref = LK.sparse_moments_ld(ua, Na, fa, all_rows=True)
            f_app = -ref["logS"][K:]                   # appended rows: f = 0 - log S
            f_l, f_s = f_app[:K], f_app[K:]
            obs = np.exp((f_l - f_s).astype(np.float64)) + floor
            tol = LK.pass_tolerances(ref, Na, plan)
            within("facade f (3K = 2100)", r["f"] - f_l.astype(np.float64),
                   tol["logS"][K:2 * K] + 4 * EPS * np.abs(f_l.astype(np.float64)))
            tobs = (tol["logS"][K:2 * K] + tol["logS"][2 * K:] + 8 * EPS * np.abs((f_l - f_s).astype(np.float64))) \
                * np.abs(obs - floor) * 1.01 + 2 * EPS * np.abs(obs)
            within("facade observables (3K = 2100)", r["observables"] - obs, tobs)
        assert len(OriginalInnerMBAR.calls) == 1
    finally:
        facade.uninstall_from(OriginalInnerMBAR)

"""Every instantiation of the fused pass (K <= 2048) against the sparse long-double reference of tests/_large_k.py.

The matrix of tests/_fused.py runs each of the 90 kernels `fused_enqueue` can launch in three sample-count regimes
(fewer stages than CTA groups, one stage per group, at least 2 NS + 1 stages per group so that every ring slot wraps)
for MODE 3 and in one of them for MODE 1, at both K edges of every (R, CL) band.  MODE 1 comes from the data: half the
sampled states carry an offset of 900 on their energies and on f, which leaves every weight as it was and puts
max c - min c near 900.  Each case runs every entry point on one context, asserts after each call that the launched
kernel is the one `fused_plan` names (a silent fall-back to the generic kernel fails), that repeated calls are
bit-identical, and holds each output to the tolerance of _large_k's reference and tolerance model with the plan's
reduction depth and the device exp's floor divided by the pass's denominator.  The K at which the last CTA of a
cluster used to read unset state constants run right after a log-domain generic pass.
"""
import numpy as np
import pytest

from tests import _fused as F
from tests import _large_k as LK
from tests import _moments as M_
from tests import test_gpu_large_k as LKT

pytestmark = pytest.mark.gpu
HEADROOM = {}
EPS = M_.EPS
OFFSET = 900.0          # MODE 1 cases: energy and f offset of every other sampled state


@pytest.fixture(scope="module")
def lib():
    import pymbar_b200
    from pymbar_b200 import _lib

    _lib.load()
    if _lib.device_count() == 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    yield pymbar_b200
    for label in sorted(HEADROOM):
        print(f"\n[fused] {label}: max |error|/tol = {HEADROOM[label]:.3g}", end="")
    print()


@pytest.fixture(scope="module")
def sm_count(lib):
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def within(label, err, tol):
    err = np.abs(np.asarray(err, np.float64))
    tol = np.asarray(tol, np.float64)
    r = float(np.max(err / tol)) if err.size else 0.0
    HEADROOM[label] = max(HEADROOM.get(label, 0.0), r)
    assert r <= 1.0, (label, r, int(np.argmax(err / tol)) if err.size else -1)


def family(plan):
    return (f"R={plan['R']} CL={plan['CL']} {'FULL' if plan['full'] else 'MASKED'} MODE={plan['mode']}"
            + (" WST" if plan["wst"] else "") + (" M=2" if plan["M"] == 2 else ""))


def expect(p, plan):
    assert plan is not None
    name = p.last_kernels()["pass_kernel"]
    assert name == plan["name"], (name, plan["name"])


# ---- cases ------------------------------------------------------------------------------------------------------------
def make_case(K, N, mode, content, seed):
    uns, gaps, N_k = F.case_sampling(K, N, content)
    n_s = K - len(uns)
    c = LK.permuted_ladder(K, N / n_s, seed, unsampled=uns, gaps=gaps, n_inf=7 if N >= K > 1 else 0)
    assert np.array_equal(c["N"], N_k) and c["u"].shape[1] == N
    u, f = c["u"], c["f"]
    if mode == 1:
        s = np.flatnonzero(N_k > 0)
        off = np.zeros(K)
        off[s[1::2]] = OFFSET
        u = u + off[:, None]
        f = f + off
    # Poisson multiplicities, zeros included, but the first sample of every sampled state counts at least once: a
    # state whose every sample has multiplicity 0 (likely at one or two samples per state) has an S that underflows,
    # and the pass rightly hands it to the log-domain kernel
    mult = c["mult"].copy()
    first = (np.cumsum(N_k) - N_k)[N_k > 0].astype(int)
    mult[first] = np.maximum(mult[first], 1.0)
    return dict(u=u, N=N_k, f=f, mult=mult if content == "mult" else None)


def c_abs(f, N_k):
    """Per row, the larger magnitude of the centred constant c_k - mid the device holds in a pass over the sampled
    rows and in an all-state pass (unsampled rows at log N = -80)."""
    s = N_k > 0
    logNe = np.where(s, np.log(np.where(s, N_k, 1.0)), F.LOG_EPS_UNSAMPLED)
    return np.maximum(np.abs(f + logNe - c_mid(f, N_k, False)), np.abs(f + logNe - c_mid(f, N_k, True)))


def c_mid(f, N_k, all_states):
    s = N_k > 0
    c = np.where(s, f + np.log(np.where(s, N_k, 1.0)), f + F.LOG_EPS_UNSAMPLED)
    c = c if all_states else c[s]
    return 0.5 * (np.max(c) + np.min(c))


def floor_bound(ref, f, N_k, mult, all_states):
    """Per row, what entries on the device exp's floor (at most 2^-1020, times E_k = e^(c_k - mid) in MODE 3) add to
    S_k once divided by D_n = e^(L'_n - mid) and N_k (e^-80 for an unsampled row of an all-state pass)."""
    mid = c_mid(f, N_k, all_states)
    s = N_k > 0
    logNe = np.where(s, np.log(np.where(s, N_k, 1.0)), F.LOG_EPS_UNSAMPLED)
    m = np.ones(len(ref["x"])) if mult is None else mult
    logD = (ref["L"].astype(np.float64) + ref["x"]) - mid
    inv = float(np.sum(m * np.exp(-logD)))
    return M_.FLOOR * np.maximum(1.0, np.exp(f + logNe - mid)) * inv / np.exp(logNe), mid


def check_pass(label, ref, plan, N_k, f, mult, S, sL, g=None, obj=None, L=None):
    s = N_k > 0
    floor, mid = floor_bound(ref, f, N_k, mult, False)
    tol = LK.pass_tolerances(ref, N_k, plan, mult, floor=floor)
    S_ref = ref["S"].astype(np.float64)
    within(f"S {label}", (S - S_ref)[s], tol["S"][s])
    assert np.all(S[~s] == 0)
    sumL_ref = float(ref["sumL"])
    tsum = LK.sumL_tolerance(ref, plan, mult, mid)
    within(f"sumL {label}", sL - sumL_ref, tsum)
    if g is not None:
        g_ref = N_k * (S_ref - 1.0)
        within(f"gradient {label}", (g - g_ref)[s], (N_k * tol["S"] + 2 * EPS * (np.abs(g_ref) + N_k))[s])
    if obj is not None:
        obj_ref = sumL_ref - np.sum(N_k * f)
        t = tsum + (len(f) + 2) * EPS * np.sum(np.abs(N_k * f)) + 2 * EPS * abs(obj_ref)
        within(f"objective {label}", obj - obj_ref, t)
    if L is not None:
        within(f"log_denominator {label}", L - ref["L"].astype(np.float64), tol["L"] + 2 * EPS * abs(mid))


def weight_floor(ref, f, N_k, mult):
    """Bound on what floored entries add to any Ghat_ij through the stored weights w_nk = sqrt(m_n) e_kn / D_n:
    each is off by at most d_n = sqrt(m_n) 2^-1020 max(1, e^(c_max - mid)) / D_n and w_nk <= sqrt(m_n), so
    Ghat_ij by at most sum_n (2 sqrt(m_n) d_n + d_n^2)."""
    mid = c_mid(f, N_k, False)
    s = N_k > 0
    cmax = float(np.max((f + np.log(np.where(s, N_k, 1.0)))[s]))
    m = np.ones(len(ref["x"])) if mult is None else mult
    logD = (ref["L"].astype(np.float64) + ref["x"]) - mid
    d = np.sqrt(m) * M_.FLOOR * max(1.0, np.exp(cmax - mid)) * np.exp(-logD)
    return float(np.sum(2 * np.sqrt(m) * d + d * d))


def check_weights(ref_G, ref, N_k, S, G, plan, f, mult):
    """streaming_pass(want_G) on the weight-storing pass: Ghat entry by entry where the reference holds it (the
    helper of tests/test_gpu_large_k.py, its absolute term raised by the floored entries the weight store divides by
    D_n), else symmetry and the row sums tied to the same call's S."""
    s = N_k > 0
    assert np.array_equal(G, G.T)
    N = plan["N"]
    label = family(plan)
    wf = weight_floor(ref, f, N_k, mult)
    if ref_G is not None:
        ref_G = dict(ref_G, drop=ref_G["drop"] + wf)
        LKT.check_sparse_G(label, G, ref_G, N_k, False, S, N)
        for key in (f"Ghat {label}", f"Ghat off support {label}", f"row sums {label}"):
            HEADROOM[key] = max(HEADROOM.get(key, 0.0), LKT.HEADROOM.pop(key))
        return
    sc = np.where(s, N_k, 0.0)
    A = ref["A"]
    rho = 16 * EPS * np.max(A) + 8 * EPS * np.sqrt(float(N)) + 64 * EPS
    lhs = (G[:, s] * sc[s][None, :]).sum(axis=1) * sc
    alpha = 4.0 * N * M_.FLOOR + float(ref["drop"]) + wf
    bound = (2 * rho + len(N_k) * EPS) * np.abs(sc * S) + len(N_k) ** 2 * alpha
    within(f"row sums {label}", (lhs - sc * S)[s], bound[s])


def sci_reference(u, N_k, f, plan, steps):
    """The stepped long-double iteration f <- f - log S, gauge on the first sampled state, with the bound the device
    is held to after each step (its own error plus twice the previous one)."""
    s = N_k > 0
    first = int(np.flatnonzero(s)[0])
    fh = f.copy()
    tol = 0.0
    out = []
    for _ in range(steps):
        ref = LK.sparse_moments_ld(u, N_k, fh, all_rows=True, c_abs=np.abs(fh + np.log(np.where(s, N_k, 1.0))
                                                                          - c_mid(f, N_k, False)))
        floor, _ = floor_bound(ref, fh, N_k, None, False)
        t = LK.pass_tolerances(ref, N_k, plan, floor=floor)
        nxt = fh - ref["logS"].astype(np.float64)
        step = np.max((t["S"] / ref["S"].astype(np.float64))[s]) * 1.01 + 4 * EPS * np.max(np.abs(nxt[s]))
        tol = 2 * tol + 2 * step
        fh = np.where(s, nxt - nxt[first], fh)
        out.append((fh.copy(), tol))
    return out


def run_case(lib, sm, K, regime, M, mode, content, monkeypatch, poison=False):
    N = F.regime_n(K, regime, M, sm)
    seed = K * 7 + F.REGIMES.index(regime) * 3 + F.CONTENTS.index(content) + 100 * mode
    c = make_case(K, N, mode, content, seed)
    u, N_k, f, mult = c["u"], c["N"], c["f"], c["mult"]
    s = N_k > 0
    n_act = int(s.sum())
    w = mult is not None
    sp = F.c_spread(f, N_k, False)
    sp_all = F.c_spread(f, N_k, True)
    assert F.mode_of(sp) == mode and sp < F.SPREAD_MAX, (sp, mode)
    kw = dict(n_active=n_act, weighted=w, sm_count=sm)
    plan = F.fused_plan(K, N, spread=sp, **kw)
    plan_u = F.fused_plan(K, N, all_states=n_act < K, spread=sp_all if n_act < K else sp, **kw)
    plan_w = F.fused_plan(K, N, want_w=True, spread=sp, **kw)
    m2c = M == 2 and F.geometry(K, 2)["CL"] > 1
    if m2c:
        monkeypatch.setenv("MBAR_B200_M2_CLUSTERS", "1")
    ca = c_abs(f, N_k)
    ref = LK.sparse_moments_ld(u, N_k, f, mult=mult, all_rows=True, c_abs=ca)
    want_G = N * K <= 4_000_000
    ref_G = LK.sparse_moments_ld(u, N_k, f, mult=mult, all_rows=False, want_G=True, c_abs=ca) if want_G else None
    with lib.DeviceProblem(u, N_k) as p:
        if poison:
            # a log-domain generic pass leaves -inf running maxima in shared memory on every SM it ran on
            assert n_act < K
            p.set_kernel("generic")
            p.self_consistent_update(f)
            assert p.last_kernels()["pass_kernel"].startswith("pass_generic_kernel<log-domain rows>")
            p.set_kernel("auto")
        if w:
            p.set_sample_weights(mult)
        S0, sL0, _ = p.streaming_pass(f)
        expect(p, plan)
        S1, sL1, _ = p.streaming_pass(f)
        g = p.gradient(f)
        expect(p, plan)
        obj = p.objective(f)
        expect(p, plan)
        L = p.log_denominator(f)
        expect(p, plan)
        fn0 = p.self_consistent_update(f)
        expect(p, plan_u)
        fn1 = p.self_consistent_update(f)
        Sw, sLw, G = p.streaming_pass(f, want_G=True)
        expect(p, plan_w)
        Sw1, sLw1, G1 = p.streaming_pass(f, want_G=True)
        assert np.array_equal(Sw, Sw1) and sLw == sLw1 and np.array_equal(G, G1)
        del G1
        multi = None
        if M == 2:
            rng = np.random.RandomState(seed)
            f2 = f + np.where(s, rng.normal(scale=0.3, size=K), 0.0)
            assert F.mode_of(F.c_spread(f2, N_k, False)) == 3
            plan_m = F.fused_plan(K, N, M=2, m2_clusters=m2c, spread=sp, **kw)
            Sm, sLm = p.pass_multi(np.stack([f, f2]))
            expect(p, plan_m)
            Sm1, sLm1 = p.pass_multi(np.stack([f, f2]))
            assert np.array_equal(Sm, Sm1) and np.array_equal(sLm, sLm1)
            multi = (f2, Sm, sLm, plan_m)
        sci = None
        if regime == "one" and not w:
            fd = p.sci_iterate(f, 3)
            expect(p, plan)
            sci = fd
    assert np.array_equal(S0, S1) and sL0 == sL1 and np.array_equal(fn0, fn1)
    fam = family(plan)
    check_pass(fam, ref, plan, N_k, f, mult, S0, sL0, g, obj, L)
    # the update: sampled rows through S, unsampled rows (all-state pass, linear sums) through log S
    floor_u, _ = floor_bound(ref, f, N_k, mult, n_act < K)
    tol_u = LK.pass_tolerances(ref, N_k, plan_u, mult, floor=floor_u)
    key = f"update {family(plan_u)}"
    LKT.check_update(fn0, f, ref, tol_u, s, key)
    HEADROOM[key] = max(HEADROOM.get(key, 0.0), LKT.HEADROOM.pop(key))
    check_pass(family(plan_w), ref, plan_w, N_k, f, mult, Sw, sLw)
    check_weights(ref_G, ref, N_k, Sw, G, plan_w, f, mult)
    if multi is not None:
        f2, Sm, sLm, plan_m = multi
        ref2 = LK.sparse_moments_ld(u, N_k, f2, mult=mult, all_rows=True, c_abs=c_abs(f2, N_k))
        check_pass(family(plan_m), ref, plan_m, N_k, f, mult, Sm[0], sLm[0])
        check_pass(family(plan_m) + " candidate 2", ref2, plan_m, N_k, f2, mult, Sm[1], sLm[1])
    if sci is not None:
        fh, t = sci_reference(u, N_k, f, plan, 3)[-1]
        within(f"sci_iterate x3 {fam}", (sci - fh)[s], np.full(int(s.sum()), t))
        assert np.array_equal(sci[~s], f[~s])


MATRIX = F.variant_matrix()


@pytest.mark.parametrize("K,regime,M,mode,content", MATRIX,
                         ids=[f"K{K}-{r}-M{m}-MODE{md}-{c}" for K, r, m, md, c in MATRIX])
def test_fused_variant(lib, sm_count, K, regime, M, mode, content, monkeypatch):
    run_case(lib, sm_count, K, regime, M, mode, content, monkeypatch)


OVERRUN = [(K, 1) for K in F.overrun_ks(1, pad=32)] + [(K, 2) for K in F.overrun_ks(2, pad=32)]


@pytest.mark.parametrize("K,M", OVERRUN, ids=[f"K{K}-M{m}" for K, m in OVERRUN])
def test_last_cta_constants_after_log_domain_pass(lib, sm_count, K, M, monkeypatch):
    """The K at which the last CTA of a cluster read state constants past the 32 it used to zero, MASKED MODE 3,
    right after a log-domain generic pass on the same context (a stale -inf or NaN constant would poison D_n and
    send the pass to the generic kernel, which the kernel-name assertion catches)."""
    run_case(lib, sm_count, K, "one", M, 3, "unsampled", monkeypatch, poison=True)

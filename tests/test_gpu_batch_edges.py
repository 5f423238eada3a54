"""The batched MBAR pass (batch.cu) at the edges of the fp64 range, against the long-double restatement of
tests/_batch_edges.py: the _moments ladders, the exponent families at their known f, requests on both sides of every
flag threshold, isolation of flagged requests, large absolute energies, the chunk geometry of more than 4096 chunks'
worth of tiles, and mbar_many end to end.  Every item runs plain and as a weighted replicate slot, with and without
all rows, with the Gram."""
import gc
import time

import numpy as np
import pytest

from pymbar_b200 import DeviceMbarBatch, DeviceProblem, estimators
from pymbar_b200.mbar_many import mbar_many
from tests import _batch_edges as BE
from tests import _edges as E
from tests import _moments as M

pytestmark = pytest.mark.gpu


def _slots_for(cases, seed):
    """One slot per case with multinomial counts (a whole chunk of zeros where the problem has three chunks)."""
    return [BE.slot_counts(c["u"].shape[1], len(c["N"]), seed + i) for i, c in enumerate(cases)]


def _verify(c, counts, d, all_rows, want_G, what):
    """Assert the flag where predict_flag is clear; hold an unflagged request to the restatement.  Returns the flag."""
    ref = BE.restate(c["u"], c["N"], c["f"], all_rows, mult=counts)
    flag, margin = BE.predict_flag(c["u"], c["N"], c["f"], all_rows, want_G, counts, ref=ref)
    if BE.is_clear(margin):
        assert d["flag"] == flag, (what, "flag", flag, margin)
    if d["flag"]:
        return True
    wmax = 1.0 if counts is None else float(np.max(counts))
    BE.check_request(d, ref, c["N"], all_rows, c["u"].shape[1], wmax=wmax, what=what)
    return False


def _run_cases(cases, extra_slots=(), want_G=True):
    """Every case plain and as a weighted slot (plus extra (case index, counts) slots), all_rows False and True.
    Returns {(name, weighted, all_rows): flag}."""
    counts = _slots_for(cases, 100)
    slot_case = list(range(len(cases))) + [i for i, _ in extra_slots]
    counts += [c for _, c in extra_slots]
    flags = {}
    with DeviceMbarBatch([c["u"] for c in cases], [c["N"] for c in cases]) as b:
        b.set_replicates(slot_case, counts)
        for all_rows in (False, True):
            plain = b.moments([c["f"] for c in cases], want_G=want_G, all_rows=all_rows)
            for c, d in zip(cases, plain):
                flags[(c["name"], False, all_rows)] = _verify(c, None, d, all_rows, want_G,
                                                              (c["name"], "plain", all_rows))
            w = b.moments([cases[i]["f"] for i in slot_case], want_G=want_G, all_rows=all_rows,
                          slots=np.arange(len(slot_case)))
            for s, (i, d) in enumerate(zip(slot_case, w)):
                key = (cases[i]["name"] + ("" if s < len(cases) else f"_slot{s}"), True, all_rows)
                flags[key] = _verify(cases[i], counts[s], d, all_rows, want_G, key)
    return flags


# ---- 1. the _moments ladders with K <= 64 ---------------------------------------------------------------------------
def test_ladders():
    cases = [BE.ladder_case(n) for n in BE.LADDERS]
    flags = _run_cases(cases)
    # mild f: nothing at a threshold, so nothing may be flagged
    assert not any(flags.values()), [k for k, v in flags.items() if v]


# ---- 2. the exponent families at their known f ----------------------------------------------------------------------
def _big_slot_case():
    """K = 3 with N = 65535 samples: (u_0, u_0 + 5, u_0 - 60), the last state empty, f known."""
    u0 = E.base_samples(BE.UINT16_MAX, 23)
    return dict(name="n65535", u=np.stack([u0, u0 + 5.0, u0 - 60.0]), N=np.array([32768.0, 32767.0, 0.0]),
                f=np.array([0.0, 5.0, -60.0]))


def test_families_at_known_f():
    cases = BE.family_cases() + [_big_slot_case()]
    big = len(cases) - 1
    flags = _run_cases(cases, extra_slots=[(big, BE.all_on_one(BE.UINT16_MAX, 40000))])
    assert not any(flags.values()), [k for k, v in flags.items() if v]
    # at the known f, S_k = 1 for every state and log S_k = 0 for the empty ones, past 1e6 included
    with DeviceMbarBatch([c["u"] for c in cases], [c["N"] for c in cases]) as b:
        out = b.moments([c["f"] for c in cases], all_rows=True)
    for c, d in zip(cases, out):
        ref = BE.restate(c["u"], c["N"], c["f"], True, want_G=False)
        assert np.max(np.abs(ref["S"].astype(float) - 1.0)) < 8 * BE.EPS * max(1.0, np.max(np.abs(c["f"]))), c["name"]
        assert np.all(np.abs(d["log_S"]) <= BE.log_s_tol(ref["A"], c["u"].shape[1], len(c["N"])) + 1e-13), \
            (c["name"], d["log_S"])


# ---- 3. the flag at each threshold -----------------------------------------------------------------------------------
def _threshold_cases():
    return [dict(name=n, u=u, N=N_k, f=f) for n, u, N_k, f in BE.threshold_cases()]


@pytest.mark.parametrize("want_G", [False, True])
def test_flag_at_each_threshold(want_G):
    cases = _threshold_cases()
    flags = _run_cases(cases, want_G=want_G)
    want = {
        "sampled_S_1e-280-0.5": True, "sampled_S_1e-280+0.5": False,
        "unsampled_S_DBL_MAX-0.5": want_G, "unsampled_S_DBL_MAX+0.5": True,
        "gram_DBL_MAX-0.5": False, "gram_DBL_MAX+0.5": want_G, "gram_400kT_below_f0": want_G,
        "unsampled_all_inf": False,
    }
    for name, flag in want.items():
        assert flags[(name, False, True)] == flag, (name, want_G)
    # with sampled rows only, no unsampled rule applies
    for name in ("unsampled_S_DBL_MAX+0.5", "gram_DBL_MAX+0.5", "gram_400kT_below_f0"):
        assert not flags[(name, False, False)], name


def test_gram_overflow_is_flagged():
    """An unsampled row whose largest weight is above e^355: S_k is finite but Ghat_kk = sum w^2 overflows.  The
    request must be flagged; an unflagged one must return a finite Gram."""
    cases = [c for c in _threshold_cases() if c["name"] in ("gram_DBL_MAX+0.5", "gram_400kT_below_f0")]
    with DeviceMbarBatch([c["u"] for c in cases], [c["N"] for c in cases]) as b:
        out = b.moments([c["f"] for c in cases], want_G=True, all_rows=True)
    for c, d in zip(cases, out):
        assert np.all(np.isfinite(d["S"])), c["name"]
        assert d["flag"] or np.all(np.isfinite(d["G"])), (c["name"], "unflagged with a Gram that is not finite")
        assert d["flag"], c["name"]


def test_unsampled_row_of_inf_only():
    c = [x for x in _threshold_cases() if x["name"] == "unsampled_all_inf"][0]
    with DeviceMbarBatch([c["u"]], [c["N"]]) as b:
        for want_G in (False, True):
            d = b.moments([c["f"]], want_G=want_G, all_rows=True)[0]
            assert not d["flag"]
            assert d["S"][2] == 0.0 and d["log_S"][2] == -np.inf
            if want_G:
                assert np.all(d["G"][2] == 0.0) and np.all(d["G"][:, 2] == 0.0)


def test_undrawn_sample_without_L_does_not_flag():
    """A sample whose sampled energies are all +inf has no L_n: the plain request is flagged (a NaN reaches the sums),
    but a replicate that never draws it has well-defined sums, which the reference computes on the drawn samples."""
    u, N_k, f, cnt = BE.undrawn_nan_case()
    c = dict(name="undrawn", u=u, N=N_k, f=f)
    with DeviceMbarBatch([u], [N_k]) as b:
        b.set_replicates([0], [cnt])
        for all_rows in (False, True):
            d = b.moments([f], want_G=True, all_rows=all_rows)[0]
            assert d["flag"]
            w = b.moments([f], want_G=True, all_rows=all_rows, slots=[0])[0]
            assert not w["flag"]
            _verify(c, cnt, w, all_rows, True, ("undrawn", all_rows))


# ---- 4. isolation and duplicates -------------------------------------------------------------------------------------
def test_flagged_requests_do_not_touch_clean_ones():
    th = {c["name"]: c for c in _threshold_cases()}
    u, N_k, f = BE.nan_case()
    dirty = [dict(name="nan", u=u, N=N_k, f=f), th["gram_DBL_MAX+0.5"], th["sampled_S_1e-280-0.5"],
             th["unsampled_S_DBL_MAX+0.5"]]
    clean = [BE.ladder_case("ladder_K17"), BE.ladder_case("ladder_K63")] + BE.family_cases()[::6]
    probs = [x for pair in zip(dirty, clean) for x in pair] + clean[len(dirty):]
    counts = _slots_for(probs, 300)
    with DeviceMbarBatch([c["u"] for c in probs], [c["N"] for c in probs]) as b:
        b.set_replicates(np.arange(len(probs)), counts)
        for weighted in (False, True):
            kw = (lambda ids: dict(slots=ids)) if weighted else (lambda ids: dict(problems=ids))
            ids = np.arange(len(probs))
            together = b.moments([c["f"] for c in probs], want_G=True, all_rows=True, **kw(ids))
            for i, c in enumerate(probs):
                alone = b.moments([c["f"]], want_G=True, all_rows=True, **kw([i]))[0]
                for k in ("S", "log_S", "G"):
                    np.testing.assert_array_equal(together[i][k], alone[k], err_msg=(c["name"], k, weighted))
                assert together[i]["sum_L"] == alone["sum_L"] or (np.isnan(alone["sum_L"]) and
                                                                 np.isnan(together[i]["sum_L"]))
                assert together[i]["flag"] == alone["flag"]
                if c in dirty:
                    assert alone["flag"] or weighted, (c["name"], weighted)
                else:
                    assert not alone["flag"], (c["name"], weighted)
            # the same problem twice in one call, at different f: each request gets its own answer
            i = 1
            c = probs[i]
            f2 = c["f"] + np.linspace(0.0, 0.3, len(c["N"]))
            two = b.moments([c["f"], f2], want_G=True, all_rows=True, **kw([i, i]))
            for g, d in zip((c["f"], f2), two):
                alone = b.moments([g], want_G=True, all_rows=True, **kw([i]))[0]
                for k in ("S", "log_S", "G"):
                    np.testing.assert_array_equal(d[k], alone[k])
                assert d["sum_L"] == alone["sum_L"]
            assert not np.array_equal(two[0]["S"], two[1]["S"])


# ---- 5. large absolute energies --------------------------------------------------------------------------------------
@pytest.mark.parametrize("scale", [1e5, 1e8])
def test_large_absolute_energies(scale):
    base = [BE.ladder_case("ladder_K16"), BE.ladder_case("ladder_K17"), BE.ladder_case("ladder_K33")]
    for fam in (E.with_unsampled(60.0, sign=-1.0), E.offset_pair(705.0), E.with_unsampled(800.0, sign=1.0)):
        base.append(dict(name="fam", u=fam["u"], N=fam["N"], f=fam["f_true"]))
    cases = []
    for i, c in enumerate(base):
        cases.append(dict(c, name=f"{c['name']}_{i}_{scale:g}", u=BE.offset_energies(c["u"], scale, 40 + i)))
    flags = _run_cases(cases)
    assert not any(flags.values()), [k for k, v in flags.items() if v]


# ---- 6. more than 4096 chunks' worth of tiles ------------------------------------------------------------------------
@pytest.fixture(scope="module", params=[131073, 135168], ids=["nT131073", "nT135168"])
def large(request):
    nT = request.param
    K = 64
    N = 32 * (nT - 1) + 19                     # not a multiple of 32
    block, f = BE.tiled_block(K)
    N_k = BE.tiled_N_k(K, N)
    counts = BE.slot_counts(N, K, 9)
    t0 = time.perf_counter()
    u = BE.tiled(block, N)
    b = DeviceMbarBatch([u], [N_k])
    del u
    gc.collect()
    b.set_replicates([0], [counts])
    yield dict(b=b, nT=nT, K=K, N=N, block=block, f=f, N_k=N_k, counts=counts, t_build=time.perf_counter() - t0)
    b.close()
    gc.collect()


def test_chunk_branch_geometry(large):
    nT, ct, nc, last = BE.geometry(large["N"], large["K"])
    assert (nT, ct) == (large["nT"], 33)
    assert (nc, last) == ((3972, 30) if nT == 131073 else (4096, 33))


@pytest.mark.parametrize("weighted", [False, True])
def test_chunk_branch_against_long_double(large, weighted):
    b, N, K, N_k = large["b"], large["N"], large["K"], large["N_k"]
    f = large["f"]
    counts = large["counts"] if weighted else None
    mult = BE.column_mult(N, counts)
    kw = dict(slots=[0]) if weighted else {}
    for all_rows in (False, True):
        d = b.moments([f], want_G=True, all_rows=all_rows, **kw)[0]
        again = b.moments([f], want_G=True, all_rows=all_rows, **kw)[0]
        for k in ("S", "log_S", "G"):
            np.testing.assert_array_equal(d[k], again[k])
        assert d["sum_L"] == again["sum_L"]
        nT = large["nT"]
        assert b.last_stats()["bytes_read"] == nT * 32 * K * 8 + (nT * 32 * 2 if weighted else 0)
        ref = BE.restate(large["block"], N_k, f, all_rows, mult=mult)
        flag, margin = BE.predict_flag(large["block"], N_k, f, all_rows, True, mult, ref=ref)
        assert BE.is_clear(margin) and not flag and not d["flag"]
        wmax = 1.0 if counts is None else float(counts.max())
        BE.check_request(d, ref, N_k, all_rows, N, wmax=wmax, what=(large["nT"], weighted, all_rows))


# ---- 7. mbar_many end to end -----------------------------------------------------------------------------------------
def _e2e_cases():
    out = []
    for d in (30.0, 705.0):
        c = E.offset_pair(d)
        out.append((f"pair_{d:g}", c["u"], c["N"], c["f_true"]))
        c = E.offset_pair(d, noisy=True)
        out.append((f"pair_noisy_{d:g}", c["u"], c["N"], None))
    for d, sign in ((400.0, -1.0), (800.0, -1.0), (1e4, 1.0)):
        c = E.with_unsampled(d, sign=sign)
        out.append((f"unsampled_{sign * d:g}", c["u"], c["N"], c["f_true"]))
    c = E.with_unsampled(60.0, sign=-1.0, noisy=True)
    out.append(("unsampled_noisy", c["u"], c["N"], None))
    c = E.offset_copies(16, 40.0)
    out.append(("copies16_40", c["u"], c["N"], c["f_true"]))
    for K in (16, 33):                         # well-overlapping ladders: f is well determined
        c = M.solve_ladder(K, K)
        out.append((f"solve_ladder_K{K}", c["u"], c["N"], None))
    return out


def test_mbar_many_end_to_end():
    cases = _e2e_cases()
    res = mbar_many([u for _, u, _, _ in cases], [n for _, _, n, _ in cases], compute_uncertainty=True)
    paths = {}
    for (name, u, N_k, f_true), r in zip(cases, res):
        assert r["success"], name
        paths[name] = r["path"]
        s = N_k > 0
        if f_true is None:
            with DeviceProblem(u, N_k) as p:
                f1, _ = p.solve_adaptive(np.zeros(len(N_k)), tol=1e-12, min_sc_iter=0)
            f1 = f1 - f1[0]
            assert np.max(np.abs((r["f_k"] - f1)[s])) <= 1e-8, name
        else:
            assert np.max(np.abs(r["f_k"] - f_true)) <= 1e-8, (name, r["f_k"] - f_true)
        with DeviceProblem(u, N_k) as p:
            _, G = p.weight_moments(r["f_k"])
        want = estimators.free_energy_differences(r["f_k"], G, N_k)["dDelta_f"]
        np.testing.assert_allclose(r["dDelta_f"], want, rtol=1e-6, atol=1e-8, err_msg=name)
        # the first all-rows update is made at the batched solve's f: sampled states converged (f[first] = 0),
        # unsampled ones at their start, 0
        f_upd = np.where(s, r["f_k"] - r["f_k"][np.flatnonzero(s)[0]], 0.0)
        flag, margin = BE.predict_flag(u, N_k, f_upd, True, False)
        if BE.is_clear(margin) and flag:
            assert r["path"] == "single", name
    print("paths:", paths)
    assert paths["unsampled_-800"] == "single" and paths["unsampled_-400"] == "batch", paths

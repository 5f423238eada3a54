"""mbar_many and DeviceMbarBatch on the GPU: parity with the reference's results, the batched sums against an
extended-precision restatement, determinism, agreement with the single-problem solver, and a 2000-problem batch."""
import os

import numpy as np
import pytest

from pymbar_b200 import DeviceMbarBatch, DeviceProblem
from pymbar_b200.mbar_many import mbar_many
from tests import _mbar_many as H
from tests._batch_edges import predict_flag
from tests._moments import entry_tol, excess, moments_ld

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", H.GOLDEN)


def test_golden_parity():
    cases = H.load(GOLDEN)
    res = mbar_many([c["u_kn"] for c in cases], [c["N_k"] for c in cases], f_k_init=[c["f_init"] for c in cases],
                    return_theta=True)
    for r, c in zip(res, cases):
        K = len(c["N_k"])
        assert r["success"], c["name"]
        if K > 64:
            assert r["path"] == "single"
        elif c["name"] != "span_750kT":
            assert r["path"] == "batch", c["name"]
        assert np.max(np.abs(r["Delta_f"] - c["Delta_f"])) < 1e-8, c["name"]
        np.testing.assert_allclose(r["dDelta_f"], c["dDelta_f"], rtol=1e-6, atol=1e-9, err_msg=c["name"])
        if K > 1:   # one state: Theta is the pseudo-inverse of a rounding residue
            np.testing.assert_allclose(r["Theta"], c["Theta"], rtol=1e-5, atol=1e-9, err_msg=c["name"])


def _mixed_batch():
    """Problems with K in {1, 2, 7, 8, 9, 31, 32, 33, 63, 64}, N around the chunk boundaries and 1e6, empty states
    first, in the middle and last."""
    rng = np.random.RandomState(5)
    probs = []
    Ks = (1, 2, 7, 8, 9, 31, 32, 33, 63, 64)
    Ns = (1, 31, 32, 33)
    for i, K in enumerate(Ks):
        ct = max(4, 2048 // K) * 32          # samples per chunk of the batched pass
        for N in Ns + (ct - 1, ct + 1):
            N = max(N, K)
            u, N_k = H.random_problem(rng, K, N)
            probs.append((u, N_k))
    for K, where in ((9, 0), (33, 16), (64, 63)):
        u, N_k = H.random_problem(rng, K, 3000)
        owner = np.repeat(np.arange(K), N_k.astype(int))
        N_k[owner[0]] += N_k[where]                 # move the samples of state `where` to another state
        N_k[where] = 0
        probs.append((u, N_k))
    u, N_k = H.random_problem(rng, 12, 1_000_000)
    probs.append((u, N_k))
    return probs


@pytest.mark.parametrize("which", ["zeros", "random"])
def test_moments_against_long_double(which):
    probs = _mixed_batch()
    rng = np.random.RandomState(11)
    fs = [np.zeros(len(N_k)) if which == "zeros" else rng.normal(scale=2.0, size=len(N_k)) for _, N_k in probs]
    with DeviceMbarBatch([u for u, _ in probs], [n for _, n in probs]) as b:
        for all_rows in (False, True):
            out = b.moments(fs, want_G=True, all_rows=all_rows)
            again = b.moments(fs[::-1], want_G=True, all_rows=all_rows, problems=np.arange(len(probs))[::-1])[::-1]
            for (u, N_k), f, d, d2 in zip(probs, fs, out, again):
                np.testing.assert_array_equal(d["G"], d2["G"])
                np.testing.assert_array_equal(d["S"], d2["S"])
                if d["flag"]:
                    assert predict_flag(u, N_k, f, all_rows, True)[0], (len(N_k), u.shape[1])
                    continue
                S, G, A = moments_ld(u, N_k, f, all_rows=all_rows)
                rows = np.ones(len(N_k), bool) if all_rows else N_k > 0
                tol = entry_tol(G, A, u.shape[1], 1.0)
                assert excess(d["G"], G, tol) <= 1.0, (len(N_k), u.shape[1])
                Stol = 8 * 2.0 ** -53 * (np.abs(A) + np.sqrt(u.shape[1]) + 8) * np.abs(S.astype(float)) + 1e-300
                assert excess(d["S"][rows], S[rows], Stol[rows]) <= 1.0, (len(N_k), u.shape[1])
                s = N_k > 0
                a = (f[s] + np.log(N_k[s]))[:, None] - u[s].astype(np.longdouble)
                m = a.max(axis=0)
                sumL = float((m + np.log(np.exp(a - m).sum(axis=0))).sum())
                assert abs(d["sum_L"] - sumL) <= 1e-12 * max(1.0, np.abs(sumL)) * np.sqrt(u.shape[1]) + 1e-9


def _problems(n, seed, Kmax=24, Nmax=3000):
    rng = np.random.RandomState(seed)
    return [H.random_problem(rng, rng.randint(2, Kmax + 1), rng.randint(50, Nmax), empty=rng.randint(0, 2))
            for _ in range(n)]


def test_determinism():
    probs = _problems(50, 3)
    us, ns = [u for u, _ in probs], [n for _, n in probs]
    full = mbar_many(us, ns, compute_uncertainty=False)
    rev = mbar_many(us[::-1], ns[::-1], compute_uncertainty=False)[::-1]
    for p in range(len(probs)):
        alone = mbar_many([us[p]], [ns[p]], compute_uncertainty=False)[0]
        assert full[p]["path"] == "batch"
        np.testing.assert_array_equal(full[p]["f_k"], alone["f_k"])
        np.testing.assert_array_equal(full[p]["f_k"], rev[p]["f_k"])


def test_same_solver_as_single_path():
    probs = _problems(30, 4)
    with DeviceMbarBatch([u for u, _ in probs], [n for _, n in probs]) as b:
        fs, status, iters = b.solve(tol=1e-12, min_sc_iter=0)
    for (u, N_k), f, st, it in zip(probs, fs, status, iters):
        assert st == 0
        with DeviceProblem(u, N_k) as p:
            f1, r = p.solve_adaptive(np.zeros(len(N_k)), tol=1e-12, min_sc_iter=0)
        s = N_k > 0
        assert np.max(np.abs((f - f1)[s])) <= 1e-10
        assert abs(int(it) - r["iterations"]) <= 1


def test_scale_2000_problems():
    rng = np.random.RandomState(2000)
    probs = []
    for _ in range(2000):
        K = rng.randint(1, 65)
        probs.append(H.random_problem(rng, K, max(K, rng.randint(1, 20001)), empty=rng.randint(0, 3) if K > 3 else 0))
    us, ns = [u for u, _ in probs], [n for _, n in probs]
    with DeviceMbarBatch(us, ns) as b:
        fs, status, iters = b.solve(tol=1e-12)
        st = b.last_stats()
    # a problem the batched loop does not finish goes through the single-problem path inside mbar_many
    assert np.mean(status == 0) >= 0.995, np.flatnonzero(status)
    assert st["launches"] == 2 * (st["iterations"] + 1)
    with DeviceMbarBatch(us[:100], ns[:100]) as b:
        b.solve(tol=1e-12)
        st100 = b.last_stats()
    assert st100["launches"] == 2 * (st100["iterations"] + 1)
    res = mbar_many(us, ns, compute_uncertainty=False)
    assert all(r["success"] for r in res)
    for p in rng.choice(np.flatnonzero(status == 0), size=20, replace=False):
        u, N_k = probs[p]
        s = N_k > 0
        with DeviceProblem(u, N_k) as d:
            f1, _ = d.solve_adaptive(np.zeros(len(N_k)), tol=1e-12, min_sc_iter=0)
            gb = np.max(np.abs(d.gradient(fs[p])[s]))
            g1 = np.max(np.abs(d.gradient(f1)[s]))
        assert gb <= 10 * max(g1, 1e-12 * N_k.sum()), (p, gb, g1)
        assert np.max(np.abs((fs[p] - f1)[s])) <= 1e-10

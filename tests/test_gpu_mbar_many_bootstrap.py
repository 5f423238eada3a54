"""mbar_many(n_bootstraps=B) and the replicate slots of DeviceMbarBatch on the GPU: weighted sums against the
extended-precision restatement, all-ones counts against the unweighted bits, replicates against bootstrap_f_k on a
DeviceProblem, parity with the reference's bootstraps, determinism across batches and waves, and a 200 x 100 run."""
import os

import numpy as np
import pytest

from pymbar_b200 import DeviceMbarBatch, DeviceProblem, bootstrap
from pymbar_b200 import mbar_many as mm
from tests import _mbar_many as H
from tests import _mbar_many_boot as W
from tests._batch_edges import predict_flag
from tests._moments import entry_tol, excess, moments_ld

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", W.GOLDEN)


def _mixed():
    """(u, N_k, counts): K in {1, 2, 7, 8, 9, 31, 32, 33, 63, 64}, N around the chunk boundaries, counts that are a
    reference draw, some with whole tiles of zero counts, and empty states first, in the middle and last."""
    rng = np.random.RandomState(7)
    out = []
    for K in (1, 2, 7, 8, 9, 31, 32, 33, 63, 64):
        ct = max(4, 2048 // K) * 32
        for N in (1, 33, ct - 1, ct + 1, 3 * ct + 5):
            u, N_k = H.random_problem(rng, K, max(N, K))
            c = np.bincount(bootstrap.bootstrap_indices(N_k.astype(np.int64), 1, rng.randint(1 << 30))[0],
                            minlength=u.shape[1])
            if u.shape[1] > 128:                    # tiles 1 and 2 hold no replicate sample
                c[0] += c[32:96].sum()
                c[32:96] = 0
            out.append((u, N_k, c))
    for K, where in ((9, 0), (33, 16), (64, 63)):
        u, N_k = H.random_problem(rng, K, 3000)
        owner = np.repeat(np.arange(K), N_k.astype(int))
        N_k[owner[0]] += N_k[where]
        N_k[where] = 0
        c = rng.multinomial(u.shape[1], np.ones(u.shape[1]) / u.shape[1])
        out.append((u, N_k, c))
    return out


@pytest.mark.parametrize("which", ["zeros", "random"])
def test_weighted_moments_against_long_double(which):
    probs = _mixed()
    rng = np.random.RandomState(11)
    fs = [np.zeros(len(N_k)) if which == "zeros" else rng.normal(scale=2.0, size=len(N_k)) for _, N_k, _ in probs]
    with DeviceMbarBatch([u for u, _, _ in probs], [n for _, n, _ in probs]) as b:
        b.set_replicates(np.arange(len(probs)), [c for _, _, c in probs])
        slots = np.arange(len(probs))
        for all_rows in (False, True):
            out = b.moments(fs, want_G=True, all_rows=all_rows, slots=slots)
            again = b.moments(fs[::-1], want_G=True, all_rows=all_rows, slots=slots[::-1])[::-1]
            checked = 0
            for (u, N_k, c), f, d, d2 in zip(probs, fs, out, again):
                np.testing.assert_array_equal(d["G"], d2["G"])
                np.testing.assert_array_equal(d["S"], d2["S"])
                assert d["sum_L"] == d2["sum_L"]
                if d["flag"]:
                    assert predict_flag(u, N_k, f, all_rows, True, counts=c)[0], (len(N_k), u.shape[1])
                    continue
                checked += 1
                S, G, A = moments_ld(u, N_k, f, mult=c, all_rows=all_rows)
                rows = np.ones(len(N_k), bool) if all_rows else N_k > 0
                tol = entry_tol(G, A, u.shape[1], float(c.max()))
                assert excess(d["G"], G, tol) <= 1.0, (len(N_k), u.shape[1])
                Stol = 8 * 2.0 ** -53 * (np.abs(A) + np.sqrt(u.shape[1]) + 8) * np.abs(S.astype(float)) + 1e-300
                assert excess(d["S"][rows], S[rows], Stol[rows]) <= 1.0, (len(N_k), u.shape[1])
                s = N_k > 0
                a = (f[s] + np.log(N_k[s]))[:, None] - u[s].astype(np.longdouble)
                m = a.max(axis=0)
                L = m + np.log(np.exp(a - m).sum(axis=0))
                sumL = float((c.astype(np.longdouble) * L).sum())
                scale = float((c * np.abs(L.astype(float))).sum())
                assert abs(d["sum_L"] - sumL) <= 1e-14 * max(1.0, scale) * np.sqrt(u.shape[1]) + 1e-9
            assert checked >= len(probs) - 2


def test_all_ones_counts_give_the_unweighted_bits():
    probs = _mixed()
    rng = np.random.RandomState(3)
    fs = [rng.normal(size=len(N_k)) for _, N_k, _ in probs]
    with DeviceMbarBatch([u for u, _, _ in probs], [n for _, n, _ in probs]) as b:
        b.set_replicates(np.arange(len(probs)), [np.ones(u.shape[1], np.uint16) for u, _, _ in probs])
        for all_rows in (False, True):
            plain = b.moments(fs, want_G=True, all_rows=all_rows)
            ones = b.moments(fs, want_G=True, all_rows=all_rows, slots=np.arange(len(probs)))
            for d, e in zip(plain, ones):
                for k in ("S", "log_S", "G"):
                    np.testing.assert_array_equal(d[k], e[k])
                assert d["sum_L"] == e["sum_L"] and d["flag"] == e["flag"]


def test_set_replicates_errors():
    u, N_k = H.random_problem(np.random.RandomState(1), 5, 300)
    with DeviceMbarBatch([u], [N_k]) as b:
        c = np.ones(u.shape[1], np.uint16)
        b.set_replicates([0], [c])
        with pytest.raises(ValueError):                      # checked before anything changes
            b.set_replicates([0], [np.full(u.shape[1], 70000)])
        assert len(b.moments([np.zeros(5)], slots=[0])) == 1
        with pytest.raises(Exception, match="sum to"):
            b.set_replicates([0], [c * 2])
        with pytest.raises(Exception, match="names problem"):
            b.set_replicates([1], [c])
        # a failed library call leaves no slot
        with pytest.raises(ValueError):
            b.moments([np.zeros(5)], slots=[0])
        b.set_replicates([0], [c])
        assert len(b.moments([np.zeros(5)], slots=[0])) == 1


def _replicate_probs(n, seed):
    rng = np.random.RandomState(seed)
    return [H.random_problem(rng, rng.randint(2, 25), rng.randint(200, 3000), empty=rng.randint(0, 2))
            for _ in range(n)]


def test_replicates_match_bootstrap_f_k():
    probs = _replicate_probs(8, 21)
    B = 6
    res = mm.mbar_many([u for u, _ in probs], [n for _, n in probs], compute_uncertainty=False, n_bootstraps=B,
                       rseed=list(range(100, 100 + len(probs))))
    protocol = (dict(method="adaptive", tol=1e-12, options=dict(min_sc_iter=0, gamma=1.0, maxiter=10000)),)
    for p, ((u, N_k), r) in enumerate(zip(probs, res)):
        assert r["boot_single"] == 0
        Ni = N_k.astype(np.int64)
        with DeviceProblem(u, N_k) as d:
            want = bootstrap.bootstrap_f_k(d, r["f_k"], Ni, rints=bootstrap.bootstrap_indices(Ni, B, 100 + p),
                                           solver_protocol=protocol)
        assert np.max(np.abs(r["f_k_boots"] - want)) <= 1e-10, p


def test_golden_parity():
    cases = W.load(GOLDEN)
    res = mm.mbar_many([c["u_kn"] for c in cases], [c["N_k"] for c in cases], f_k_init=[c["f_init"] for c in cases],
                       uncertainty_method="bootstrap", n_bootstraps=cases[0]["B"], rseed=[c["seed"] for c in cases])
    for r, c in zip(res, cases):
        assert np.max(np.abs(r["f_k_boots"] - c["f_k_boots"])) < 1e-8, c["name"]
        assert np.max(np.abs(r["dDelta_f"] - c["dDelta_f"])) < 1e-8, c["name"]
        if len(c["N_k"]) > 64:
            assert r["boot_single"] == c["B"]


def test_determinism_across_batches_and_waves(monkeypatch):
    probs = _replicate_probs(50, 4)
    us, ns = [u for u, _ in probs], [n for _, n in probs]
    seeds = list(range(500, 550))
    kw = dict(compute_uncertainty=False, n_bootstraps=4)
    full = mm.mbar_many(us, ns, rseed=seeds, **kw)
    rev = mm.mbar_many(us[::-1], ns[::-1], rseed=seeds[::-1], **kw)[::-1]
    monkeypatch.setattr(mm, "BOOT_WAVE_BYTES", 1)
    for p in (0, 17, 49):
        alone = mm.mbar_many([us[p]], [ns[p]], rseed=[seeds[p]], **kw)[0]
        np.testing.assert_array_equal(full[p]["f_k_boots"], alone["f_k_boots"])
    waves = mm.mbar_many(us[:10], ns[:10], rseed=seeds[:10], **kw)
    for p in range(50):
        assert full[p]["boot_single"] == 0
        np.testing.assert_array_equal(full[p]["f_k_boots"], rev[p]["f_k_boots"])
        if p < 10:
            np.testing.assert_array_equal(full[p]["f_k_boots"], waves[p]["f_k_boots"])


def test_scale_200_problems_100_replicates(monkeypatch):
    rng = np.random.RandomState(200)
    probs = [H.random_problem(rng, rng.randint(8, 33), rng.randint(1000, 4000)) for _ in range(200)]
    stats = []
    orig = DeviceMbarBatch.solve_replicates

    def solve_replicates(self, *a, **kw):
        out = orig(self, *a, **kw)
        stats.append((self.last_stats(), len(self.slot_problems)))
        return out

    monkeypatch.setattr(DeviceMbarBatch, "solve_replicates", solve_replicates)
    monkeypatch.setattr(mm, "BOOT_WAVE_BYTES", 256 << 20)
    res = mm.mbar_many([u for u, _ in probs], [n for _, n in probs], uncertainty_method="bootstrap",
                       n_bootstraps=100, rseed=list(range(200)))
    assert len(stats) > 1 and sum(n for _, n in stats) == 200 * 100
    for st, _ in stats:
        assert st["launches"] == 2 * (st["iterations"] + 1)
    assert sum(r["boot_single"] for r in res) <= 0.005 * 200 * 100
    assert all(np.all(np.isfinite(r["f_k_boots"])) and np.all(np.isfinite(r["dDelta_f"])) for r in res)

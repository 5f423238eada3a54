"""MbarMany's estimators and DeviceMbarBatch.augmented_moments on the GPU: parity with the reference's results, the
batched path against the single-problem path, the augmented sums against a long-double restatement, bit identity
whichever problems share a call or a wave, and the Gram-overflow flag."""
import os

import numpy as np
import pytest

from pymbar_b200 import DeviceMbarBatch, DeviceProblem
from pymbar_b200 import expectations as ex
from pymbar_b200 import mbar_many as mm
from tests import _mbar_many as H
from tests import _mbar_many_expectations as E
from tests._batch_edges import LOG_DBL_MAX, is_clear, log_s_tol, predict_flag, restate
from tests._mbar_many_expectations import check_case, run_all
from tests._moments import entry_tol, excess

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", E.GOLDEN)


def test_golden_parity():
    cases = E.load(GOLDEN)
    with mm.MbarMany([c["u_kn"] for c in cases], [c["N_k"] for c in cases]) as m:
        out = run_all(m, cases)
    for i, c in enumerate(cases):
        check_case(c, *(o[i] for o in out))
        want = "single" if len(c["N_k"]) > 64 else "batch"
        assert [o[i]["path"] for o in out] == [want] * 6, c["name"]


def _near(a, b, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    fin = np.isfinite(b)
    assert np.array_equal(fin, np.isfinite(a)), what
    assert np.all(np.abs(a[fin] - b[fin]) <= 1e-10 * np.maximum(1.0, np.abs(b[fin]))), what


def _rel(a, b, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    fin = np.isfinite(b)
    assert np.all(np.abs(a[fin] - b[fin]) <= 1e-8 * np.abs(b[fin]) + 1e-300), what


def test_batch_matches_single_path():
    cases = [c for c in E.load(GOLDEN) if len(c["N_k"]) <= 64]
    with mm.MbarMany([c["u_kn"] for c in cases], [c["N_k"] for c in cases]) as m:
        reqs = [E.requests(c["u_kn"]) for c in cases]
        ent = m.compute_entropy_and_enthalpy()
        pert = m.compute_perturbed_free_energies([r[2] for r in reqs])
        avg = m.compute_expectations([r[0] for r in reqs])
        for p, c in enumerate(cases):
            assert ent[p]["path"] == pert[p]["path"] == avg[p]["path"] == "batch", c["name"]
            u, N_k, f = c["u_kn"], c["N_k"], m.results[p]["f_k"]
            K = len(N_k)
            with DeviceProblem(u, N_k) as q:
                inner = ex.expectations_inner(u, N_k, f, u, u, np.array([np.arange(K), np.arange(K)]),
                                              return_theta=True, problem=q)
                single_ent = ex.entropy_enthalpy_result(inner, K)
                inner = ex.expectations_inner(u, N_k, f, np.array([0.0]), reqs[p][2], np.arange(len(reqs[p][2])),
                                              return_theta=True, problem=q)
                single_pert = ex.perturbed_result(inner, True, 1e-10)
                inner = ex.expectations_inner(u, N_k, f, reqs[p][0], u, ex.expectation_state_map(K, False),
                                              return_theta=True, problem=q)
                single_avg = ex.expectations_result(inner, K, "averages", True, False, 1e-10)
            for k in ("Delta_f", "Delta_u", "Delta_s"):
                _near(ent[p][k], single_ent[k], c["name"] + " " + k)
                _rel(ent[p]["d" + k], single_ent["d" + k], c["name"] + " d" + k)
            _near(pert[p]["Delta_f"], single_pert["Delta_f"], c["name"] + " pert")
            _rel(pert[p]["dDelta_f"], single_pert["dDelta_f"], c["name"] + " pert d")
            _near(avg[p]["mu"], single_avg["mu"], c["name"] + " mu")
            _rel(avg[p]["sigma"], single_avg["sigma"], c["name"] + " sigma")


def _augmented_case(K, M, N, seed, far=False, inf_rows=0):
    """(u [K, N], N_k, extra [M, N]): a harmonic problem with K states and M appended harmonic rows between and
    beyond its centres (or 45 widths away, weights about e^-900), the last inf_rows of them all +inf."""
    rng = np.random.RandomState(seed)
    u, N_k = H.harmonic(K, max(N // K, 1), seed, spacing=0.5)
    if u.shape[1] != N:                           # exactly N samples: top up the last state
        extra_n = N - u.shape[1]
        x = 0.5 * (K - 1) + rng.normal(size=extra_n)
        u = np.hstack([u, 0.5 * (x[None, :] - 0.5 * np.arange(K)[:, None]) ** 2])
        N_k[-1] += extra_n
    # the sample positions, from u_1 - u_0 = 0.125 - x / 2 (one state: |x| only, which still gives valid rows)
    x = 0.25 - 2.0 * (u[1] - u[0]) if K > 1 else np.sqrt(2 * u[0])
    centres = np.linspace(-0.25, 0.5 * K + 0.25, M) + (45.0 + 0.5 * K if far else 0.0)
    extra = 0.5 * (x[None, :] - centres[:, None]) ** 2
    if inf_rows:
        extra[-inf_rows:] = np.inf
    return u, N_k, extra


def _normalised_f(dev, p, K, M):
    """The solved, normalised f of problem p with its appended rows' f from the self-consistent update."""
    f_list, status, _ = dev.solve(tol=1e-12)
    f = f_list[p] - dev.moments([f_list[p]], all_rows=True, problems=[p])[0]["log_S"]
    f = f - f[0]
    f0 = np.concatenate([f, np.zeros(M)])
    m = dev.augmented_moments([f0], problems=[p])[0]
    fa = f0.copy()
    fa[K:] = (f0 - m["log_S"])[K:]
    return np.where(np.isfinite(fa), fa, 0.0)


@pytest.mark.parametrize("K,M,N", [(1, 1, 1), (1, 1, 1000), (2, 61, 777), (32, 32, 4097), (33, 32, 3000),
                                   (64, 1, 2049), (64, 64, 1500), (64, 127, 700), (64, 128, 1100),
                                   (2, 1, 1_000_000), (8, 24, 200_003), (16, 176, 40_001)])
def test_augmented_moments_against_long_double(K, M, N):
    u, N_k, extra = _augmented_case(K, M, N, seed=K * 1000 + M)
    with DeviceMbarBatch([u], [N_k]) as dev:
        dev.set_unsampled([0], [extra])
        f = _normalised_f(dev, 0, K, M)
        d = dev.augmented_moments([f], want_G=True)[0]
    ua = np.vstack([u, extra])
    Na = np.concatenate([N_k, np.zeros(M)])
    ref = restate(ua, Na, f, True)
    assert not d["flag"]
    tol = entry_tol(ref["G"], ref["A"], N, 1.0)
    assert excess(d["G"], ref["G"], tol) <= 1.0, (K, M, N)
    app = np.arange(K, K + M)
    err = np.abs(d["log_S"][app] - ref["logS"][app].astype(np.float64))
    assert np.all(err <= log_s_tol(ref["A"][app], N, K + M)), (K, M, N, err.max())


def test_appended_rows_of_inf_and_far_away():
    u, N_k, extra = _augmented_case(6, 6, 5000, seed=3, far=True, inf_rows=2)
    with DeviceMbarBatch([u], [N_k]) as dev:
        dev.set_unsampled([0], [extra])
        f = np.concatenate([dev.solve(tol=1e-12)[0][0], np.zeros(6)])
        d = dev.augmented_moments([f], want_G=True)[0]
    ref = restate(np.vstack([u, extra]), np.concatenate([N_k, np.zeros(6)]), f, True)
    assert not d["flag"]
    assert np.all(d["log_S"][-2:] == -np.inf) and np.all(d["S"][-2:] == 0.0)
    assert np.all(d["G"][-2:] == 0.0) and np.all(d["G"][:, -2:] == 0.0)
    far = np.arange(6, 10)
    assert np.all(ref["logS"][far] < -800)
    err = np.abs(d["log_S"][far] - ref["logS"][far].astype(np.float64))
    assert np.all(err <= log_s_tol(ref["A"][far], 5000, 12))
    tol = entry_tol(ref["G"], ref["A"], 5000, 1.0)
    assert excess(d["G"], ref["G"], tol) <= 1.0


def _campaign(n, seed):
    rng = np.random.RandomState(seed)
    return [H.random_problem(rng, int(rng.choice([3, 12, 21, 22, 32, 64])), int(rng.choice([200, 2500, 9000])),
                             empty=int(rng.randint(0, 2))) for _ in range(n)]


def _bits(res):
    return [None if r is None else {k: np.asarray(v).tobytes() for k, v in r.items()} for r in res]


def test_bit_identity_alone_batch_reversed_and_waves(monkeypatch):
    probs = _campaign(50, 11)
    us, nks = [p[0] for p in probs], [p[1] for p in probs]
    with mm.MbarMany(us, nks) as m:
        full = _bits(m.compute_entropy_and_enthalpy())
        assert all(r["path"] == "batch" for r in m.compute_entropy_and_enthalpy())
    with mm.MbarMany(us[::-1], nks[::-1]) as m:
        rev = _bits(m.compute_entropy_and_enthalpy())[::-1]
    monkeypatch.setattr(mm, "AUG_WAVE_BYTES", 1)
    with mm.MbarMany(us, nks) as m:
        waves = _bits(m.compute_entropy_and_enthalpy())
    for p in (0, 17, 49):
        with mm.MbarMany([us[p]], [nks[p]]) as m:
            assert _bits(m.compute_entropy_and_enthalpy())[0] == full[p]
    assert rev == full
    assert waves == full


def test_augmented_requests_keep_their_bits_in_any_company():
    probs = _campaign(12, 5)
    us, nks = [p[0] for p in probs], [p[1] for p in probs]
    rng = np.random.RandomState(2)
    extras = [u[rng.randint(0, u.shape[0], size=u.shape[0] // 2 + 1)] + rng.uniform(0, 1) for u in us]
    with DeviceMbarBatch(us, nks) as dev:
        f_list, _, _ = dev.solve()
        f = [np.concatenate([fk, np.zeros(e.shape[0])]) for fk, e in zip(f_list, extras)]
        dev.set_unsampled(list(range(12)), extras)
        together = dev.augmented_moments(f, want_G=True)
        again = dev.augmented_moments(f[::-1], want_G=True, problems=list(range(12))[::-1])[::-1]
        dev.set_unsampled([7], [extras[7]])
        alone = dev.augmented_moments([f[7]], want_G=True, problems=[7])[0]
        st = dev.last_stats()
    assert st["launches"] == 3
    for a, b in zip(together, again):
        for k in ("S", "log_S", "G"):
            assert a[k].tobytes() == b[k].tobytes()
    for k in ("S", "log_S", "G"):
        assert alone[k].tobytes() == together[7][k].tobytes()


def test_gram_overflow_flag_is_predicted():
    u, N_k, extra = _augmented_case(4, 2, 3000, seed=9)
    ua, Na = np.vstack([u, extra]), np.concatenate([N_k, np.zeros(2)])
    with DeviceMbarBatch([u], [N_k]) as dev:
        dev.set_unsampled([0], [extra])
        f = _normalised_f(dev, 0, 4, 2)
        base = restate(ua, Na, f, True, want_G=False)
        # raise the last appended row's f until its Ghat_kk crosses DBL_MAX: log Ghat_kk grows by 2 per unit of f
        t0 = (LOG_DBL_MAX - float(base["logGd"][-1])) / 2
        seen = set()
        for dt in (-0.5, -0.25, 0.25, 0.5):
            fx = f.copy()
            fx[-1] += t0 + dt
            want, margin = predict_flag(ua, Na, fx, True, True)
            assert is_clear(margin)
            d = dev.augmented_moments([fx], want_G=True)[0]
            assert d["flag"] == want, dt
            seen.add(want)
            s = dev.augmented_moments([fx])[0]
            assert not s["flag"]             # without the Gram only S decides, and S is finite
    assert seen == {False, True}


def test_errors():
    u, N_k, extra = _augmented_case(4, 3, 500, seed=1)
    from pymbar_b200._lib import MbarB200Error

    with DeviceMbarBatch([u, u], [N_k, N_k]) as dev:
        bad = extra.copy()
        bad[1, 3] = np.nan
        for problems, rows, status in (([0], [bad], "ERR_NAN"), ([0], [-np.inf * extra], "ERR_NAN"),
                                       ([2], [extra], "ERR_INVALID"), ([0, 0], [extra, extra], "ERR_INVALID"),
                                       ([0], [np.zeros((189, 500))], "ERR_INVALID")):
            with pytest.raises(MbarB200Error, match=status):
                dev.set_unsampled(problems, rows)
            with pytest.raises(MbarB200Error, match="no appended rows"):    # a failed call leaves none: R = K
                dev.augmented_moments([np.zeros(4)], problems=[0])
        dev.set_unsampled([1], [np.zeros((188, 500))])     # K + M = 192, the limit
        assert dev.augmented_moments([np.zeros(192)], problems=[1])[0]["S"].shape == (192,)
        dev.set_unsampled([], [])
        with pytest.raises(MbarB200Error, match="no appended rows"):
            dev.augmented_moments([np.zeros(4)], problems=[1])

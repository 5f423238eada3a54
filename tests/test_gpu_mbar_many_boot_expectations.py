"""MbarMany's estimators with uncertainty_method="bootstrap" and DeviceMbarBatch.augmented_moments(..., slots=) on the
GPU: parity with the reference's bootstrap results, the batched path against the single-problem path, the weighted
augmented sums against a long-double restatement, bit identity whichever problems share a call or a wave, the entry
point's errors and a campaign-sized case."""
import ctypes as C
import os

import numpy as np
import pytest

from pymbar_b200 import DeviceMbarBatch, DeviceProblem
from pymbar_b200 import expectations as ex
from pymbar_b200 import mbar_many as mm
from pymbar_b200._lib import MbarB200Error, check
from tests import _mbar_many as H
from tests import _mbar_many_boot_expectations as BE
from tests import _mbar_many_expectations as E
from tests._batch_edges import check_request, restate, slot_counts
from tests.test_gpu_mbar_many_expectations import _augmented_case, _normalised_f

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", BE.GOLDEN)
BOOT_KEYS = ("bootstrapped_observables", "bootstrapped_f")


def _many(us, nks, B, seeds, **kw):
    return mm.MbarMany(us, nks, compute_uncertainty=False, n_bootstraps=B, rseed=seeds, **kw)


def test_golden_parity():
    cases = BE.load(GOLDEN)
    with _many([c["u_kn"] for c in cases], [c["N_k"] for c in cases], cases[0]["B"], [c["seed"] for c in cases]) as m:
        out = BE.run_boot(m, cases)
    worst = {}
    for i, c in enumerate(cases):
        for k, v in BE.max_errors(c, *(o[i] for o in out)).items():
            worst[k] = max(worst.get(k, 0.0), v)
    print("largest differences from the reference:", worst)
    for i, c in enumerate(cases):
        BE.check_boot_case(c, *(o[i] for o in out))
        want = "single" if len(c["N_k"]) > 64 else "batch"
        assert [o[i]["path"] for o in out] == [want] * 4, c["name"]


def _close(a, b, what, rel=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.array_equal(np.isfinite(a), np.isfinite(b)), what
    fin = np.isfinite(b)
    err = np.abs(a[fin] - b[fin]) / np.maximum(1.0, np.abs(b[fin]))
    assert np.all(err <= rel), (what, float(err.max()))


def test_batch_matches_single_path():
    rng = np.random.RandomState(21)
    Ks = [2, 3, 7, 16, 21, 33, 48, 64]
    probs = [H.random_problem(rng, K, int(rng.choice([500, 3000, 8000])), empty=int(rng.randint(0, 2))) for K in Ks]
    us, nks = [p[0] for p in probs], [p[1] for p in probs]
    B = 6
    with _many(us, nks, B, list(range(100, 100 + len(Ks)))) as m:
        avg = m.compute_expectations([u[-1] for u in us], uncertainty_method="bootstrap")
        ent = m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap")
        for p, (u, N_k) in enumerate(probs):
            assert avg[p]["path"] == ent[p]["path"] == "batch", Ks[p]
            K = len(N_k)
            counts = np.array([m._draws[p].counts(b) for b in range(B)])
            reps = (m.results[p]["f_k_boots"], counts)
            f = m.results[p]["f_k"]
            with DeviceProblem(u, N_k) as q:
                a = ex.expectations_inner(u, N_k, f, u[-1], u, ex.expectation_state_map(K, False), problem=q,
                                          replicates=reps)
                e = ex.expectations_inner(u, N_k, f, u, u, np.array([np.arange(K), np.arange(K)]), problem=q,
                                          replicates=reps)
            for k in BOOT_KEYS:
                _close(avg[p][k], a[k], (K, "avg", k))
                _close(ent[p][k], e[k], (K, "ent", k))


@pytest.mark.parametrize("K,M,N", [(1, 1, 1000), (2, 61, 777), (32, 32, 4097), (64, 1, 2049), (64, 128, 1100),
                                   (2, 1, 1_000_000), (8, 24, 200_003), (16, 176, 40_001)])
def test_weighted_augmented_moments_against_long_double(K, M, N):
    u, N_k, extra = _augmented_case(K, M, N, seed=K * 1000 + M, inf_rows=1 if M > 1 else 0)
    with DeviceMbarBatch([u], [N_k]) as dev:
        dev.set_unsampled([0], [extra])
        f = _normalised_f(dev, 0, K, M)
    counts = slot_counts(N, K + M, seed=N + M)
    # sample 0: undrawn, with every sampled energy +inf; the pass must not flag the slot for it
    counts[np.flatnonzero(counts)[-1]] += counts[0]
    counts[0] = 0
    u[:, 0] = np.inf
    assert counts.max() <= 65535
    with DeviceMbarBatch([u], [N_k]) as dev:
        dev.set_unsampled([0], [extra])
        dev.set_replicates([0], [counts])
        d = dev.augmented_moments([f], slots=[0])[0]
        st = dev.last_stats()
    assert st["launches"] == 2
    nT = -(-N // 32)
    assert st["bytes_read"] == nT * 32 * (K + M) * 8 + nT * 32 * 2
    ua, Na = np.vstack([u, extra]), np.concatenate([N_k, np.zeros(M)])
    ref = restate(ua, Na, f, True, mult=counts, want_G=False)
    assert not d["flag"]
    check_request(d, ref, Na, True, N, wmax=float(counts.max()), what=(K, M, N))
    if M > 1:
        assert d["S"][-1] == 0.0 and d["log_S"][-1] == -np.inf


def test_all_ones_counts_give_the_unweighted_bits():
    probs = [H.random_problem(np.random.RandomState(s), K, N) for s, (K, N) in enumerate([(5, 3000), (40, 9000)])]
    us, nks = [p[0] for p in probs], [p[1] for p in probs]
    rng = np.random.RandomState(4)
    extras = [u[rng.randint(0, u.shape[0], size=u.shape[0] + 3)] + 0.5 for u in us]
    with DeviceMbarBatch(us, nks) as dev:
        f_list, _, _ = dev.solve()
        f = [np.concatenate([fk, np.zeros(e.shape[0])]) for fk, e in zip(f_list, extras)]
        dev.set_unsampled([0, 1], extras)
        plain = dev.augmented_moments(f)
        dev.set_replicates([1, 0], [np.ones(u.shape[1], np.uint16) for u in us[::-1]])
        ones = dev.augmented_moments(f[::-1], slots=[0, 1])[::-1]
    for a, b in zip(plain, ones):
        assert not a["flag"] and not b["flag"]
        for k in ("S", "log_S", "sum_L"):
            assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


def _bits(res):
    return [None if r is None else {k: np.asarray(v).tobytes() for k, v in r.items()} for r in res]


def test_bit_identity_alone_among_many_reversed_waves_and_repeat(monkeypatch):
    rng = np.random.RandomState(11)
    probs = [H.random_problem(rng, int(rng.choice([3, 12, 21, 32, 64])), int(rng.choice([200, 2500, 6000])),
                              empty=int(rng.randint(0, 2))) for _ in range(50)]
    us, nks = [p[0] for p in probs], [p[1] for p in probs]
    seeds = list(range(500, 550))
    B = 4
    with _many(us, nks, B, seeds) as m:
        full = _bits(m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap"))
        again = _bits(m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap"))
        paths = [r["path"] for r in m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap")]
    assert paths == ["batch"] * 50
    assert again == full
    with _many(us[::-1], nks[::-1], B, seeds[::-1]) as m:
        rev = _bits(m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap"))[::-1]
    assert rev == full
    monkeypatch.setattr(mm, "BOOT_WAVE_BYTES", 1)
    with _many(us, nks, B, seeds) as m:
        waves = _bits(m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap"))
    assert waves == full
    for p in (0, 17, 49):
        with _many([us[p]], [nks[p]], B, [seeds[p]]) as m:
            assert _bits(m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap"))[0] == full[p]


def test_errors():
    u, N_k, extra = _augmented_case(4, 3, 500, seed=1)
    with DeviceMbarBatch([u, u], [N_k, N_k]) as dev:
        dev.set_unsampled([0], [extra])
        dev.set_replicates([0, 1], [np.ones(500, np.uint16)] * 2)
        f = np.zeros(7)
        assert not dev.augmented_moments([f], slots=[0])[0]["flag"]
        with pytest.raises(MbarB200Error, match="no appended rows"):       # slot 1's problem holds none
            dev.augmented_moments([np.zeros(4)], slots=[1])
        with pytest.raises(ValueError):
            dev.augmented_moments([f], want_G=True, slots=[0])
        with pytest.raises(ValueError):
            dev.augmented_moments([f], problems=[0], slots=[0])
        # a slot out of range, through the entry point itself (the wrapper rejects it before the call)
        out = [np.empty(7), np.empty(7), np.empty(1)]
        flag = np.empty(1, np.int32)
        for slot in (2, -1):
            ids = np.array([slot], np.int32)
            with pytest.raises(MbarB200Error, match="ERR_INVALID"):
                check(dev._lib.mbar_b200_batch_replicate_augmented_moments(
                    dev._h, 1, ids.ctypes.data_as(C.POINTER(C.c_int32)), f.ctypes.data_as(C.POINTER(C.c_double)),
                    *(o.ctypes.data_as(C.POINTER(C.c_double)) for o in out), flag.ctypes.data_as(C.POINTER(C.c_int32))))
        dev.set_unsampled([], [])
        with pytest.raises(MbarB200Error, match="no appended rows"):       # none left: R = K
            dev.augmented_moments([np.zeros(4)], slots=[0])


def test_campaign_scale(monkeypatch):
    rng = np.random.RandomState(7)
    probs = [H.random_problem(rng, int(rng.randint(8, 33)), int(rng.choice([1000, 3000, 6000]))) for _ in range(200)]
    us, nks = [p[0] for p in probs], [p[1] for p in probs]
    launches = []
    count = mm.MbarMany._count

    def recording(self):
        launches.append(self._dev.last_stats()["launches"])
        count(self)

    monkeypatch.setattr(mm.MbarMany, "_count", recording)
    with _many(us, nks, 50, list(range(200))) as m:
        res = m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap")
    assert [r["path"] for r in res] == ["batch"] * 200
    assert len(launches) >= 2 and set(launches) == {2}
    for r, (u, _) in zip(res, probs):
        K = u.shape[0]
        assert r["bootstrapped_observables"].shape == (50, K) and r["dDelta_s"].shape == (K, K)
        assert np.all(np.isfinite(r["dDelta_u"])) and np.all(np.isfinite(r["dDelta_s"]))

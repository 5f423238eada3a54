"""MbarMany's estimators with uncertainty_method="bootstrap" without a GPU, over numpy stand-ins of the weighted batch
with appended rows (tests/_mbar_many_boot_expectations): the reference's bootstrap results in
tests/golden/mbar_many_boot_expectations.npz, the regenerated replicate counts, routing, waves, skipped problems and the
argument checks."""
import os

import numpy as np
import pytest

from pymbar_b200 import bootstrap
from pymbar_b200 import mbar_many as mm
from pymbar_b200 import mbar_solvers as ms
from pymbar_b200.utils import ParameterError
from tests import _mbar_many as H
from tests import _mbar_many_boot as W
from tests import _mbar_many_boot_expectations as BE
from tests import _mbar_many_expectations as E

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", BE.GOLDEN)


@pytest.fixture
def oracle(monkeypatch):
    monkeypatch.setattr(mm, "DeviceMbarBatch", BE.BootOracleBatch)
    monkeypatch.setattr(mm, "DeviceProblem", BE.BootOracleProblem)
    monkeypatch.setattr(ms, "solve_mbar_for_all_states", H.oracle_all_states)
    monkeypatch.setattr(bootstrap, "bootstrap_f_k", W.oracle_bootstrap_f_k)
    monkeypatch.setattr(BE.BootOracleBatch, "flagged", ())
    monkeypatch.setattr(BE.BootOracleBatch, "aug_flagged", ())
    monkeypatch.setattr(BE.BootOracleBatch, "slot_flagged", ())
    monkeypatch.setattr(BE.BootOracleBatch, "flagged_counts", set())
    BE.BootOracleBatch.created.clear()
    BE.BootOracleBatch.calls.clear()
    BE.BootOracleBatch.uploads.clear()
    BE.BootOracleProblem.created.clear()
    BE.BootOracleProblem.replicate_calls.clear()
    return BE.BootOracleBatch


def _many(cases, B=None, **kw):
    return mm.MbarMany([c["u_kn"] for c in cases], [c["N_k"] for c in cases], compute_uncertainty=False,
                       n_bootstraps=cases[0]["B"] if B is None else B, rseed=[c["seed"] for c in cases], **kw)


def _bits(res):
    return [None if r is None else {k: np.asarray(v).tobytes() for k, v in r.items()} for r in res]


def test_golden_through_stand_in(oracle):
    cases = BE.load(GOLDEN)
    with _many(cases) as m:
        out = BE.run_boot(m, cases)
        for r, c in zip(m.results, cases):
            np.testing.assert_allclose(r["f_k_boots"], c["f_k_boots"], rtol=0, atol=1e-8, err_msg=c["name"])
    for i, c in enumerate(cases):
        BE.check_boot_case(c, *(o[i] for o in out))
        want = "single" if len(c["N_k"]) > 64 else "batch"
        assert [o[i]["path"] for o in out] == [want] * 4, c["name"]
        B, K = c["B"], len(c["N_k"])
        assert out[0][i]["bootstrapped_observables"].shape == (B, K)
        assert out[2][i]["dDelta_f"].shape == (K - 1,) and "bootstrapped_observables" not in out[2][i]
        assert out[3][i]["bootstrapped_f"].shape == (B, K)


def test_regenerated_counts_are_the_reference_draws(oracle):
    cases = [BE.load(GOLDEN)[i] for i in (0, 2, 7)]
    B = 5
    with _many(cases, B=B) as m:
        oracle.uploads.clear()
        m.compute_expectations([c["u_kn"][0] for c in cases], uncertainty_method="bootstrap")
        uploads = list(oracle.uploads)
    got = {}
    for problems, counts in uploads[:-1]:                 # the last call drops the slots
        for p, c in zip(problems, counts):
            got.setdefault(int(p), []).append(c)
    assert uploads[-1][0].size == 0
    for p, c in enumerate(cases):
        want = bootstrap.bootstrap_indices(c["N_k"].astype(np.int64), B, c["seed"])
        N = c["u_kn"].shape[1]
        np.testing.assert_array_equal(np.array(got[p]), [np.bincount(r, minlength=N) for r in want])


def test_other_keys_are_those_of_the_analytic_call(oracle):
    cases = [BE.load(GOLDEN)[i] for i in (0, 1, 7, 8)]  # K = 2, 9, 6, 7
    reqs = [E.requests(c["u_kn"]) for c in cases]
    with _many(cases) as m:
        for method in (None, "bootstrap"):
            for k, v in (("avg", m.compute_expectations([r[0] for r in reqs], uncertainty_method=method,
                                                        return_theta=True)),
                         ("diff", m.compute_expectations([r[1] for r in reqs], output="differences",
                                                         state_dependent=True, uncertainty_method=method)),
                         ("pert", m.compute_perturbed_free_energies([r[2] for r in reqs],
                                                                    uncertainty_method=method)),
                         ("ent", m.compute_entropy_and_enthalpy(uncertainty_method=method))):
                if method is None:
                    ref = {k: v} if k == "avg" else dict(ref, **{k: v})
                    continue
                for a, b in zip(ref[k], v):
                    for key in a:
                        if key == "sigma" or key.startswith("dDelta"):
                            assert key in b
                            continue
                        assert np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes(), (k, key)


def test_routing_to_the_single_path(oracle, monkeypatch):
    cases = BE.load(GOLDEN)
    pick = [1, 5, 6, 7]                                   # K = 9, 64, 65, 6
    sub = [cases[i] for i in pick]
    with _many(sub) as m:
        clean = m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap")
        # K = 64 with 2K + 1 appended rows exceeds the row limit
        u64 = sub[1]["u_kn"]
        A = np.vstack([u64, u64[:1]])
        r = m.compute_expectations([None, A, None, None], u_ln_list=[None, A, None, None], state_dependent=True,
                                   uncertainty_method="bootstrap")
        assert r[1]["path"] == "single" and r[1]["bootstrapped_observables"].shape == (sub[0]["B"], 65)
    assert [e["path"] for e in clean] == ["batch", "batch", "single", "batch"]
    # a flagged replicate sends the whole problem (batch index 2: the K = 6 problem) to the single path
    monkeypatch.setattr(oracle, "slot_flagged", (2,))
    oracle.calls.clear()
    BE.BootOracleProblem.replicate_calls.clear()
    with _many(sub) as m:
        flagged = m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap")
    assert [e["path"] for e in flagged] == ["batch", "batch", "single", "single"]
    assert any(kind == "replicate_augmented_moments" and 2 in probs for kind, probs in oracle.calls)
    assert len(BE.BootOracleProblem.replicate_calls) == 2          # K = 65 and the flagged problem
    for a, b in zip(clean, flagged):
        for k in a:
            if k != "path":
                np.testing.assert_allclose(b[k], a[k], rtol=1e-9, atol=1e-9, err_msg=k)


def test_none_skips_a_problem(oracle):
    cases = BE.load(GOLDEN)[:3]
    with _many(cases) as m:
        oracle.calls.clear()
        r = m.compute_perturbed_free_energies([None, E.requests(cases[1]["u_kn"])[2], None],
                                              uncertainty_method="bootstrap")
        assert r[0] is None and r[2] is None and r[1]["path"] == "batch"
        assert all(probs == [1] * len(probs) for kind, probs in oracle.calls if kind != "set_unsampled" and probs)
        r = m.compute_entropy_and_enthalpy([cases[0]["u_kn"], None, None], uncertainty_method="bootstrap")
        assert r[1] is None and r[2] is None and r[0]["path"] == "batch"


def test_waves_give_the_same_bits(oracle, monkeypatch):
    cases = [BE.load(GOLDEN)[i] for i in (0, 1, 7, 8)]  # K = 2, 9, 6, 7
    with _many(cases) as m:
        one = _bits(m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap"))
    calls_one = [c for c in oracle.calls if c[0] == "replicate_augmented_moments"]
    assert len(calls_one) == 1
    oracle.calls.clear()
    monkeypatch.setattr(mm, "BOOT_WAVE_BYTES", 1)
    monkeypatch.setattr(mm, "AUG_WAVE_BYTES", 1)
    with _many(cases) as m:
        many = _bits(m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap"))
    calls = [c for c in oracle.calls if c[0] == "replicate_augmented_moments"]
    assert calls == [("replicate_augmented_moments", [p]) for p in range(4) for _ in range(cases[0]["B"])]
    assert one == many


def test_boot_wave_bytes_follow_the_geometry():
    # K = 32, N = 160000, M = 96: counts, pass partials, output and f of one weighted request
    nT, R = 5000, 128
    nc = -(-nT // max(max(2048 // R, 4), -(-nT // 4096)))
    assert mm.boot_augmented_bytes(32, 160000, 96) == 2 * nT * 32 + 8 * (nc * (2 * R + 2) + 2 * R + 2 + R)


def test_errors_before_device_work(oracle):
    cases = BE.load(GOLDEN)[:2]
    us = [c["u_kn"] for c in cases]
    with _many(cases, B=0) as m:
        oracle.calls.clear()
        with pytest.raises(ParameterError, match="without any bootstraps"):
            m.compute_expectations([u[0] for u in us], uncertainty_method="bootstrap")
        with pytest.raises(ParameterError, match="without any bootstraps"):
            m.compute_perturbed_free_energies([u[:1] for u in us], uncertainty_method="bootstrap")
        with pytest.raises(ParameterError, match="without any bootstraps"):
            m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap")
        assert oracle.calls == []
    with _many(cases, B=3) as m:
        oracle.calls.clear()
        BE.BootOracleProblem.created.clear()
        with pytest.raises(ParameterError, match="svd"):
            m.compute_expectations([u[0] for u in us], uncertainty_method="svd")
        with pytest.raises(ParameterError, match="problem 1.*states"):
            m.compute_entropy_and_enthalpy([us[0], us[1][:3]], uncertainty_method="bootstrap")
        m._overflow = {1}
        with pytest.raises(ParameterError, match="problem 1.*65535"):
            m.compute_perturbed_free_energies([u[:2] for u in us], uncertainty_method="bootstrap")
        r = m.compute_perturbed_free_energies([us[0][:2], None], uncertainty_method="bootstrap")
        assert r[1] is None and r[0]["bootstrapped_f"].shape == (3, 2)
    assert not any(kind == "augmented_moments" and 1 in probs for kind, probs in oracle.calls)

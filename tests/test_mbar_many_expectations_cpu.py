"""MbarMany's estimators without a GPU: routing, waves, skipped problems, validation and the host algebra, over numpy
stand-ins of the batch with appended rows (tests/_mbar_many_expectations), checked against the reference's results in
tests/golden/mbar_many_expectations.npz."""
import os

import numpy as np
import pytest

from pymbar_b200 import mbar_many as mm
from pymbar_b200 import mbar_solvers as ms
from pymbar_b200.utils import ParameterError
from tests import _mbar_many as H
from tests import _mbar_many_expectations as E
from tests._mbar_many_expectations import _close, check_case, run_all

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", E.GOLDEN)


@pytest.fixture
def oracle(monkeypatch):
    monkeypatch.setattr(mm, "DeviceMbarBatch", E.AugOracleBatch)
    monkeypatch.setattr(mm, "DeviceProblem", E.AugOracleProblem)
    monkeypatch.setattr(ms, "solve_mbar_for_all_states", H.oracle_all_states)
    monkeypatch.setattr(E.AugOracleBatch, "flagged", ())
    monkeypatch.setattr(E.AugOracleBatch, "aug_flagged", ())
    E.AugOracleBatch.created.clear()
    E.AugOracleBatch.calls.clear()
    E.AugOracleProblem.created.clear()
    return E.AugOracleBatch


def test_golden_through_stand_in(oracle):
    cases = E.load(GOLDEN)
    with mm.MbarMany([c["u_kn"] for c in cases], [c["N_k"] for c in cases]) as m:
        out = run_all(m, cases)
    for i, c in enumerate(cases):
        check_case(c, *(o[i] for o in out))
        K = len(c["N_k"])
        want = "single" if K > 64 else "batch"
        assert [o[i]["path"] for o in out] == [want] * 6, c["name"]


def test_results_are_those_of_mbar_many(oracle):
    cases = E.load(GOLDEN)[:4]
    args = ([c["u_kn"] for c in cases], [c["N_k"] for c in cases])
    ref = mm.mbar_many(*args, return_theta=True)
    with mm.MbarMany(*args, return_theta=True) as m:
        for a, b in zip(ref, m.results):
            assert a.keys() == b.keys()
            for k in a:
                np.testing.assert_array_equal(a[k], b[k])


def test_routing_rows_flags_and_skips(oracle, monkeypatch):
    cases = E.load(GOLDEN)
    pick = [1, 4, 5, 6, 2]                         # K = 2, 22, 33, 64, 9
    monkeypatch.setattr(oracle, "aug_flagged", (4,))   # the fifth problem of the batch: K = 9
    with mm.MbarMany([cases[i]["u_kn"] for i in pick], [cases[i]["N_k"] for i in pick]) as m:
        # entropy and enthalpy: 3K rows, 66 for K = 22, 99 for K = 33, 192 for K = 64 (all batched)
        ent = m.compute_entropy_and_enthalpy([cases[i]["u_kn"] if i != 1 else None for i in pick])
        assert ent[0] is None
        assert [e["path"] for e in ent[1:]] == ["batch", "batch", "batch", "single"]
        for e, i in zip(ent[1:], pick[1:]):
            for k in ("Delta_f", "Delta_u", "Delta_s"):
                _close(e[k], cases[i]["ent"][k], 0, 1e-8, cases[i]["name"])
        # K = 64 with 2K + 1 appended rows exceeds the row limit and takes the single path
        u64 = cases[6]["u_kn"]
        A = np.vstack([u64, u64[:1]])
        r = m.compute_expectations([None, None, None, A, None], u_ln_list=[None, None, None, A, None],
                                   state_dependent=True)
        assert r[:3] == [None, None, None] and r[4] is None
        assert r[3]["path"] == "single"
    # the flagged problem was sent to the device, then solved alone
    assert any(kind == "augmented_moments" and 4 in probs for kind, probs in oracle.calls)


def test_single_path_from_the_solve(oracle, monkeypatch):
    cases = E.load(GOLDEN)
    pick = [2, 6, 3]                               # K = 9, 64, 21
    monkeypatch.setattr(oracle, "flagged", (0,))
    with mm.MbarMany([cases[i]["u_kn"] for i in pick], [cases[i]["N_k"] for i in pick]) as m:
        assert [r["path"] for r in m.results] == ["single", "batch", "batch"]
        reqs = [E.requests(cases[i]["u_kn"]) for i in pick]
        pert = m.compute_perturbed_free_energies([r[2] for r in reqs])
        ovl = m.compute_overlap()
    assert [p["path"] for p in pert] == ["single", "batch", "batch"]
    assert [o["path"] for o in ovl] == ["single", "batch", "batch"]
    for p, o, i in zip(pert, ovl, pick):
        _close(p["Delta_f"], cases[i]["pert"]["Delta_f"], 0, 1e-8, cases[i]["name"])
        _close(p["dDelta_f"], cases[i]["pert"]["dDelta_f"], 1e-5, 1e-8, cases[i]["name"])
        _close(o["matrix"], cases[i]["ovl"]["matrix"], 1e-6, 1e-9, cases[i]["name"])


def test_waves_give_the_same_bits(oracle, monkeypatch):
    cases = E.load(GOLDEN)[:8]
    args = ([c["u_kn"] for c in cases], [c["N_k"] for c in cases])
    with mm.MbarMany(*args) as m:
        one = m.compute_entropy_and_enthalpy()
        waves_one = sum(1 for kind, _ in oracle.calls if kind == "set_unsampled")
    oracle.calls.clear()
    monkeypatch.setattr(mm, "AUG_WAVE_BYTES", 1)
    with mm.MbarMany(*args) as m:
        many = m.compute_entropy_and_enthalpy()
    sets = [probs for kind, probs in oracle.calls if kind == "set_unsampled"]
    batched = [i for i, c in enumerate(cases) if len(c["N_k"]) <= 64]
    assert waves_one == 2                           # one wave, then the drop
    assert sets == [[i] for i in batched] + [[]]    # one problem per wave, in problem order
    for a, b in zip(one, many):
        assert a["path"] == b["path"]
        for k in a:
            if k != "path":
                np.testing.assert_array_equal(a[k], b[k])


def test_wave_bytes_follow_the_geometry():
    # K = 32, N = 160000, M = 64: appended tiles, L_n, pass and Gram partials, output, f
    nT = 5000
    R = 96
    nc = -(-nT // max(max(2048 // R, 4), -(-nT // 4096)))
    want = 8 * (nT * 32 * 65 + nc * (2 * R + 2) + 6 * 10 * 1024 + 2 * R + 2 + R * R + R)
    assert mm.augmented_bytes(32, 160000, 64) == want


def test_validation_before_device_work(oracle):
    cases = E.load(GOLDEN)
    pick = [2, 3]
    us = [cases[i]["u_kn"] for i in pick]
    with mm.MbarMany(us, [cases[i]["N_k"] for i in pick]) as m:
        good = [E.requests(u)[2] for u in us]
        bad_shape = [good[0], good[1][:, :-1]]
        with pytest.raises(ParameterError, match="problem 1"):
            m.compute_perturbed_free_energies(bad_shape)
        nan = good[1].copy()
        nan[0, 5] = np.nan
        shape0 = [good[0][:, :7], nan]
        with pytest.raises(ParameterError, match="problem 0"):
            m.compute_perturbed_free_energies(shape0)
        with pytest.raises(ParameterError, match="problem 1.*NaN"):
            m.compute_expectations([us[0][0], nan[0]])
        with pytest.raises(ParameterError, match="bootstrap"):
            m.compute_expectations([us[0][0], us[1][0]], uncertainty_method="bootstrap")
        with pytest.raises(ParameterError, match="svd"):
            m.compute_entropy_and_enthalpy(uncertainty_method="svd")
        with pytest.raises(ParameterError, match="output"):
            m.compute_expectations([us[0][0], us[1][0]], output="ratios")
        with pytest.raises(ParameterError, match="rows"):
            m.compute_expectations([us[0], us[1][0]], state_dependent=False)
        with pytest.raises(ValueError):
            m.compute_perturbed_free_energies([good[0]])
        assert oracle.calls == []
        # None skips a problem everywhere
        r = m.compute_perturbed_free_energies([None, good[1]])
        assert r[0] is None and r[1]["path"] == "batch"
        assert oracle.calls[0] == ("set_unsampled", [1])


def test_closed_object_keeps_results(oracle):
    c = E.load(GOLDEN)[2]
    m = mm.MbarMany([c["u_kn"]], [c["N_k"]])
    res = m.results
    m.close()
    assert res[0]["path"] == "batch" and m.results is res

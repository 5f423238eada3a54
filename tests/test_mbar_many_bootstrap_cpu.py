"""mbar_many(n_bootstraps=B) without a GPU, over a weighted numpy stand-in of DeviceMbarBatch
(tests/_mbar_many_boot.WeightedOracleBatch): the replicate draws, the seeds, waves, the single replicate path, the
bootstrap uncertainty and the argument checks, against the reference's results in tests/golden/mbar_many_bootstrap.npz."""
import os

import numpy as np
import pytest

from pymbar_b200 import bootstrap
from pymbar_b200 import mbar_many as mm
from pymbar_b200 import mbar_solvers as ms
from pymbar_b200.utils import ParameterError
from tests import _mbar_many as H
from tests import _mbar_many_boot as W

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", W.GOLDEN)


@pytest.fixture
def oracle(monkeypatch):
    monkeypatch.setattr(mm, "DeviceMbarBatch", W.WeightedOracleBatch)
    monkeypatch.setattr(mm, "DeviceProblem", W.WeightedOracleProblem)
    monkeypatch.setattr(ms, "solve_mbar_for_all_states", H.oracle_all_states)
    monkeypatch.setattr(bootstrap, "bootstrap_f_k", W.oracle_bootstrap_f_k)
    monkeypatch.setattr(W.WeightedOracleBatch, "flagged", ())
    monkeypatch.setattr(W.WeightedOracleBatch, "flagged_counts", set())
    W.WeightedOracleBatch.created.clear()
    W.WeightedOracleBatch.uploads.clear()
    W.WeightedOracleProblem.opened.clear()
    return W.WeightedOracleBatch


def _cases(pick):
    cases = W.load(GOLDEN)
    return [cases[i] for i in pick]


def _run(cases, **kw):
    kw.setdefault("n_bootstraps", cases[0]["B"])
    kw.setdefault("rseed", [c["seed"] for c in cases])
    return mm.mbar_many([c["u_kn"] for c in cases], [c["N_k"] for c in cases],
                        f_k_init=[c["f_init"] for c in cases], **kw)


def test_golden_through_stand_in(oracle):
    cases = _cases(range(13))
    res = _run(cases, uncertainty_method="bootstrap")
    for r, c in zip(res, cases):
        assert r["f_k_boots"].shape == (c["B"], len(c["N_k"]))
        np.testing.assert_allclose(r["f_k_boots"], c["f_k_boots"], rtol=0, atol=1e-8, err_msg=c["name"])
        np.testing.assert_allclose(r["dDelta_f"], c["dDelta_f"], rtol=0, atol=1e-8, err_msg=c["name"])
        assert r["boot_single"] == (c["B"] if len(c["N_k"]) > 64 else 0), c["name"]


def test_counts_are_the_reference_draws(oracle):
    cases = _cases([1, 3, 9, 10])
    B = 7
    _run(cases, n_bootstraps=B, compute_uncertainty=False)
    got = {}
    for problems, counts in oracle.uploads:
        for p, c in zip(problems, counts):
            got.setdefault(int(p), []).append(c)
    for p, c in enumerate(cases):
        want = bootstrap.bootstrap_indices(c["N_k"].astype(np.int64), B, c["seed"])
        want = np.array([np.bincount(r, minlength=c["u_kn"].shape[1]) for r in want])
        np.testing.assert_array_equal(np.array(got[p]), want, err_msg=c["name"])


def test_rseed_none_draws_one_seed_per_problem(oracle):
    cases = _cases([1, 3, 5])
    np.random.seed(123)
    res = _run(cases, rseed=None, compute_uncertainty=False)
    after = np.random.randint(1 << 30)
    np.random.seed(123)
    seeds = [np.random.randint(np.iinfo(np.int32).max) for _ in cases]
    assert np.random.randint(1 << 30) == after
    want = _run(cases, rseed=seeds, compute_uncertainty=False)
    for r, w in zip(res, want):
        np.testing.assert_array_equal(r["f_k_boots"], w["f_k_boots"])
    # n_bootstraps = 0 leaves np.random alone
    np.random.seed(5)
    _run(cases, n_bootstraps=0, rseed=None, compute_uncertainty=False)
    now = np.random.randint(1 << 30)
    np.random.seed(5)
    assert np.random.randint(1 << 30) == now


def test_bootstrap_std_formula(oracle):
    (c,) = _cases([5])
    r = _run([c], uncertainty_method="bootstrap", return_theta=True)[0]
    fb = r["f_k_boots"]
    diffm = np.array([f - np.vstack(f) for f in fb])
    np.testing.assert_array_equal(r["dDelta_f"], np.std(diffm, axis=0))
    assert r["Theta"].shape == (16, 16)
    svd = _run([c], n_bootstraps=0, rseed=None, uncertainty_method="svd-ew", return_theta=True)[0]
    np.testing.assert_allclose(r["Theta"], svd["Theta"], rtol=1e-12, atol=1e-15)
    plain = _run([c], uncertainty_method="svd-ew")[0]
    assert plain["f_k_boots"].shape == fb.shape and not np.array_equal(plain["dDelta_f"], r["dDelta_f"])


def test_wave_size_does_not_change_results(oracle, monkeypatch):
    cases = _cases([1, 3, 5, 10])
    full = _run(cases, compute_uncertainty=False)
    n_full = len(oracle.uploads)
    oracle.uploads.clear()
    monkeypatch.setattr(mm, "BOOT_WAVE_BYTES", 1)            # one slot per wave
    small = _run(cases, compute_uncertainty=False)
    assert n_full == 1 and len(oracle.uploads) == sum(c["B"] for c in cases)
    assert all(len(p) == 1 for p, _ in oracle.uploads)
    for a, b in zip(full, small):
        np.testing.assert_array_equal(a["f_k_boots"], b["f_k_boots"])
    oracle.uploads.clear()
    monkeypatch.setattr(mm, "BOOT_WAVE_BYTES", 3 * mm.slot_bytes(*cases[1]["u_kn"].shape))
    mid = _run(cases, compute_uncertainty=False)
    assert 1 < len(oracle.uploads) < sum(c["B"] for c in cases)
    for a, b in zip(full, mid):
        np.testing.assert_array_equal(a["f_k_boots"], b["f_k_boots"])


def test_flagged_replicate_alone_goes_single(oracle):
    cases = _cases([1, 3, 8, 5])                 # K = 2, 8, 65, 16
    B = cases[0]["B"]
    ref = _run(cases, compute_uncertainty=False)
    # flag replicate 4 of the second problem (batch problem 1)
    rints = bootstrap.bootstrap_indices(cases[1]["N_k"].astype(np.int64), B, cases[1]["seed"])
    c4 = np.bincount(rints[4], minlength=cases[1]["u_kn"].shape[1]).astype(np.uint16)
    oracle.flagged_counts = {(1, c4.tobytes())}
    res = _run(cases, compute_uncertainty=False)
    assert [r["boot_single"] for r in res] == [0, 1, B, 0]
    for r, w in zip(res, ref):
        np.testing.assert_allclose(r["f_k_boots"], w["f_k_boots"], rtol=0, atol=1e-9)
    # the single path opened one problem per problem that needed it, in input order
    assert [p.u.shape for p in W.WeightedOracleProblem.opened[-2:]] == [cases[1]["u_kn"].shape,
                                                                       cases[2]["u_kn"].shape]


def test_no_bootstraps_is_unchanged(oracle):
    cases = _cases([1, 5])
    r = _run(cases, n_bootstraps=0, rseed=None, return_theta=True)
    assert all("f_k_boots" not in x and "boot_single" not in x for x in r)
    assert oracle.uploads == []


def test_validation(oracle):
    cases = _cases([1, 5])
    for bad in (-1, 2.0, True, "3"):
        with pytest.raises(ParameterError, match="n_bootstraps"):
            _run(cases, n_bootstraps=bad)
    with pytest.raises(ParameterError, match="single seed"):
        _run(cases, rseed=7)
    with pytest.raises(ParameterError, match="one seed per problem"):
        _run(cases, rseed=[1])
    with pytest.raises(ParameterError, match="Cannot request bootstrap sampling"):
        _run(cases, n_bootstraps=0, rseed=None, uncertainty_method="bootstrap")
    assert oracle.created == []

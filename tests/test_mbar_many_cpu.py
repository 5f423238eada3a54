"""mbar_many without a GPU: validation, routing, result order and post-processing over a numpy stand-in of
DeviceMbarBatch (tests/_mbar_many.OracleBatch), checked against the reference's results in tests/golden/mbar_many.npz."""
import os

import numpy as np
import pytest

from pymbar_b200 import mbar_many as mm
from pymbar_b200 import mbar_solvers as ms
from pymbar_b200.utils import ParameterError
from tests import _mbar_many as H

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", H.GOLDEN)


@pytest.fixture
def oracle(monkeypatch):
    monkeypatch.setattr(mm, "DeviceMbarBatch", H.OracleBatch)
    monkeypatch.setattr(mm, "DeviceProblem", H.OracleProblem)
    monkeypatch.setattr(ms, "solve_mbar_for_all_states", H.oracle_all_states)
    monkeypatch.setattr(H.OracleBatch, "flagged", ())
    H.OracleBatch.created.clear()
    return H.OracleBatch


def _check(r, c):
    K = len(c["N_k"])
    assert r["f_k"].shape == (K,)
    np.testing.assert_allclose(r["Delta_f"], c["Delta_f"], rtol=0, atol=1e-8, err_msg=c["name"])
    np.testing.assert_allclose(r["dDelta_f"], c["dDelta_f"], rtol=1e-6, atol=1e-9, err_msg=c["name"])
    if K > 1:   # one state: Theta is the pseudo-inverse of a rounding residue, in the reference as here
        np.testing.assert_allclose(r["Theta"], c["Theta"], rtol=1e-5, atol=1e-9, err_msg=c["name"])


def test_golden_through_stand_in(oracle):
    cases = H.load(GOLDEN)
    res = mm.mbar_many([c["u_kn"] for c in cases], [c["N_k"] for c in cases], f_k_init=[c["f_init"] for c in cases],
                       return_theta=True)
    assert len(res) == len(cases)
    for r, c in zip(res, cases):
        _check(r, c)
        assert r["success"]
        assert r["path"] == ("single" if len(c["N_k"]) > 64 else "batch"), c["name"]
    # one batch object held every problem with K <= 64, in input order
    (b,) = oracle.created
    assert [u.shape for u in b.u] == [c["u_kn"].shape for c in cases if len(c["N_k"]) <= 64]


def test_flagged_problem_goes_single_and_order_is_kept(oracle, monkeypatch):
    cases = H.load(GOLDEN)
    pick = [1, 8, 3, 5]                      # K = 2, 65, 8, 16
    monkeypatch.setattr(oracle, "flagged", (1,))  # the second problem of the batch: K = 8
    res = mm.mbar_many([cases[i]["u_kn"] for i in pick], [cases[i]["N_k"] for i in pick], return_theta=True)
    assert [r["path"] for r in res] == ["batch", "single", "single", "batch"]
    for r, i in zip(res, pick):
        _check(r, cases[i])
    assert res[1]["iterations"] is None and res[0]["iterations"] >= 0


def test_uncertainty_options(oracle):
    c = H.load(GOLDEN)[5]
    r = mm.mbar_many([c["u_kn"]], [c["N_k"]], compute_uncertainty=False)[0]
    assert "dDelta_f" not in r and "Theta" not in r
    r = mm.mbar_many([c["u_kn"]], [c["N_k"]], uncertainty_method="approximate", return_theta=True)[0]
    assert r["Theta"].shape == (16, 16)
    with pytest.raises(ParameterError):
        mm.mbar_many([c["u_kn"]], [c["N_k"]], uncertainty_method="svd")
    with pytest.raises(ParameterError):
        mm.mbar_many([c["u_kn"]], [c["N_k"]], uncertainty_method="bootstrap")


def test_validation_lowest_index_first(oracle):
    c = H.load(GOLDEN)[2]
    good_u, good_N = c["u_kn"], c["N_k"]
    bad_sum = good_N.copy()
    bad_sum[0] += 1
    with pytest.raises(ParameterError, match="sums to"):
        mm.mbar_many([good_u, good_u, good_u[:, :10]], [good_N, bad_sum, good_N])
    with pytest.raises(ValueError, match="shape"):
        mm.mbar_many([good_u, good_u[:, :10], good_u], [good_N, good_N[:3], bad_sum])
    with pytest.raises(ParameterError, match="numpy array"):
        mm.mbar_many([good_u.tolist()], [good_N])
    nan = good_u.copy()
    nan[1, 3] = np.nan
    with pytest.raises(ParameterError, match="NaN"):
        mm.mbar_many([good_u, nan], [good_N, good_N])
    with pytest.raises(ValueError):
        mm.mbar_many([good_u], [good_N, good_N])
    # nothing reached the device before the error
    assert oracle.created == []
    assert mm.mbar_many([], []) == []


def test_default_options_are_the_adaptive_stage(oracle, monkeypatch):
    seen = {}
    orig = oracle.solve

    def solve(self, f_list=None, **kw):
        seen.update(kw)
        return orig(self, f_list, **kw)

    monkeypatch.setattr(oracle, "solve", solve)
    c = H.load(GOLDEN)[3]
    mm.mbar_many([c["u_kn"]], [c["N_k"]])
    assert seen == dict(tol=1e-12, maxiter=10000, min_sc_iter=0, gamma=1.0)
    mm.mbar_many([c["u_kn"]], [c["N_k"]], solver_tolerance=1e-10, options=dict(maxiter=50))
    assert seen["tol"] == 1e-10 and seen["maxiter"] == 50 and seen["min_sc_iter"] == 0

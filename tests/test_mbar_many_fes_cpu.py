"""MbarMany's histogram FES without a GPU: routing, waves, skipped problems, validation and the host algebra, over
numpy stand-ins of the batch's bin_moments (tests/_mbar_many_fes), checked against the reference's results in
tests/golden/mbar_many_fes.npz."""
import numpy as np
import pytest

from pymbar_b200 import mbar_many as mm
from pymbar_b200 import mbar_solvers as ms
from pymbar_b200.utils import ParameterError
from tests import _mbar_many as H
from tests import _mbar_many_fes as F


@pytest.fixture
def oracle(monkeypatch):
    monkeypatch.setattr(mm, "DeviceMbarBatch", F.FesOracleBatch)
    monkeypatch.setattr(mm, "DeviceProblem", F.FesOracleProblem)
    monkeypatch.setattr(ms, "solve_mbar_for_all_states", H.oracle_all_states)
    monkeypatch.setattr(F.FesOracleBatch, "flagged", ())
    monkeypatch.setattr(F.FesOracleBatch, "bin_flagged", ())
    monkeypatch.setattr(F.FesOracleBatch, "bin_flagged_C", ())
    F.FesOracleBatch.created.clear()
    F.FesOracleBatch.calls.clear()
    F.FesOracleProblem.created.clear()
    return F.FesOracleBatch


def _bin_calls(oracle):
    return [c[1:] for c in oracle.calls if c[0] == "bin_moments"]


def _args(cases):
    return [c["u_kn"] for c in cases], [c["N_k"].astype(np.float64) for c in cases]


def test_golden_through_stand_in(oracle):
    cases = F.load()
    with mm.MbarMany(*_args(cases)) as m:
        out = F.run_all(m, cases)
        for i, c in enumerate(cases):
            F.check_case(c, m.histogram_datas[i], {k: v[i] for k, v in out.items()})
            want = "single" if len(c["N_k"]) > 64 else "batch"
            assert all(v[i]["path"] == want for v in out.values()), c["name"]
    # one call for f, one for C and D (the first analytical query), each over the five batched problems
    assert _bin_calls(oracle) == [([0, 1, 2, 3, 4], False), ([0, 1, 2, 3, 4], True)]


def test_routing_flags_and_skips(oracle, monkeypatch):
    cases = F.load()
    monkeypatch.setattr(oracle, "flagged", (1,))          # problem 1 takes the single path in the solve
    monkeypatch.setattr(oracle, "bin_flagged", (2,))      # problem 2's f request is flagged
    monkeypatch.setattr(oracle, "bin_flagged_C", (3,))    # problem 3's C and D request is flagged
    with mm.MbarMany(*_args(cases)) as m:
        assert [r["path"] for r in m.results] == ["batch", "single", "batch", "batch", "batch", "single"]
        out = F.run_all(m, cases, skip=(4,))
        for i, c in enumerate(cases):
            if i == 4:
                assert m.histogram_datas[i] is None
                assert all(v[i] is None for v in out.values())
                continue
            F.check_case(c, m.histogram_datas[i], {k: v[i] for k, v in out.items()})
        assert [out[("lowest", "none")][i]["path"] for i in (0, 1, 2, 3, 5)] == \
            ["batch", "single", "single", "batch", "single"]
        assert [out[("lowest", "analytical")][i]["path"] for i in (0, 1, 2, 3, 5)] == \
            ["batch", "single", "single", "single", "single"]
    assert _bin_calls(oracle) == [([0, 2, 3], False), ([0, 3], True)]


def test_theta_is_computed_once(oracle):
    cases = F.load()[:3]
    with mm.MbarMany(*_args(cases)) as m:
        F.run_all(m, cases)
        n = len(_bin_calls(oracle))
        m.get_fes([c["queries"] for c in cases], uncertainty_method="analytical")
        assert len(_bin_calls(oracle)) == n
        # a new surface drops its problem's Theta: the next analytical query asks for that problem alone
        c = cases[1]
        m.generate_fes([None, c["u_n"], None], [None, c["x_n"], None],
                       histogram_parameters={"bin_edges": c["bin_edges"]})
        m.get_fes([c["queries"] for c in cases], uncertainty_method="analytical")
        assert _bin_calls(oracle)[n:] == [([1], False), ([1], True)]


def test_waves_give_the_same_bits(oracle, monkeypatch):
    cases = F.load()
    with mm.MbarMany(*_args(cases)) as m:
        one = F.run_all(m, cases)
    assert len(_bin_calls(oracle)) == 2
    oracle.calls.clear()
    monkeypatch.setattr(mm, "FES_WAVE_BYTES", 1)
    with mm.MbarMany(*_args(cases)) as m:
        many = F.run_all(m, cases)
    assert _bin_calls(oracle) == [([i], False) for i in range(5)] + [([i], True) for i in range(5)]
    for k in one:
        for a, b in zip(one[k], many[k]):
            assert a.keys() == b.keys()
            for key in a:
                np.testing.assert_array_equal(a[key], b[key])


def test_wave_bytes_follow_the_geometry():
    # K = 32, N = 160000, 2500 bins: the sums pass has 64 sample chunks of 79 tiles; the moments pass, 6 bin chunks
    # of 418 and, under the 4 MB cap of partials, 6 sample chunks of 834 tiles
    nT, K, nb = 5000, 32, 2500
    assert mm._bin_geometry(nT, 1, nb) == (2500, 1, 64)
    assert mm._bin_geometry(nT, K + 1, nb) == (418, 6, 6)
    want = 20 * nT * 32 + 40 * nb + 8 * 6 * (K + 1) * nb + 8 * (K + 1) * nb + 8 * K + 164
    assert mm.bin_bytes(K, 160000, nb, True) == want
    assert mm.bin_bytes(K, 160000, nb, False) == 20 * nT * 32 + 40 * nb + 8 * 64 * nb + 8 * K + 164


def test_single_value_and_per_problem_arguments(oracle):
    cases = [F.load()[i] for i in (1, 4)]                # two 1-D problems
    with mm.MbarMany(*_args(cases)) as m:
        edges = cases[0]["bin_edges"]
        m.generate_fes([c["u_n"] for c in cases], [c["x_n"] for c in cases], histogram_parameters={"bin_edges": edges})
        assert all(np.array_equal(h["bins"][0], edges) for h in m.histogram_datas)
        q = [edges[1:3]] * 2
        one = m.get_fes(q, reference_point="from-specified", fes_reference=0.05)
        per = m.get_fes(q, reference_point="from-specified", fes_reference=[0.05, 0.05])
        for a, b in zip(one, per):
            np.testing.assert_array_equal(a["f_i"], b["f_i"])


def test_validation_before_device_work(oracle):
    cases = F.load()[:2]
    with mm.MbarMany(*_args(cases)) as m:
        u = [c["u_n"] for c in cases]
        x = [c["x_n"] for c in cases]
        hp = [{"bin_edges": c["bin_edges"]} for c in cases]
        with pytest.raises(ParameterError, match="fes_type"):
            m.generate_fes(u, x, fes_type="kde", histogram_parameters=hp)
        with pytest.raises(ParameterError, match="u_n_list must hold one entry"):
            m.generate_fes(u[:1], x, histogram_parameters=hp)
        with pytest.raises(ParameterError, match="x_n_list must hold one entry"):
            m.generate_fes(u, x + x, histogram_parameters=hp)
        with pytest.raises(ParameterError, match="problem 1: u_n has shape"):
            m.generate_fes([u[0], u[1][:-1]], x, histogram_parameters=hp)
        nan = u[1].copy()
        nan[3] = np.nan
        with pytest.raises(ParameterError, match="problem 1: u_n holds NaN"):
            m.generate_fes([u[0], nan], x, histogram_parameters=hp)
        with pytest.raises(ParameterError, match="problem 0: x_n has shape"):
            m.generate_fes(u, [np.stack([x[0], x[0]], axis=1), x[1]], histogram_parameters=hp)
        with pytest.raises(ParameterError, match="problem 1: give both"):
            m.generate_fes([u[0], None], x, histogram_parameters=hp)
        with pytest.raises(ParameterError, match="bin_edges"):
            m.generate_fes(u, x, histogram_parameters=None)
        with pytest.raises(ParameterError, match="problem 0: get_fes before generate_fes"):
            m.get_fes([c["queries"] for c in cases])
        assert _bin_calls(oracle) == []
        m.generate_fes([None, u[1]], [None, x[1]], histogram_parameters=hp)
        assert _bin_calls(oracle) == [([1], False)]
        with pytest.raises(ParameterError, match="problem 0: get_fes before generate_fes"):
            m.get_fes([c["queries"] for c in cases])
        q = [None, cases[1]["queries"]]
        with pytest.raises(ParameterError, match="bootstrap"):
            m.get_fes(q, uncertainty_method="bootstrap")
        with pytest.raises(ParameterError, match="x_list must hold one entry"):
            m.get_fes(q[1:])
        with pytest.raises(Exception, match="all-differences"):
            m.get_fes(q, reference_point="all-differences", uncertainty_method="analytical")
        with pytest.raises(Exception, match="from-normalization"):
            m.get_fes(q, reference_point="from-normalization", uncertainty_method="analytical")
        with pytest.raises(Exception, match="Specified reference point"):
            m.get_fes(q, reference_point="from-specified")
        assert _bin_calls(oracle) == [([1], False)]
        r = m.get_fes(q)
        assert r[0] is None and r[1]["path"] == "batch"


def test_single_path_errors_name_the_problem(oracle, monkeypatch):
    cases = F.load()

    def boom(*args, **kwargs):
        raise RuntimeError("device failure")

    monkeypatch.setattr(F.FesOracleProblem, "bin_moments", boom)
    with mm.MbarMany(*_args(cases)) as m:
        with pytest.raises(RuntimeError, match="device failure") as e:
            F.run_all(m, cases)
    assert any("problem 5" in note for note in e.value.__notes__)

"""MbarMany's KDE surfaces without a GPU: golden parity, the draw stream, routing, waves, the byte model, validation,
atomicity and the reference's quirks, over numpy stand-ins of the batch's log_weights and of DeviceKdeMany
(tests/_mbar_many_fes_kde), checked against the reference's results in tests/golden/mbar_many_fes_kde.npz."""
import numpy as np
import pytest

from pymbar_b200 import bootstrap
from pymbar_b200 import fes_bootstrap as fb
from pymbar_b200 import mbar_many as mm
from pymbar_b200 import mbar_solvers as ms
from pymbar_b200.utils import ParameterError
from tests import _mbar_many as H
from tests import _mbar_many_boot as W
from tests import _mbar_many_fes_kde as FK

pytest.importorskip("sklearn")


@pytest.fixture
def oracle(monkeypatch):
    monkeypatch.setattr(mm, "DeviceMbarBatch", FK.KdeOracleBatch)
    monkeypatch.setattr(mm, "DeviceProblem", FK.KdeOracleProblem)
    monkeypatch.setattr(mm, "DeviceKdeMany", FK.NumpyKdeMany)
    monkeypatch.setattr(ms, "solve_mbar_for_all_states", H.oracle_all_states)
    monkeypatch.setattr(bootstrap, "bootstrap_f_k", W.oracle_bootstrap_f_k)
    for name in ("flagged", "bin_flagged", "bin_flagged_C", "rep_bin_flagged", "lw_flagged"):
        monkeypatch.setattr(FK.KdeOracleBatch, name, ())
    monkeypatch.setattr(FK.KdeOracleBatch, "flagged_counts", set())
    FK.KdeOracleBatch.calls.clear()
    FK.NumpyKdeMany.calls.clear()
    state = np.random.get_state()
    yield FK.KdeOracleBatch
    np.random.set_state(state)


@pytest.fixture(scope="module")
def golden():
    return FK.load()


PLAIN = [i for i in range(len(FK.SPECS)) if i not in FK.RAISES]


def _lw_calls(oracle):
    return [c[1] for c in oracle.calls if c[0] == "log_weights"]


def test_golden_plain(oracle, golden):
    cases, _ = golden
    with mm.MbarMany(*FK.args(cases)) as m:
        FK.generate(m, cases, range(len(cases)))
        assert m.fes_types == ["kde"] * len(cases)
        # one log_weights call for the batched problems (batch slots); the K = 70 problem takes the single path
        assert _lw_calls(oracle) == [[0, 1, 2, 3, 4, 5]]
        assert [m._kde[p]["path"] for p in range(len(cases))] == ["batch"] * 5 + ["single", "batch"]
        for tag, rp in FK.REFS:
            out = FK.query(m, cases, PLAIN, rp)
            for i in PLAIN:
                FK.check_plain(cases[i], out[i], tag)
                assert out[i]["path"] == m._kde[i]["path"]
        assert len(FK.NumpyKdeMany.calls) == 3 and all(len(c) == len(PLAIN) for c in FK.NumpyKdeMany.calls)
        # the epanechnikov problem: KernelDensity.sample raises, as in the reference
        with pytest.raises(NotImplementedError):
            FK.query(m, cases, FK.RAISES, "from-lowest")
        e = FK.RAISES[0]
        k = m._kde[e]
        got = FK.NumpyKdeMany([cases[e]["x_n"]]).log_sum([0], ["epanechnikov"], [k["settings"]["h"]], [k["w"]],
                                                              [cases[e]["queries"]])[0]
        from pymbar_b200 import fes as hist

        score = got + hist.kde_log_norm("epanechnikov", 1, k["settings"]["h"]) - k["log_sum_w"]
        want = cases[e]["score"]
        np.testing.assert_array_equal(np.isinf(score), np.isinf(want))
        np.testing.assert_allclose(score[np.isfinite(want)], want[np.isfinite(want)], rtol=0, atol=1e-8)


@pytest.mark.parametrize("run", FK.RUNS)
def test_golden_bootstrap(oracle, golden, run):
    cases, stream_next = golden
    with mm.MbarMany(*FK.args(cases)) as m:
        if run == "seeded":
            FK.generate(m, cases, FK.BOOT, FK.B, seed=[FK.SEED0 + i if i in FK.BOOT else None
                                                       for i in range(len(cases))])
        else:
            np.random.seed(FK.STREAM_SEED)
            FK.generate(m, cases, FK.BOOT, FK.B)
            assert np.random.randint(2 ** 31 - 1) == stream_next
        for tag, rp in FK.BOOT_REFS:
            FK.NumpyKdeMany.calls.clear()
            out = FK.query(m, cases, FK.BOOT, rp, "bootstrap")
            for i in FK.BOOT:
                FK.check_boot(cases[i], out[i], run, tag)
            # one log_sum call: b = 0 and every replicate of every problem
            assert FK.NumpyKdeMany.calls == [list(range(len(FK.BOOT))) + [s for s in range(len(FK.BOOT))
                                                                          for _ in range(FK.B)]]


def test_waves_of_one_request(oracle, golden, monkeypatch):
    cases, _ = golden
    keep = FK.BOOT[:3]
    with mm.MbarMany(*FK.args(cases)) as m:
        FK.generate(m, cases, keep, 3, seed=[7, 8, 9, None, None, None, None])
        a = FK.query(m, cases, keep, "from-specified", "bootstrap")
        FK.NumpyKdeMany.calls.clear()
        monkeypatch.setattr(mm, "KDE_WAVE_BYTES", mm.KDE_PART_BYTES + 1)
        b = FK.query(m, cases, keep, "from-specified", "bootstrap")
        assert len(FK.NumpyKdeMany.calls) == 3 * 4 and all(len(c) == 1 for c in FK.NumpyKdeMany.calls)
        for i in keep:
            np.testing.assert_array_equal(a[i]["f_i"], b[i]["f_i"])
            np.testing.assert_array_equal(a[i]["df_i"], b[i]["df_i"])


def test_byte_model():
    # N = 5000: nPad 5120, 2 chunks; Q = 100 queries in D = 2: one piece
    assert mm._kde_chunks(5000) == (5120, 2)
    assert mm.kde_bytes(5000, 2, 100) == 8 * 5120 + 8 * 2 * 100 + 8 * 100 + 2 * 112
    # 1024 chunks: pieces of 4096 queries
    N = 1024 * 4096 * 2
    assert mm._kde_chunks(N)[1] == 1024
    assert mm.kde_bytes(N, 1, 4097) == 8 * N + 16 * 4097 + 2 * 112 * 2
    assert mm.log_weight_bytes(8, 100) == 8 * 128 + 64 + 4 + 164


def test_routing_and_flags(oracle, golden, monkeypatch):
    cases, _ = golden
    monkeypatch.setattr(FK.KdeOracleBatch, "lw_flagged", (1,))
    with mm.MbarMany(*FK.args(cases)) as m:
        FK.generate(m, cases, [0, 1, 5])
        assert [m._kde[p]["path"] for p in (0, 1, 5)] == ["batch", "single", "single"]
        out = FK.query(m, cases, [0, 1, 5], "from-lowest")
        for i in (0, 1, 5):
            FK.check_plain(cases[i], out[i], "lowest")
            assert out[i]["path"] == m._kde[i]["path"]


def test_validation_before_any_work(oracle, golden):
    cases, _ = golden
    sel = cases[:2]
    with mm.MbarMany(*FK.args(sel)) as m:
        u = [c["u_n"] for c in sel]
        x = [c["x_n"] for c in sel]
        kp = [c["kde_parameters"] for c in sel]
        state = np.random.get_state()

        def bad(match, **kw):
            a = dict(u_n_list=u, x_n_list=x, fes_type="kde", kde_parameters=kp, n_bootstraps=3)
            a.update(kw)
            with pytest.raises(ParameterError, match=match):
                m.generate_fes(**a)

        bad("Warning: nope is not a parameter", kde_parameters=[{"nope": 1}, kp[1]])
        bad("problem 1: fes_type 'kde' needs kde_parameters", kde_parameters=[kp[0], None])
        bad("problem 0: .* are not served", kde_parameters={"metric": "manhattan"})
        bad("problem 0: .* are not served", kde_parameters={"metric_params": {"p": 1}})
        bad("problem 1: .* are not served", kde_parameters=[kp[0], {"bandwidth": -1.0}])
        bad("problem 1: .* are not served", x_n_list=[x[0], np.tile(x[1][:, None], (1, 5))])
        nan = x[1].copy()
        nan[4] = np.inf
        bad("problem 1: x_n holds NaN or infinite", x_n_list=[x[0], nan])
        bad("problem 0: x_n has shape", x_n_list=[x[0][:-1], x[1]])
        bad("problem 1: u_n has shape", u_n_list=[u[0], u[1][:-2]])
        bad("seed must hold one entry", seed=[1])
        with pytest.raises(ValueError, match="n_bootstraps"):
            m.generate_fes(u, x, fes_type="kde", kde_parameters=kp, n_bootstraps=1)
        assert np.array_equal(np.random.get_state()[1], state[1])
        assert FK.KdeOracleBatch.calls == [] or all(c[0] != "log_weights" for c in FK.KdeOracleBatch.calls)
        assert FK.NumpyKdeMany.created == 0 or FK.NumpyKdeMany.calls == []
        assert m.fes_types == [None, None]


def test_empty_state_and_atomicity(oracle, golden, monkeypatch):
    cases, _ = golden
    uns = FK.NAMES.index("1d_unsampled")
    with mm.MbarMany(*FK.args(cases)) as m:
        FK.generate(m, cases, [0])
        before = m._kde[0]
        state = np.random.get_state()
        with pytest.raises(ParameterError, match=f"problem {uns}: a state without samples"):
            FK.generate(m, cases, [0, uns], 3)
        # an error after the first draw: the generator is restored and no surface changes
        calls = []

        def boom(N_k, n, each=None):
            calls.append(1)
            if len(calls) == 2:
                np.random.randint(5)
                raise RuntimeError("boom")
            return real(N_k, n, each)

        real = fb.draw_replicates
        monkeypatch.setattr(fb, "draw_replicates", boom)
        with pytest.raises(RuntimeError, match="boom"):
            FK.generate(m, cases, [0, 1], 3)
        assert np.array_equal(np.random.get_state()[1], state[1])
        assert m._kde[0] is before and 1 not in m._kde
        assert m.fes_types[:2] == ["kde", None]


def test_mixed_histogram_and_kde(oracle, golden):
    from tests import _mbar_many_fes as F

    hcases = F.load()[:2]
    cases, _ = golden
    sel = [hcases[0], cases[1]]
    with mm.MbarMany([c["u_kn"] for c in sel], [c["N_k"] for c in sel]) as m:
        m.generate_fes([hcases[0]["u_n"], None], [hcases[0]["x_n"], None],
                       histogram_parameters={"bin_edges": hcases[0]["bin_edges"]})
        m.generate_fes([None, cases[1]["u_n"]], [None, cases[1]["x_n"]], fes_type="kde",
                       kde_parameters=cases[1]["kde_parameters"])
        assert m.fes_types == ["histogram", "kde"]
        out = m.get_fes([hcases[0]["queries"], cases[1]["queries"]], reference_point="from-lowest")
        FK.check_plain(cases[1], out[1], "lowest")
        assert "df_i" not in out[0] and np.isfinite(out[0]["f_i"]).any()
        # a histogram surface replaces problem 1's KDE surface, and the reverse
        m.generate_fes([hcases[0]["u_n"], None], [hcases[0]["x_n"], None], fes_type="kde",
                       kde_parameters={"bandwidth": 0.1})
        assert m.fes_types == ["kde", "kde"] and m.histogram_datas[0] is None
        assert m.kde_settings[0] == {"kernel": "gaussian", "h": 0.1, "D": 1}


def test_query_quirks(oracle, golden):
    cases, _ = golden
    keep = [0, 3]
    with mm.MbarMany(*FK.args(cases)) as m:
        FK.generate(m, cases, keep, 2, seed=[1, None, None, 2, None, None, None])
        q = FK.select(cases, keep, "queries")
        # gaussian and tophat draw one uniform and D normals per query, as KernelDensity.sample does
        np.random.seed(5)
        m.get_fes(q, reference_point="from-lowest")
        got = np.random.get_state()[1].copy()
        np.random.seed(5)
        for D in (1, 2):
            np.random.uniform(0, 1, size=1)
            np.random.normal(size=(1, D))
        assert np.array_equal(got, np.random.get_state()[1])
        with pytest.raises(ParameterError, match="analytical for kde is not implemented"):
            m.get_fes(q, reference_point="from-lowest", uncertainty_method="analytical")
        with pytest.raises(ParameterError, match="from-normalization"):
            m.get_fes(q, reference_point="from-normalization", uncertainty_method="bootstrap")
        with pytest.raises(ParameterError, match="reference point choice nope"):
            m.get_fes(q, reference_point="nope")
        from pymbar_b200.fes import _kde_errors

        DataError = _kde_errors()[0]
        state = np.random.get_state()
        with pytest.raises(DataError, match="inconsistent dimension"):
            m.get_fes([q[3]] + q[1:], reference_point="from-lowest")
        assert np.array_equal(np.random.get_state()[1], state[1])      # restored
        FK.generate(m, cases, [0])
        with pytest.raises(ParameterError, match="Cannot calculate bootstrap error"):
            m.get_fes([q[0]] + [None] * 6, uncertainty_method="bootstrap")
    with pytest.raises(ParameterError, match="freed by close"):
        m.get_fes([q[0]] + [None] * 6)
    assert FK.NumpyKdeMany.closed >= 2

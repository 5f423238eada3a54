"""MbarMany's bootstrap histogram FES without a GPU: the draw stream, waves, routing, validation, atomicity and the host
algebra, over numpy stand-ins of the batch's replicate slots and weighted bin pass (tests/_mbar_many_fes_bootstrap),
checked against the reference's results in tests/golden/mbar_many_fes_bootstrap.npz."""
import numpy as np
import pytest

from pymbar_b200 import bootstrap
from pymbar_b200 import fes_bootstrap as fb
from pymbar_b200 import mbar_many as mm
from pymbar_b200 import mbar_solvers as ms
from pymbar_b200.utils import ParameterError
from tests import _mbar_many as H
from tests import _mbar_many_boot as W
from tests import _mbar_many_fes as F
from tests import _mbar_many_fes_bootstrap as FB


@pytest.fixture
def oracle(monkeypatch):
    monkeypatch.setattr(mm, "DeviceMbarBatch", FB.FesBootOracleBatch)
    monkeypatch.setattr(mm, "DeviceProblem", FB.FesBootOracleProblem)
    monkeypatch.setattr(ms, "solve_mbar_for_all_states", H.oracle_all_states)
    monkeypatch.setattr(bootstrap, "bootstrap_f_k", W.oracle_bootstrap_f_k)
    for name in ("flagged", "bin_flagged", "bin_flagged_C", "rep_bin_flagged"):
        monkeypatch.setattr(FB.FesBootOracleBatch, name, ())
    monkeypatch.setattr(FB.FesBootOracleBatch, "flagged_counts", set())
    FB.FesBootOracleBatch.calls.clear()
    state = np.random.get_state()
    yield FB.FesBootOracleBatch
    np.random.set_state(state)


@pytest.fixture(scope="module")
def golden():
    return FB.load()


def _calls(oracle, kind):
    return [c[1:] for c in oracle.calls if c[0] == kind]


def _draw_calls(oracle):
    return _calls(oracle, "replicate_bin_moments") + _calls(oracle, "bin_moments")


@pytest.mark.parametrize("run", FB.RUNS)
def test_golden_through_stand_in(oracle, golden, run):
    cases, stream_next = golden
    with mm.MbarMany(*FB.args(cases)) as m:
        out, nxt = FB.run(m, cases, run)
        for i, c in enumerate(cases):
            FB.check_case(c, run, m, i, out)
        assert m.fes_boot_single == [0, 0, 0, 0, FB.B]       # the K = 70 problem takes the single path
    if run == "stream":
        assert nxt == stream_next
    # one wave: every replicate of the four batched problems in one replicate_bin_moments call
    assert _calls(oracle, "replicate_bin_moments") == [([0, 1, 2, 3], [p for p in range(4) for _ in range(FB.B)])]


def _expected_state(cases, seeds, B):
    """numpy's global generator after P reference generate_fes calls, from fes_bootstrap.draw_replicates."""
    for c, s in zip(cases, seeds):
        if c is None:
            continue
        if s is not None and s >= 0:
            np.random.seed(s)
        fb.draw_replicates(c["N_k"], B)
    return np.random.get_state()


@pytest.mark.parametrize("mode", ["per_problem", "stream", "mixed"])
def test_generator_ends_where_the_reference_leaves_it(oracle, golden, mode):
    cases = golden[0][:3]
    seeds = {"per_problem": [5, 6, 7], "stream": None, "mixed": [5, -1, None]}[mode]
    skip = (1,) if mode == "mixed" else ()
    sel = [None if i in skip else c for i, c in enumerate(cases)]
    np.random.seed(99)
    want = _expected_state(sel, [None] * 3 if seeds is None else seeds, 3)
    with mm.MbarMany(*FB.args(cases)) as m:
        np.random.seed(99)
        u, x, hp = FB.fes_args(cases)
        m.generate_fes([None if c is None else v for c, v in zip(sel, u)],
                       [None if c is None else v for c, v in zip(sel, x)], histogram_parameters=hp, n_bootstraps=3,
                       seed=seeds)
        got = np.random.get_state()
        assert m.replicate_histogram_datas[1] is None if skip else len(m.replicate_histogram_datas[1]) == 3
    assert got[0] == want[0] and np.array_equal(got[1], want[1]) and got[2:] == want[2:]


def test_replicates_follow_the_draw_stream(oracle, golden):
    # replicate b of problem p regenerates the indices fes_bootstrap.replicate_indices gives from its kept state
    cases = golden[0][:2]
    with mm.MbarMany(*FB.args(cases)) as m:
        u, x, hp = FB.fes_args(cases)
        m.generate_fes(u, x, histogram_parameters=hp, n_bootstraps=2, seed=[3, 4])
        np.random.seed(3)
        states = fb.draw_replicates(cases[0]["N_k"], 2)
        h = m.replicate_histogram_datas[0][1]
        idx = fb.replicate_indices(states[1], cases[0]["N_k"])
        np.testing.assert_array_equal(h["sample_label"], m.histogram_datas[0]["sample_label"][idx])
        np.testing.assert_array_equal(h["bin_n"], m.histogram_datas[0]["bin_n"][idx])


def test_non_bootstrap_outputs_keep_their_bits(oracle, golden):
    cases = golden[0]
    with mm.MbarMany(*FB.args(cases)) as m:
        u, x, hp = FB.fes_args(cases)
        m.generate_fes(u, x, histogram_parameters=hp)
        plain = [dict(h) for h in m.histogram_datas]
        q0 = {(rp, unc): m.get_fes([c["queries"] for c in cases], reference_point=rp,
                                   fes_reference=[c["fes_reference"] for c in cases], uncertainty_method=unc)
              for _, rp in FB.TAGS for unc in (None, "analytical")}
        state = np.random.get_state()
        m.generate_fes(u, x, histogram_parameters=hp, n_bootstraps=0, seed=[1] * len(cases))
        after = np.random.get_state()
        assert np.array_equal(state[1], after[1]) and state[2:] == after[2:]     # B = 0 draws nothing
        assert m.replicate_histogram_datas == [None] * len(cases)
        m.generate_fes(u, x, histogram_parameters=hp, n_bootstraps=3, seed=FB.seeds(cases))
        for a, b in zip(plain, m.histogram_datas):
            np.testing.assert_array_equal(a["f"], b["f"])
            np.testing.assert_array_equal(a["sample_label"], b["sample_label"])
        for (rp, unc), want in q0.items():
            got = m.get_fes([c["queries"] for c in cases], reference_point=rp,
                            fes_reference=[c["fes_reference"] for c in cases], uncertainty_method=unc)
            for a, b in zip(want, got):
                assert a.keys() == b.keys()
                for k in a:
                    np.testing.assert_array_equal(a[k], b[k])
        # a later plain generate_fes resets the problem's replicates, as the reference does
        m.generate_fes([u[0]] + [None] * 4, [x[0]] + [None] * 4, histogram_parameters=hp)
        assert m.replicate_histogram_datas[0] is None and len(m.replicate_histogram_datas[1]) == 3
        with pytest.raises(ParameterError, match="problem 0: Can't calculate uncertainties via bootstrap"):
            m.get_fes([c["queries"] for c in cases], uncertainty_method="bootstrap")


def test_routing_and_single_counts(oracle, golden, monkeypatch):
    cases = golden[0]
    B = 4
    monkeypatch.setattr(oracle, "flagged", (1,))             # problem 1: single path in the solve
    monkeypatch.setattr(oracle, "bin_flagged", (3,))         # problem 3: its b = 0 request is flagged
    monkeypatch.setattr(oracle, "rep_bin_flagged", (2,))     # problem 2: every replicate's bin request is flagged
    # problem 0: replicate 1's batched solve reports status 2
    np.random.seed(FB.SEED0)
    c1 = []
    fb.draw_replicates(cases[0]["N_k"], 2, lambda b, idx: c1.append(np.bincount(idx, minlength=800)))
    monkeypatch.setattr(oracle, "flagged_counts", {(0, c1[1].astype(np.uint16).tobytes())})
    with mm.MbarMany(*FB.args(cases)) as m:
        u, x, hp = FB.fes_args(cases)
        m.generate_fes(u, x, histogram_parameters=hp, n_bootstraps=B, seed=FB.seeds(cases))
        assert m.fes_boot_single == [1, B, B, B, B]
        ref = [c.copy() for c in cases]
        # every replicate matches the single path run from the same state
        for i, c in enumerate(ref):
            with FB.FesBootOracleProblem(c["u_kn"], c["N_k"].astype(float)) as q:
                np.random.seed(FB.SEED0 + i)
                states = fb.draw_replicates(c["N_k"], B)
                want = fb.histogram_replicates(q, m.results[i]["f_k"], c["N_k"], c["u_n"], m.histogram_datas[i],
                                               states, fb.solver_protocol(ms.DEFAULT_SOLVER_PROTOCOL))
            for a, b in zip(want, m.replicate_histogram_datas[i]):
                np.testing.assert_allclose(b["f"], a["f"], rtol=0, atol=1e-9, err_msg=c["name"])
    # only problems 0 and 2 reach the weighted bin pass; replicate 1 of problem 0 never does
    assert _calls(oracle, "replicate_bin_moments") == [([0, 2], [0] * (B - 1) + [2] * B)]


def test_one_slot_waves_give_the_same_bits(oracle, golden, monkeypatch):
    cases = golden[0][:4]
    with mm.MbarMany(*FB.args(cases)) as m:
        one, _ = FB.run(m, cases, "seeded")
        f_one = [[h["f"] for h in r] for r in m.replicate_histogram_datas]
    assert len(_calls(oracle, "replicate_bin_moments")) == 1
    oracle.calls.clear()
    monkeypatch.setattr(mm, "BOOT_WAVE_BYTES", 1)
    with mm.MbarMany(*FB.args(cases)) as m:
        many, _ = FB.run(m, cases, "seeded")
        f_many = [[h["f"] for h in r] for r in m.replicate_histogram_datas]
    calls = _calls(oracle, "replicate_bin_moments")
    assert calls == [([p], [p]) for p in range(4) for _ in range(FB.B)]
    for a, b in zip(f_one, f_many):
        for x, y in zip(a, b):
            np.testing.assert_array_equal(x, y)
    for tag in one:
        for a, b in zip(one[tag], many[tag]):
            for k in a:
                np.testing.assert_array_equal(a[k], b[k])


def test_rep_bin_bytes_follow_the_geometry():
    # K = 32, N = 160000, 100 bins: one bin chunk, 64 sample chunks of 79 tiles; f, two request records and a flag
    nT, K, nb = 5000, 32, 100
    assert mm._bin_geometry(nT, 1, nb) == (100, 1, 64)
    assert mm.rep_bin_bytes(K, 160000, nb) == 32 * nT * 32 + 40 * nb + 8 * 64 * nb + 8 * K + 180
    # a tiny problem: one sample chunk
    assert mm.rep_bin_bytes(1, 10, 3) == 32 * 32 + 40 * 3 + 8 * 3 + 8 + 180


def test_validation_before_any_device_work_or_draw(oracle, golden):
    cases = golden[0][:2]
    u, x, hp = FB.fes_args(cases)
    with mm.MbarMany(*FB.args(cases)) as m:
        oracle.calls.clear()
        state = np.random.get_state()
        for bad in (1, -2, 2.0, True, "3", None):
            with pytest.raises(ValueError, match="n_bootstraps must be an integer of 0 or >=2"):
                m.generate_fes(u, x, histogram_parameters=hp, n_bootstraps=bad)
        with pytest.raises(ParameterError, match="single seed"):
            m.generate_fes(u, x, histogram_parameters=hp, n_bootstraps=2, seed=5)
        with pytest.raises(ParameterError, match="one entry per problem"):
            m.generate_fes(u, x, histogram_parameters=hp, n_bootstraps=2, seed=[5])
        for bad in (-2, 1.5, True):
            with pytest.raises(ParameterError, match="problem 1: seed must be"):
                m.generate_fes(u, x, histogram_parameters=hp, n_bootstraps=2, seed=[5, bad])
        with pytest.raises(ParameterError, match="problem 1: u_n has shape"):
            m.generate_fes([u[0], u[1][:-1]], x, histogram_parameters=hp, n_bootstraps=2, seed=[1, 2])
        after = np.random.get_state()
        assert np.array_equal(state[1], after[1]) and state[2:] == after[2:]
        assert oracle.calls == []
        m.get_fes([None, None], uncertainty_method="bootstrap")          # nothing asked: nothing to check
        with pytest.raises(ParameterError, match="problem 0: get_fes before generate_fes"):
            m.get_fes([c["queries"] for c in cases], uncertainty_method="bootstrap")


def test_empty_state_raises_before_any_draw(oracle):
    rng = np.random.RandomState(3)
    x = rng.normal(0, 0.3, 400)
    edges = np.linspace(-0.5, 0.5, 5)
    u_kn, u_n = FB._fes.umbrella_energies(x, np.array([[-0.2], [0.0], [0.2]]), 4.0, 10.0)
    with mm.MbarMany([u_kn, u_kn], [np.array([200.0, 200.0, 0.0]), np.array([200.0, 0.0, 200.0])]) as m:
        oracle.calls.clear()
        state = np.random.get_state()
        with pytest.raises(ParameterError, match="problem 0: a state without samples"):
            m.generate_fes([u_n, u_n], [x, x], histogram_parameters={"bin_edges": edges}, n_bootstraps=2)
        assert np.array_equal(state[1], np.random.get_state()[1]) and oracle.calls == []
        m.generate_fes([u_n, None], [x, None], histogram_parameters={"bin_edges": edges})     # B = 0 is fine
        assert m.histogram_datas[0] is not None


def test_uncovered_replicate_restores_everything(oracle, golden):
    cases = golden[0][:2]
    u, x, hp = FB.fes_args(cases)
    with mm.MbarMany(*FB.args(cases)) as m:
        m.generate_fes(u, x, histogram_parameters=hp, n_bootstraps=2, seed=[1, 2])
        before = ([h["f"].copy() for h in m.histogram_datas],
                  [[r["f"].copy() for r in reps] for reps in m.replicate_histogram_datas], list(m.fes_boot_single))
        # a surface whose outermost bin holds one sample of problem 1: some replicate misses it
        x1 = x[1].copy()
        x1[np.argmax(x1)] = 10.0
        edges = np.concatenate([hp[1]["bin_edges"], [9.0, 11.0]])
        np.random.seed(5)
        state = np.random.get_state()
        with pytest.raises(ParameterError, match=r"problem 1: bootstrap replicate \d+ draws no sample"):
            m.generate_fes([u[0], u[1]], [x[0], x1], histogram_parameters=[hp[0], {"bin_edges": edges}],
                           n_bootstraps=30)
        after = np.random.get_state()
        assert np.array_equal(state[1], after[1]) and state[2:] == after[2:]
        for a, h in zip(before[0], m.histogram_datas):
            np.testing.assert_array_equal(a, h["f"])
        for a, reps in zip(before[1], m.replicate_histogram_datas):
            assert len(a) == len(reps)
            for f, r in zip(a, reps):
                np.testing.assert_array_equal(f, r["f"])
        assert m.fes_boot_single == before[2]


def test_single_path_errors_name_the_problem(oracle, golden, monkeypatch):
    cases = golden[0]

    def boom(*args, **kwargs):
        raise RuntimeError("device failure")

    with mm.MbarMany(*FB.args(cases)) as m:
        m.generate_fes(*FB.fes_args(cases)[:2], histogram_parameters=FB.fes_args(cases)[2])
        monkeypatch.setattr(fb, "histogram_replicates", boom)
        state = np.random.get_state()
        with pytest.raises(RuntimeError, match="device failure") as e:
            m.generate_fes(*FB.fes_args(cases)[:2], histogram_parameters=FB.fes_args(cases)[2], n_bootstraps=2)
        assert np.array_equal(state[1], np.random.get_state()[1])
        assert m.replicate_histogram_datas == [None] * len(cases)
    assert any("problem 4" in note for note in e.value.__notes__)


def test_mbar_many_bootstraps_keep_their_bits(monkeypatch):
    """_bootstraps through the shared per-wave solve (_solve_slots) gives f_k_boots in any wave split."""
    monkeypatch.setattr(mm, "DeviceMbarBatch", W.WeightedOracleBatch)
    monkeypatch.setattr(mm, "DeviceProblem", W.WeightedOracleProblem)
    monkeypatch.setattr(ms, "solve_mbar_for_all_states", H.oracle_all_states)
    rng = np.random.RandomState(8)
    probs = [H.random_problem(rng, K, 60) for K in (2, 3)]
    one = mm.mbar_many([p[0] for p in probs], [p[1] for p in probs], n_bootstraps=3, rseed=[1, 2])
    monkeypatch.setattr(mm, "BOOT_WAVE_BYTES", 1)
    many = mm.mbar_many([p[0] for p in probs], [p[1] for p in probs], n_bootstraps=3, rseed=[1, 2])
    for a, b in zip(one, many):
        np.testing.assert_array_equal(a["f_k_boots"], b["f_k_boots"])
        assert a["boot_single"] == b["boot_single"] == 0

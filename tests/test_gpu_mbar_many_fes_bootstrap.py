"""mbar_b200_batch_replicate_bin_moments on the GPU: every replicate's f_bin against a long-double restatement with
the multiplicities, all-ones counts against batch_bin_moments' bits, agreement with the single-problem weighted bin
pass, bit identity alone / among 50 problems / reversed / in one-slot waves / repeated, the documented errors and
flags, the launch count of a large call, and MbarMany.generate_fes(..., n_bootstraps=B) end to end against the
single-problem path and the unmodified reference's outputs (tests/golden/mbar_many_fes_bootstrap.npz)."""
import numpy as np
import pytest

from pymbar_b200 import DeviceProblem
from pymbar_b200 import fes_bootstrap as fb
from pymbar_b200 import mbar_many as mm
from pymbar_b200 import mbar_solvers as ms
from pymbar_b200._lib import MbarB200Error
from pymbar_b200.problem import DeviceMbarBatch
from tests import _fes
from tests import _mbar_many as H
from tests import _mbar_many_fes_bootstrap as FB
from tests.test_gpu_mbar_many_fes import SHAPES, _problem

pytestmark = pytest.mark.gpu

pytest.importorskip("tests._moments")


def _replicate(c, seed):
    """Counts [N] summing to N for problem c, drawn with replacement, with one sample repeated N/3 times (a large
    multiplicity), every bin holding a drawn sample of finite u_n, and (N > 10) an undrawn sample whose sampled
    energies are all +inf and a second row with +inf entries.  Modifies c's u and u_n in place."""
    rng = np.random.RandomState(seed)
    u, u_n, bins = c["u"], c["u_n"], c["bins"]
    N = u.shape[1]
    idx = rng.randint(0, N, size=N)
    heavy = int(rng.randint(N))
    idx[:N // 3] = heavy
    counts = np.bincount(idx, minlength=N)
    u_n[heavy] = min(u_n[heavy], 4.0)
    for i in range(c["nbins"]):
        members = np.flatnonzero(bins == i)
        if not np.any((counts[members] > 0) & np.isfinite(u_n[members])):
            j = members[0]
            u_n[j] = 2.0
            if counts[j] == 0:
                counts[np.argmax(counts)] -= 1
                counts[j] += 1
    zero = np.flatnonzero(counts == 0)
    if N > 10 and zero.size:                          # (one sample per bin draws every sample)
        u[c["N_k"] > 0, int(zero[0])] = np.inf        # L_n is NaN: must not flag, since it is not drawn
    sampled = np.flatnonzero(c["N_k"] > 0)
    if N > 10 and u.shape[0] > 1 and (c["N_k"][1] == 0 or sampled.size > 1):
        drawn = np.flatnonzero((counts > 0) & (np.arange(N) != heavy))[:5]
        u[1, drawn] = np.inf                          # +inf entries of drawn samples: weight 0 in that row
    assert counts.sum() == N and counts.max() <= 65535 and counts.min() >= 0
    c["counts"] = counts
    c["f"] = np.where(c["N_k"] > 0, rng.normal(0.0, 0.3, size=u.shape[0]), rng.normal(0.0, 0.3, size=u.shape[0]))
    return c


@pytest.fixture(scope="module")
def batch():
    cases = [_replicate(_problem(*s, seed=10 + i), 50 + i) for i, s in enumerate(SHAPES)]
    rng = np.random.RandomState(5)
    while len(cases) < 50:                            # small problems, so that a request shares the call with 50
        K = int(rng.randint(1, 9))
        c = _problem(K, int(rng.randint(40, 400)), int(rng.randint(1, 12)), "scattered", 0, seed=100 + len(cases))
        cases.append(_replicate(c, 200 + len(cases)))
    with DeviceMbarBatch([c["u"] for c in cases], [c["N_k"] for c in cases]) as dev:
        dev.set_replicates(list(range(len(cases))), [c["counts"] for c in cases])
        yield dev, cases


def _call(dev, cases, slots, targets=None):
    """replicate_bin_moments of the resident slots `slots` (slot s is problem s), each problem's target once."""
    probs = list(dict.fromkeys(slots)) if targets is None else targets
    t = {p: i for i, p in enumerate(probs)}
    return dev.replicate_bin_moments(probs, [cases[p]["u_n"] for p in probs], [cases[p]["bins"] for p in probs],
                                     [cases[p]["nbins"] for p in probs], slots, [t[s] for s in slots],
                                     [cases[s]["f"] for s in slots])


def test_entries_match_long_double(batch):
    dev, cases = batch
    ids = list(range(len(SHAPES)))
    out, flags = _call(dev, cases, ids)
    assert not flags.any()
    st = dev.last_stats()
    assert st["launches"] == 5 and st["ms"] > 0
    assert st["bytes_read"] == sum(-(-cases[i]["u"].shape[1] // 32) * 32 * (8 * cases[i]["u"].shape[0] + 2)
                                   for i in ids)
    for i, f_bin in zip(ids, out):
        c = cases[i]
        with np.errstate(all="ignore"):
            rf = _fes.bin_moments_ld(c["u"], c["N_k"], c["f"], c["u_n"], c["bins"], c["nbins"], mult=c["counts"])[0]
        np.testing.assert_allclose(f_bin, np.asarray(rf, np.float64), rtol=0, atol=1e-10, err_msg=str(SHAPES[i]))


def test_all_ones_counts_give_the_unweighted_bits(batch):
    dev, cases = batch
    ids = list(range(len(SHAPES)))
    try:
        dev.set_replicates(ids, [np.ones(cases[i]["u"].shape[1], np.uint16) for i in ids])
        ones, flags = _call(dev, cases, ids)
    finally:
        dev.set_replicates(list(range(len(cases))), [c["counts"] for c in cases])
    plain, plain_flags = dev.bin_moments(ids, [cases[i]["f"] for i in ids], [cases[i]["u_n"] for i in ids],
                                         [cases[i]["bins"] for i in ids], [cases[i]["nbins"] for i in ids],
                                         want_C=False)
    # every sample is drawn now, the one whose sampled energies are all +inf too: both flag the same requests
    np.testing.assert_array_equal(flags, plain_flags)
    for a, (b, _, _) in zip(ones, plain):
        np.testing.assert_array_equal(a, b)


def test_against_the_single_problem_weighted_pass(batch):
    dev, cases = batch
    ids = list(range(len(SHAPES)))
    out, _ = _call(dev, cases, ids)
    for i, f_bin in zip(ids, out):
        c = cases[i]
        # the single-problem upload refuses a sample whose sampled energies are all +inf; it is undrawn, so any
        # finite energies give it the same (zero) weight
        u = c["u"].copy()
        u[:, np.all(np.isinf(u[c["N_k"] > 0]), axis=0)] = 0.0
        with DeviceProblem(u, c["N_k"]) as p:
            p.set_sample_weights(c["counts"].astype(np.float64))
            sf, _, _ = p.bin_moments(c["f"], c["u_n"], c["bins"], c["nbins"], want_C=False)
        np.testing.assert_allclose(f_bin, sf, rtol=1e-12, atol=1e-13, err_msg=str(SHAPES[i]))


def test_bit_identical_alone_among_50_reversed_in_waves_and_repeated(batch):
    dev, cases = batch
    ids = list(range(len(cases)))
    mixed, _ = _call(dev, cases, ids)
    again, _ = _call(dev, cases, ids)
    reverse, _ = _call(dev, cases, ids[::-1])
    for i in ids:
        alone, _ = _call(dev, cases, [i])
        for other in (again[i], reverse[len(ids) - 1 - i], alone[0]):
            np.testing.assert_array_equal(mixed[i], other)
    try:
        for i in range(len(SHAPES)):                   # one-slot waves: the slot is slot 0 of its own upload
            dev.set_replicates([i], [cases[i]["counts"]])
            one, _ = dev.replicate_bin_moments([i], [cases[i]["u_n"]], [cases[i]["bins"]], [cases[i]["nbins"]], [0],
                                               [0], [cases[i]["f"]])
            np.testing.assert_array_equal(mixed[i], one[0])
    finally:
        dev.set_replicates(ids, [c["counts"] for c in cases])


def test_documented_errors_and_flags(batch):
    dev, cases = batch
    c = cases[3]
    good, _ = _call(dev, cases, [0])

    def call(bins=None, nbins=None, u_n=None, slot=3, target=0, tprob=3, f=None, counts=None):
        return dev.replicate_bin_moments([tprob, 0], [c["u_n"] if u_n is None else u_n, cases[0]["u_n"]],
                                         [c["bins"] if bins is None else bins, cases[0]["bins"]],
                                         [c["nbins"] if nbins is None else nbins, cases[0]["nbins"]],
                                         [slot, 0], [target, 1], [c["f"] if f is None else f, cases[0]["f"]])

    for kw in (dict(slot=len(cases)), dict(slot=-1), dict(target=2), dict(slot=4), dict(tprob=len(cases)),
               dict(nbins=0, bins=np.zeros_like(c["bins"]))):
        with pytest.raises((MbarB200Error, ValueError)) as e:
            call(**kw)
        if isinstance(e.value, MbarB200Error):
            assert e.value.status == -1, kw
    for bad in (c["nbins"], -1):
        b = c["bins"].copy()
        b[5] = bad
        with pytest.raises(MbarB200Error) as e:
            call(bins=b)
        assert e.value.status == -1
    u_nan = c["u_n"].copy()
    u_nan[7] = np.nan
    with pytest.raises(MbarB200Error) as e:
        call(u_n=u_nan)
    assert e.value.status == -5
    # flags, as the long-double restatement predicts them: a bin nobody is drawn from (an extra, empty bin); a bin
    # whose drawn samples all have u_n = +inf; a drawn sample whose sampled energies are all +inf (L_n NaN)
    u_inf = c["u_n"].copy()
    drawn = c["counts"] > 0
    u_inf[(c["bins"] == 4) & drawn] = np.inf
    for kw in (dict(nbins=c["nbins"] + 1), dict(u_n=u_inf)):
        out, flags = call(**kw)
        assert flags.tolist() == [True, False], kw
        np.testing.assert_array_equal(out[1], good[0])
    with np.errstate(all="ignore"):
        rf = _fes.bin_moments_ld(c["u"], c["N_k"], c["f"], u_inf, c["bins"], c["nbins"], mult=c["counts"])[0]
    assert not np.isfinite(np.asarray(rf, np.float64)[4])
    # the batch still answers, with the same bits
    again, flags = _call(dev, cases, [0])
    assert not flags.any()
    np.testing.assert_array_equal(again[0], good[0])


def test_nan_denominator_of_a_drawn_sample_flags():
    rng = np.random.RandomState(4)
    u, N_k = H.random_problem(rng, 3, 200)
    N = u.shape[1]
    u[:, 17] = np.inf
    bins = (np.arange(N) % 4).astype(np.int32)
    u_n = rng.uniform(0, 2, N)
    counts = np.ones(N, np.uint16)
    undrawn = counts.copy()
    undrawn[17] = 0
    undrawn[18] += 1
    f = np.array([0.0, 0.1, -0.2])
    with DeviceMbarBatch([u], [N_k]) as dev:
        dev.set_replicates([0, 0], [counts, undrawn])
        _, flags = dev.replicate_bin_moments([0], [u_n], [bins], [4], [0, 1], [0, 0], [f, f])
    assert flags.tolist() == [True, False]


def test_one_call_of_200_problems_by_50_replicates_takes_five_launches():
    rng = np.random.RandomState(11)
    probs = [H.random_problem(rng, 4, 200) for _ in range(200)]
    with DeviceMbarBatch([p[0] for p in probs], [p[1] for p in probs]) as dev:
        slots, counts = [], []
        for p, (u, _) in enumerate(probs):
            N = u.shape[1]
            for _ in range(50):
                slots.append(p)
                counts.append(np.bincount(rng.randint(0, N, N), minlength=N))
        dev.set_replicates(slots, counts)
        N = [u.shape[1] for u, _ in probs]
        out, flags = dev.replicate_bin_moments(list(range(200)), [rng.uniform(0, 1, n) for n in N],
                                               [(np.arange(n) % 10).astype(np.int32) for n in N], [10] * 200,
                                               list(range(len(slots))), slots, [np.zeros(4)] * len(slots))
        assert len(out) == 10000 and dev.last_stats()["launches"] == 5
        assert not flags.any()


def test_batch_matches_the_single_path_end_to_end():
    cases, _ = FB.load()
    u, x, hp = FB.fes_args(cases)
    with mm.MbarMany(*FB.args(cases)) as m:
        m.generate_fes(u, x, histogram_parameters=hp, n_bootstraps=FB.B, seed=FB.seeds(cases))
        assert m.fes_boot_single == [0, 0, 0, 0, FB.B]
        protocol = tuple(dict(st, tol=1e-12) for st in fb.solver_protocol(ms.DEFAULT_SOLVER_PROTOCOL))
        for i, c in enumerate(cases[:4]):
            N_k = c["N_k"]
            np.random.seed(FB.SEED0 + i)
            states = fb.draw_replicates(N_k, FB.B)
            with DeviceProblem(c["u_kn"], N_k.astype(np.float64)) as q:
                want = fb.histogram_replicates(q, m.results[i]["f_k"], N_k, c["u_n"], m.histogram_datas[i], states,
                                               protocol)
                # at equal replicate f, the bin free energies agree to 1e-12 relative
                base = m.histogram_datas[i]
                dense = _fes_dense(base)
                for b, st in enumerate(states[:2]):
                    idx = fb.replicate_indices(st, N_k)
                    cnt = np.bincount(idx, minlength=len(c["u_n"]))
                    from pymbar_b200.bootstrap import bootstrap_f_k
                    f_b = bootstrap_f_k(q, m.results[i]["f_k"], N_k, rints=idx[None], solver_protocol=protocol)[0]
                    q.set_sample_weights(cnt.astype(np.float64))
                    sf, _, _ = q.bin_moments(f_b, c["u_n"], dense, len(base["bin_order"]), want_C=False)
                    q.set_sample_weights(None)
                    m._dev.set_replicates([m._slot[i]], [cnt.astype(np.uint16)])
                    bf, flags = m._dev.replicate_bin_moments([m._slot[i]], [c["u_n"]], [dense],
                                                             [len(base["bin_order"])], [0], [0], [f_b])
                    assert not flags.any()
                    np.testing.assert_allclose(bf[0], sf, rtol=1e-12, atol=0)
            for a, h in zip(want, m.replicate_histogram_datas[i]):
                np.testing.assert_allclose(h["f"], a["f"], rtol=0, atol=1e-9, err_msg=c["name"])


def _fes_dense(base):
    from pymbar_b200 import fes as hist

    return hist.dense_bins(base["sample_label"], base["bin_order"])


@pytest.mark.parametrize("run", FB.RUNS)
def test_mbar_many_fes_bootstrap_against_the_reference(run):
    cases, stream_next = FB.load()
    state = np.random.get_state()
    try:
        with mm.MbarMany(*FB.args(cases)) as m:
            out, nxt = FB.run(m, cases, run)
            for i, c in enumerate(cases):
                FB.check_case(c, run, m, i, out)
            errs = [FB.max_errors(c, run, m, i, out) for i, c in enumerate(cases)]
            print(run, "largest difference from the reference:", max(max(e.values()) for e in errs))
            assert m.device_stats["launches"] > 0
        if run == "stream":
            assert nxt == stream_next
    finally:
        np.random.set_state(state)

"""mbar_b200_batch_bin_moments on the GPU: f_bin, C and D of every request entry by entry against a long-double
restatement, against the single-problem DeviceProblem.bin_moments, bit identity alone / mixed / repeated, the
documented errors and flags, and MbarMany.generate_fes / get_fes end to end against the unmodified reference's outputs
(tests/golden/mbar_many_fes.npz)."""
import numpy as np
import pytest

from pymbar_b200 import DeviceProblem
from pymbar_b200 import mbar_many as mm
from pymbar_b200._lib import MbarB200Error
from pymbar_b200.problem import DeviceMbarBatch
from tests import _fes
from tests import _mbar_many as H
from tests import _mbar_many_fes as F

pytestmark = pytest.mark.gpu

_moments = pytest.importorskip("tests._moments")

# (K_p, N_p, nbins, layout, unsampled states): "blocked" puts each bin's samples together (large groups inside a
# warp), "scattered" spreads them at random (mostly groups of one or two)
SHAPES = [(1, 1, 1, "blocked", 0), (2, 31, 3, "scattered", 0), (5, 33, 3, "blocked", 1), (33, 5000, 100, "blocked", 0),
          (33, 5000, 2500, "scattered", 3), (64, 100000, 5000, "blocked", 0), (64, 100000, 100, "scattered", 2),
          (5, 5000, 5000, "scattered", 0), (2, 100000, 1, "scattered", 0)]


def _problem(K, N, nbins, layout, empty, seed):
    rng = np.random.RandomState(seed)
    u, N_k = H.random_problem(rng, K, N, empty=empty)
    N = u.shape[1]
    bins = (np.arange(N) * nbins // N).astype(np.int32)
    if layout == "scattered":
        bins = rng.permutation(bins).astype(np.int32)
    u_n = rng.uniform(0.0, 5.0, size=N)
    if N > 10:
        u_n[rng.choice(N, size=3, replace=False)] = np.inf       # weight exactly 0
        for i in range(nbins):                                   # keep every bin with a sample of finite weight
            idx = np.flatnonzero(bins == i)
            if not np.isfinite(u_n[idx]).any():
                u_n[idx[0]] = 1.0
    return dict(u=u, N_k=N_k, u_n=u_n, bins=bins, nbins=nbins)


@pytest.fixture(scope="module")
def batch():
    cases = [_problem(*s, seed=10 + i) for i, s in enumerate(SHAPES)]
    with DeviceMbarBatch([c["u"] for c in cases], [c["N_k"] for c in cases]) as dev:
        f_list, status, _ = dev.solve()
        assert all(s == 0 for s in status)
        for c, f in zip(cases, f_list):
            c["f"] = f
        yield dev, cases


def _call(dev, cases, ids, want_C=True):
    return dev.bin_moments(ids, [cases[i]["f"] for i in ids], [cases[i]["u_n"] for i in ids],
                           [cases[i]["bins"] for i in ids], [cases[i]["nbins"] for i in ids], want_C=want_C)


def test_entries_match_long_double(batch):
    dev, cases = batch
    ids = list(range(len(cases)))
    out, flags = _call(dev, cases, ids)
    assert not flags.any()
    st = dev.last_stats()
    assert st["launches"] == 7 and st["bytes_read"] > 0 and st["ms"] > 0
    for i, (f_bin, C, D) in zip(ids, out):
        c = cases[i]
        rf, rC, rD, A_C, A_D = _fes.bin_moments_ld(c["u"], c["N_k"], c["f"], c["u_n"], c["bins"], c["nbins"])
        np.testing.assert_allclose(f_bin, np.asarray(rf, np.float64), rtol=0, atol=1e-10, err_msg=str(SHAPES[i]))
        N = len(c["u_n"])
        errC = float((np.abs(C.astype(_moments.LD) - rC) / _fes.moment_tol(rC, A_C, A_D, N)).max())
        errD = float((np.abs(D.astype(_moments.LD) - rD) / _fes.moment_tol(rD, A_D, A_D, N)).max())
        assert errC <= 1.0 and errD <= 1.0, (SHAPES[i], errC, errD)
        unsampled = np.flatnonzero(c["N_k"] == 0)
        if unsampled.size:
            assert np.any(C[unsampled] > 0)


def test_against_the_single_problem_path(batch):
    dev, cases = batch
    out, _ = _call(dev, cases, list(range(len(cases))))
    for c, (f_bin, C, D) in zip(cases, out):
        with DeviceProblem(c["u"], c["N_k"]) as p:
            sf, sC, sD = p.bin_moments(c["f"], c["u_n"], c["bins"], c["nbins"])
        # entries far below the largest carry the relative error of their large exponents (up to ~500 here)
        np.testing.assert_allclose(f_bin, sf, rtol=1e-13, atol=1e-13)
        np.testing.assert_allclose(C, sC, rtol=1e-13, atol=1e-13 * np.abs(sC).max())
        np.testing.assert_allclose(D, sD, rtol=1e-13, atol=1e-13 * np.abs(sD).max())


def test_bit_identical_alone_mixed_and_repeated(batch):
    dev, cases = batch
    ids = list(range(len(cases)))
    mixed, _ = _call(dev, cases, ids)
    again, _ = _call(dev, cases, ids)
    reverse, _ = _call(dev, cases, ids[::-1] + [3, 3])
    f_only, _ = _call(dev, cases, ids, want_C=False)
    assert dev.last_stats()["launches"] == 5
    for i in ids:
        alone, _ = _call(dev, cases, [i])
        for other in (again[i], reverse[len(ids) - 1 - i], alone[0]):
            for a, b in zip(mixed[i], other):
                np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(f_only[i][0], mixed[i][0])
        assert f_only[i][1] is None and f_only[i][2] is None
    np.testing.assert_array_equal(reverse[-1][1], mixed[3][1])


def test_documented_errors_and_flags(batch):
    dev, cases = batch
    c = cases[3]

    def call(f=None, u_n=None, bins=None, nbins=None, problem=3):
        return dev.bin_moments([problem, 0], [c["f"] if f is None else f, cases[0]["f"]],
                               [c["u_n"] if u_n is None else u_n, cases[0]["u_n"]],
                               [c["bins"] if bins is None else bins, cases[0]["bins"]],
                               [c["nbins"] if nbins is None else nbins, 1])

    for bad in (c["nbins"], -1):
        b = c["bins"].copy()
        b[5] = bad
        with pytest.raises(MbarB200Error) as e:
            call(bins=b)
        assert e.value.status == -1
    with pytest.raises(MbarB200Error) as e:
        call(nbins=0, bins=np.zeros_like(c["bins"]))
    assert e.value.status == -1
    with pytest.raises(MbarB200Error) as e:
        call(problem=len(cases))
    assert e.value.status == -1
    u_nan = c["u_n"].copy()
    u_nan[7] = np.nan
    with pytest.raises(MbarB200Error) as e:
        call(u_n=u_nan)
    assert e.value.status == -5
    # flags: an empty bin, a bin of +inf energies, an unsampled row's exponent above 700; the other request is served
    good, _ = _call(dev, cases, [0])
    u_inf = c["u_n"].copy()
    u_inf[c["bins"] == 4] = np.inf
    e_cases = cases[4]
    far = e_cases["f"].copy()
    far[np.flatnonzero(e_cases["N_k"] == 0)[0]] += 1500.0
    for kw in (dict(nbins=c["nbins"] + 1), dict(u_n=u_inf)):
        out, flags = call(**kw)
        assert flags.tolist() == [True, False]
        for a, b in zip(out[1], good[0]):
            np.testing.assert_array_equal(a, b)
    out, flags = dev.bin_moments([4], [far], [e_cases["u_n"]], [e_cases["bins"]], [e_cases["nbins"]])
    assert flags.tolist() == [True]
    # the batch still answers
    again, flags = _call(dev, cases, [0])
    assert not flags.any()
    for a, b in zip(again[0], good[0]):
        np.testing.assert_array_equal(a, b)


def test_mbar_many_fes_against_the_reference():
    cases = F.load()
    with mm.MbarMany([c["u_kn"] for c in cases], [c["N_k"].astype(np.float64) for c in cases]) as m:
        out = F.run_all(m, cases)
        stats = dict(m.device_stats)
        for i, c in enumerate(cases):
            F.check_case(c, m.histogram_datas[i], {k: v[i] for k, v in out.items()})
            want = "single" if len(c["N_k"]) > 64 else "batch"
            assert all(v[i]["path"] == want for v in out.values()), c["name"]
    assert stats["calls"] >= 2 and stats["launches"] >= 12

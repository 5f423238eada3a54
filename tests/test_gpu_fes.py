"""mbar_b200_bin_moments on the GPU: f_bin, C and D entry by entry against a long-double restatement, the
multiplicities, determinism, the documented errors, and the histogram FES end to end against the unmodified
reference's outputs (tests/golden/fes_hist_*.npz)."""
import numpy as np
import pytest

from pymbar_b200 import DeviceProblem
from pymbar_b200 import fes as hist
from pymbar_b200._lib import MbarB200Error
from tests import _fes

pytestmark = pytest.mark.gpu

_moments = pytest.importorskip("tests._moments")

# (K, nbins, layout): layout "blocked" puts each bin's samples together (large groups inside a warp), "scattered"
# spreads them at random (mostly groups of one or two)
SHAPES = [(1, 3, "scattered"), (2, 1, "blocked"), (5, 100, "scattered"), (64, 3, "blocked"), (96, 100, "blocked"),
          (256, 100, "scattered"), (300, 5000, "scattered"), (513, 100, "blocked"), (2100, 3, "scattered"),
          (64, 5000, "blocked")]


def _case(K, nbins, layout, unsampled=(), seed=0):
    n_per = max(5 if K < 100 else 3, -(-int(1.1 * nbins) // K))
    c = _moments.ladder(K, n_per, unsampled=unsampled, seed=seed + K)
    N = c["u"].shape[1]
    assert N % 32 and N >= nbins
    rng = np.random.RandomState(seed + 7)
    bins = (np.arange(N) * nbins // N).astype(np.int32)
    if layout == "scattered":
        bins = rng.permutation(bins).astype(np.int32)
    # the target state: energies of a few kT per sample; a few samples of weight zero
    u_n = rng.uniform(0.0, 5.0, size=N)
    u_n[rng.choice(N, size=min(3, N // 10), replace=False)] = np.inf
    # keep every bin's samples from being all +inf
    for i in range(nbins):
        idx = np.flatnonzero(bins == i)
        if not np.isfinite(u_n[idx]).any():
            u_n[idx[0]] = 1.0
    return dict(c, u_n=u_n, bins=bins, nbins=nbins)


def _check(p, case, mult=None, f=None):
    f = case["f"] if f is None else f
    f_bin, C, D = p.bin_moments(f, case["u_n"], case["bins"], case["nbins"])
    u = p.download() if p.K != case["u"].shape[0] else case["u"]
    N_k = p.N_k
    rf, rC, rD, A_C, A_D = _fes.bin_moments_ld(u, N_k, f, case["u_n"], case["bins"], case["nbins"], mult)
    np.testing.assert_allclose(f_bin, np.asarray(rf, np.float64), rtol=0, atol=1e-10)
    N = len(case["u_n"])
    tolC = _fes.moment_tol(rC, A_C, A_D, N)
    tolD = _fes.moment_tol(rD, A_D, A_D, N)
    errC = float((np.abs(C.astype(_moments.LD) - rC) / tolC).max())
    errD = float((np.abs(D.astype(_moments.LD) - rD) / tolD).max())
    assert errC <= 1.0 and errD <= 1.0, (errC, errD)
    return f_bin, C, D


@pytest.mark.parametrize("K,nbins,layout", SHAPES)
def test_bin_moments_match_long_double(K, nbins, layout):
    case = _case(K, nbins, layout)
    with DeviceProblem(case["u"], case["N"]) as p:
        first = _check(p, case)
        again = p.bin_moments(case["f"], case["u_n"], case["bins"], case["nbins"])
        for a, b in zip(first, again):
            np.testing.assert_array_equal(a, b)                # deterministic: bit-identical


@pytest.mark.parametrize("K,unsampled", [(17, (0,)), (129, (64, 128)), (257, (0, 128, 256))])
def test_unsampled_states_enter_C(K, unsampled):
    case = _case(K, 100, "blocked", unsampled=unsampled)
    with DeviceProblem(case["u"], case["N"]) as p:
        _, C, _ = _check(p, case)
        assert np.any(C[list(unsampled)] > 0)       # (a row whose neighbours lie e^-700 away may underflow to 0)


def test_augmented_context():
    case = _case(64, 100, "scattered")
    rng = np.random.RandomState(3)
    extra = case["u"][[3, 40]] + rng.uniform(0, 2, size=(2, case["u"].shape[1]))
    with DeviceProblem(case["u"], case["N"]) as base, base.augmented(extra) as p:
        f = np.concatenate([case["f"], [0.1, -0.2]])
        _check(p, dict(case, f=f), f=f)


def test_integer_multiplicities_equal_gathered_columns():
    case = _case(96, 100, "blocked")
    mult = case["mult"]
    keep = np.repeat(np.arange(len(mult)), mult.astype(int))
    with DeviceProblem(case["u"], case["N"]) as p:
        p.set_sample_weights(mult)
        fw, Cw, Dw = _check(p, case, mult=mult)
    g = dict(case, u=np.ascontiguousarray(case["u"][:, keep]), u_n=case["u_n"][keep], bins=case["bins"][keep])
    with DeviceProblem(g["u"], case["N"]) as q:
        fg, Cg, Dg = q.bin_moments(case["f"], g["u_n"], g["bins"], g["nbins"])
    np.testing.assert_allclose(fw, fg, rtol=0, atol=1e-10)
    np.testing.assert_allclose(Cw, Cg, rtol=1e-10, atol=1e-300)
    np.testing.assert_allclose(Dw, Dg, rtol=1e-10, atol=1e-300)


def test_bin_chunks_forced_by_large_K_times_nbins():
    """K + 1 = 2101 rows and 3000 bins do not fit one shared-memory accumulator: several chunks answer."""
    case = _case(2100, 3000, "blocked")
    with DeviceProblem(case["u"], case["N"]) as p:
        _check(p, case)


def test_documented_errors():
    case = _case(64, 100, "scattered")
    with DeviceProblem(case["u"], case["N"]) as p:
        bad = case["bins"].copy()
        bad[5] = case["nbins"]
        with pytest.raises(MbarB200Error) as e:
            p.bin_moments(case["f"], case["u_n"], bad, case["nbins"])
        assert e.value.status == -1
        bad[5] = -1
        with pytest.raises(MbarB200Error) as e:
            p.bin_moments(case["f"], case["u_n"], bad, case["nbins"])
        assert e.value.status == -1
        u_nan = case["u_n"].copy()
        u_nan[7] = np.nan
        with pytest.raises(MbarB200Error) as e:
            p.bin_moments(case["f"], u_nan, case["bins"], case["nbins"])
        assert e.value.status == -5
        # a sampled state's W_nk stays below 1 / N_k at any f (it is in the denominator); an unsampled one's does not
        far = case["f"].copy()
        far[10] += 800.0
        _check(p, case, f=far)
    empty = _case(64, 100, "scattered", unsampled=(5,))
    with DeviceProblem(empty["u"], empty["N"]) as p:
        far = empty["f"].copy()
        far[5] += 1500.0                                       # W_nk of unsampled state 5 near e^1250
        with pytest.raises(MbarB200Error) as e:
            p.bin_moments(far, empty["u_n"], empty["bins"], empty["nbins"])
        assert e.value.status == -6
    with DeviceProblem(case["u"], case["N"]) as p:
        with pytest.raises(MbarB200Error) as e:                # an empty bin has no free energy
            p.bin_moments(case["f"], case["u_n"], case["bins"], case["nbins"] + 1)
        assert e.value.status == -6
        u_inf = case["u_n"].copy()
        u_inf[case["bins"] == 4] = np.inf                      # every sample of bin 4 has weight 0
        with pytest.raises(MbarB200Error) as e:
            p.bin_moments(case["f"], u_inf, case["bins"], case["nbins"])
        assert e.value.status == -6
        # the context still answers after the errors
        _check(p, case)
    with DeviceProblem(case["u"], case["N"]) as p:
        try:
            p.comm_init(1, 0, DeviceProblem.comm_unique_id())
        except MbarB200Error as err:
            pytest.skip(f"no communicator on this machine: {err}")
        with pytest.raises(MbarB200Error) as e:
            p.bin_moments(case["f"], case["u_n"], case["bins"], case["nbins"])
        assert e.value.status == -1


@pytest.mark.parametrize("name", _fes.FIXTURES)
def test_histogram_fes_against_the_reference(name):
    z = _fes.load(name)
    with DeviceProblem(z["u_kn"], z["N_k"]) as p:
        edges = z["bin_edges"]
        hd = hist.histogram_fes(p, z["f_k"], z["u_n"], z["x_n"], edges)
        np.testing.assert_array_equal(hd["sample_label"], z["sample_label"])
        np.testing.assert_allclose(hd["f"], z["f"], rtol=0, atol=1e-8)
        Theta = hist.histogram_theta(p, z["f_k"], z["N_k"], z["u_n"], hd)
    K = len(z["N_k"])
    ref = z["fes_reference"].tolist() if z["fes_reference"].ndim else float(z["fes_reference"])
    for tag, rp in (("lowest", "from-lowest"), ("specified", "from-specified")):
        r = hist.query(hd, z["queries"], rp, ref, lambda j: hist.bin_uncertainties(Theta, K, j, len(hd["f"])))
        np.testing.assert_allclose(r["f_i"], z[f"f_i_{tag}"], rtol=0, atol=1e-8)
        np.testing.assert_allclose(r["df_i"], z[f"df_i_{tag}"], rtol=1e-5, atol=1e-12)


@pytest.mark.parametrize("name", _fes.FIXTURES)
def test_facade_on_the_gpu_backend(name):
    from pymbar_b200 import facade
    from pymbar_b200 import mbar_solvers as ms
    from tests.test_driver_logic_cpu import StandInMBAR

    StandInMBAR.solvers = ms
    _fes.StandInFES.mbar_class = StandInMBAR
    facade.install_on(StandInMBAR)
    facade.install_fes_on(_fes.StandInFES)
    try:
        _fes.check_fes_facade(_fes.StandInFES, _fes.load(name))
    finally:
        facade.uninstall_from(_fes.StandInFES)
        facade.uninstall_from(StandInMBAR)
        ms.clear_cache()

"""FES bootstrap replicates on the GPU: mbar_b200_kde_log_sum_replicates against mbar_b200_kde_log_sum run replicate by
replicate (D = 1..4, all six kernels, B not a multiple of the batch width, N not a multiple of a tile or a chunk, zero
weights, replicates without weight, queries far from the data), bit-identical repeats, the documented errors, and
the histogram and KDE bootstrap surfaces end to end through the facade against the unmodified reference's outputs
(tests/golden/fes_bootstrap.npz)."""
import numpy as np
import pytest

from pymbar_b200 import DeviceKde
from pymbar_b200._lib import MbarB200Error
from pymbar_b200.fes import KDE_KERNELS

pytestmark = pytest.mark.gpu


def _replicates(N, D, B, seed):
    """Samples, b = 0 weights spanning 16 decades with zeros, and the weights V [B, N] of B bootstrap replicates
    (V_bn = sum of w over the positions drawn as sample n); replicate 3 has no weight at all."""
    rng = np.random.RandomState(seed)
    x = rng.normal(size=(N, D))
    w = 10.0 ** rng.uniform(-8, 8, size=N)
    w[rng.uniform(size=N) < 0.05] = 0.0
    w[0] = 1.0
    V = np.array([np.bincount(rng.randint(N, size=N), weights=w, minlength=N) for _ in range(B)])
    V[3] = 0.0
    return x, w, V


def _queries(Q, D, x, seed):
    rng = np.random.RandomState(seed + 1)
    y = rng.normal(scale=1.3, size=(Q, D))
    y[:3] = x[rng.randint(len(x), size=3)] + 1e-3
    y[3] = 40.0                                          # far from the data: gaussian terms near -8e4 at h = 0.2
    return y


@pytest.mark.parametrize("kernel", KDE_KERNELS)
@pytest.mark.parametrize("D", [1, 2, 3, 4])
def test_log_sum_replicates_matches_log_sum(kernel, D):
    for N, B, Q, h in ((1, 4, 5, 0.7), (9001, 11, 300, 0.2), (20011, 17, 40, 0.5)):
        x, w, V = _replicates(N, D, B, seed=N + D)
        y = _queries(Q, D, x, seed=N)
        with DeviceKde(x, w) as kde:
            kde.set_replicates(V)
            got = kde.log_sum_replicates(kernel, h, y)
            assert got.shape == (B, Q) and kde.last_stats()["ms"] > 0
            np.testing.assert_array_equal(kde.log_sum_replicates(kernel, h, y), got)      # repeat: bit-identical
        for b in range(B):
            if not np.any(V[b] > 0):
                assert np.all(got[b] == -np.inf)
                continue
            with DeviceKde(x, V[b]) as one:
                want = one.log_sum(kernel, h, y)
            np.testing.assert_array_equal(np.isneginf(got[b]), np.isneginf(want))
            fin = np.isfinite(want)
            err = np.abs(got[b][fin] - want[fin])
            assert np.all(err <= 1e-12 * np.maximum(1.0, np.abs(want[fin]))), (b, float(err.max()))


def test_replicate_errors():
    x, w, V = _replicates(500, 2, 5, seed=3)
    y = _queries(6, 2, x, seed=3)
    with DeviceKde(x, w) as kde:
        with pytest.raises(MbarB200Error) as e:
            kde.log_sum_replicates("gaussian", 0.3, y)
        assert e.value.status == -4                       # no replicates uploaded
        for bad in (np.where(np.arange(2500).reshape(5, 500) == 7, -1.0, V),
                    np.where(np.arange(2500).reshape(5, 500) == 9, np.nan, V),
                    np.where(np.arange(2500).reshape(5, 500) == 11, np.inf, V)):
            with pytest.raises(MbarB200Error) as e:
                kde.set_replicates(bad)
            assert e.value.status == -1 and kde.B == 0
        with pytest.raises(ValueError):
            kde.set_replicates(V[:, :10])
        kde.set_replicates(V)
        want = kde.log_sum_replicates("gaussian", 0.3, y)
        for kernel, h, q, status in (("gaussian", 0.0, y, -1), ("box", 0.3, y, -1),
                                     ("gaussian", 0.3, np.where(np.arange(12).reshape(6, 2) == 3, np.nan, y), -5)):
            with pytest.raises(MbarB200Error) as e:
                kde.log_sum_replicates(kernel, h, q)
            assert e.value.status == status
        np.testing.assert_array_equal(kde.log_sum_replicates("gaussian", 0.3, y), want)
        with DeviceKde(x, w) as fresh:                 # b = 0's weights are untouched by the replicates
            np.testing.assert_array_equal(kde.log_sum("gaussian", 0.3, y), fresh.log_sum("gaussian", 0.3, y))


def _agrees_with_log_sum(x, V, y, kernel, h, got):
    for b in range(len(V)):
        if not np.any(V[b] > 0):
            assert np.all(got[b] == -np.inf)
            continue
        with DeviceKde(x, V[b]) as one:
            want = one.log_sum(kernel, h, y)
        np.testing.assert_array_equal(np.isneginf(got[b]), np.isneginf(want))
        fin = np.isfinite(want)
        err = np.abs(got[b][fin] - want[fin])
        assert np.all(err <= 1e-12 * np.maximum(1.0, np.abs(want[fin]))), (b, float(err.max()))


def test_scaled_out_entries_are_recomputed_exactly():
    """Entries the batch's shared scale cuts short come back exact.  (1) One chunk, 1-D gaussian, h = 1, query 0,
    samples with x^2 / 2 = 710 (replicate A), 583 (B), 0 (A), 595 (B) in that order: B's e^-583 is accumulated
    within 128 of the scale set by A's e^-710, A's e^0 then raises the scale by 710 and the rescale flushes B's sum;
    B's pass alone reads -595 where its log sum is -583.  (2) A far query (40, 40, 40) at h = 0.2, where replicates'
    nearest samples differ by more than 700 in the log."""
    x = np.sqrt(2.0 * np.array([710.0, 583.0, 0.0, 595.0])).reshape(-1, 1)
    V = np.array([[1.0, 0.0, 1.0, 0.0], [0.0, 1.0, 0.0, 1.0]])
    y = np.zeros((1, 1))
    with DeviceKde(x, np.ones(4)) as kde:
        kde.set_replicates(V)
        got = kde.log_sum_replicates("gaussian", 1.0, y)
    assert abs(got[1, 0] - np.logaddexp(-583.0, -595.0)) < 1e-12 * 583
    _agrees_with_log_sum(x, V, y, "gaussian", 1.0, got)
    x, w, V = _replicates(9001, 3, 11, seed=9004)
    y = _queries(300, 3, x, seed=9001)
    with DeviceKde(x, w) as kde:
        kde.set_replicates(V)
        got = kde.log_sum_replicates("gaussian", 0.2, y)
    _agrees_with_log_sum(x, V, y, "gaussian", 0.2, got)


@pytest.fixture()
def gpu_boot_fes():
    pytest.importorskip("sklearn")
    from pymbar_b200 import facade
    from pymbar_b200 import mbar_solvers as ms
    from tests import _kde
    from tests.test_driver_logic_cpu import StandInMBAR

    StandInMBAR.solvers = ms
    cls = _kde.kde_stand_in()
    cls.mbar_class = StandInMBAR
    facade.install_on(StandInMBAR)
    facade.install_fes_on(cls)
    yield cls
    facade.uninstall_from(cls)
    facade.uninstall_from(StandInMBAR)
    ms.clear_cache()


def _cases():
    from tests.test_fes_bootstrap_cpu import CASES

    return CASES


@pytest.mark.parametrize("source,seed", _cases())
def test_histogram_bootstrap_on_the_gpu_backend(gpu_boot_fes, source, seed):
    from tests.test_fes_bootstrap_cpu import check_histogram_bootstrap

    check_histogram_bootstrap(gpu_boot_fes, source, seed, atol_f=1e-7)


@pytest.mark.parametrize("source,seed", _cases())
def test_kde_bootstrap_on_the_gpu_backend(gpu_boot_fes, source, seed):
    from pymbar_b200 import facade
    from tests.test_fes_bootstrap_cpu import check_kde_bootstrap

    p0 = facade.STATS["fes_boot_passes"]
    fes = check_kde_bootstrap(gpu_boot_fes, source, seed)
    assert facade.STATS["fes_boot_passes"] == p0 + 4          # gaussian and tophat, two reference points each
    assert isinstance(fes.__dict__["_b200_kde_dev"][0], DeviceKde)

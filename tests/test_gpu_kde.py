"""mbar_b200_kde_log_sum on the GPU: l_q entry by entry against the long-double restatement (tests/_kde.py) for all
six kernels, D = 1..4, N from 1 to 2e5 and Q from 1 to 40000; weights with zeros spanning 600 decades, queries far
beyond the fp64 range of the linear sum, compact kernels with nothing in reach and samples on the support boundary;
batch independence and bit-identical repeats; the documented errors; a full-size case; and the KDE free-energy
surface end to end through the facade against the unmodified reference's outputs (tests/golden/fes_kde_*.npz)."""
import numpy as np
import pytest

from pymbar_b200 import DeviceKde, DeviceProblem
from pymbar_b200._lib import MbarB200Error
from pymbar_b200.fes import KDE_KERNELS
from tests import _kde

pytestmark = pytest.mark.gpu

if np.finfo(np.longdouble).nmant < 63:
    pytest.skip("the long-double reference needs an 80-bit long double", allow_module_level=True)


def _samples(N, D, seed):
    rng = np.random.RandomState(seed)
    x = rng.normal(size=(N, D))
    w = 10.0 ** rng.uniform(-300, 300, size=N)           # 600 decades
    w[rng.uniform(size=N) < 0.05] = 0.0
    if not np.any(w > 0):
        w[0] = 1.0
    return x, w


def _queries(Q, D, x, seed):
    rng = np.random.RandomState(seed + 1)
    y = rng.normal(scale=1.3, size=(Q, D))
    y[: min(Q, 3)] = x[rng.randint(len(x), size=min(Q, 3))] + 1e-3       # next to a sample
    return y


def _check(kde, kernel, h, x, w, y, n_check=48, seed=0):
    got = kde.log_sum(kernel, h, y)
    idx = np.arange(len(y))
    if len(y) > n_check:
        idx = np.random.RandomState(seed).choice(len(y), n_check, replace=False)
    _kde.check_against_ld(got[idx], kernel, h, x, w, y[idx])
    return got


@pytest.mark.parametrize("kernel", KDE_KERNELS)
@pytest.mark.parametrize("D", [1, 2, 3, 4])
def test_log_sum_matches_long_double(kernel, D):
    for N, Q, h in ((1, 7, 0.7), (777, 1, 0.3), (4097, 1000, 0.25), (40001, 7, 0.1), (200003, 40000, 0.05)):
        if N == 200003 and D > 2:
            continue
        x, w = _samples(N, D, seed=N + D)
        y = _queries(Q, D, x, seed=N)
        with DeviceKde(x, w) as kde:
            got = _check(kde, kernel, h, x, w, y)
            np.testing.assert_array_equal(kde.log_sum(kernel, h, y), got)          # repeat: bit-identical
            st = kde.last_stats()
            assert st["chunks"] >= 1 and st["ms"] > 0


@pytest.mark.parametrize("kernel", ["gaussian", "exponential"])
def test_queries_far_below_the_fp64_range(kernel):
    """Every term of these queries lies below e^-745: the linear sum underflows, the log sum does not."""
    x, w = _samples(5000, 2, seed=3)
    w = np.where(w > 0, 1.0, 0.0)
    y = np.array([[60.0, 0.0], [0.0, -1000.0], [400.0, 400.0]])
    with DeviceKde(x, w) as kde:
        got = _check(kde, kernel, 0.05, x, w, y)
    assert np.all(np.isfinite(got)) and np.all(got < -745)


@pytest.mark.parametrize("kernel", ["tophat", "epanechnikov", "linear", "cosine"])
def test_compact_kernels_with_nothing_in_reach_are_minus_inf(kernel):
    x, w = _samples(3000, 2, seed=4)
    i = int(np.flatnonzero(w > 0)[0])
    y = np.array([[10.0, 0.0], [0.0, 8.0], x[i]])
    with DeviceKde(x, w) as kde:
        got = _check(kde, kernel, 0.2, x, w, y)
    assert got[0] == -np.inf and got[1] == -np.inf and np.isfinite(got[2])


@pytest.mark.parametrize("D", [1, 2])
@pytest.mark.parametrize("kernel", ["tophat", "epanechnikov", "linear", "cosine"])
def test_support_on_boundary_sets(kernel, D):
    """Samples at distance exactly h from a query and at the neighbouring doubles: the device's support is the
    restatement's (sklearn's d < h on its rounded distance), query by query."""
    rng = np.random.RandomState(9)
    h = 0.37
    ys, xs = [], []
    for t in range(1200):
        y = rng.uniform(-1, 1, size=D) + 10.0 * t             # 10 apart: each query reaches only its own sample
        if D == 1:
            b = y[0] + h
            cand = [[b], [np.nextafter(b, -np.inf)], [np.nextafter(b, np.inf)]]
        else:
            phi = rng.uniform(0, 2 * np.pi)
            p = y + h * np.array([np.cos(phi), np.sin(phi)])
            cand = [p, [np.nextafter(p[0], -np.inf), p[1]], [np.nextafter(p[0], np.inf), p[1]]]
        ys.append(y)
        xs.append(cand[t % 3])
    ys, xs = np.array(ys), np.array(xs)
    with DeviceKde(xs, np.ones(len(xs))) as kde:
        got = kde.log_sum(kernel, h, ys)
    d = np.sqrt(np.array([_kde.distance_sq(ys[i:i + 1], xs[i:i + 1])[0, 0] for i in range(len(ys))]))
    np.testing.assert_array_equal(np.isfinite(got), d < h)
    inside = d < h
    assert 0 < inside.sum() < len(d)
    ref = np.array([_kde.log_sum_ld(kernel, h, xs[i:i + 1], np.ones(1), ys[i:i + 1])[0][0]
                    for i in np.flatnonzero(inside)])
    err = np.abs(got[inside].astype(np.longdouble) - ref).astype(np.float64)
    assert np.all(err <= _kde.tolerance(1, np.abs(ref.astype(np.float64))))


def test_batch_independence_and_repeats():
    x, w = _samples(20011, 2, seed=5)
    g = np.linspace(-2.5, 2.5, 100)
    grid = np.array([[a, b] for a in g for b in g])
    perm = np.random.RandomState(0).permutation(len(grid))
    with DeviceKde(x, w) as kde:
        for kernel in ("gaussian", "epanechnikov"):
            one = kde.log_sum(kernel, 0.2, grid)
            np.testing.assert_array_equal(kde.log_sum(kernel, 0.2, grid), one)
            np.testing.assert_array_equal(kde.log_sum(kernel, 0.2, grid[perm]), one[perm])
            each = np.array([kde.log_sum(kernel, 0.2, grid[i:i + 1])[0] for i in range(len(grid))])
            np.testing.assert_array_equal(each, one)


def test_documented_errors_leave_the_object_usable():
    x, w = _samples(1000, 2, seed=6)
    y = _queries(5, 2, x, seed=6)
    for bad_x, status in ((np.where(np.arange(2000).reshape(1000, 2) == 7, np.nan, x), -5),
                          (np.where(np.arange(2000).reshape(1000, 2) == 9, np.inf, x), -5)):
        with pytest.raises(MbarB200Error) as e:
            DeviceKde(bad_x, w)
        assert e.value.status == status
    for bad_w in (np.where(np.arange(1000) == 3, -1.0, w), np.where(np.arange(1000) == 3, np.nan, w),
                  np.zeros(1000)):
        with pytest.raises(MbarB200Error) as e:
            DeviceKde(x, bad_w)
        assert e.value.status == -1
    with pytest.raises(MbarB200Error) as e:
        DeviceKde(np.zeros((10, 5)), np.ones(10))
    assert e.value.status == -1
    with DeviceKde(x, w) as a, DeviceKde(x[:500, :1], w[:500]) as b, \
            DeviceProblem(np.random.RandomState(0).uniform(size=(4, 64)), np.full(4, 16.0)) as p:
        want = a.log_sum("gaussian", 0.3, y)
        for kernel, h, q, status in (("gaussian", 0.0, y, -1), ("gaussian", -1.0, y, -1),
                                     ("gaussian", np.inf, y, -1), ("gaussian", np.nan, y, -1), ("box", 0.3, y, -1),
                                     ("gaussian", 0.3, np.where(np.arange(10).reshape(5, 2) == 3, np.nan, y), -5),
                                     ("gaussian", 0.3, np.where(np.arange(10).reshape(5, 2) == 4, -np.inf, y), -5)):
            with pytest.raises(MbarB200Error) as e:
                a.log_sum(kernel, h, q)
            assert e.value.status == status
        np.testing.assert_array_equal(a.log_sum("gaussian", 0.3, y), want)
        _check(b, "linear", 0.5, x[:500, :1], w[:500], y[:, :1])
        S, _, _ = p.streaming_pass(np.zeros(4))
        assert np.all(np.isfinite(S))
        np.testing.assert_array_equal(a.log_sum("gaussian", 0.3, y), want)


def test_full_size():
    """N = 1e7 samples in 2-D against long double on 16 queries."""
    rng = np.random.RandomState(7)
    N = 10_000_000
    x = rng.normal(size=(N, 2))
    w = rng.uniform(size=N)
    y = rng.normal(scale=1.5, size=(16, 2))
    with DeviceKde(x, w) as kde:
        got = kde.log_sum("gaussian", 0.02, y)
        assert kde.last_stats()["chunks"] > 100
    _kde.check_against_ld(got, "gaussian", 0.02, x, w, y)


@pytest.mark.parametrize("name", ["fes_kde_1d", "fes_kde_2d"])
def test_facade_on_the_gpu_backend(name):
    pytest.importorskip("sklearn")
    from pymbar_b200 import facade
    from pymbar_b200 import mbar_solvers as ms
    from tests import _fes
    from tests.test_driver_logic_cpu import StandInMBAR
    from tests.test_kde_cpu import check_kde_facade

    StandInMBAR.solvers = ms
    cls = _kde.kde_stand_in()
    _fes.StandInFES.mbar_class = StandInMBAR
    facade.install_on(StandInMBAR)
    facade.install_fes_on(cls)
    try:
        q0 = facade.STATS["fes_kde_queries"]
        fes = check_kde_facade(cls, name)
        assert facade.STATS["fes_kde_queries"] > q0
        assert isinstance(fes.__dict__["_b200_kde_dev"][0], DeviceKde)
    finally:
        facade.uninstall_from(cls)
        facade.uninstall_from(StandInMBAR)
        ms.clear_cache()

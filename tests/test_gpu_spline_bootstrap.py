"""Spline bootstrap replicate sums on the H100 (mbar_b200_bspline_set_replicates / _replicate_sums): every row against
the long-double restatement within the bound of tests/_spline.py with w = V_b, and against the single-replicate
moments; bit-identical repeats, and rows that do not depend on the other rows or on B; the documented errors; the full
size; and the spline bootstrap surfaces end to end through the facade against the unmodified reference's outputs
(tests/golden/fes_spline_bootstrap.npz)."""
import numpy as np
import pytest

from pymbar_b200 import DeviceBSpline
from pymbar_b200._lib import MbarB200Error
from tests import _spline

pytestmark = pytest.mark.gpu
LD_OK = np.finfo(np.longdouble).nmant >= 63
needs_ld = pytest.mark.skipif(not LD_OK, reason="long double is plain fp64 here")
KINDS = ("clamped", "nonuniform", "repeated")


def _replicates(N, B, seed):
    """Replicate weights V [B, N]: multiplicities times weights spanning 8 decades (so entries are often 0); row 1 is
    all zero."""
    rng = np.random.RandomState(seed)
    w = rng.uniform(0, 1, size=N) * np.exp(rng.uniform(-4, 4, size=N))
    V = np.array([np.bincount(rng.randint(N, size=N), minlength=N) * w for _ in range(B)])
    if B > 1:
        V[1] = 0.0
    return V


def _check_rows(R, t, k, x, V, factor=1.0):
    assert R.shape == (len(V), len(t) - k - 1)
    for b, v in enumerate(V):
        _, A_ld = _spline.moments_ld(t, k, x, v)
        _, _, TA, nA = _spline.bounds(t, k, x, v)
        np.testing.assert_array_equal(R[b][nA == 0], 0.0)
        err = np.abs(R[b].astype(np.longdouble) - A_ld).astype(np.float64)
        assert np.all(err <= factor * _spline.tolerance(k, TA, nA)), (b, k)


@needs_ld
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("k", range(8))
def test_against_long_double(k, kind):
    """Degrees 0-7, the three knot kinds, N in {1, 31, 33, 4097}; B = 7 (not a multiple of a batch)."""
    t = _spline.knots(kind, k, k + 12, seed=k)
    for N in (1, 31, 33, 4097):
        x = _spline.samples_with_edges(t, N, seed=N + k)
        V = _replicates(N, 7, seed=N)
        with DeviceBSpline(x) as d:
            d.set_replicates(V)
            R = d.replicate_sums(t, k)
            assert d.B == 7 and d.last_stats()["ms"] > 0
        _check_rows(R, t, k, x, V)


def _passes(B, k, nb):
    """Replicate passes of one call (DESIGN.md 3.5c'): 8 warps, halved while 8 nb + n_knots exceeds 13824 doubles,
    then floor((13824 - n_knots) / (warps nb)) replicates per pass."""
    nk, warps = nb + k + 1, 8
    while warps > 1 and warps * nb + nk > 13824:
        warps //= 2
    rows = max(1, min(B, (13824 - nk) // (warps * nb)))
    return -(-B // rows)


@needs_ld
@pytest.mark.parametrize("k,nb", [(0, 9), (3, 20), (7, 30), (3, 500), (3, 1000), (2, 2000)])
def test_large_n_and_several_batches(k, nb):
    """N = 200003; at nb = 500 a pass holds 3 replicates, so B = 7 takes three passes (7 at nb = 1000, and at nb =
    2000, where a CTA has 4 warps).  Each row also agrees with the single-replicate moments of DeviceBSpline(x, V_b)
    within twice the bound (both lie within it)."""
    t = _spline.knots("nonuniform", k, nb, seed=nb)
    x = _spline.samples_with_edges(t, 200003, seed=k)
    V = _replicates(len(x), 7, seed=k)
    with DeviceBSpline(x) as d:
        d.set_replicates(V)
        R = d.replicate_sums(t, k)
        passes = d.last_stats()["chunks"]
    assert passes == _passes(7, k, nb) == {500: 3, 1000: 7, 2000: 7}.get(nb, 1)
    _check_rows(R, t, k, x, V)
    for b, v in enumerate(V):
        with DeviceBSpline(x, v) as one:
            A = one.moments(t, k, want_S=False)[1]
        _, _, TA, nA = _spline.bounds(t, k, x, v)
        assert np.all(np.abs(R[b] - A) <= 2 * _spline.tolerance(k, TA, nA)), b


def test_rows_do_not_depend_on_the_others():
    """Repeat calls are bit-identical, and every row is the same bits uploaded alone, among fewer rows, or after
    another knot vector."""
    t = _spline.knots("repeated", 3, 25, seed=1)
    x = _spline.samples_with_edges(t, 100003, seed=2)
    V = _replicates(len(x), 11, seed=3)
    with DeviceBSpline(x) as d:
        d.set_replicates(V)
        R = d.replicate_sums(t, 3)
        np.testing.assert_array_equal(d.replicate_sums(t, 3), R)
        d.replicate_sums(_spline.knots("clamped", 5, 40), 5)
        np.testing.assert_array_equal(d.replicate_sums(t, 3), R)
        for b in (0, 1, 6, 10):
            d.set_replicates(V[b:b + 1])
            np.testing.assert_array_equal(d.replicate_sums(t, 3)[0], R[b])
        d.set_replicates(V[4:9])
        np.testing.assert_array_equal(d.replicate_sums(t, 3), R[4:9])
    with DeviceBSpline(x) as fresh:
        fresh.set_replicates(V[::-1])
        np.testing.assert_array_equal(fresh.replicate_sums(t, 3), R[::-1])


def test_errors_leave_the_object_usable():
    t = _spline.knots("clamped", 3, 12)
    x = _spline.samples_with_edges(t, 5000, seed=2)
    rng = np.random.RandomState(0)
    w = rng.uniform(size=len(x))
    s = np.repeat(np.arange(4), len(x) // 4 + 1)[:len(x)]
    V = _replicates(len(x), 5, seed=4)
    with DeviceBSpline(x, w, s, K=4) as d:
        S0, A0 = d.moments(t, 3)
        with pytest.raises(MbarB200Error) as e:
            d.replicate_sums(t, 3)
        assert e.value.status == -4                      # no replicates uploaded
        for bad in (np.where(np.arange(V.size).reshape(V.shape) == 7, -1.0, V),
                    np.where(np.arange(V.size).reshape(V.shape) == 9, np.nan, V),
                    np.where(np.arange(V.size).reshape(V.shape) == 11, np.inf, V), V[:0]):
            d.set_replicates(V)
            with pytest.raises(MbarB200Error) as e:
                d.set_replicates(bad)
            assert e.value.status == -1 and d.B == 0
            with pytest.raises(MbarB200Error) as e:
                d.replicate_sums(t, 3)
            assert e.value.status == -4                  # the failed upload left no replicates
        with pytest.raises(ValueError):
            d.set_replicates(V[:, :10])
        d.set_replicates(V)
        want = d.replicate_sums(t, 3)
        for tk, k in ((t, 8), (t, -1), (t[::-1], 3), (t[:7], 3), (np.where(t > 0.5, np.inf, t), 3),
                      (np.where(t > 0.5, np.nan, t), 3), (np.zeros(12), 3)):
            with pytest.raises(MbarB200Error) as e:
                d.replicate_sums(tk, k)
            assert e.value.status == -1
            np.testing.assert_array_equal(d.replicate_sums(t, 3), want)
        # b = 0's weights and labels are untouched by the replicates
        S1, A1 = d.moments(t, 3)
        np.testing.assert_array_equal(S1, S0)
        np.testing.assert_array_equal(A1, A0)


def test_full_size():
    """N = 1e7, B = 50, nspline = 20, cubic: small multiplicities times normalised weights, against a chunked fp64 host
    sum, within the bound with the host sum's own rounding added."""
    N, B, k, nb, K = 10_000_000, 50, 3, 20, 64
    rng = np.random.RandomState(0)
    centres = np.linspace(-2, 2, K)
    s = np.repeat(np.arange(K), N // K + 1)[:N]
    x = centres[s] + 0.15 * rng.standard_normal(N)
    w = np.exp(-2.0 * x ** 2)
    w /= w.sum()
    t = _spline.knots("clamped", k, nb, lo=-2.3, hi=2.3)
    V = np.empty((B, N))
    for b in range(B):
        V[b] = rng.randint(0, 3, size=N) * w
    with DeviceBSpline(x) as d:
        d.set_replicates(V)
        R = d.replicate_sums(t, k)
        assert d.last_stats()["ms"] > 0
    chunk = 1_000_000
    R_h, T = np.zeros((B, nb)), np.zeros((B, nb))
    for n0 in range(0, N, chunk):
        first, h = _spline.basis_values(t, k, x[n0:n0 + chunk])
        _, habs = _spline.basis_values(t, k, x[n0:n0 + chunk], absolute=True)
        cols = (first[None, :] + np.arange(k + 1)[:, None]).ravel()
        for b in range(B):
            v = V[b, n0:n0 + chunk]
            R_h[b] += np.bincount(cols, weights=(h * v[None, :]).ravel(), minlength=nb)
            T[b] += np.bincount(cols, weights=(habs * v[None, :]).ravel(), minlength=nb)
    assert np.all(np.abs(R - R_h) <= 2 * _spline.tolerance(k, T, float(N)))


@pytest.fixture()
def gpu_boot_spline():
    from pymbar_b200 import facade
    from pymbar_b200 import mbar_solvers as ms
    from tests.test_driver_logic_cpu import StandInMBAR
    from tests.test_fes_spline_bootstrap_cpu import boot_stand_in

    StandInMBAR.solvers = ms
    cls = boot_stand_in()
    cls.mbar_class = StandInMBAR
    facade.install_on(StandInMBAR)
    facade.install_fes_on(cls)
    yield cls
    facade.uninstall_from(cls)
    facade.uninstall_from(StandInMBAR)
    ms.clear_cache()


def _facade_cases():
    from tests.test_fes_spline_bootstrap_cpu import CASES

    return CASES


@pytest.mark.parametrize("name,seed", _facade_cases())
def test_spline_bootstrap_on_the_gpu_backend(gpu_boot_spline, monkeypatch, name, seed):
    from tests.test_fes_spline_bootstrap_cpu import ReplicateNumpyBSpline, check_spline_bootstrap

    # the device's DeviceBSpline, with its replicate weights kept for the comparison with the reference's
    orig_set = DeviceBSpline.set_replicates

    def keep(self, V):
        ReplicateNumpyBSpline.last_V = np.array(V)
        return orig_set(self, V)

    monkeypatch.setattr(DeviceBSpline, "set_replicates", keep)
    monkeypatch.setattr(ReplicateNumpyBSpline, "replicate_calls", 0)
    calls = []
    orig_sums = DeviceBSpline.replicate_sums

    def count(self, t, k):
        ReplicateNumpyBSpline.replicate_calls += 1
        calls.append(self)
        return orig_sums(self, t, k)

    monkeypatch.setattr(DeviceBSpline, "replicate_sums", count)
    check_spline_bootstrap(gpu_boot_spline, name, seed)
    assert len(calls) == 1 and isinstance(calls[0], DeviceBSpline)

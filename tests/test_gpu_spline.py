"""B-spline basis sums on the H100 (mbar_b200_bspline_*): S and A against the long-double restatement entry by entry
within the bound of tests/_spline.py, bit-identity across repeats, S-only / A-only / both and earlier knot vectors,
the documented errors, the full size, and the spline FES facade end to end on the device."""
import numpy as np
import pytest

from pymbar_b200 import DeviceBSpline
from pymbar_b200._lib import MbarB200Error
from tests import _spline

pytestmark = pytest.mark.gpu
LD_OK = np.finfo(np.longdouble).nmant >= 63
needs_ld = pytest.mark.skipif(not LD_OK, reason="long double is plain fp64 here")


def _problem(N, K, k, nb, kind="clamped", shuffled=False, zero_w=False, seed=0):
    t = _spline.knots(kind, k, nb, seed=seed)
    x = _spline.samples_with_edges(t, N, seed=seed)
    rng = np.random.RandomState(seed + 1)
    w = rng.uniform(0, 1, size=N) * np.exp(rng.uniform(-4, 4, size=N))
    if zero_w:
        w[rng.rand(N) < 0.3] = 0.0
    # contiguous labels with uneven state sizes; the last state of three or more is empty
    live = max(K - 1, 1) if K >= 3 else K
    cuts = np.sort(rng.randint(0, N + 1, size=live - 1))
    s = np.searchsorted(cuts, np.arange(N), side="right").astype(np.int64)
    if shuffled:
        s = rng.permutation(s)
    return t, x, w, s


def _check(N, K, k, nb, **kw):
    t, x, w, s = _problem(N, K, k, nb, **kw)
    with DeviceBSpline(x, w, s, K=K) as d:
        S, A = d.moments(t, k)
        stats = d.last_stats()
    assert stats["ms"] > 0 and stats["chunks"] >= 1
    _spline.check_against_ld(S, A, t, k, x, w, s, K)
    return stats


@needs_ld
@pytest.mark.parametrize("N", [1, 31, 32, 33, 4097, 200003])
@pytest.mark.parametrize("k", range(8))
def test_against_long_double_every_degree(N, k):
    _check(N, 3, k, k + 12, kind=("clamped", "nonuniform", "repeated")[k % 3], seed=k)


@needs_ld
@pytest.mark.parametrize("K,nb", [(1, 20), (256, 20), (256, 1000), (2100, 20)])
@pytest.mark.parametrize("shuffled", [False, True])
def test_against_long_double_many_states(K, nb, shuffled):
    stats = _check(200003, K, 3, nb, shuffled=shuffled, zero_w=True, seed=K)
    if K * nb + 1 > 13824 - nb - 4:
        assert stats["chunks"] > 1                # state chunking
    else:
        assert stats["chunks"] == 1


def test_bit_identity_across_requests():
    t, x, w, s = _problem(100003, 7, 3, 25, shuffled=True, seed=5)
    t2 = _spline.knots("nonuniform", 5, 40, seed=9)
    with DeviceBSpline(x, w, s, K=7) as d:
        S, A = d.moments(t, 3)
        S2, A2 = d.moments(t, 3)
        S_only, none = d.moments(t, 3, want_A=False)
        none2, A_only = d.moments(t, 3, want_S=False)
        d.moments(t2, 5)                          # another knot vector in between
        S3, A3 = d.moments(t, 3)
    assert none is None and none2 is None
    for a, b in ((S, S2), (S, S_only), (S, S3), (A, A2), (A, A_only), (A, A3)):
        np.testing.assert_array_equal(a, b)
    # one object per kind of upload gives the same bits as well
    with DeviceBSpline(x, None, s, K=7) as d:
        np.testing.assert_array_equal(d.moments(t, 3, want_A=False)[0], S)
    with DeviceBSpline(x, w) as d:
        np.testing.assert_array_equal(d.moments(t, 3, want_S=False)[1], A)


def test_errors_leave_the_object_usable():
    t, x, w, s = _problem(5000, 4, 3, 12, seed=2)
    for bad, status in ((dict(w_n=-w), -1), (dict(w_n=np.where(x > 0, np.nan, w)), -1),
                        (dict(w_n=np.where(x > 0, np.inf, w)), -1),
                        (dict(state_n=np.where(np.arange(len(s)) == 7, 4, s)), -1),
                        (dict(state_n=np.where(np.arange(len(s)) == 7, -1, s)), -1)):
        args = dict(w_n=w, state_n=s, K=4)
        args.update(bad)
        with pytest.raises(MbarB200Error) as e:
            DeviceBSpline(x, **args)
        assert e.value.status == status
    for v in (np.nan, np.inf, -np.inf):
        xb = x.copy()
        xb[17] = v
        with pytest.raises(MbarB200Error) as e:
            DeviceBSpline(xb, w, s, K=4)
        assert e.value.status == -5
    with DeviceBSpline(x, w, s, K=4) as d:
        want = d.moments(t, 3)
        bad_knots = [(t, 8), (t, -1), (t[::-1], 3), (t[:7], 3), (np.where(t > 0.5, np.inf, t), 3),
                     (np.where(t > 0.5, np.nan, t), 3), (np.zeros(12), 3)]
        for tk, k in bad_knots:
            with pytest.raises(MbarB200Error) as e:
                d.moments(tk, k)
            assert e.value.status == -1
            got = d.moments(t, 3)
            np.testing.assert_array_equal(got[0], want[0])
            np.testing.assert_array_equal(got[1], want[1])
    with DeviceBSpline(x, w) as d:                # no labels: S cannot be asked for
        with pytest.raises(MbarB200Error):
            d.moments(t, 3)
        assert d.moments(t, 3, want_S=False)[1] is not None


def test_full_size():
    """N = 1e7, K = 256, nspline = 20, cubic: against a chunked fp64 host sum (scipy's basis values, summed per
    chunk), within the bound of tests/_spline.py with the host sum's own rounding added."""
    N, K, k, nb = 10_000_000, 256, 3, 20
    rng = np.random.RandomState(0)
    centres = np.linspace(-2, 2, K)
    s = np.repeat(np.arange(K), N // K + 1)[:N]
    x = centres[s] + 0.15 * rng.standard_normal(N)
    w = np.exp(-2.0 * x ** 2)
    w /= w.sum()
    t = _spline.knots("clamped", k, nb, lo=-2.3, hi=2.3)
    with DeviceBSpline(x, w, s, K=K) as d:
        S, A = d.moments(t, k)
        ms = d.last_stats()["ms"]
    S_h, A_h = np.zeros((K, nb)), np.zeros(nb)
    TS, TA = np.zeros((K, nb)), np.zeros(nb)
    for n0 in range(0, N, 1_000_000):
        sl = slice(n0, n0 + 1_000_000)
        Sc, Ac = _spline.moments(t, k, x[sl], w[sl], s[sl], K)
        TSc, _, TAc, _ = _spline.bounds(t, k, x[sl], w[sl], s[sl], K)
        S_h += Sc
        A_h += Ac
        TS += TSc
        TA += TAc
    nS = np.full_like(TS, N / K)
    tolS = 2 * _spline.tolerance(k, TS, nS)
    tolA = 2 * _spline.tolerance(k, TA, float(N))
    assert np.all(np.abs(S - S_h) <= tolS)
    assert np.all(np.abs(A - A_h) <= tolA)
    assert ms > 0


def test_facade_on_the_gpu_backend():
    from pymbar_b200 import facade
    from pymbar_b200 import mbar_solvers as ms
    from tests import _fes
    from tests.test_driver_logic_cpu import StandInMBAR
    from tests.test_spline_cpu import _load, check_case, golden

    StandInMBAR.solvers = ms
    cls = _spline.spline_stand_in()
    _fes.StandInFES.mbar_class = StandInMBAR
    facade.install_on(StandInMBAR)
    facade.install_fes_on(cls)
    g, z = golden(), _load()
    from scipy.interpolate import BSpline

    calls = []
    orig_call = BSpline.__call__

    def watch(self, x, *a, **k):
        calls.append(np.size(x))
        return orig_call(self, x, *a, **k)

    BSpline.__call__ = watch
    try:
        for i in range(len(_spline.SPLINE_CASES)):
            m0 = facade.STATS["fes_spline_moments"]
            fes, x = check_case(cls, i, g, z, served=True)
            assert facade.STATS["fes_spline_moments"] == m0 + 1
            assert isinstance(fes.__dict__["_b200_spline"], facade.SplineMoments)
        assert max(calls) < int(np.min(z["N_k"]))
    finally:
        BSpline.__call__ = orig_call
        facade.uninstall_from(cls)
        facade.uninstall_from(StandInMBAR)
        ms.clear_cache()

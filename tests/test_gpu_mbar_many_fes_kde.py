"""DeviceKdeMany and DeviceMbarBatch.log_weights on the GPU: bit identity with DeviceKde, the errors, the launch counts,
the log weights against long double and the single path, and MbarMany's KDE surfaces end to end against
tests/golden/mbar_many_fes_kde.npz and the single-problem device path."""
import numpy as np
import pytest

from pymbar_b200 import _lib
from pymbar_b200 import fes_bootstrap as fb
from pymbar_b200.fes import KDE_KERNELS
from tests import _mbar_many_fes_kde as FK

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from pymbar_b200 import build

    build.build()
    if _lib.device_count() == 0:
        pytest.skip("no GPU")
    return _lib


def _sets(rng):
    """(x, w) sample sets with N from 1 to above 10^5 in D = 1..4, some zero weights."""
    out = []
    for N, D in ((1, 1), (255, 2), (4097, 3), (20000, 4), (130001, 1), (9000, 2)):
        x = rng.normal(size=(N, D))
        w = rng.exponential(size=N)
        w[rng.random(N) < 0.1] = 0.0
        w[0] = 1.0
        out.append((x, w))
    return out


def _queries(rng, D, Q):
    y = rng.normal(size=(Q, D)) * 1.5
    y[: min(Q, 3)] += 40.0          # far from the data: -inf beyond the compact supports, deep tails otherwise
    return y


def test_bit_identical_to_device_kde(lib):
    from pymbar_b200 import DeviceKde, DeviceKdeMany

    rng = np.random.default_rng(11)
    sets = _sets(rng)
    reqs, want = [], []
    for s, (x, w) in enumerate(sets):
        with DeviceKde(x, w) as k:
            for kern in KDE_KERNELS:
                for Q in (1, 300):
                    y = _queries(rng, x.shape[1], Q)
                    h = 0.3 + 0.1 * s
                    reqs.append((s, kern, h, w, y))
                    want.append(k.log_sum(kern, h, y))
    with DeviceKdeMany([x for x, _ in sets]) as km:
        got = km.log_sum(*zip(*reqs))
        for g, e in zip(got, want):
            np.testing.assert_array_equal(g, e)
        assert any(np.isneginf(e).any() for e in want)
        # alone, shuffled, repeated
        perm = rng.permutation(len(reqs))
        shuffled = km.log_sum(*zip(*[reqs[i] for i in perm]))
        for i, g in zip(perm, shuffled):
            np.testing.assert_array_equal(g, want[i])
        for i in (0, 7, len(reqs) - 1):
            np.testing.assert_array_equal(km.log_sum(*zip(reqs[i]))[0], want[i])
        again = km.log_sum(*zip(*reqs))
        for g, e in zip(again, want):
            np.testing.assert_array_equal(g, e)


def test_large_query_counts_and_sub_batches(lib):
    from pymbar_b200 import DeviceKde, DeviceKdeMany

    rng = np.random.default_rng(12)
    x = rng.normal(size=(1200000, 1))
    w = rng.exponential(size=1200000)
    y = _queries(rng, 1, 15000)
    with DeviceKde(x, w) as k:
        want = k.log_sum("gaussian", 0.2, y)
        want_t = k.log_sum("tophat", 0.2, y[:500])
    with DeviceKdeMany([x, x[:1000]]) as km:
        # 293 chunks x 15000 queries x 16 B is over 64 MiB: the call splits into sub-batches
        got = km.log_sum([0, 1, 0], ["gaussian", "gaussian", "tophat"], [0.2, 0.2, 0.2], [w, w[:1000], w],
                         [y, y[:5], y[:500]])
        assert km.last_stats()["launches"] > 3
        np.testing.assert_array_equal(got[0], want)
        np.testing.assert_array_equal(got[2], want_t)
        one = km.log_sum([0], ["gaussian"], [0.2], [w], [y])[0]
        np.testing.assert_array_equal(one, want)


def test_launches_and_errors(lib):
    from pymbar_b200 import DeviceKdeMany

    rng = np.random.default_rng(13)
    xs = [rng.normal(size=(500, 1)), rng.normal(size=(700, 1)), rng.normal(size=(300, 2))]
    ws = [np.ones(500), np.ones(700), np.ones(300)]
    y = rng.normal(size=(20, 1))
    with DeviceKdeMany(xs) as km:
        km.log_sum([0, 1, 0], ["gaussian"] * 3, [0.2] * 3, [ws[0], ws[1], ws[0] * 2], [y, y, y])
        s = km.last_stats()
        assert s["launches"] == 2 and s["pairs"] == 20 * (500 + 700 + 500)
        km.log_sum([0, 2], ["gaussian", "gaussian"], [0.2, 0.2], [ws[0], ws[2]], [y, np.hstack([y, y])])
        assert km.last_stats()["launches"] == 3
        good = km.log_sum([0], ["gaussian"], [0.2], [ws[0]], [y])[0]

        def err(status, *a, match=None):
            with pytest.raises(_lib.MbarB200Error, match=match) as e:
                km.log_sum(*a)
            assert e.value.status == status

        INV, NAN = -1, -5          # MBAR_B200_ERR_INVALID, MBAR_B200_ERR_NAN
        err(INV, [3], ["gaussian"], [0.2], [ws[0]], [y])
        err(INV, [0], [17], [0.2], [ws[0]], [y])
        err(INV, [0], ["gaussian"], [0.0], [ws[0]], [y])
        err(INV, [0], ["gaussian"], [np.inf], [ws[0]], [y])
        for bad in (-1.0, np.nan, np.inf):
            w = ws[0].copy()
            w[5] = bad
            err(INV, [0], ["gaussian"], [0.2], [w], [y])
        err(INV, [0], ["gaussian"], [0.2], [np.zeros(500)], [y])
        yn = y.copy()
        yn[3] = np.nan
        err(NAN, [0], ["gaussian"], [0.2], [ws[0]], [yn])
        np.testing.assert_array_equal(km.log_sum([0], ["gaussian"], [0.2], [ws[0]], [y])[0], good)
    with pytest.raises(_lib.MbarB200Error) as e:
        DeviceKdeMany([rng.normal(size=(10, 5))])
    assert e.value.status == -1
    xn = rng.normal(size=(10, 1))
    xn[2] = np.inf
    with pytest.raises(_lib.MbarB200Error) as e:
        DeviceKdeMany([xn])
    assert e.value.status == -5


def _umbrella(rng, K, n, shift=0.0):
    from tests._fes import umbrella_energies

    c = np.linspace(-2, 2, K)
    x = np.concatenate([rng.normal(0.8 * c[k], 0.3, size=n) for k in range(K)])
    u_kn, u_n = umbrella_energies(x, c, 4.0, 30.0)
    return x, u_kn, u_n + shift, np.full(K, n)


def test_log_weights(lib):
    from pymbar_b200 import DeviceMbarBatch, DeviceProblem

    rng = np.random.default_rng(14)
    probs = [_umbrella(rng, K, n) for K, n in ((1, 50), (8, 400), (33, 1000), (64, 90))]
    N_k = [p[3].astype(float) for p in probs]
    N_k[1][3] = 0.0
    us = [p[1].copy() for p in probs]
    us[1] = np.delete(us[1], np.s_[1200:1600], axis=1)
    xs = [p[0] for p in probs]
    un = [p[2].copy() for p in probs]
    un[1] = np.delete(un[1], np.s_[1200:1600])
    un[2][[5, 17]] = np.inf
    f = [rng.normal(size=len(n)) for n in N_k]
    with DeviceMbarBatch(us, N_k) as b:
        out, flags = b.log_weights([0, 1, 2, 3], f, un)
        assert b.last_stats()["launches"] == 1 and not flags.any()
        for p in range(4):
            s = N_k[p] > 0
            LD = np.longdouble
            a = LD(1) * f[p][s, None] + np.log(N_k[p][s, None].astype(LD)) - us[p][s].astype(LD)
            m = a.max(axis=0)
            L = m + np.log(np.exp(a - m).sum(axis=0))
            want = (-un[p].astype(LD) - L).astype(np.float64)
            fin = np.isfinite(want)
            np.testing.assert_array_equal(np.isneginf(out[p]), ~fin)
            tol = 1e-13 * np.abs(want[fin]).max()
            np.testing.assert_allclose(out[p][fin], want[fin], rtol=1e-13, atol=tol)
            with DeviceProblem(us[p], N_k[p]) as q:
                single = -un[p] - q.log_denominator(f[p])
            np.testing.assert_allclose(out[p][fin], single[fin], rtol=1e-13, atol=tol)
        # a NaN log w_n flags its request and the call succeeds; errors leave the batch usable
        with DeviceMbarBatch(us[:1] + [np.vstack([us[1][:1], np.full((1, us[1].shape[1]), np.inf)])],
                             [N_k[0], np.array([0.0, float(us[1].shape[1])])]) as b2:
            _, fl = b2.log_weights([0, 1], [f[0], np.zeros(2)], [un[0], un[1]])
            assert fl.tolist() == [False, True]
        with pytest.raises(_lib.MbarB200Error) as e:
            b.log_weights([4], [f[0]], [un[0]])
        assert e.value.status == -1
        nanu = un[0].copy()
        nanu[3] = np.nan
        with pytest.raises(_lib.MbarB200Error) as e:
            b.log_weights([0], [f[0]], [nanu])
        assert e.value.status == -5
        again, _ = b.log_weights([2], [f[2]], [un[2]])
        np.testing.assert_array_equal(again[0], out[2])


def test_mbar_many_golden_and_single_path(lib):
    from pymbar_b200 import DeviceKde, DeviceProblem
    from pymbar_b200.mbar_many import MbarMany

    cases, stream_next = FK.load()
    plain = [i for i in range(len(cases)) if i not in FK.RAISES]
    with MbarMany(*FK.args(cases)) as m:
        FK.generate(m, cases, range(len(cases)))
        for tag, rp in FK.REFS:
            out = FK.query(m, cases, plain, rp)
            for i in plain:
                FK.check_plain(cases[i], out[i], tag)
        # per query: one log_sum call, a partial launch for each (D, kernel) of the six problems and one combine
        assert m.kde_stats["calls"] == 3 and m.kde_stats["launches"] == 3 * 4
        np.random.seed(FK.STREAM_SEED)
        FK.generate(m, cases, FK.BOOT, FK.B)
        assert np.random.randint(2 ** 31 - 1) == stream_next
        worst_f = worst_df = 0.0
        for tag, rp in FK.BOOT_REFS:
            out = FK.query(m, cases, FK.BOOT, rp, "bootstrap")
            for i in FK.BOOT:
                c = cases[i]
                FK.check_boot(c, out[i], "stream", tag)
                # the single-problem device path: DeviceProblem log weights, DeviceKde and log_sum_replicates
                k = m._kde[i]
                with DeviceProblem(c["u_kn"], c["N_k"].astype(float)) as q:
                    lw = -c["u_n"] - q.log_denominator(m.results[i]["f_k"])
                w = np.exp(lw - np.max(lw))
                w = w / np.sum(w)
                with DeviceKde(c["x_n"], w) as dk:
                    dk.set_replicates(k["V"])
                    x = np.asarray(c["queries"], float)
                    x = x.reshape(-1, 1) if x.ndim == 1 else x
                    want = fb.kde_bootstrap_query(dk, k["settings"], x, rp, c["fes_reference"],
                                                  float(np.log(np.sum(w))))
                fin = np.isfinite(want["f_i"])
                np.testing.assert_allclose(out[i]["f_i"][fin], want["f_i"][fin], rtol=1e-12, atol=1e-12)
                np.testing.assert_allclose(out[i]["df_i"], want["df_i"], rtol=1e-12, atol=1e-12)
                worst_f = max(worst_f, float(np.max(np.abs(out[i]["f_i"][fin] - want["f_i"][fin]))))
                worst_df = max(worst_df, float(np.max(np.abs(out[i]["df_i"] - want["df_i"]))))
        print(f"largest difference from the single path: f_i {worst_f:.3g}, df_i {worst_df:.3g}")

"""The extended-precision reference of tests/_moments.py (no GPU): against mpmath, against the oracle's Hessian, the
tolerance formula on hand-made inputs, and the claims the ladder cases make about themselves."""
import mpmath
import numpy as np
import pytest

from oracle import mbar_oracle as orc
from tests import _moments as M


def _mp_moments(u, N_k, f, mult, all_rows):
    mpmath.mp.dps = 40
    K, N = u.shape
    S = [mpmath.mpf(0)] * K
    G = [[mpmath.mpf(0)] * K for _ in range(K)]
    for n in range(N):
        W = [mpmath.exp(mpmath.mpf(f[k]) - mpmath.mpf(u[k, n])) if np.isfinite(u[k, n]) else mpmath.mpf(0)
             for k in range(K)]
        D = mpmath.fsum(N_k[j] * W[j] for j in range(K) if N_k[j] > 0)
        W = [x / D for x in W]
        w = [W[k] * N_k[k] if N_k[k] > 0 else (W[k] if all_rows else mpmath.mpf(0)) for k in range(K)]
        for i in range(K):
            S[i] += mult[n] * W[i]
            for j in range(K):
                G[i][j] += mult[n] * w[i] * w[j]
    return S, G


def _mp(x):
    """A long double as an mpf, exactly."""
    m, e = np.frexp(M.LD(x))
    return mpmath.mpf(int(m * M.LD(2) ** 64)) * mpmath.mpf(2) ** (int(e) - 64)


@pytest.mark.parametrize("all_rows", [False, True])
def test_reference_against_mpmath(all_rows):
    """Entries below 1e-300, an unsampled state, a +inf energy and a zero multiplicity, at 40 digits."""
    u = np.array([[0.1, 0.5, 710.0, 715.0, 1.3],
                  [708.0, 712.0, 0.2, 0.9, 703.0],
                  [350.0, 360.0, 340.0, 355.0, np.inf],
                  [0.3, 1.1, 1.2, 0.4, 0.8]])
    N_k = np.array([2.0, 2.0, 0.0, 1.0])
    f = np.array([0.0, 0.4, -0.3, 1.2])
    mult = np.array([1.0, 0.0, 2.0, 1.0, 3.0])
    S, G, A = M.moments_ld(u, N_k, f, mult=mult, all_rows=all_rows)
    Sm, Gm = _mp_moments(u, N_k, f, mult, all_rows)
    assert 0 < float(min(x for row in Gm for x in row if x > 0)) < 1e-300
    for k in range(4):
        assert abs(_mp(S[k]) - Sm[k]) <= 1e-16 * abs(Sm[k]), (k, S[k], Sm[k])
        for j in range(4):
            assert abs(_mp(G[k, j]) - Gm[k][j]) <= 1e-16 * abs(Gm[k][j]), (k, j, G[k, j], Gm[k][j])
    if not all_rows:
        assert np.all(G[2] == 0) and np.all(G[:, 2] == 0)
    assert np.all(A >= 0) and A.max() < 710


def test_reference_against_oracle_hessian():
    u, N_k = (a.astype(float) for a in __import__("oracle.testsystems", fromlist=["x"]).oscillators(6, 40, seed=2))
    f = np.random.RandomState(0).normal(scale=0.3, size=6)
    S, G, _ = M.moments_ld(u, N_k, f)
    H = orc.mbar_hessian(u, N_k, f)
    G_or = -H + np.diag(N_k * orc.mbar_W_nk(u, N_k, f).sum(0))
    np.testing.assert_allclose(G.astype(float), G_or, rtol=1e-13, atol=0)
    np.testing.assert_allclose(S.astype(float), orc.mbar_W_nk(u, N_k, f).sum(0), rtol=1e-13)


def test_reference_refuses_fp64_long_double():
    assert np.finfo(M.LD).nmant >= 63


def test_entry_tol_by_hand():
    G = np.array([[4.0, 1e-300], [1e-300, 0.0]], M.LD)
    t = M.entry_tol(G, np.array([10.0, 0.0]), N=100, wmax=0.5)
    eps = 2.0 ** -53
    alpha = 400 * 2.0 ** -1020
    assert float(t[0, 0]) == pytest.approx((160 * eps + 80 * eps + 64 * eps) * 4.0 + alpha, rel=1e-15)
    assert float(t[1, 1]) == pytest.approx(alpha, rel=1e-15)
    assert float(t[0, 1]) == pytest.approx(alpha + (80 * eps + 80 * eps + 64 * eps) * 1e-300, rel=1e-12)
    # wmax above 1 scales the floor term; a scalar A applies to every state
    t2 = M.entry_tol(G, 5.0, N=100, wmax=8.0)
    assert float(t2[1, 1]) == pytest.approx(8 * alpha, rel=1e-15)
    assert float(t2[0, 0]) == pytest.approx((80 * eps + 80 * eps + 64 * eps) * 4.0 + 8 * alpha, rel=1e-15)
    # a dropped sample (relative 1/N) or tile (32/N) is far outside the band
    assert float(t[0, 0]) < 4.0 / 100 * 1e-9
    assert M.excess(G + t, G, t) == pytest.approx(1.0)


@pytest.mark.parametrize("name", [n for n in M.cases() if n != "ladder_K2100"])
def test_ladders_reach_the_edges(name):
    """What the cases are for: entries spanning the fp64 range, weights on both sides of the exp floor, subnormal
    products, N not a multiple of 32."""
    c = M.build(name)
    K = len(c["N"])
    assert c["u"].shape[1] % 32 != 0
    S, G, A = M.moments_ld(c["u"], c["N"], c["f"])
    s = c["N"] > 0
    normal = G[G >= 2.0 ** -1022]
    span = float(np.log10(normal.max()) - np.log10(normal.min()))
    if K >= 33:
        assert span > 300, span
    if K >= 16:
        assert np.any((G > 0) & (G < 2.0 ** -1022)), "no subnormal entry"
    if K >= 5 and name != "ladder_K5_tiny":
        assert np.any((A > 600)), A.max()
    np.testing.assert_allclose(S[s].astype(float), 1.0, atol=0.3)
    assert np.all(G == G.T)

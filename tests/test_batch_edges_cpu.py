"""The cases and the flag restatement of tests/_batch_edges.py, without a GPU: every builder lands where it claims,
the tiled-column reference equals the direct one, the chunk geometry of the large cases, and predict_flag on
hand-built arrays."""
import numpy as np
import pytest

from pymbar_b200 import mbar_many as mm
from tests import _batch_edges as BE
from tests import _edges as E
from tests._moments import moments_ld


def _by_name():
    return {n: (u, N_k, f) for n, u, N_k, f in BE.threshold_cases()}


@pytest.mark.parametrize("side", [-0.5, 0.5])
def test_threshold_builders_land_where_they_claim(side):
    th = _by_name()
    u, N_k, f = th[f"sampled_S_1e-280{side:+g}"]
    r = BE.restate(u, N_k, f, False, want_G=False)
    assert abs(float(r["logS"][1]) - (BE.LOG_S_LO + side)) < 1e-9
    assert float(r["logS"][0]) > -1 and float(r["logG"]) < 10
    u, N_k, f = th[f"unsampled_S_DBL_MAX{side:+g}"]
    r = BE.restate(u, N_k, f, True, want_G=False)
    assert abs(float(r["logS"][2]) - (BE.LOG_DBL_MAX + side)) < 1e-9
    u, N_k, f = th[f"gram_DBL_MAX{side:+g}"]
    r = BE.restate(u, N_k, f, True, want_G=False)
    assert abs(float(r["logGd"][2]) - (BE.LOG_DBL_MAX + side)) < 1e-9
    assert float(r["logS"][2]) < BE.LOG_DBL_MAX - 300           # S_k itself is far from overflow
    # the largest weight of that row sits near e^355, the square root of DBL_MAX
    w = float(np.max(f[2] - u[2] - (f[0] + np.log(N_k[0]) - u[0] + np.log1p(np.exp(f[1] - u[1] + u[0] - f[0])))))
    assert abs(w - BE.LOG_DBL_MAX / 2) < 3
    for s in (False, True):
        for G in (False, True):
            flag, margin = BE.predict_flag(*th[f"gram_DBL_MAX{side:+g}"], s, G)
            assert flag == (side > 0 and s and G) and (margin >= 0.5 - 1e-9 or not (s and G))


def test_gram_400kT_example_and_inf_row():
    th = _by_name()
    u, N_k, f = th["gram_400kT_below_f0"]
    r = BE.restate(u, N_k, f, True, want_G=False)
    assert abs(float(r["logS"][2]) - 400) < 1e-9                  # S finite
    assert float(r["logGd"][2]) > BE.LOG_DBL_MAX + 50              # Ghat_22 overflows
    assert BE.predict_flag(u, N_k, f, True, True) == (True, pytest.approx(float(r["logGd"][2]) - BE.LOG_DBL_MAX))
    assert not BE.predict_flag(u, N_k, f, True, False)[0]
    u, N_k, f = th["unsampled_all_inf"]
    r = BE.restate(u, N_k, f, True)
    assert r["S"][2] == 0 and r["logS"][2] == -np.inf and np.all(r["G"][2] == 0)
    flag, margin = BE.predict_flag(u, N_k, f, True, True)
    assert not flag and BE.is_clear(margin)


def test_families_are_normalised_at_their_f():
    for c in BE.family_cases():
        r = BE.restate(c["u"], c["N"], c["f"], True, want_G=False)
        # exact up to the rounding of the energies passed: eps per unit of |f|
        assert np.max(np.abs(r["logS"].astype(float))) < 8 * BE.EPS * max(1.0, np.max(np.abs(c["f"]))), c["name"]
        flag, margin = BE.predict_flag(c["u"], c["N"], c["f"], True, True)
        assert not flag and BE.is_clear(margin), c["name"]
    names = [c["name"] for c in BE.family_cases()]
    assert "unsampled_below_1e+08" in names and "unsampled_above_2e+06" in names


def test_restate_matches_moments_ld():
    for name in BE.LADDERS:
        c = BE.ladder_case(name)
        for all_rows in (False, True):
            S, G, _ = moments_ld(c["u"], c["N"], c["f"], all_rows=all_rows)
            r = BE.restate(c["u"], c["N"], c["f"], all_rows)
            rows = np.ones(len(c["N"]), bool) if all_rows else c["N"] > 0
            np.testing.assert_allclose(r["S"][rows].astype(float), S[rows].astype(float), rtol=1e-15, atol=1e-300)
            np.testing.assert_allclose(r["G"].astype(float), G.astype(float), rtol=1e-15, atol=1e-300)


def test_tiled_reference_equals_direct():
    block, f = BE.tiled_block(8, seed=8)
    N = 3 * BE.BLOCK + 40
    u = BE.tiled(block, N)
    N_k = BE.tiled_N_k(8, N)
    assert N_k.sum() == N and np.array_equal(u[:, BE.BLOCK + 5], block[:, 5])
    counts = BE.multinomial_counts(N, 1)
    for cnt in (None, counts):
        for all_rows in (False, True):
            a = BE.restate(u, N_k, f, all_rows, mult=cnt)
            b = BE.restate(block, N_k, f, all_rows, mult=BE.column_mult(N, cnt))
            for k in ("S", "G"):
                np.testing.assert_allclose(a[k].astype(float), b[k].astype(float), rtol=1e-16, atol=0)
            assert abs(float(a["sumL"] - b["sumL"])) <= 1e-14 * abs(float(a["sumL"]))
            assert a["absx"] == pytest.approx(b["absx"], rel=1e-12)
    # one tile dropped moves S far beyond the tolerance at 4 million samples
    N = 32 * 131072 + 19
    m = BE.column_mult(N)
    drop = m - BE.column_mult(32, width=BE.BLOCK)
    block, f = BE.tiled_block(64)
    N_k = BE.tiled_N_k(64, N)
    a = BE.restate(block, N_k, f, False, mult=m)
    b = BE.restate(block, N_k, f, False, mult=drop)
    s = N_k > 0
    rel = np.max(np.abs((a["S"][s] - b["S"][s]) / a["S"][s]).astype(float))
    assert rel > 1e-6 and rel > 100 * np.max(BE.s_tol(a["S"], a["A"], N)[s] / a["S"][s].astype(float))


def test_chunk_tiles_of_the_large_cases():
    for nT, nc, last in ((131073, 3972, 30), (135168, 4096, 33)):
        assert mm._chunk_tiles(nT, 64) == BE.chunk_tiles(nT, 64) == 33
        N = 32 * (nT - 1) + 19
        assert BE.geometry(N, 64) == (nT, 33, nc, last)
    # the 2048 / K branch below it, and the floor of 4 tiles
    assert mm._chunk_tiles(131072, 64) == 32 and mm._chunk_tiles(10, 64) == 32 and mm._chunk_tiles(10, 1000) == 4


def test_counts():
    c = BE.multinomial_counts(5000, 2, zero=((64, 128),))
    assert c.sum() == 5000 and np.all(c[64:128] == 0)
    nT, ct, nc, _ = BE.geometry(20000, 7)
    s = BE.slot_counts(20000, 7, 1)
    assert nc >= 3 and s.sum() == 20000 and np.all(s[ct * 32:2 * ct * 32] == 0)
    c = BE.all_on_one(BE.UINT16_MAX, 40000)
    assert c.sum() == 65535 and c.max() == 65535
    with pytest.raises(AssertionError):
        BE.all_on_one(65536, 0)


def test_predict_flag_hand_built():
    inf = np.inf
    # 2 states x 3 samples, both sampled; at f = 0 every S_k is near 1
    u = np.array([[0.0, 1.0, 2.0], [0.5, 0.0, 1.0]])
    N_k = np.array([2.0, 1.0])
    assert BE.predict_flag(u, N_k, np.zeros(2), False, True)[0] is False
    # a sample with +inf in every sampled state: NaN
    v = u.copy()
    v[:, 1] = inf
    assert BE.predict_flag(v, N_k, np.zeros(2), False, False) == (True, inf)
    # ... unless it is not drawn
    flag, _ = BE.predict_flag(v, N_k, np.zeros(2), False, False, counts=np.array([2, 0, 1]))
    assert not flag
    # state 1 far above every sample: S_1 ~ e^-700 < 1e-280
    w = u.copy()
    w[1] += 700.0
    flag, margin = BE.predict_flag(w, N_k, np.zeros(2), False, False)
    assert flag and margin > 50
    # the same when every draw falls on samples state 1 does not see
    x = np.array([[0.0, 1.0, 2.0], [0.5, inf, inf]])
    assert BE.predict_flag(x, N_k, np.zeros(2), False, False, counts=np.array([0, 2, 1]))[0]
    assert not BE.predict_flag(x, N_k, np.zeros(2), False, False)[0]
    # an empty third state 800 below: S overflows only with all rows; at 400 below only the Gram does
    for d, s_over in ((800.0, True), (400.0, False)):
        y = np.vstack([u, u[0] - d])
        Nk3 = np.array([2.0, 1.0, 0.0])
        assert BE.predict_flag(y, Nk3, np.zeros(3), False, True)[0] is False
        assert BE.predict_flag(y, Nk3, np.zeros(3), True, False)[0] is s_over
        assert BE.predict_flag(y, Nk3, np.zeros(3), True, True)[0] is True
    # an empty row of +inf only: no flag
    z = np.vstack([u, np.full(3, inf)])
    flag, margin = BE.predict_flag(z, np.array([2.0, 1.0, 0.0]), np.zeros(3), True, True)
    assert not flag and margin > 100


def test_offset_energies_keep_the_answer():
    c = E.with_unsampled(60.0, sign=-1.0)
    for scale in (1e5, 1e8):
        u = BE.offset_energies(c["u"], scale, 3)
        r0 = BE.restate(c["u"], c["N"], c["f_true"], True)
        r1 = BE.restate(u, c["N"], c["f_true"], True)
        # the rounding of u + o moves each entry by up to eps * scale, hence S by about that relative
        np.testing.assert_allclose(r1["S"].astype(float), r0["S"].astype(float), rtol=64 * BE.EPS * scale)
        assert r1["absx"] > 0.9 * scale * u.shape[1]

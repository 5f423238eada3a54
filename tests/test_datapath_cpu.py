"""Checks of the data-path restatements in tests/_datapath.py (no GPU needed)."""
import numpy as np
import pytest

from oracle import mbar_oracle as orc
from oracle import testsystems as ots
from tests import _datapath as D
from tests import _edges as E


def _case(seed=3):
    u, N = ots.oscillators(5, 40, seed=seed)
    N = N.astype(float)
    N[2] = 0.0
    u = u.copy()
    u[2] -= 30.0                         # an unsampled row below the sampled minimum
    u[4, 7] = np.inf
    return u, N


def test_upload_image_matches_edges_shift():
    u, N = _case()
    im = D.upload_image(u, N)
    np.testing.assert_array_equal(im["up"], E.shifted(u, N))
    assert np.all(im["up"][N > 0] >= 0.0)
    assert im["rowmin"][2] == np.floor(E.shifted(u, N)[2].min()) < -29.0
    assert np.all(im["rowmin"][N > 0] == 0.0)
    assert not im["clamped"].any()              # +inf is not a clamped finite energy
    u2 = u.copy()
    u2[2] += 2.0e6
    u2[3, 0] = u2[0, 0] + 999300.0
    u2[1, 5] = u2[0, 5] + 999100.0                # a sampled row; just below the flag
    assert D.upload_image(u2, N)["clamped"].tolist() == [False, False, True, True, False]
    assert D.upload_image(u2, N)["far"].tolist() == [False, False, True, False, False]
    u2[2] = np.inf
    assert D.upload_image(u2, N)["allinf"].tolist() == [False, False, True, False, False]


def test_download_image_is_one_rounding_from_u():
    u, N = _case()
    back = D.download_image(u, N)
    fin = np.isfinite(u)
    x = D.upload_image(u, N)["x"]
    # (u - x) + x differs from u by at most one rounding of each operation
    assert np.all(np.abs(back - u)[fin] <= 2 * D.EPS * (np.abs(u) + np.abs(x))[fin])
    assert np.all(back[~fin] == D.U_CLAMP + x[np.nonzero(~fin)[1]])


def test_passes_on_image_match_raw():
    u, N = _case()
    up = D.upload_image(u, N)["up"]
    f = np.array([0.0, 0.3, -1.0, 0.8, 1.1])
    s = N > 0
    np.testing.assert_allclose(orc.self_consistent_update(up, N, f), orc.self_consistent_update(u, N, f),
                               rtol=0, atol=1e-12)
    np.testing.assert_allclose(orc.mbar_gradient(up[s], N[s], f[s]), orc.mbar_gradient(u[s], N[s], f[s]),
                               rtol=0, atol=1e-12)
    lw_up, lw = orc.mbar_log_W_nk(up, N, f), orc.mbar_log_W_nk(u, N, f)
    fin = np.isfinite(lw)
    np.testing.assert_allclose(lw_up[fin], lw[fin], rtol=0, atol=1e-12)


@pytest.mark.parametrize("K,N,up,down", [(384, 3 * 21824 + 45, 4, 6), (5, 1677696 + 1000, 2, 3)])
def test_chunk_geometry(K, N, up, down):
    assert D.upload_chunks(K, N) == up
    assert D.download_chunks(K, N) == down


def test_chunk_sizes_of_the_gpu_shapes():
    assert D.upload_stage_cols(384, 3 * 21824 + 45) == 21824
    assert D.download_cols(384, 10 ** 6) == 10944
    assert D.logw_rows_per_chunk(384, 10 ** 6) == 21824
    assert D.logw_chunks(384, 3 * 21824 + 45) == 4
    assert D.upload_stage_cols(5, 1677696 + 1000) == 1677696
    assert D.upload_serial_pack(5, 1677696 + 1000, 1) and not D.upload_serial_pack(5, 1677696 + 1000, 0)
    assert D.upload_serial_pack(384, 3 * 21824 + 45, 3) and not D.upload_serial_pack(384, 3 * 21824 + 45, 2)
    assert D.append_cols(200, 10 ** 6) == 20960
    assert D.append_chunks(200, 3 * 20960 + 17) == 4
    # the download slices of the GPU test: one, two and three chunks
    assert [D.download_chunks(384, n) for n in (10944, 10945, 2 * 10944 + 77)] == [1, 2, 3]


def test_philox_known_answers():
    """Random123's known-answer vectors for Philox-4x32-10."""
    z = D.philox4x32_10([0], [0], [0], [0], 0, 0)
    assert [int(v[0]) for v in z] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    m = 0xFFFFFFFF
    f = D.philox4x32_10([m], [m], [m], [m], m, m)
    assert [int(v[0]) for v in f] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    p = D.philox4x32_10([0x243F6A88], [0x85A308D3], [0x13198A2E], [0x03707344], 0xA4093822, 0x299F31D0)
    assert [int(v[0]) for v in p] == [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


def test_cospi():
    """Relative accuracy against long double everywhere, near the zeros included."""
    t = np.concatenate([np.linspace(0.0, 2.0, 100001), 0.5 + np.ldexp(1.0, -np.arange(1, 50)),
                        1.5 - np.ldexp(1.0, -np.arange(1, 50))])
    pi = np.arccos(np.longdouble(-1.0))
    tl = t.astype(np.longdouble)
    tl = np.where(tl > 1, 2 - tl, tl)                 # exact; then cos(pi t) = sin(pi (1/2 - t)), |1/2 - t| <= 1/2
    ref = np.sin(pi * (np.longdouble(0.5) - tl))
    assert np.all(np.abs(D.cospi(t) - ref) <= 2 * D.EPS * np.abs(ref))
    assert D.cospi(np.array([0.5, 1.5]))[0] == 0.0 and D.cospi(np.array([1.0]))[0] == -1.0


@pytest.mark.parametrize("N_k", [[0, 300, 250, 0, 190, 0], [1001], [3, 0, 0, 7, 1, 0, 0, 0, 5]])
def test_synth_blocks(N_k):
    N_k = np.array(N_k, float)
    K, N = len(N_k), int(N_k.sum())
    O, k = np.linspace(1, 5, K), np.linspace(1, 3, K)
    _, aux = D.synth(O, k, N_k, 7, 0, N, N)
    assert np.bincount(aux["state"], minlength=K).tolist() == N_k.astype(int).tolist()
    assert np.all(np.diff(aux["state"]) >= 0)


def test_synth_slice_equals_columns_of_the_whole():
    N_k = np.array([0, 300, 250, 0, 190, 0], float)
    N = int(N_k.sum())
    O, k = np.linspace(1, 5, 6), np.linspace(1, 3, 6)
    whole, _ = D.synth(O, k, N_k, 11, 0, N, N)
    for n0, n in ((0, 299), (299, 2), (37, 500), (N - 33, 33)):
        part, _ = D.synth(O, k, N_k, 11, n0, n, N)
        np.testing.assert_array_equal(part, whole[:, n0:n0 + n])
    other, _ = D.synth(O, k, N_k, 12, 0, N, N)
    assert not np.array_equal(other, whole)


def test_synth_moments_match_the_harmonic_family():
    K, per = 4, 20000
    O, k = np.array([0.0, 1.0, 2.5, -3.0]), np.array([1.0, 4.0, 0.5, 2.0])
    N_k = np.full(K, float(per))
    u, aux = D.synth(O, k, N_k, 5, 0, K * per, K * per)
    x_ref, u_ref, _ = ots.harmonic_u_kn(O, k, N_k.astype(int), seed=5)
    for s in range(K):
        blk = slice(s * per, (s + 1) * per)
        sd = k[s] ** -0.5
        se = sd / np.sqrt(per)
        assert abs(aux["x"][blk].mean() - O[s]) < 5 * se
        assert abs(aux["x"][blk].mean() - x_ref[blk].mean()) < 7 * se
        assert abs(aux["x"][blk].std() / sd - 1.0) < 5 / np.sqrt(2 * per)
        # mean energy of the state in its own samples: 1/2 kT
        assert abs(u[s, blk].mean() - 0.5) < 5 * np.sqrt(0.5 / per)
        assert abs(u[s, blk].mean() - u_ref[s, blk].mean()) < 7 * np.sqrt(0.5 / per)


def test_synth_tolerance_is_tight():
    N_k = np.array([0, 300, 250, 0, 190, 0], float)
    N = int(N_k.sum())
    u, aux = D.synth(np.linspace(1, 5, 6), np.linspace(1, 3, 6), N_k, 11, 0, N, N)
    tol = D.synth_tolerance(aux)
    assert np.all(tol > 0) and np.all(tol <= 1e-12 * (1.0 + np.abs(u)))
    # a sample placed in the neighbouring state is far outside the bound
    assert np.all(np.abs(np.diff(np.linspace(1, 5, 6))) > 1e6 * tol.max())

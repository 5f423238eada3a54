"""mbar_b200_replicate_unsampled on the H100 against the per-replicate path on the same context
(set_sample_weights(c_b) + self_consistent_update(F_b)) and a long-double host restatement, its bit-identity rules and
errors, and MBAR bootstrap replicates through the facade against tests/golden/mbar_bootstrap.npz."""
import numpy as np
import pytest

from tests import _cases
from tests import _mbar_boot as mb

pytestmark = pytest.mark.gpu


def _ld_restatement(u_kn, N_k, counts, F):
    """-log sum_n c_bn exp(-u_jn - L_bn) in long double, every sum with an exact max shift."""
    u = np.asarray(u_kn, dtype=np.longdouble)
    s = np.asarray(N_k) > 0
    out = np.empty((len(counts), int(np.sum(~s))))
    logN = np.log(np.asarray(N_k, dtype=np.longdouble)[s])
    for b in range(len(counts)):
        a = np.asarray(F[b], dtype=np.longdouble)[s, None] + logN[:, None] - u[s]
        m = a.max(axis=0)
        L = m + np.log(np.exp(a - m).sum(axis=0))
        c = np.asarray(counts[b], dtype=np.longdouble)
        for q, j in enumerate(np.flatnonzero(~s)):
            keep = c > 0
            v = -u[j, keep] - L[keep] + np.log(c[keep])
            mv = v.max()
            out[b, q] = np.inf if not np.isfinite(mv) else float(-(mv + np.log(np.exp(v - mv).sum())))
    return out


def _problem(K_s, n_unsampled, N, seed, far=False, inf_row=False):
    from oracle import testsystems as ots
    from pymbar_b200 import DeviceProblem

    rng = np.random.default_rng(seed)
    per = max(1, N // K_s)
    u_kn, N_k = ots.oscillators(K_s, per, seed=seed)
    N_k = N_k.copy()
    N_k[-1] += N - u_kn.shape[1]
    extra = u_kn[rng.integers(0, K_s, n_unsampled)] + rng.normal(0, 0.5, (n_unsampled, u_kn.shape[1]))
    if N > u_kn.shape[1]:
        more = u_kn[:, rng.integers(0, u_kn.shape[1], N - u_kn.shape[1])]
        u_kn = np.hstack([u_kn, more])
        extra = np.hstack([extra, extra[:, rng.integers(0, extra.shape[1], N - extra.shape[1])]])
    u_kn, extra = u_kn[:, :N], extra[:, :N]
    if inf_row:
        extra[0] = np.inf
    if far:
        extra[-1] = u_kn.min(0) + 2.0e6
    u = np.vstack([u_kn, extra])
    Nf = np.concatenate([N_k.astype(float), np.zeros(n_unsampled)])
    return DeviceProblem(u, Nf, device=0), u, Nf


def _replicates(p, Nf, B, seed, zero_tiles=0):
    rng = np.random.default_rng(seed)
    s = Nf > 0
    f0 = p.self_consistent_update(np.zeros(len(Nf)))
    F = np.tile(f0, (B, 1)) + rng.normal(0, 0.05, (B, len(Nf)))
    F[:, ~s] = 0.0
    counts = rng.poisson(1.0, (B, p.N)).astype(np.uint16)
    counts[:, :32 * zero_tiles] = 0
    counts[:, -1] = np.maximum(counts[:, -1], 1)
    return F, counts


def _oracle(p, counts, F):
    s = p.N_k > 0
    out = []
    try:
        for c, f in zip(counts, F):
            p.set_sample_weights(c.astype(np.float64))
            out.append(p.self_consistent_update(f)[~s])
    finally:
        p.set_sample_weights(None)
    return np.array(out)


def _close(got, want):
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin) and np.all(got[~fin] == want[~fin])
    err = np.abs(got[fin] - want[fin]) / np.maximum(1.0, np.abs(want[fin]))
    assert err.size == 0 or err.max() < 1e-12, err.max()


@pytest.mark.parametrize("K_s, n_u, N, B, zero_tiles", [
    (5, 3, 29, 1, 0),          # N < 32, B = 1
    (6, 34, 1000, 11, 3),      # N not a multiple of 32, B not a multiple of the batch, whole tiles of zero counts
    (1, 4, 300, 9, 0),         # one sampled state
    (8, 32, 2049, 8, 0),       # K_total = 40
    (8, 2992, 300, 10, 1),     # K_total = 3000: two rows per thread, several row chunks
])
def test_against_oracle_and_long_double(K_s, n_u, N, B, zero_tiles):
    p, u, Nf = _problem(K_s, n_u, N, seed=K_s + n_u)
    with p:
        F, counts = _replicates(p, Nf, B, seed=N, zero_tiles=zero_tiles)
        got = p.replicate_unsampled(counts, F)
        assert got.shape == (B, n_u)
        _close(got, _oracle(p, counts, F))
        _close(got, _ld_restatement(u, Nf, counts, F))
        st = p.last_replicate_stats()
        assert st["batches"] == (B + 7) // 8 and st["ms"] > 0.0
        chunks = (n_u + (511 if n_u > 256 else 255)) // (512 if n_u > 256 else 256)
        assert st["exps"] == int(np.count_nonzero(counts)) * (K_s * chunks + n_u)
        # bit-identical: row b alone, inside a larger B, and on a repeat call
        again = p.replicate_unsampled(counts, F)
        assert np.array_equal(again, got)
        b = B // 2
        alone = p.replicate_unsampled(counts[b:b + 1], F[b:b + 1])
        assert np.array_equal(alone[0], got[b])


def test_inf_row_and_far_row():
    from pymbar_b200._lib import MbarB200Error

    p, u, Nf = _problem(4, 3, 200, seed=3, inf_row=True)
    with p:
        F, counts = _replicates(p, Nf, 3, seed=1)
        got = p.replicate_unsampled(counts, F)
        assert np.all(got[:, 0] == np.inf) and np.all(np.isfinite(got[:, 1:]))
        _close(got, _oracle(p, counts, F))
    p, u, Nf = _problem(4, 3, 200, seed=4, far=True)
    with p:
        F = np.zeros((2, len(Nf)))
        counts = np.ones((2, p.N), np.uint16)
        with pytest.raises(MbarB200Error) as e1:
            p.self_consistent_update(F[0])
        with pytest.raises(MbarB200Error) as e2:
            p.replicate_unsampled(counts, F)
        assert e1.value.status == e2.value.status == -6
        # the context stays usable, and invalid calls are refused
        counts[1] = 0
        with pytest.raises(MbarB200Error) as e3:
            p.replicate_unsampled(counts, F)
        assert e3.value.status in (-1, -6)


def test_invalid_counts():
    from pymbar_b200._lib import MbarB200Error

    p, u, Nf = _problem(4, 2, 100, seed=5)
    with p:
        F, counts = _replicates(p, Nf, 3, seed=2)
        counts[1] = 0
        with pytest.raises(MbarB200Error) as e:
            p.replicate_unsampled(counts, F)
        assert e.value.status == -1
        counts[1] = 1
        assert np.all(np.isfinite(p.replicate_unsampled(counts, F)))


@pytest.fixture()
def gpu_boot_mbar():
    from pymbar_b200 import facade
    from pymbar_b200 import mbar_solvers as ms

    mb.BootMBAR.solvers = ms
    facade.install_on(mb.BootMBAR)
    yield mb.BootMBAR
    facade.uninstall_from(mb.BootMBAR)
    ms.clear_cache()


@pytest.mark.parametrize("name", ["small_osc_8x40", "small_empty_first", "ref_suite_ho_4"])
def test_facade_against_golden(gpu_boot_mbar, name):
    from pymbar_b200 import facade

    g = mb.golden()
    seed = int(g["seeds"][0])
    NB = int(g["n_bootstraps"])
    z = _cases.load(name)
    s0 = dict(facade.STATS)
    m = gpu_boot_mbar(z["u_kn"], z["N_k"], n_bootstraps=NB, rseed=seed)
    assert facade.STATS["mbar_boot_solves"] == s0["mbar_boot_solves"] + NB
    mb.check_case(m, g, name, seed, rtol_obs=1e-8, rtol_sigma=1e-6, atol_sigma=1e-9, tol_f=1e-8)
    assert facade.STATS["redeemed"] == s0["redeemed"]
    assert facade.STATS["expectations_boot"] == s0["expectations_boot"] + 7
    assert m.rng.random() == g[f"{name}_s{seed}_after"]


def test_construction_uploads_u_kn_once(gpu_boot_mbar):
    from oracle import testsystems as ots
    from pymbar_b200 import facade
    from pymbar_b200 import mbar_solvers as ms

    ms.clear_cache()
    u_kn, N_k = ots.oscillators(16, 2000, seed=9)
    K, N = u_kn.shape
    B = 12
    s0 = dict(facade.STATS)
    m = gpu_boot_mbar(u_kn, N_k, n_bootstraps=B, rseed=3)
    with ms._borrow(m.u_kn, np.asarray(m.N_k, dtype=np.float64)) as p:
        h2d = p.counters()["h2d_bytes"]
    want = 8 * K * N + B * 8 * N
    assert want <= h2d < 1.05 * want + 1_000_000, (h2d, want)
    assert h2d < B * 8 * K * N
    m.compute_expectations_inner(np.arange(N, dtype=float)[None], m.u_kn, np.array([[0, 1], [0, 0]]),
                                 uncertainty_method="bootstrap")
    m.compute_free_energy_differences(uncertainty_method="bootstrap", return_theta=True)
    assert facade.STATS["redeemed"] == s0["redeemed"]

"""CPU checks of tests/_large_k.py (the generic pass's plan, the permuted ladders, the sparse long-double reference)
and of the facade's fall-through for augmented problems the device cannot hold."""
import numpy as np
import pytest

from tests import _large_k as LK
from tests import _moments as M
from tests.test_driver_logic_cpu import OracleProblem, StandInMBAR

# warps per CTA of the generic pass and the K range of each, as DESIGN 3.2 states them
W_TABLE = [(8, 1, 1070), (7, 1071, 1298), (6, 1299, 1602), (5, 1603, 2028), (4, 2029, 2668), (3, 2669, 3733),
           (2, 3734, 5864), (1, 5865, 8192)]


def test_plan_bands_match_the_table():
    assert LK.w_bands() == W_TABLE


def test_plan_fits_for_every_k():
    for K in range(1, LK.K_MAX + 1):
        p = LK.generic_plan(K, 1000)
        assert 1 <= p["W"] <= 8 and p["smem"] <= 200 * 1024, p
        assert (p["ctas_per_sm"] == 2) == (p["smem"] <= 100 * 1024)
    assert LK.generic_plan(270, 32)["ctas_per_sm"] == 2 and LK.generic_plan(271, 32)["ctas_per_sm"] == 1


def test_chosen_ks_straddle_every_w_change():
    ks = LK.generic_ks()
    for W, first, last in W_TABLE:
        assert last in ks, (W, last)
        if first > 1:
            assert first in ks, (W, first)
    assert LK.K_MAX in ks
    assert any(LK.generic_plan(K, 32)["ctas_per_sm"] == 2 for K in ks)


@pytest.mark.parametrize("K", [200, 1070, 2029, 2669, 3734, 5865, 8192])
def test_regimes_reach_their_tile_counts(K):
    few, one, sev = (LK.generic_plan(K, LK.regime_n(K, r)) for r in LK.REGIMES)
    for p in (few, one, sev):
        assert p["N"] % 32 != 0
    assert few["n_tiles"] < few["W"] or (few["W"] <= 2 and few["N"] < 32)
    assert one["tiles_per_warp"] == 1 and one["grid"] == one["max_grid"]
    assert sev["tiles_per_warp"] == 3 and sev["grid"] == sev["max_grid"]


def test_permuted_ladder_shape_and_permutation():
    K = 300
    c = LK.permuted_ladder(K, 2, seed=3, unsampled=(0, 150, 299), n_inf=20)
    assert c["u"].shape == (K, int(c["N"].sum())) and c["mult"].shape == (c["u"].shape[1],)
    assert c["N"][[0, 150, 299]].sum() == 0 and int(c["N"].sum()) % 32 != 0
    assert np.isinf(c["u"]).sum() > 0 and np.any(c["mult"] == 0)
    # neighbours on the ladder are not neighbours in the index order: their 128-blocks differ for most states
    perm = LK.permutation(K, 3)
    blocks = perm.argsort() // 128
    assert np.mean(blocks[:-1] != blocks[1:]) > 0.3
    frac = LK.permuted_ladder(K, 0.5, seed=3)
    assert abs(frac["N"].sum() - K * 0.5) <= 1 and set(np.unique(frac["N"])) <= {0.0, 1.0, 2.0}


CASES = {
    "first": dict(K=40, n_per=3, seed=1, unsampled=(0,)),
    "middle_inf": dict(K=70, n_per=2, seed=2, unsampled=(35,), n_inf=60),
    "last": dict(K=129, n_per=2, seed=4, unsampled=(128,)),
    "three": dict(K=257, n_per=1, seed=5, unsampled=(0, 128, 256)),
}


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("all_rows", [False, True])
@pytest.mark.parametrize("name", list(CASES))
def test_sparse_reference_equals_dense(name, all_rows, weighted):
    c = LK.permuted_ladder(**CASES[name])
    mult = c["mult"] if weighted else None
    S, G, A = M.moments_ld(c["u"], c["N"], c["f"], mult=mult, all_rows=all_rows)
    r = LK.sparse_moments_ld(c["u"], c["N"], c["f"], mult=mult, all_rows=all_rows, want_G=True, chunk=37)
    K = len(c["N"])
    drop = r["drop"]                          # what the cut may drop (below e^-1500: no fp64 sees it)
    assert np.all(np.abs(r["S"] - S) <= 1e-15 * S + drop)
    rows = np.ones(K, bool) if all_rows else c["N"] > 0
    Gs = LK.dense_G(r, K)
    assert np.all(np.abs(Gs - G) <= 1e-15 * G + drop)
    assert np.all(Gs[G > drop] > 0)                 # everything above the bound is on the support
    assert np.all(Gs[~rows] == 0)
    np.testing.assert_array_equal(r["A"], A)
    ref_L = dense_L(c)
    assert np.max(np.abs(r["L"] - ref_L)) < 1e-15 * np.max(np.abs(ref_L)) + 1e-17
    m = np.ones(len(ref_L)) if mult is None else mult
    assert abs(r["sumL"] - (m * ref_L).sum()) <= 1e-15 * np.abs(m * ref_L).sum()
    # the error budget is finite and at least the exp's own bound
    assert np.all(np.isfinite(r["dL"])) and np.all(r["dL"] >= (K + 2) * M.EPS)


def dense_L(c):
    s = c["N"] > 0
    a = (c["f"][s].astype(M.LD) + np.log(c["N"][s].astype(M.LD)))[:, None] - c["u"][s].astype(M.LD)
    top = a.max(axis=0)
    return top + np.log(np.exp(a - top).sum(axis=0))


@pytest.mark.parametrize("cut", [5.0, 20.0])
def test_cut_bound_holds(cut):
    """What the cut drops: at most K e^-cut relative of each D_n, and at most M e^-cut of every N_k S_k and Ghat_ij."""
    c = LK.permuted_ladder(60, 3, seed=9, unsampled=(7,), gaps=(1.0, 2.5))
    K = 60
    full = LK.sparse_moments_ld(c["u"], c["N"], c["f"], mult=c["mult"], all_rows=True, want_G=True, cut=1e9)
    part = LK.sparse_moments_ld(c["u"], c["N"], c["f"], mult=c["mult"], all_rows=True, want_G=True, cut=cut)
    assert part["Gv"].size < full["Gv"].size                        # the cut drops something
    assert np.all(np.abs(part["L"] - full["L"]) <= K * np.exp(-cut))
    Nd = np.where(c["N"] > 0, c["N"], 1.0)
    assert np.all(np.abs(part["S"] - full["S"]) * Nd <= part["drop"])
    dG = np.abs(LK.dense_G(part, K) - LK.dense_G(full, K))
    assert dG.max() <= part["drop"] and dG.max() > 0


def test_pass_tolerances_shapes():
    c = LK.permuted_ladder(50, 3, seed=2, unsampled=(3,))
    N = c["u"].shape[1]
    r = LK.sparse_moments_ld(c["u"], c["N"], c["f"], all_rows=True)
    t = LK.pass_tolerances(r, c["N"], LK.generic_plan(50, N))
    s = c["N"] > 0
    S = r["S"].astype(np.float64)
    assert np.all(t["S"][s] > 0) and np.all(t["S"][~s] == 0)
    # the budget is a small multiple of eps relative: big enough for the kernel's rounding, far below any slip
    assert np.all(t["S"][s] / S[s] < 1e-12) and np.all(t["logS"] < 1e-11)
    assert np.all(t["L"] < 1e-11) and 0 < LK.sumL_tolerance(r, LK.generic_plan(50, N)) < 1e-8 * N


# ---- the facade past the size of a context ----------------------------------------------------------------------
class CappedOracleProblem(OracleProblem):
    """OracleProblem whose augmented problems stop at the library's size limit with ERR_INVALID, as the library's
    create_augmented does."""

    def augmented(self, u_extra):
        from pymbar_b200 import _lib

        u_extra = np.atleast_2d(u_extra)
        if self.K + len(u_extra) > _lib.MAX_STATES:
            raise _lib.MbarB200Error(-1, f"n_extra={len(u_extra)}")
        return super().augmented(u_extra)


class OriginalInnerMBAR(StandInMBAR):
    """StandInMBAR whose own compute_expectations_inner (the original the facade may fall through to) records its
    calls."""

    calls = []

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)

    def compute_expectations_inner(self, A_n, u_ln, state_map, uncertainty_method=None, warning_cutoff=1.0e-10,
                                   return_theta=False):
        type(self).calls.append((np.shape(u_ln), np.shape(state_map)))
        return {"original": True}


@pytest.fixture()
def capped_facade(monkeypatch):
    import pymbar_b200
    from pymbar_b200 import facade
    from pymbar_b200 import mbar_solvers as ours

    monkeypatch.setattr(ours, "DeviceProblem", CappedOracleProblem)
    monkeypatch.setenv("PYMBAR_B200_CACHE", "0")
    monkeypatch.setattr(pymbar_b200._lib, "load", lambda: None)
    OriginalInnerMBAR.solvers = ours
    OriginalInnerMBAR.calls = []
    facade.install_on(OriginalInnerMBAR)
    yield OriginalInnerMBAR
    facade.uninstall_from(OriginalInnerMBAR)
    ours.clear_cache()


def test_expectations_past_the_cap_call_the_original(capped_facade):
    from pymbar_b200 import _lib
    from pymbar_b200 import expectations as ex
    from pymbar_b200 import facade
    from tests import _cases

    z = _cases.load("small_osc_8x40")
    m = capped_facade(z["u_kn"], z["N_k"])
    K, N = m.u_kn.shape
    rng = np.random.RandomState(0)
    s0 = dict(facade.STATS)
    # states of interest plus one observable per state: K + L + L rows
    for L, served in ((5, True), ((_lib.MAX_STATES - K) // 2, True), ((_lib.MAX_STATES - K) // 2 + 1, False)):
        u_ln = m.u_kn[rng.randint(0, K, size=L)] + rng.normal(scale=0.01, size=(L, N))
        table = np.array([np.arange(L), np.zeros(L, int)])
        assert ex.augmented_states(K, table) == K + 2 * L
        r = m.compute_expectations_inner(z["x_n"].copy(), u_ln, table)
        assert ("original" in r) != served, L
    assert facade.STATS["expectations"] == s0["expectations"] + 2
    assert facade.STATS["expectations_fallbacks"] == s0["expectations_fallbacks"] + 1
    assert capped_facade.calls == [((L, N), (2, L))]
    # free energies only: K + L rows
    L = _lib.MAX_STATES - K + 1
    r = m.compute_expectations_inner(np.array([0.0]), np.repeat(m.u_kn[:1], L, axis=0), np.arange(L))
    assert r == {"original": True} and facade.STATS["expectations_fallbacks"] == s0["expectations_fallbacks"] + 2

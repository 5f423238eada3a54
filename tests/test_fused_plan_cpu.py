"""The fused pass's launch plan (tests/_fused.py) without a GPU: the variant matrix reaches all 90 instantiations, the
sample-count regimes give the stage counts they name, a plan worked by hand comes out right, and no CTA reads a state
constant it did not initialise."""
import pytest

from tests import _fused as F


def test_ninety_instantiations_reachable():
    inst = F.instantiations()
    assert len(inst) == 90
    assert not [k for k, ks in inst.items() if not ks]
    # the ids of fused_enqueue: 0..91 less the two unused after the M = 2 table (50, 51)
    ids = set()
    for K, regime, M, mode, content in F.variant_matrix():
        N = F.regime_n(K, regime, M)
        for _, plan in F.case_plans(K, N, M, mode, content):
            if plan is not None:
                ids.add(plan["which"])
    assert ids == set(range(92)) - {50, 51}


@pytest.mark.parametrize("sm_count", [132, 114])
def test_matrix_covers_every_instantiation_in_its_regimes(sm_count):
    rows = F.variant_matrix(sm_count)
    cov = F.matrix_coverage(rows, sm_count)
    inst = F.instantiations()
    missing = [k for k in inst if k not in cov]
    assert not missing, missing
    # MODE 3 in every regime, except where no K of the instantiation has a sample per state in that regime: the
    # FULL weight-storing pass and the FULL two-candidate pass need every state sampled (neither runs all states)
    for k, v in cov.items():
        if k[3] != 3:
            continue
        for regime in set(F.REGIMES) - v:
            R, CL, full, mode, wst, M = k
            assert full and (wst or M == 2), (k, regime)
            assert all(F.regime_n(K, regime, M, sm_count) < K for K in inst[k]), (k, regime)
    # every K of the matrix is reached by its instantiation's K list
    for (K, regime, M, mode, content) in rows:
        for _, plan in F.case_plans(K, F.regime_n(K, regime, M, sm_count), M, mode, content, sm_count):
            if plan is not None:
                assert K in inst[plan["inst"]], (K, plan["inst"])


@pytest.mark.parametrize("sm_count", [132, 114])
@pytest.mark.parametrize("M", [1, 2])
def test_regimes_give_their_stage_counts(sm_count, M):
    for (R, CL, k0, k1) in F.bands(M):
        for K in sorted({k0, k1, (k0 + k1) // 2}):
            for regime in F.REGIMES:
                N = F.regime_n(K, regime, M, sm_count)
                assert N % 32 != 0, (K, regime, N)
                plan = F.fused_plan(K, N, M=M, sm_count=sm_count, m2_clusters=True)
                G = sm_count // plan["CL"]
                if regime == "few":
                    assert plan["n_stages"] < G and plan["groups"] == plan["n_stages"], (K, plan["n_stages"], G)
                elif regime == "one":
                    assert plan["n_stages"] == G and plan["stages_per_group"] == 1, (K, plan["n_stages"])
                else:
                    assert plan["groups"] == G
                    assert plan["n_stages"] // G >= 2 * plan["NS"] + 1, (K, plan["n_stages"], plan["NS"])
                # the samples never fill the last stage
                assert N < 32 * plan["tiles_per_stage"] * plan["n_stages"], (K, regime, N)
                assert plan["grid"] == plan["groups"] * plan["CL"] <= sm_count


def test_hand_worked_plan_k256():
    """DESIGN 3.1: K = 256, N = 1e7 runs 8 warps x 32 states on one CTA per SM (R = 32, FULL, MODE = 3, CL = 1),
    one 64 KB tile per stage in a 3-deep ring."""
    p = F.fused_plan(256, 10 ** 7)
    assert (p["R"], p["full"], p["mode"], p["CL"], p["Wk"], p["Rw"]) == (32, True, 3, 1, 8, 32)
    assert (p["TPW"], p["stageBytes"], p["NS"], p["grid"]) == (1, 65536, 3, 132)
    assert p["name"] == ("pass_fused_kernel<R=32, FULL, CW=8, BATCH=8, MODE=3 (LDS table + multiplicative state "
                         "constant), CL=1> grid=132 NS=3 TPW=1")


def test_plan_declines_where_fused_prepare_does():
    assert F.fused_plan(2049, 1000) is None
    assert F.fused_plan(64, 1000, spread=1200.0) is None
    assert F.fused_plan(64, 1000, spread=700.0)["mode"] == 1
    assert F.fused_plan(129, 1000, M=2) is None                       # clusters only with the switch
    assert F.fused_plan(129, 1000, M=2, m2_clusters=True) is not None
    assert F.fused_plan(64, 1000, M=2, all_states=True) is None
    assert F.fused_plan(64, 1000, M=2, spread=700.0) is None
    assert F.fused_plan(1025, 1000, M=2, m2_clusters=True) is None
    assert F.fused_plan(1, 1000, M=2) is None
    # an all-state pass stores no weights; a weighted pass is MASKED
    assert not F.fused_plan(64, 1000, want_w=True, all_states=True, n_active=63)["wst"]
    assert not F.fused_plan(64, 1000, weighted=True)["full"]
    assert F.fused_plan(64, 1000, all_states=True, n_active=63)["full"]
    assert not F.fused_plan(64, 1000, n_active=63)["full"]


@pytest.mark.parametrize("M", [1, 2])
def test_no_cta_reads_an_uninitialised_state_constant(M):
    """Every CTA zeroes its state constants past Kl far enough for the highest constant any of its warps reads, and
    that stays inside the K + 32 entries fused_smem_header gives c_s (and c_s2).  The zeroing is the one the kernel
    source compiles."""
    pad = F.kernel_zeroing()
    top = 1024 if M == 2 else F.K_MAX
    for K in range(2 if M == 2 else 1, top + 1):
        for read, init in F.constant_reads(K, M, pad=pad):
            assert read <= init, (K, M, read, init)
            assert init < K + 32, (K, M, init)


def test_fixed_32_entry_zeroing_left_reads_uninitialised():
    """The zeroing of a fixed 32 entries past Kl left the last CTA of a cluster reading unset constants at these K."""
    assert F.overrun_ks(1, pad=32) == [1025, 1026, 1027, 1041, 1153, 1537, 1538, 1539, 1553, 1665]
    assert F.overrun_ks(2, pad=32) == [513, 514, 515, 529, 641]
    # K = 1025: CL = 8, Kh = 130, last CTA Kl = 115, Rw = 18, R = 24: warp 7 reads c_s[126..149]
    g = F.geometry(1025)
    assert (g["CL"], g["Kh"], g["Rw"], g["R"]) == (8, 130, 18, 24)
    assert F.constant_reads(1025, pad=32)[-1] == (149, 146)

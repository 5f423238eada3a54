"""The exponent-edge cases of tests/_edges.py really sit in the bands they are built for (no GPU needed).

A case that drifted into the easy middle of the exponent range would let tests/test_gpu_exponent_edges.py
pass without exercising anything; these checks recompute each band from the inputs alone."""
import numpy as np
import pytest

from tests import _edges as E

FLOOR_ARG = -707.7     # exp arguments below this are floored by scale2 (binary exponent < -1021)


@pytest.mark.parametrize("delta", E.A_DELTAS)
@pytest.mark.parametrize("start", E.A_STARTS)
def test_floor_band_pairs(delta, start):
    case = E.offset_pair(delta)
    f = np.array([0.0, start])
    b = E.bands(case["u"], case["N"], f, all_states=False)
    # state 1 is state 0 plus delta: its shifted energies are exactly delta, state 0's exactly 0
    assert np.allclose(b["umin"], [0.0, delta]) and np.allclose(b["umax"], [0.0, delta])
    assert b["spread"] == pytest.approx(start)
    assert b["kernel"] == ("fused" if start < E.FUSED_SPREAD else "generic")
    if start < E.FUSED_SPREAD:
        assert b["mode"] == (3 if start <= E.MULT_SPREAD else 1)
        arg = -delta if b["mode"] == 3 else start / 2 - delta      # exp argument of state 1's entries
        if b["mode"] == 3:
            assert (arg < FLOOR_ARG) == (delta >= 709.0)          # these entries are floored on the device
        else:
            assert (arg < FLOOR_ARG) == (delta == 1100.0 and start == 650.0)
        # the truth S_1 = 2 e^x / (1 + e^x), x = start - delta: tiny, so floored entries could dominate it
        x = start - delta
        assert b["logS"][1] == pytest.approx(x + np.log(2) - np.log1p(np.exp(x)), abs=1e-9)
        if b["answer"] == "fused":
            assert b["logS"][1] > b["logthr"][1]


def test_floor_band_mode1_reaches_the_floor():
    """MBAR_B200_FUSED_MODE=1 with delta = 1100 and start 650: the argument c - mid - u' is below the floor."""
    case = E.offset_pair(1100.0)
    b = E.bands(case["u"], case["N"], np.array([0.0, 650.0]), all_states=False, mode_env=1)
    assert b["kernel"] == "fused" and b["mode"] == 1
    assert 650.0 / 2 - 1100.0 < FLOOR_ARG


@pytest.mark.parametrize("K", E.K_SHAPES)
def test_copies_bands(K):
    case = E.offset_copies(K, 800.0)
    b = E.bands(case["u"], case["N"], np.where(np.arange(K) % 2 == 1, 100.0, 0.0), all_states=False)
    assert np.allclose(b["umin"][1::2], 800.0) and np.allclose(b["umax"][0::2], 0.0)
    assert b["kernel"] == "fused" and b["mode"] == 3 and b["spread"] == pytest.approx(100.0)
    assert b["answer"] == "generic"        # S of the odd states is e^-700: below the floor-aware threshold


@pytest.mark.parametrize("delta", E.B_BELOW)
def test_wrap_band(delta):
    case = E.with_unsampled(delta, -1.0)
    f0 = np.zeros(3)
    b = E.bands(case["u"], case["N"], f0, all_states=True)
    assert b["umin"][2] == pytest.approx(-delta) and b["umax"][2] == pytest.approx(-delta)
    c = np.array([np.log(64), np.log(64), E.LOG_EPS_UNSAMPLED])
    assert b["spread"] == pytest.approx(c.max() - c.min())
    assert b["mode"] == 3
    # MODE=3: the unsampled row's exp argument is -u' = +delta; above 700 the host must not use the fused pass
    assert b["kernel"] == ("generic" if delta > E.WRAP_ARG - 1 else "fused")
    if b["kernel"] == "fused":
        assert b["wrap_arg"] == pytest.approx(np.ceil(delta))


@pytest.mark.parametrize("delta", E.B_ABOVE)
def test_unsampled_above_band(delta):
    case = E.with_unsampled(delta, +1.0)
    b = E.bands(case["u"], case["N"], np.zeros(3), all_states=True)
    assert b["umin"][2] == pytest.approx(delta) and b["kernel"] == "fused"
    assert b["wrap_arg"] <= 0.0
    # S of the unsampled state is about e^(80 - delta): tiny, so the pass is answered by the log-domain kernel
    assert b["answer"] == "generic"


@pytest.mark.parametrize("spread", E.C_SPREADS)
def test_mode_boundaries(spread):
    case = E.spread_pair(spread)
    b = E.bands(case["u"], case["N"], case["f"], all_states=False)
    assert b["spread"] == pytest.approx(spread)
    want = "generic" if spread >= E.FUSED_SPREAD else "fused"
    assert b["kernel"] == want
    if want == "fused":
        assert b["mode"] == (3 if spread <= E.MULT_SPREAD else 1)
        # with mid in the middle of the spread, a sample's D_n is about e^(-spread / 2): 1e-130 .. 1e-261
        assert b["logD_min"] == pytest.approx(-spread / 2 + np.log(2), abs=1e-6)


def test_noisy_variants_stay_in_band():
    p = E.offset_pair(800.0, noisy=True)
    b = E.bands(p["u"], p["N"], np.array([0.0, 100.0]), all_states=False)
    assert b["umin"][1] > 790 and b["kernel"] == "fused" and b["mode"] == 3
    q = E.with_unsampled(2500.0, -1.0, noisy=True)
    b = E.bands(q["u"], q["N"], np.zeros(3), all_states=True)
    assert b["umin"][2] < -2490 and b["kernel"] == "generic"


@pytest.mark.parametrize("spread,answer", [(1149.0, "fused"), (1150.0, "fused"), (1155.0, "generic"),
                                           (1157.0, "generic")])
def test_range_flag_band(spread, answer):
    """D_n = 2 e^(-spread/2) with c centred on mid: within a factor 10 of 1e-250, on the side the answer says."""
    case = E.spread_pair(spread)
    b = E.bands(case["u"], case["N"], case["f"], all_states=False)
    assert b["logD_min"] == pytest.approx(-spread / 2 + np.log(2), abs=1e-6)
    assert abs(b["logD_min"] - np.log(1e-250)) < np.log(10.0)
    assert b["mode"] == 1 and b["answer"] == answer
    assert (b["logD_min"] > np.log(1e-250)) == (answer == "fused")


def test_fused_band_next_to_spread_limit():
    case = E.offset_pair(1144.9)
    b = E.bands(case["u"], case["N"], np.array([0.0, 1199.9]), all_states=False)
    assert b["mode"] == 1 and b["answer"] == "fused" and b["margin"] > 10
    assert E.bands(case["u"], case["N"], np.array([0.0, 1200.1]), all_states=False)["kernel"] == "generic"


@pytest.mark.parametrize("delta", [d for d in E.B_BELOW if d <= 1000.0])
def test_wrap_band_fused_at_the_answer(delta):
    """At f_true the all-state pass of an empty copy u_0 - delta is the fused kernel's (MODE=1 above ~520)."""
    case = E.with_unsampled(delta, -1.0)
    b = E.bands(case["u"], case["N"], case["f_true"], all_states=True)
    assert b["answer"] == "fused" and b["margin"] > 1 and b["wrap_arg"] < E.WRAP_ARG

"""CPU checks of tests/_adaptive.py, the restatement the device-resident adaptive loop is held to: in fp64 it walks the
oracle's adaptive() step for step; a numpy model of newton_kernel's arithmetic passes its backward-error bound at
every Newton size the GPU tests run, and fails it under each of four small faults of that arithmetic."""
import numpy as np
import pytest

from oracle import mbar_oracle as orc
from tests import _adaptive as AD
from tests import _cases
from tests import _moments as M

# Newton sizes n = sampled states - 1: both sides of the shared-memory limit (n <= 158) and of the CTA-size bands
# (256 threads below 32, 512 below 96), K <= 128 (one candidate-batched pass) and the L2-resident kernel up to 2047
SHAPES = (1, 2, 31, 32, 95, 96, 157, 158, 159, 160, 255, 511, 1023, 1024, 2047)


@pytest.mark.parametrize("min_sc_iter", [0, 2])
@pytest.mark.parametrize("name", _cases.SMALL + ["osc_50x100", "golden_example"])
def test_fp64_restatement_walks_the_oracle(name, min_sc_iter):
    """Same choices, same iterates and the same iteration count as oracle.adaptive on the sampled states, wherever
    the choice and the stop rule are decided above rounding level."""
    z = _cases.load(name)
    u, N = z["u_kn"], z["N_k"].astype(float)
    s = N > 0
    ref = orc.adaptive(u[s], N[s], np.zeros(int(s.sum())), tol=1e-12,
                       options=dict(min_sc_iter=min_sc_iter, maxiter=200))
    f = np.zeros(len(N))
    choices, decided, sci = [], [], 0
    noise = (1e-12 * N.sum()) ** 2        # squared gradient norms at rounding level: the choice is a coin toss
    for _ in range(200):
        it = AD.iteration(u, N, f, tol=1e-12, min_sc_iter=min_sc_iter, sci_done=sci, precision="fp64")
        choices.append(it["choice"])
        hi = max(it["gn_sci"], it["gn_nr"])
        decided.append(sci < min_sc_iter or (hi > noise and abs(it["gn_sci"] - it["gn_nr"]) > 0.5 * hi))
        sci += it["choice"] == "sci"
        assert np.all(it["f_new"][~s] == f[~s])          # unsampled states are carried through
        f = it["f_new"]
        if it["stop"]:
            break
    # the stop rule at rounding level may take one step more or less
    assert abs(len(choices) - len(ref["history"])) <= 1
    assert all(c == r for c, r, d in zip(choices, ref["history"], decided) if d)
    assert sum(decided) >= len(choices) - 2      # (Newton: the last two steps sit at rounding level)
    assert ref["success"] and it["stop"]
    np.testing.assert_allclose(f[s], ref["x"], rtol=0, atol=1e-10)


@pytest.mark.parametrize("n", SHAPES)
def test_newton_model_passes_backward_bound(n):
    """newton_kernel's arithmetic (left-looking, quad-split dot products, the kernel's solve order) in numpy on an
    MBAR-like system: its step satisfies the backward-error bound the device is held to, with the fp64 rounding
    of A and g as the input error."""
    T, A64, g, active = AD.synthetic_system(n, seed=n)
    rng = np.random.RandomState(n)
    f = rng.normal(scale=3.0, size=n + 1)
    f[0] = 0.0
    gamma = 0.5
    f_nr = AD.newton_model(A64, g, active, f, gamma)
    assert f_nr is not None
    x = AD.recover_step(f, f_nr, active[1:], gamma)
    normA = float(AD.row_abs_sums(T).max())
    ratio, res, bound = AD.backward_ratio(T, g[1:], x, f, f_nr, gamma, dA=AD.EPS * normA,
                                          dg=AD.EPS * float(np.abs(g).max()))
    assert ratio <= 1.0, (n, ratio, res, bound)
    # the bound is not vacuous: the step solves the system to far better than its own size
    assert bound < 1e-9 * normA * float(np.abs(x).max())


@pytest.mark.parametrize("fault", AD.FAULTS)
@pytest.mark.parametrize("n", [31, 160])
def test_newton_model_faults_fail_backward_bound(n, fault):
    """Each fault costs a Newton step only accuracy, never convergence of the loop, and is caught here."""
    T, A64, g, active = AD.synthetic_system(n, seed=n)
    rng = np.random.RandomState(n)
    f = rng.normal(scale=3.0, size=n + 1)
    f[0] = 0.0
    f_nr = AD.newton_model(A64, g, active, f, 0.5, fault=fault)
    if f_nr is None:          # a fault may make the factorisation fail outright: caught as well
        return
    x = AD.recover_step(f, f_nr, active[1:], 0.5)
    normA = float(AD.row_abs_sums(T).max())
    ratio, _, _ = AD.backward_ratio(T, g[1:], x, f, f_nr, 0.5, dA=AD.EPS * normA, dg=AD.EPS * float(np.abs(g).max()))
    assert ratio > 10.0, (fault, ratio)


@pytest.mark.parametrize("K, unsampled, mult", [(6, (0,), False), (40, (3, 20, 39), True)])
def test_fp64_step_lies_within_the_long_double_bounds(K, unsampled, mult):
    """The bounds are not tighter than an honest fp64 computation: the oracle-style fp64 candidates of one
    iteration fall inside the long-double iteration's bounds (self-consistent candidate, Newton backward error)."""
    case = M.ladder(K, 30, gaps=(1.5,), unsampled=unsampled, seed=K, f_noise=0.5)
    u, N, f = case["u"], case["N"], case["f"].copy()
    s = N > 0
    f -= f[np.flatnonzero(s)[0]]
    f[~s] = 0.0
    m = case["mult"] if mult else None
    it = AD.iteration(u, N, f, gamma=0.5, mult=m)
    if m is None:
        it64 = AD.iteration(u, N, f, gamma=0.5, precision="fp64")
        d = np.abs(it64["f_sci"] - it["f_sci"].astype(np.float64))
        assert np.all(d[s] <= it["tol_fsci"][s]), (d[s] / it["tol_fsci"][s]).max()
        ratio, _, _ = AD.newton_backward(it, f, it64["f_nr"], 0.5)
        assert ratio <= 1.0, ratio
    # the long-double candidate itself, rounded to fp64, passes its own check
    ratio, _, _ = AD.newton_backward(it, f, it["f_nr"].astype(np.float64), 0.5)
    assert ratio <= 1e-2, ratio
    assert it["inv_norm"] > 0 and np.isfinite(it["inv_norm"])

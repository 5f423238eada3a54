"""Inputs at the edges of the fp64 exponent range, with the band each one claims to be in.

Every case is built from a state that is a constant offset of another: a sampled copy u_0 + D has f = D, an
empty or appended copy u_0 - D has f = -D against state 0, so the answer is known without a solver.  One noisy
variant per family checks that the exact structure is not special.

`bands()` restates, in numpy, what the host decides for one pass of the library (`fused_applicable`,
`fused_prepare` and the checks on the pass's results in pass_fused.cu / api.cu):
  * the spread of c = f + log N over the states that enter the pass, the centring `mid`;
  * the minimum and maximum shifted energy u'_kn = u_kn - min_{sampled j} u_jn of every row;
  * the kernel and mode the host launches (fused MODE=3, fused MODE=1 or generic);
  * which kernel answers: the fused pass's result is discarded when a denominator leaves [1e-250, 1e250], when
    a state's S_k lies below the floor-aware underflow threshold, or when an unsampled state's S leaves
    (1e-250, 1e12).
tests/test_edges_cpu.py recomputes these from the inputs; tests/test_gpu_exponent_edges.py asserts them
against the device.
"""
import numpy as np
from scipy.special import logsumexp

from oracle import testsystems as ots

LOG_EPS_UNSAMPLED = -80.0
FUSED_SPREAD = 1200.0
MULT_SPREAD = 600.0
WRAP_ARG = 700.0           # largest exp argument an unsampled row may present to the fused pass
U_CLAMP = 1.0e6
# a raw sum sum_n e_kn / D_n below 2^53 * N * 2^-1020 * e^(mid - c_min), c_min over the sampled states, may be made
# of floored entries (pass_fused.cu)
LOG_FLOOR = -967.0 * np.log(2.0)

A_DELTAS = (650.0, 705.0, 709.0, 712.0, 750.0, 800.0, 1100.0)
A_STARTS = (0.0, 30.0, 70.0, 100.0, 300.0, 590.0, 650.0, 1150.0)
B_BELOW = (300.0, 650.0, 705.0, 709.5, 710.0, 712.0, 720.0, 800.0, 1000.0, 1500.0, 2500.0, 5000.0, 2e4, 9.9e4,
           1.01e5)
B_ABOVE = (700.0, 712.0, 800.0, 1500.0, 5000.0, 2e4, 1.01e5, 9e5)
C_SPREADS = (599.9, 600.1, 1199.9, 1200.1)
K_SHAPES = (64, 96, 300, 1100)


def base_samples(n, seed):
    """Energies of n samples of one harmonic state (oracle/testsystems.py, fixed seed)."""
    _, u, _ = ots.harmonic_u_kn([1.0], [2.0], [n], seed=seed)
    return u[0]


def offset_pair(delta, n=64, noisy=False, seed=11):
    """K = 2, both sampled: u_1 = u_0 + delta.  f = (0, delta) unless noisy."""
    u0 = base_samples(2 * n, seed)
    u1 = u0 + delta
    if noisy:
        u1 = u1 + 0.3 * np.random.RandomState(seed + 1).normal(size=u0.size)
    return dict(u=np.stack([u0, u1]), N=np.array([n, n], float), f_true=None if noisy else np.array([0.0, delta]))


def offset_copies(K, delta, n_per=4, seed=13):
    """K copies of one state, every odd one offset by delta, all sampled: f_k = delta * (k odd)."""
    u0 = base_samples(K * n_per, seed)
    off = np.where(np.arange(K) % 2 == 1, delta, 0.0)
    return dict(u=u0[None, :] + off[:, None], N=np.full(K, float(n_per)), f_true=off.copy())


def with_unsampled(delta, sign=-1.0, n=64, noisy=False, seed=17):
    """Two sampled states (u_0, u_0 + 5) and one empty state u_0 + sign * delta: f = (0, 5, sign * delta)."""
    u0 = base_samples(2 * n, seed)
    extra = u0 + sign * delta
    if noisy:
        extra = extra + 0.3 * np.random.RandomState(seed + 1).normal(size=u0.size)
    u = np.stack([u0, u0 + 5.0, extra])
    return dict(u=u, N=np.array([n, n, 0.0]), f_true=None if noisy else np.array([0.0, 5.0, sign * delta]))


def spread_pair(spread, n=64, seed=19):
    """K = 2 at f = (0, spread): c has exactly that spread; u_1 = u_0 + spread keeps S near 1."""
    case = offset_pair(spread, n=n, seed=seed)
    case["f"] = np.array([0.0, spread])
    return case


def shifted(u, N):
    """u'_kn = min(u_kn - min_{sampled j} u_jn, 1e6), as uploaded."""
    x = u[N > 0].min(axis=0)
    return np.minimum(u - x, U_CLAMP)


def bands(u, N, f, all_states, mode_env=None):
    """What the host does with one pass at f (see the module docstring)."""
    u, N, f = np.asarray(u, float), np.asarray(N, float), np.asarray(f, float)
    s = N > 0
    K = len(N)
    all_states = bool(all_states) and not s.all()
    rows = np.ones(K, bool) if all_states else s
    with np.errstate(divide="ignore"):
        logNeff = np.where(s, np.log(np.where(s, N, 1.0)), LOG_EPS_UNSAMPLED)
    c = f + logNeff
    up = shifted(u, N)
    out = dict(spread=float(c[rows].max() - c[rows].min()), umin=up.min(axis=1), umax=up.max(axis=1))
    lo, hi = c[rows].min(), c[rows].max()
    mid = 0.5 * (lo + hi)
    out["mid"] = mid
    if K > 2048 or hi - lo >= FUSED_SPREAD or max(abs(lo), abs(hi)) > 1e6:
        out.update(kernel="generic", mode=None, answer="generic", reason="spread")
        return out
    mode = 3 if mode_env is None else (int(mode_env) & 3) | 1
    if hi - lo > MULT_SPREAD:
        mode = 1
    out["mode"] = mode
    cp = c - mid
    if all_states:
        # largest exp argument of an unsampled row in the chosen mode (the host rounds the row minimum down)
        arg = (cp if mode == 1 else 0.0) - np.minimum(np.floor(out["umin"]), 0.0)
        out["wrap_arg"] = float(arg[~s].max())
        if out["wrap_arg"] > WRAP_ARG:
            out.update(kernel="generic", answer="generic", reason="wrap")
            return out
    out["kernel"] = "fused"
    logD = logsumexp(cp[rows, None] - up[rows], axis=0)
    logS = logsumexp(cp[:, None] - up - logD[None, :], axis=1) - logNeff
    cmin = cp[s].min()          # D_n >= e^(c_min - mid) over the sampled states
    logthr = LOG_FLOOR + np.log(N.sum()) - logNeff - cmin + (cp if mode == 3 else 0.0)
    out.update(logD_min=float(logD.min()), logD_max=float(logD.max()), logS=logS, logthr=logthr)
    margin = [np.log(1e250) - logD.max(), logD.min() - np.log(1e-250)]
    margin.append(np.min((logS - logthr)[rows]))
    margin.append(np.min(logS[s]) - np.log(1e-280))
    if all_states:
        margin += [np.min(logS[~s]) - np.log(1e-250), np.log(1e12) - np.max(logS[~s])]
    out["margin"] = float(min(margin))
    out["answer"] = "fused" if out["margin"] > 0 else "generic"
    out["reason"] = None if out["margin"] > 0 else "checks"
    return out

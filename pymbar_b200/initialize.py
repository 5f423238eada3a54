"""Initial guess for the MBAR solve from pairwise BAR (SURVEY.md 8f row N4; MBAR(initialize="BAR"),
mbar.py:1936-1988).

For consecutive sampled states k -> l the reference collects the forward work of the samples drawn from k and
the reverse work of the samples drawn from l with boolean masks over all N samples per pair and calls
`pymbar.other_estimators.bar` (bisection to a relative tolerance of 1e-5).  Here the samples are grouped by
state of origin once, the work vectors are plain slices, and Bennett's implicit equation

    sum_F 1 / (1 + T_F/T_R exp(w_F - dF))  =  sum_R 1 / (1 + T_R/T_F exp(w_R + dF))

(monotone in dF) is bracketed by the two one-sided exponential averages and solved with Brent's method to the
same 1e-5 relative tolerance.  The result only seeds the solver: the converged f_k does not depend on it.
"""
from __future__ import annotations

import logging

import numpy as np
import scipy.optimize
from scipy.special import logsumexp

logger = logging.getLogger(__name__)


def _log_fermi_sum(x):
    """log sum_i 1 / (1 + exp(x_i)), stable for any sign of x."""
    return logsumexp(-np.logaddexp(0.0, x))


def bar_delta_f(w_F, w_R, guess=0.0, rtol=1.0e-5, maxiter=100):
    """Bennett acceptance ratio estimate of the free energy difference from forward / reverse work values."""
    w_F = np.asarray(w_F, dtype=np.float64)
    w_R = np.asarray(w_R, dtype=np.float64)
    M = np.log(len(w_F) / len(w_R))

    def imbalance(dF):
        return _log_fermi_sum(M + w_F - dF) - _log_fermi_sum(-M + w_R + dF)

    # one-sided exponential averages bound the root from both sides (Jensen)
    hi = -(logsumexp(-w_F) - np.log(len(w_F)))
    lo = logsumexp(-w_R) - np.log(len(w_R))
    if lo > hi:
        lo, hi = hi, lo
    pad = 1.0e-6 + 1.0e-9 * max(abs(lo), abs(hi))
    lo, hi = lo - pad, hi + pad
    flo, fhi = imbalance(lo), imbalance(hi)
    grow = 1.0
    for _ in range(60):                       # widen until the sign changes (never needed for finite data)
        if flo * fhi <= 0.0:
            break
        lo, hi = lo - grow, hi + grow
        flo, fhi = imbalance(lo), imbalance(hi)
        grow *= 2.0
    else:
        raise RuntimeError("BAR: could not bracket the root")
    if flo == 0.0:
        return lo
    if fhi == 0.0:
        return hi
    return scipy.optimize.brentq(imbalance, lo, hi, xtol=1e-14, rtol=max(rtol, 4 * np.finfo(float).eps),
                                 maxiter=maxiter, disp=False)


def initialize_with_bar(u_kn, N_k, x_kindices, f_k_init=None, columns=None):
    """f_k seeded by BAR along the chain of sampled states (mbar.py:1936-1988).  `x_kindices[n]` is the state
    sample n was drawn from (mbar.py:264-268).

    `columns` [N] (a bootstrap replicate's rints) makes it BAR on the gathered u_kn[:, columns] without the gather:
    position p keeps its label x_kindices[p] and reads the energies of sample columns[p], and only the two rows of each
    adjacent pair are read at those columns (what mbar.py:436 and :1957-1960 compute on the gathered matrix)."""
    u_kn = np.asarray(u_kn)
    N_k = np.asarray(N_k)
    K = len(N_k)
    f = np.zeros(K) if f_k_init is None else np.array(f_k_init, dtype=np.float64)
    start = f.copy()
    order = np.flatnonzero(N_k > 0)
    # group the sample indices by state of origin once (stable: keeps the order inside each state)
    idx = np.argsort(np.asarray(x_kindices), kind="stable")
    counts = np.bincount(np.asarray(x_kindices, dtype=np.int64), minlength=K)
    first = np.concatenate([[0], np.cumsum(counts)])
    members = lambda k: idx[first[k]:first[k + 1]]           # noqa: E731
    for k, l in zip(order[:-1], order[1:]):
        nk, nl = members(k), members(l)
        if columns is not None:
            nk, nl = np.asarray(columns)[nk], np.asarray(columns)[nl]
        if len(nk) == 0 or len(nl) == 0:
            f[l] = 0.0
            continue
        w_F = u_kn[l, nk] - u_kn[k, nk]
        w_R = u_kn[k, nl] - u_kn[l, nl]
        try:
            f[l] = f[k] + bar_delta_f(w_F, w_R, guess=start[l] - start[k])
        except (RuntimeError, ValueError):
            logger.warning("WARNING: BAR did not converge to within tolerance")
            f[l] = f[k]
    return f

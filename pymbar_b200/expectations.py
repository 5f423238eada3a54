"""Expectations and perturbed free energies without the N x K weight matrix (SURVEY.md 8f, row N2).

pymbar computes <A> and the free energies of new states by appending columns to the host-resident
``Log_W_nk`` (mbar.py:886-940): one column per new state l (energies u_ln) and one per observable
(log A_n added to that state's log-weights), then takes the asymptotic covariance of the augmented
N x (K + NL + S) matrix.  Every appended column is an *unsampled state* of an augmented MBAR problem:

    new state l            energies  u_ln
    observable i at state l  energies  u_ln - log(A_in - A_min_i + logfactor_i)

so the existing kernels do all of it: the all-state self-consistent update returns the appended states'
free energies (``log_C_a`` / ``f_k[sa]`` of mbar.py:924-940) and ``weight_moments`` returns the
(K + NL + S)^2 second moments that Theta needs.  The K x K algebra on top is the reference's.
"""
from __future__ import annotations

import numpy as np

from . import estimators as est
from .utils import ParameterError


def _as_rows(a):
    a = np.array(a, dtype=np.float64)
    return a.reshape(1, -1) if a.ndim == 1 else a


def _appended(state_map):
    """(of_state, of_obs, wanted_states) of a state map: the u_ln row and the observable of every (state, observable)
    pair, and the distinct states of interest.  The augmented problem appends one row per wanted state and one per
    pair."""
    table = np.asarray(state_map)
    if table.ndim >= 2:
        of_state, of_obs = table[0].astype(int), table[1].astype(int)
    else:
        of_state, of_obs = table.astype(int), np.zeros(0, dtype=int)
    return of_state, of_obs, np.unique(of_state)


def augmented_states(K, state_map):
    """K plus the rows expectations_inner appends for `state_map`.  A context holds at most `_lib.MAX_STATES`
    states."""
    _, of_obs, wanted = _appended(state_map)
    return int(K) + len(wanted) + len(of_obs)


def augmentation(K, A_n, u_ln, state_map):
    """The rows expectations_inner appends to a problem with K states: a dict with `extra` [E, N] (the states of
    interest, then one row per (state, observable) pair), `rows_l` and `rows_s` (each pair's state row and its own row
    in the augmented problem) and `shift` (each pair's observable floor, given back at the end)."""
    energies = _as_rows(u_ln)
    obs = _as_rows(A_n)
    of_state, of_obs, wanted_states = _appended(state_map)     # wanted: rows of u_ln that become appended states
    n_pairs = len(of_obs)
    n_states = len(wanted_states)

    # observables must be positive to live in the exponent: shift each one used by its minimum (plus a guard
    # of a few ulp so the smallest value does not become log 0), and give the shift back at the end
    guard = 4.0 * np.finfo(np.float64).eps
    floor = {}
    for i in np.unique(of_obs):
        lo = obs[i].min()
        floor[i] = lo - abs(guard * lo)
    # appended rows: the states of interest, then one row per (state, observable) pair whose "energy" is
    # u_l - log(A_i - floor_i): its unsampled-state free energy is -log sum_n (A_i - floor_i) e^{-u_l} / D_n
    extra = np.empty((n_states + n_pairs, energies.shape[1]))
    for pos, l in enumerate(wanted_states):
        extra[pos] = energies[l]
    with np.errstate(divide="ignore"):
        for s in range(n_pairs):
            extra[n_states + s] = energies[of_state[s]] - np.log(obs[of_obs[s]] - floor[of_obs[s]])
    row_of_state = {int(l): K + pos for pos, l in enumerate(wanted_states)}
    rows_l = np.array([row_of_state[int(l)] for l in of_state], dtype=int)
    rows_s = K + n_states + np.arange(n_pairs)
    return dict(extra=extra, rows_l=rows_l, rows_s=rows_s, shift=np.array([floor[i] for i in of_obs]))


def finish(plan, f_aug, G, N_aug, uncertainty_method=None, return_theta=False):
    """The keys 'observables', 'f', 'Theta' and 'Amin' of expectations_inner from the augmented problem's free
    energies f_aug and, with return_theta, its Gram G = W^T W (N_aug: the augmented N_k, zeros on appended rows)."""
    rows_l, rows_s, shift = plan["rows_l"], plan["rows_s"], plan["shift"]
    n_pairs = len(rows_s)
    out = {}
    if n_pairs:
        out["observables"] = np.exp(f_aug[rows_l] - f_aug[rows_s]) + shift      # mbar.py:943-953
    out["f"] = f_aug[rows_l]
    if return_theta:
        Theta = est.asymptotic_covariance(G, N_aug, method=uncertainty_method)
        pick = np.concatenate([rows_s, rows_l]).astype(int)        # observables first, then their states
        out["Theta"] = Theta[np.ix_(pick, pick)]
        if n_pairs:
            out["Amin"] = shift
    return out


def expectations_inner(u_kn, N_k, f_k, A_n, u_ln, state_map, uncertainty_method=None, return_theta=False,
                       device=0, problem=None, replicates=None):
    """MBAR.compute_expectations_inner (mbar.py:766-1012).

    Same contract as the reference: A_n [I, N] observables, u_ln [L, N] energies of the states of interest,
    state_map either a 1-D list of states (free energies only) or a [2, S] table whose columns are
    (row of u_ln, row of A_n).  Returns the keys 'observables', 'f', 'Theta', 'Amin'.

    The appended rows (`augmentation`) form an augmented problem on top of the RESIDENT u_kn
    (`DeviceProblem.augmented`): only those rows are uploaded.  `problem` may name the resident DeviceProblem of
    (u_kn, N_k); otherwise the residency cache of `mbar_solvers` provides it.  `finish` turns the augmented free
    energies and Gram into the result; `mbar_many.MbarMany` runs the same two host steps around its batched pass.

    `replicates` = (F [B, K], counts [B, N]) adds the bootstrap keys of mbar.py:962-971: replicate b is the samples
    drawn counts[b, n] times with free energies F[b] (MBAR.f_k_boots[b]).  One `replicate_unsampled` call on the same
    augmented problem gives every replicate's appended rows, from which 'bootstrapped_observables' [B, S] and
    'bootstrapped_f' [B, len(state_list)] follow as for b = 0.  Theta stays the svd-ew one of b = 0, as the reference
    computes it for uncertainty_method="bootstrap" (mbar.py:1796)."""
    from . import mbar_solvers as ms

    u_kn = np.asarray(u_kn)
    f_k = np.asarray(f_k, dtype=np.float64)
    K = u_kn.shape[0]
    plan = augmentation(K, A_n, u_ln, state_map)
    extra = plan["extra"]
    n_extra = extra.shape[0]

    f_aug = np.concatenate([f_k, np.zeros(n_extra)])
    N_aug = np.concatenate([np.asarray(N_k, dtype=np.float64), np.zeros(n_extra)])

    boot = {}

    def run(base):
        with base.augmented(extra) as q:
            f_new = q.self_consistent_update(f_aug)        # appended rows: -logsumexp_n(-v_an - L_n)
            f_aug[K:] = f_new[K:]
            if replicates is not None:
                F, counts = replicates
                F = np.asarray(F, dtype=np.float64)
                F_aug = np.concatenate([F, np.zeros((F.shape[0], n_extra))], axis=1)
                # the appended rows are the last unsampled states of the augmented problem
                F_aug[:, K:] = q.replicate_unsampled(counts, F_aug)[:, -n_extra:]
                boot["f"] = F_aug
            return q.weight_moments(f_aug)[1] if return_theta else None

    if problem is not None:
        G = run(problem)
    else:
        with ms._borrow(u_kn, N_aug[:K]) as base:
            G = run(base)

    out = finish(plan, f_aug, G, N_aug, uncertainty_method=uncertainty_method, return_theta=return_theta)
    if replicates is not None:
        out.update(bootstrap_keys(plan, boot["f"]))
    return out


def bootstrap_keys(plan, F_aug):
    """'bootstrapped_observables' [B, S] and 'bootstrapped_f' [B, len(state_list)] of expectations_inner from every
    replicate's augmented free energies F_aug [B, K + E] (mbar.py:962-971)."""
    rows_l, rows_s, shift = plan["rows_l"], plan["rows_s"], plan["shift"]
    obs_b = np.exp(F_aug[:, rows_l] - F_aug[:, rows_s]) + shift if len(rows_s) else np.zeros((len(F_aug), 0))
    return {"bootstrapped_observables": obs_b, "bootstrapped_f": F_aug[:, rows_l]}


def std_of_differences(X):
    """The standard deviation over replicates b of X_b - X_b^T, [i, j] = X_bj - X_bi, for X [B, K]: the bootstrap
    uncertainty of a difference matrix (mbar.py:706-714, :1298-1303, :1623-1643)."""
    X = np.asarray(X)
    return np.std(X[:, None, :] - X[:, :, None], axis=0)


def expectation_state_map(Ks, state_dependent):
    """The state map of compute_expectations with Ks states of interest (mbar.py:1262-1272)."""
    state_map = np.zeros((2, Ks), int)
    state_map[0] = np.arange(Ks)
    state_map[1] = np.arange(Ks) if state_dependent else 0
    return state_map


def expectations_result(inner, Ks, output, compute_uncertainty, return_theta, warning_cutoff,
                        uncertainty_method=None):
    """compute_expectations' result from expectations_inner's (mbar.py:1274-1312).  uncertainty_method="bootstrap":
    sigma from inner's 'bootstrapped_observables', and Theta (return_theta) is still the b = 0 one."""
    out = {}
    boot = uncertainty_method == "bootstrap"
    if (compute_uncertainty and not boot) or return_theta:
        diag = np.ones(2 * Ks)
        diag[:Ks] = diag[Ks:] = inner["observables"] - inner["Amin"]
        Theta = np.diag(diag) @ inner["Theta"] @ np.diag(diag)
        covA = Theta[:Ks, :Ks] + Theta[Ks:, Ks:] - Theta[:Ks, Ks:] - Theta[Ks:, :Ks]
    if output == "averages":
        out["mu"] = inner["observables"]
        if compute_uncertainty and boot:
            out["sigma"] = np.std(inner["bootstrapped_observables"], axis=0)
        elif compute_uncertainty:
            out["sigma"] = np.sqrt(covA.diagonal())
    elif output == "differences":
        A = inner["observables"]
        out["mu"] = A - np.vstack(A)
        if compute_uncertainty and boot:
            out["sigma"] = std_of_differences(inner["bootstrapped_observables"])
        elif compute_uncertainty:
            out["sigma"] = est.error_of_differences(covA, warning_cutoff=warning_cutoff)
    else:
        raise ParameterError(f"output={output!r} must be 'averages' or 'differences'")
    if return_theta:
        out["Theta"] = Theta
    return out


def perturbed_result(inner, compute_uncertainty, warning_cutoff, uncertainty_method=None):
    """compute_perturbed_free_energies' result from expectations_inner's (mbar.py:1505-1521).  uncertainty_method=
    "bootstrap": dDelta_f is the standard deviation over replicates of inner's 'bootstrapped_f', a vector [L] as the
    reference returns it, not the [L, L] matrix of the analytic methods."""
    f = inner["f"]
    out = {"Delta_f": f - np.vstack(f)}
    if compute_uncertainty and uncertainty_method == "bootstrap":
        out["dDelta_f"] = np.std(inner["bootstrapped_f"], axis=0)
    elif compute_uncertainty:
        out["dDelta_f"] = est.error_of_differences(inner["Theta"], warning_cutoff=warning_cutoff)
    return out


def entropy_enthalpy_result(inner, K, warning_cutoff=1.0e-10, f_k_boots=None):
    """compute_entropy_and_enthalpy's result (mbar.py:1600-1681) from expectations_inner's with A_n = u_ln = u_kn and
    the state map (k, k).  Analytic uncertainties: the reference's 3K x 3K Theta, whose last K rows and columns
    repeat the states' block, scaled by the observables.  Bootstrap (f_k_boots [B, K], the problem's replicates): the
    reference's branch of :1623-1643, dDelta_f from f_k_boots, dDelta_u from inner's 'bootstrapped_observables' and
    dDelta_s from their difference; inner needs no Theta."""
    out = {}
    f_k = inner["f"]
    out["Delta_f"] = f_k - np.vstack(f_k)
    u_k = inner["observables"]
    out["Delta_u"] = u_k - np.vstack(u_k)
    s_k = u_k - f_k
    out["Delta_s"] = s_k - np.vstack(s_k)
    if f_k_boots is not None:
        u_b = inner["bootstrapped_observables"]
        out["dDelta_f"] = std_of_differences(f_k_boots)
        out["dDelta_u"] = std_of_differences(u_b)
        out["dDelta_s"] = std_of_differences(u_b - f_k_boots)
        return out
    Theta = np.zeros([3 * K, 3 * K], dtype=np.float64)
    Theta[0:2 * K, 0:2 * K] = inner["Theta"]
    Theta[2 * K:3 * K, :] = Theta[K:2 * K, :]
    Theta[:, 2 * K:3 * K] = Theta[:, K:2 * K]
    diag = np.ones(3 * K, dtype=np.float64)
    diag[0:K] = diag[K:2 * K] = inner["observables"] - inner["Amin"]
    Adiag = np.zeros([3 * K, 3 * K], dtype=np.float64)
    np.fill_diagonal(Adiag, diag)
    Theta = Adiag @ Theta @ Adiag
    covf = Theta[2 * K:3 * K, 2 * K:3 * K]
    out["dDelta_f"] = est.error_of_differences(covf, warning_cutoff=warning_cutoff)
    covu = Theta[0:K, 0:K] + Theta[K:2 * K, K:2 * K] - Theta[0:K, K:2 * K] - Theta[K:2 * K, 0:K]
    out["dDelta_u"] = est.error_of_differences(covu, warning_cutoff=warning_cutoff)
    # s = u - f: cov(u, u) + cov(f, f) + A cov(ln C_a, ln c_a) + A cov(ln c_a, ln C_a) - 2 A cov(ln c_a, ln c_a)
    covs = (covu + covf + Theta[0:K, 2 * K:3 * K] + Theta[2 * K:3 * K, 0:K] - Theta[K:2 * K, 2 * K:3 * K]
            - Theta[2 * K:3 * K, K:2 * K])
    out["dDelta_s"] = est.error_of_differences(covs, warning_cutoff=warning_cutoff)
    return out


def compute_expectations(u_kn, N_k, f_k, A_n, u_ln=None, output="averages", state_dependent=False,
                         compute_uncertainty=True, uncertainty_method=None, warning_cutoff=1.0e-10,
                         return_theta=False, device=0):
    """MBAR.compute_expectations (mbar.py:1124-1312) with 2-D inputs: A_n [N] (or [K, N] when
    state_dependent), optional u_ln [L, N] for states other than the sampled set."""
    if uncertainty_method == "bootstrap":
        raise ParameterError("bootstrap uncertainties are served by pymbar_b200.bootstrap, not here")
    u_kn = np.asarray(u_kn, dtype=np.float64)
    u = u_kn if u_ln is None else np.asarray(u_ln, dtype=np.float64)
    if u.ndim == 1:
        u = u.reshape(1, -1)
    Ks = u.shape[0]
    inner = expectations_inner(u_kn, N_k, f_k, A_n, u, expectation_state_map(Ks, state_dependent),
                               uncertainty_method=uncertainty_method,
                               return_theta=compute_uncertainty or return_theta, device=device)
    return expectations_result(inner, Ks, output, compute_uncertainty, return_theta, warning_cutoff)


def compute_perturbed_free_energies(u_kn, N_k, f_k, u_ln, compute_uncertainty=True, uncertainty_method=None,
                                    warning_cutoff=1.0e-10, device=0):
    """MBAR.compute_perturbed_free_energies (mbar.py:1442-1521): free energies of L new states."""
    u_ln = np.asarray(u_ln, dtype=np.float64)
    if u_ln.ndim == 1:
        u_ln = u_ln.reshape(1, -1)
    L = u_ln.shape[0]
    inner = expectations_inner(u_kn, N_k, f_k, np.array([0.0]), u_ln, np.arange(L),
                               uncertainty_method=uncertainty_method, return_theta=compute_uncertainty,
                               device=device)
    return perturbed_result(inner, compute_uncertainty, warning_cutoff)

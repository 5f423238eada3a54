"""`mbar_many`: many independent small MBAR problems solved in lockstep on one GPU (DESIGN.md 3.5g).

A relative-free-energy campaign has hundreds of edges, each a small MBAR problem (K of 12 to 32 states, 10^3 to 10^4
samples per state).  Solved one at a time, such a problem costs one upload, one adaptive loop with its own launches
and host polls, and one `weight_moments` call, and the loop over problems is bound by those fixed costs rather than by
the GPU.  Here every problem with at most 64 states lives in one `DeviceMbarBatch`: the adaptive solver steps all of
them with one moments call (two launches, one synchronisation) per iteration, then one call gives every problem's
all-state update and one more every problem's second moments for the uncertainties.

Each problem follows `solve_mbar_for_all_states` with the adaptive stage of the reference's solver protocols
(`min_sc_iter=0`, `gamma=1`, `maxiter=10000`): the sampled states are solved, one self-consistent update then covers
every state, and f is shifted so that f[0] = 0.  The uncertainties come from the all-rows Gram at the converged f
through `estimators.free_energy_differences`.

A problem goes through the single-problem path (`mbar_solvers.solve_mbar_for_all_states` with the default protocol,
then `DeviceProblem.weight_moments`) and reports path="single" when it has more than 64 states, or when the batched
sums flag one of its iterates (a sum the linear-domain batch cannot represent, a non-finite candidate) or its batched
solve does not converge.  The rule depends only on the inputs and those flags.
"""
from __future__ import annotations

import numpy as np

from . import estimators
from . import mbar_solvers as ms
from .utils import ParameterError

DeviceMbarBatch = None     # the device classes; resolved on first use (a test may put stand-ins here)
DeviceProblem = None

MAX_BATCH_K = 64
UNCERTAINTY_METHODS = (None, "svd-ew", "approximate")
DEFAULT_OPTIONS = dict(min_sc_iter=0, gamma=1.0, maxiter=10000)


def _classes():
    global DeviceMbarBatch, DeviceProblem
    if DeviceMbarBatch is None:
        from .problem import DeviceMbarBatch as B

        DeviceMbarBatch = B
    if DeviceProblem is None:
        DeviceProblem = ms.DeviceProblem
    return DeviceMbarBatch, DeviceProblem


def _validate(u_kn, N_k, f_k):
    """The checks of mbar_solvers.validate_inputs, and N_k must count the samples of u_kn."""
    if not isinstance(u_kn, np.ndarray) or u_kn.ndim != 2:
        raise ParameterError(f"u_kn must be a two-dimensional numpy array, got {type(u_kn).__name__} "
                             f"of shape {np.shape(u_kn)}")
    K, N = u_kn.shape
    if K < 1 or N < 1:
        raise ParameterError(f"u_kn must have at least one state and one sample, got shape {u_kn.shape}")
    f_k = np.zeros(K) if f_k is None else f_k
    u_kn, N_k, f_k = ms.validate_inputs(u_kn, np.asarray(N_k), np.asarray(f_k, dtype=np.float64))
    if np.any(N_k < 0) or not np.all(np.isfinite(N_k)):
        raise ParameterError("N_k must hold non-negative sample counts")
    if np.sum(N_k) != N:
        raise ParameterError(f"N_k sums to {np.sum(N_k)}, but u_kn holds {N} samples")
    if np.isnan(u_kn).any():
        raise ParameterError("u_kn holds NaN")
    return u_kn, N_k, f_k


def _gram_to_G(Ghat, N_k):
    """W^T W from the N-scaled Gram of all rows (unsampled rows scaled by 1), as DeviceProblem.weight_moments gives."""
    s = np.where(N_k > 0, N_k, 1.0)
    return Ghat / np.outer(s, s)


def _result(f, G, N_k, path, iterations, success, compute_uncertainty, uncertainty_method, return_theta):
    out = dict(f_k=f, Delta_f=f - np.vstack(f), path=path, iterations=iterations, success=bool(success))
    if compute_uncertainty or return_theta:
        d = estimators.free_energy_differences(f, G, N_k, uncertainty_method=uncertainty_method,
                                               return_theta=return_theta)
        if compute_uncertainty:
            out["dDelta_f"] = d["dDelta_f"]
        if return_theta:
            out["Theta"] = d["Theta"]
    return out


def _single(u_kn, N_k, f_k, tol, want_G):
    """(f, G or None) of the single-problem path."""
    _, Prob = _classes()
    protocol = tuple(dict(s, tol=tol) for s in ms.DEFAULT_SOLVER_PROTOCOL)
    sws = np.flatnonzero(N_k > 0)
    f = ms.solve_mbar_for_all_states(u_kn, N_k, f_k, sws, protocol)
    G = None
    if want_G:
        with Prob(u_kn, N_k, device=ms._DEVICE) as p:
            _, G = p.weight_moments(f)
    return f, G


def mbar_many(u_kn_list, N_k_list, f_k_init=None, compute_uncertainty=True, uncertainty_method=None,
              return_theta=False, solver_tolerance=1.0e-12, options=None):
    """MBAR on every problem (u_kn_list[p], N_k_list[p]): one dict per problem, in input order, with f_k, Delta_f,
    dDelta_f (compute_uncertainty), Theta (return_theta), iterations (of the batched solve; None on the single path),
    success and path ("batch" or "single").

    f_k_init: None (zeros) or one starting vector per problem.  options update the adaptive solver's defaults
    (min_sc_iter=0, gamma=1, maxiter=10000).  uncertainty_method: None, "svd-ew" or "approximate".  Every problem is
    validated before any device work; an invalid problem raises for the lowest failing index."""
    if uncertainty_method not in UNCERTAINTY_METHODS:
        raise ParameterError(f"uncertainty_method {uncertainty_method!r} is not supported by mbar_many "
                             f"(one of {UNCERTAINTY_METHODS})")
    if len(u_kn_list) != len(N_k_list):
        raise ValueError("u_kn_list and N_k_list must have the same length")
    P = len(u_kn_list)
    if f_k_init is not None and len(f_k_init) != P:
        raise ValueError("f_k_init must hold one vector per problem")
    opts = dict(DEFAULT_OPTIONS)
    opts.update(options or {})
    probs = [_validate(u_kn_list[p], N_k_list[p], None if f_k_init is None else f_k_init[p]) for p in range(P)]
    want_G = bool(compute_uncertainty or return_theta)
    results = [None] * P
    batch = [p for p in range(P) if probs[p][0].shape[0] <= MAX_BATCH_K]
    single = [p for p in range(P) if probs[p][0].shape[0] > MAX_BATCH_K]
    if batch:
        Batch, _ = _classes()
        with Batch([probs[p][0] for p in batch], [probs[p][1] for p in batch], device=ms._DEVICE) as dev:
            f_list, status, iters = dev.solve([probs[p][2] for p in batch], tol=solver_tolerance,
                                              maxiter=int(opts["maxiter"]), min_sc_iter=int(opts["min_sc_iter"]),
                                              gamma=float(opts["gamma"]))
            ok = [i for i in range(len(batch)) if status[i] == 0]
            single += [batch[i] for i in range(len(batch)) if status[i] != 0]
            # every state: one self-consistent update, then the gauge f[0] = 0 (solve_mbar_for_all_states)
            f_final = {}
            if ok:
                sums = dev.moments([f_list[i] for i in ok], all_rows=True, problems=ok)
                for i, m in zip(ok, sums):
                    if m["flag"]:
                        single.append(batch[i])
                        continue
                    f = f_list[i] - m["log_S"]
                    f_final[i] = f - f[0]
            ok = [i for i in ok if i in f_final]
            G = {}
            if ok and want_G:
                sums = dev.moments([f_final[i] for i in ok], want_G=True, all_rows=True, problems=ok)
                for i, m in zip(ok, sums):
                    if m["flag"]:
                        single.append(batch[i])
                        continue
                    G[i] = _gram_to_G(m["G"], probs[batch[i]][1])
            for i in ok:
                if want_G and i not in G:
                    continue
                p = batch[i]
                results[p] = _result(f_final[i], G.get(i), probs[p][1], "batch", int(iters[i]), True,
                                     compute_uncertainty, uncertainty_method, return_theta)
    for p in sorted(single):
        u, N_k, f0 = probs[p]
        f, G = _single(u, N_k, f0, solver_tolerance, want_G)
        success = bool(np.all(np.isfinite(f)))
        results[p] = _result(f, G, N_k, "single", None, success, compute_uncertainty, uncertainty_method,
                             return_theta)
    return results

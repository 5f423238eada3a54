"""H100 backend with the interface of ``pymbar.mbar_solvers`` (same names, arguments, errors).

``pymbar.MBAR`` reaches its solver only through module attributes of ``pymbar.mbar_solvers``
(mbar.py:413, :437, :455, :910); this module offers the same callables with the arithmetic done
by libmbar_b200.so on the GPU.  ``pymbar_b200.install()`` rebinds those attributes so an
unmodified ``pymbar.MBAR`` runs on it.  There is no numpy/JAX fallback in here: without the
compiled library and an H100 every call raises.

Residency.  The reference functions are pure functions of host arrays.  Re-uploading u_kn for
every call would turn a 3 ms pass into a PCIe transfer, so calls are served from a small cache of
:class:`DeviceProblem` objects keyed on the identity (address, shape, strides), the N_k vector and
a 64-bit hash of the WHOLE array (``mbar_b200_host_hash``: threaded, memory-bandwidth bound, far
cheaper than the upload it saves) — an in-place edit of u_kn can therefore never be answered from a
stale device copy.  Entries die with their host array (weakref) or through :func:`invalidate` /
:func:`clear_cache`; ``PYMBAR_B200_CACHE=0`` disables the cache (every call uploads).  The drivers
(``solve_mbar*``) hold one problem explicitly for the whole protocol.
"""
from __future__ import annotations

import ctypes
import logging
import os
import warnings
import weakref
from collections import OrderedDict

import numpy as np
import scipy.optimize

from .problem import DeviceAcf, DeviceBSpline, DeviceKde, DeviceProblem, DeviceWork  # noqa: F401  (DeviceKde, DeviceBSpline, DeviceAcf, DeviceWork: looked up here by the facade)
from .utils import ParameterError, ensure_type

logger = logging.getLogger(__name__)

# Protocol constants, identical in value to mbar_solvers.py:102-117 (read by mbar.py:55-58).
JAX_SOLVER_PROTOCOL = (
    dict(method="BFGS", continuation=True),
    dict(method="adaptive", options=dict(min_sc_iter=0)),
)
DEFAULT_SOLVER_PROTOCOL = (
    dict(method="hybr", continuation=True),
    dict(method="adaptive", options=dict(min_sc_iter=0)),
)
ROBUST_SOLVER_PROTOCOL = (
    dict(method="adaptive", options=dict(maxiter=1000)),
    dict(method="L-BFGS-B", options=dict(maxiter=1000)),
)
BOOTSTRAP_SOLVER_PROTOCOL = (dict(method="adaptive", options=dict(min_sc_iter=0)),)

# mbar_solvers.py:120-139
scipy_minimize_options = ["L-BFGS-B", "dogleg", "CG", "BFGS", "Newton-CG", "TNC", "trust-ncg",
                          "trust-krylov", "trust-exact", "SLSQP"]
scipy_nohess_options = ["L-BFGS-B", "BFGS", "CG", "TNC", "SLSQP"]
scipy_root_options = ["hybr", "lm"]

use_jit = False  # attribute read by callers of the reference module

_DEVICE = int(os.environ.get("PYMBAR_B200_DEVICE", os.environ.get("LOCAL_RANK", "0")))


# ---------------------------------------------------------------------------------------------
# residency cache
# ---------------------------------------------------------------------------------------------
_CACHE: "OrderedDict[tuple, DeviceProblem]" = OrderedDict()
_CACHE_SLOTS = int(os.environ.get("PYMBAR_B200_CACHE_SLOTS", "2"))


def _cache_enabled():
    return os.environ.get("PYMBAR_B200_CACHE", "1").lower() not in ("0", "false", "no")


def _content_hash(u_kn):
    """Exact-content key: 64-bit hash of every byte of the (possibly row-strided) array."""
    from . import _lib

    if u_kn.size == 0:
        return 0
    if u_kn.ndim != 2 or u_kn.strides[1] != u_kn.itemsize or u_kn.strides[0] < u_kn.shape[1] * u_kn.itemsize:
        u_kn = np.ascontiguousarray(u_kn)
    h = ctypes.c_uint64(0)
    _lib.check(_lib.load().mbar_b200_host_hash(ctypes.c_void_p(u_kn.ctypes.data), u_kn.shape[0],
                                               u_kn.shape[1] * u_kn.itemsize, u_kn.strides[0], ctypes.byref(h)))
    return h.value


def clear_cache():
    while _CACHE:
        _, p = _CACHE.popitem()
        p.close()


def invalidate(u_kn=None):
    """Drop the cached device copies of `u_kn` (or all of them)."""
    if u_kn is None:
        return clear_cache()
    addr = np.asarray(u_kn).__array_interface__["data"][0]
    for key in [k for k in _CACHE if k[0] == addr]:
        _CACHE.pop(key).close()


def _evict(key):
    prob = _CACHE.pop(key, None)
    if prob is not None:
        prob.close()


def _problem_for(u_kn, N_k):
    """DeviceProblem holding (u_kn, N_k), from the cache when the same host array WITH THE SAME CONTENTS is
    seen again."""
    if not _cache_enabled():
        return DeviceProblem(u_kn, N_k, device=_DEVICE), False
    key = (u_kn.__array_interface__["data"][0], u_kn.shape, u_kn.strides,
           np.asarray(N_k, np.float64).tobytes(), _content_hash(u_kn))
    prob = _CACHE.get(key)
    if prob is None:
        # a different content at the same address supersedes the old entry (the caller edited in place)
        for stale in [k for k in _CACHE if k[:3] == key[:3]]:
            _CACHE.pop(stale).close()
        prob = DeviceProblem(u_kn, N_k, device=_DEVICE)
        _CACHE[key] = prob
        try:
            # the device copy must not outlive the host array it mirrors
            prob._host_ref = weakref.ref(u_kn, lambda _r, key=key: _evict(key))
        except TypeError:
            pass
        while len(_CACHE) > _CACHE_SLOTS:
            _, old = _CACHE.popitem(last=False)
            old.close()
    else:
        _CACHE.move_to_end(key)
    return prob, True


class _borrow:
    """Context manager: cached problems stay alive, uncached ones are closed on exit."""

    def __init__(self, u_kn, N_k):
        self.prob, self.cached = _problem_for(u_kn, N_k)

    def __enter__(self):
        return self.prob

    def __exit__(self, *exc):
        if not self.cached:
            self.prob.close()


# ---------------------------------------------------------------------------------------------
# primitives (mbar_solvers.py:174-507, :697-735)
# ---------------------------------------------------------------------------------------------
def validate_inputs(u_kn, N_k, f_k):
    """mbar_solvers.py:174-203."""
    n_states, n_samples = u_kn.shape
    u_kn = ensure_type(u_kn, "float", 2, "u_kn or Q_kn", shape=(n_states, n_samples))
    N_k = ensure_type(N_k, "float", 1, "N_k", shape=(n_states,), warn_on_cast=False)
    f_k = ensure_type(f_k, "float", 1, "f_k", shape=(n_states,))
    return u_kn, N_k, f_k


def _prep(u_kn, N_k, f_k):
    u_kn = np.asarray(u_kn)
    if u_kn.dtype != np.float64:
        u_kn = u_kn.astype(np.float64)
    return u_kn, np.asarray(N_k, dtype=np.float64), np.asarray(f_k, dtype=np.float64)


def self_consistent_update(u_kn, N_k, f_k, states_with_samples=None):
    """Eq. C3 (mbar_solvers.py:206-257).  All K states get a value; states with N_k = 0 do not
    enter the denominator."""
    u_kn, N_k, f_k = _prep(u_kn, N_k, f_k)
    if states_with_samples is not None:
        sws = np.asarray(states_with_samples)
        u_kn, N_k, f_k = u_kn[sws], N_k[sws], f_k[sws]
    with _borrow(u_kn, N_k) as p:
        return p.self_consistent_update(f_k)


def mbar_gradient(u_kn, N_k, f_k):
    """Eq. C6 (mbar_solvers.py:260-292)."""
    u_kn, N_k, f_k = _prep(u_kn, N_k, f_k)
    with _borrow(u_kn, N_k) as p:
        return p.gradient(f_k)


def mbar_objective(u_kn, N_k, f_k):
    """mbar_solvers.py:295-338."""
    u_kn, N_k, f_k = _prep(u_kn, N_k, f_k)
    with _borrow(u_kn, N_k) as p:
        return p.objective(f_k)


def mbar_objective_and_gradient(u_kn, N_k, f_k):
    """mbar_solvers.py:341-392."""
    u_kn, N_k, f_k = _prep(u_kn, N_k, f_k)
    with _borrow(u_kn, N_k) as p:
        return p.objective_and_gradient(f_k)


def mbar_hessian(u_kn, N_k, f_k):
    """Eq. C9 (mbar_solvers.py:395-436)."""
    u_kn, N_k, f_k = _prep(u_kn, N_k, f_k)
    with _borrow(u_kn, N_k) as p:
        return p.hessian(f_k)


def mbar_log_W_nk(u_kn, N_k, f_k):
    """Eq. 9, [N, K] (mbar_solvers.py:439-473).  While `MBAR.__init__` runs under the installed facade the
    matrix is not produced yet: the caller receives a ticket that `MBAR.Log_W_nk` redeems on first use."""
    from . import facade

    if facade.deferring():
        return facade.LogWeightTicket(u_kn, N_k, f_k)
    u_kn, N_k, f_k = _prep(u_kn, N_k, f_k)
    with _borrow(u_kn, N_k) as p:
        return p.log_W_nk(f_k)


def mbar_W_nk(u_kn, N_k, f_k):
    """mbar_solvers.py:476-507."""
    u_kn, N_k, f_k = _prep(u_kn, N_k, f_k)
    with _borrow(u_kn, N_k) as p:
        return p.log_W_nk(f_k, exponentiate=True)


def precondition_u_kn(u_kn, N_k, f_k):
    """mbar_solvers.py:710-735.  The device stores u_kn already shifted per sample, so nothing in
    this backend needs the materialised array; it is provided for API completeness and computed
    from the device's per-sample log-denominators."""
    u_kn, N_k, f_k = _prep(u_kn, N_k, f_k)
    shifted = u_kn - u_kn.min(0)
    with _borrow(shifted, N_k) as p:
        L = p.log_denominator(f_k)
    return shifted + (L - np.dot(N_k, f_k) / N_k.sum())


# jax_* aliases exist in the reference namespace and are what MBAR-level monkeypatching would hit
jax_self_consistent_update = self_consistent_update
jax_mbar_gradient = mbar_gradient
jax_mbar_objective = mbar_objective
jax_mbar_objective_and_gradient = mbar_objective_and_gradient
jax_mbar_hessian = mbar_hessian
jax_mbar_log_W_nk = mbar_log_W_nk
jax_mbar_W_nk = mbar_W_nk
jax_precondition_u_kn = precondition_u_kn


# ---------------------------------------------------------------------------------------------
# drivers (mbar_solvers.py:510-1017) on an explicit DeviceProblem
# ---------------------------------------------------------------------------------------------
def _adaptive_on(problem, f_k, tol, options):
    options = {} if options is None else options
    options.setdefault("verbose", False)
    options.setdefault("maxiter", 10000)
    options.setdefault("print_warning", False)
    options.setdefault("gamma", 1.0)
    options.setdefault("min_sc_iter", 2)
    if tol < 4.0 * np.finfo(float).eps:
        logger.info("Tolerance may be too close to machine precision to converge.")
    f, r = problem.solve_adaptive(f_k, tol=tol, maxiter=options["maxiter"],
                                  min_sc_iter=options["min_sc_iter"], gamma=options["gamma"])
    if r["success"]:
        message = "Convergence achieved by change in f with respect to previous guess."
        if options["verbose"]:
            logger.info(f"Converged to tolerance of {r['max_delta']:e} in {r['iterations']:d} iterations.")
            logger.info(f"Of {r['iterations']:d} iterations, {r['nr_iterations']:d} were Newton-Raphson "
                        f"iterations and {r['sci_iterations']:d} were self-consistent iterations")
    else:
        message = "Did not converge."
        logger.warning("WARNING: Did not converge to within specified tolerance.")
        logger.warning(f"max_delta = {r['max_delta']:e}, tol = {tol:e}, maximum_iterations = "
                       f"{options['maxiter']:d}, iterations completed = {r['iterations']:d}")
    results = dict(success=bool(r["success"]), message=message, x=f)
    results.update({"b200_" + k: v for k, v in r.items()})
    return results


def adaptive(u_kn, N_k, f_k, tol=1.0e-8, options=None):
    """Newton-Raphson / self-consistent adaptive solver (mbar_solvers.py:510-667), run natively
    (mbar_b200_solve_adaptive): same step-selection and convergence rules, 3 streaming passes +
    1 Hessian pass per iteration instead of the reference's 4 + 1."""
    u_kn, N_k, f_k = _prep(u_kn, N_k, f_k)
    with _borrow(u_kn, N_k) as p:
        return _adaptive_on(p, f_k, tol, options)


def _solve_once_on(problem, f_full, method="adaptive", tol=1e-12, continuation=None, options=None):
    """solve_mbar_once (mbar_solvers.py:738-883) on a resident problem.  f_full has K entries;
    unsampled states (N_k = 0) are carried through untouched, the unknowns handed to scipy are the
    sampled states minus the gauge state."""
    act = np.flatnonzero(problem.N_k > 0)
    f_full = np.array(f_full, dtype=np.float64)
    f_full[act] -= f_full[act[0]]
    free = act[1:]

    def expand(x):
        f = f_full.copy()
        f[free] = x
        return f

    grad = lambda x: problem.gradient(expand(x))[free]
    hess = lambda x: problem.hessian(expand(x))[np.ix_(free, free)]
    # the reference preconditions u_kn so that the objective is ~0 at the starting point
    # (mbar_solvers.py:793, :726-734); the same offset keeps scipy's ftol logic comparable
    obj0 = [None]

    def grad_and_obj(x):
        o, g = problem.objective_and_gradient(expand(x))
        if obj0[0] is None:
            obj0[0] = o
        return np.array(o - obj0[0]), np.array(g[free])

    with warnings.catch_warnings(record=True) as w:
        if method in scipy_minimize_options:
            results = scipy.optimize.minimize(
                grad_and_obj, f_full[free], jac=True,
                hess=None if method in scipy_nohess_options else hess,
                method=method, tol=tol, options=options)
            f_full = expand(results["x"])
        elif method == "adaptive":
            results = _adaptive_on(problem, f_full, tol, options)
            f_full = np.array(results["x"])
        elif method in scipy_root_options:
            results = scipy.optimize.root(grad, f_full[free], jac=hess, method=method, tol=tol,
                                          options=options)
            f_full = expand(results["x"])
        else:
            raise ParameterError(f"Method {method} for solution of free energies not recognized")
    shown = [m for m in w if "Unknown solver options" not in str(m.message)]
    for m in shown:
        warnings.showwarning(m.message, m.category, m.filename, m.lineno, m.file, "")
    if shown:
        # mbar_solvers.py:874-881: weights must still be normalised
        S, _, _ = problem.streaming_pass(f_full)
        if not np.allclose(S[act], 1.0, atol=1e-4):
            raise ParameterError("Warning: Should have \\sum_n W_nk = 1.  Actual column sum for state "
                                 f"{int(act[np.argmax(np.abs(S[act] - 1))])} was "
                                 f"{S[act][np.argmax(np.abs(S[act] - 1))]:f}.")
        logger.warning("MBAR weights converged within tolerance, despite the SciPy Warnings. "
                       "Please validate your results.")
    return f_full, results


def _solve_protocol_on(problem, f_full, solver_protocol=None):
    """solve_mbar (mbar_solvers.py:886-974) on a resident problem."""
    if solver_protocol is None:
        solver_protocol = DEFAULT_SOLVER_PROTOCOL
    all_fks, all_gnorms, all_results = [], [], []
    for solver in solver_protocol:
        f_res, results = _solve_once_on(problem, f_full, **solver)
        all_fks.append(f_res)
        all_gnorms.append(np.linalg.norm(problem.gradient(f_res)))
        all_results.append(results)
        if results["success"]:
            best_gnorm = all_gnorms[-1]
            logger.info(f"Reached a solution to within tolerance with {solver['method']}")
            break
        logger.warning(f"Failed to reach a solution to within tolerance with {solver['method']}: "
                       "trying next method")
        logger.info(f"Ending gnorm of method {solver['method']} = {all_gnorms[-1]:e}")
        if solver.get("continuation"):
            f_full = f_res
            logger.info("Will continue with results from previous method")
    if results["success"]:
        logger.info("Solution found within tolerance!")
    else:
        i_best = int(np.argmin(all_gnorms))
        best_gnorm = all_gnorms[i_best]
        logger.warning("No solution found to within tolerance.")
        logger.warning(f"The solution with the smallest gradient {best_gnorm:e} norm is "
                       f"{solver_protocol[i_best]['method']}")
        f_res = all_fks[i_best]
        logger.warning("Please exercise caution with this solution and consider alternative methods "
                       "or a different tolerance.")
    logger.info(f"Final gradient norm: {best_gnorm:.3g}")
    return f_res, all_results


def solve_mbar_once(u_kn_nonzero, N_k_nonzero, f_k_nonzero, method="adaptive", tol=1e-12,
                    continuation=None, options=None):
    """mbar_solvers.py:738-883."""
    u_kn_nonzero, N_k_nonzero, f_k_nonzero = validate_inputs(u_kn_nonzero, N_k_nonzero, f_k_nonzero)
    with _borrow(u_kn_nonzero, N_k_nonzero) as p:
        return _solve_once_on(p, f_k_nonzero, method=method, tol=tol, continuation=continuation,
                              options=options)


def solve_mbar(u_kn_nonzero, N_k_nonzero, f_k_nonzero, solver_protocol=None):
    """mbar_solvers.py:886-974."""
    u_kn_nonzero, N_k_nonzero, f_k_nonzero = _prep(u_kn_nonzero, N_k_nonzero, f_k_nonzero)
    with _borrow(u_kn_nonzero, N_k_nonzero) as p:
        return _solve_protocol_on(p, f_k_nonzero, solver_protocol)


def solve_mbar_for_all_states(u_kn, N_k, f_k, states_with_samples, solver_protocol):
    """mbar_solvers.py:977-1017 — the call MBAR.__init__ makes (mbar.py:413).

    u_kn is uploaded ONCE with all K states; the sampled-state solve, the final all-state
    self-consistent update (:1012) and the gauge shift (:1015) run against that resident copy
    (the reference slices u_kn[states_with_samples] into a second full copy, :1003)."""
    u_kn, N_k_f, f_k = _prep(u_kn, N_k, f_k)
    f_k = np.array(f_k, dtype=np.float64)
    with _borrow(u_kn, N_k_f) as p:
        if len(states_with_samples) > 1:
            f_k, _ = _solve_protocol_on(p, f_k, solver_protocol)
        else:
            f_k[np.asarray(states_with_samples)] = 0.0
        f_k = p.self_consistent_update(f_k)
    f_k -= f_k[0]
    return f_k

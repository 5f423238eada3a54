"""What `pymbar_b200.install()` does to the `pymbar.MBAR` class itself (SURVEY.md 8f rows N1 / N2).

Rebinding `pymbar.mbar_solvers` moves the solve to the GPU, but `MBAR.__init__` then still asks for the full
N x K `Log_W_nk` on the host (mbar.py:455; 20.5 GB at K=256, N=1e7) and every estimator reduces that matrix on
the CPU.  With the facade installed:

* `MBAR.Log_W_nk` becomes LAZY: inside `MBAR.__init__` the backend's `mbar_log_W_nk` hands back a ticket
  instead of the array; the first read of `mbar.Log_W_nk` (property) downloads it, so code that really wants
  the matrix still gets a plain writable ndarray, and code that never looks at it never pays for it;
* `compute_effective_sample_number` (mbar.py:496-561), `compute_overlap` (:563-617) and
  `compute_free_energy_differences` (:620-760) are answered from the K x K second moments
  G = W^T W that the Hessian kernels produce on the device (`weight_moments`), through
  `pymbar_b200.estimators`;
* `compute_expectations_inner` (:766-1012) — the one routine behind compute_expectations,
  compute_multiple_expectations, compute_perturbed_free_energies and compute_entropy_and_enthalpy — is
  answered by the augmented-problem formulation of `pymbar_b200.expectations`.

* `_initialize_with_bar` (:1936-1988, `MBAR(initialize="BAR")`) uses `pymbar_b200.initialize` (samples grouped by
  state once, Brent on Bennett's equation).

* `_computeUnnormalizedLogWeights` (:1919-1934) is -u_n - L_n with L_n from the device's log denominators.

* `MBAR(..., n_bootstraps=B)` with B a positive int runs the original constructor with n_bootstraps=0, then draws the
  replicates from `self.rng` as mbar.py:424-433 does and solves each with one weighted solve on the resident problem
  (`bootstrap.bootstrap_f_k`; BAR on the replicate's columns under initialize="BAR").  `bootstrap_rints` becomes lazy:
  the generator state before each replicate is kept and the rows are regenerated on first read.
  `compute_free_energy_differences` and `compute_expectations_inner` with `uncertainty_method="bootstrap"` answer from
  `f_k_boots`, the replicates' counts and one `DeviceProblem.replicate_unsampled` call on the augmented problem
  (`expectations.expectations_inner(..., replicates=...)`).  A replicate whose device solve fails is solved on the
  gathered `u_kn[:, rints]` (`STATS["mbar_boot_*"]`).

Anything outside what the device path implements (`uncertainty_method="svd"`, an augmented problem of more than
`_lib.MAX_STATES` states, bootstrap requests without device replicates or with a count above 65535) calls the
original method, which then reads `self.Log_W_nk` and materialises it.  `uninstall()` restores the class.

`install_fes_on` does the same for `pymbar.FES` (fes.py): `generate_fes` without bootstraps takes its log weights
from the device and, for fes_type="histogram", builds the bin free energies with `pymbar_b200.fes.histogram_fes`;
`FES.w_kn` (np.exp(mbar.Log_W_nk), fes.py:416) becomes lazy like `Log_W_nk`.  `_get_fes_histogram` with
`uncertainty_method="analytical"` takes Theta from `pymbar_b200.fes.histogram_theta` (K x nbins moments on the
device) instead of the N x (K + nbins) augmented weight matrix (fes.py:1382-1406).

For fes_type="kde" (sklearn parameters the device serves, `pymbar_b200.fes.kde_settings`) `generate_fes` uploads x_n
and w_n to a `DeviceKde` instead of fitting sklearn's tree, and `_get_fes_kde` without uncertainties answers from
it (`pymbar_b200.fes.kde_query`).  `FES.kde` becomes lazy: the first read by anything else (`get_kde()`, the original
methods) fits it exactly as fes.py:696 does.

For fes_type="spline" with 1-D samples, `generate_fes` makes one pass over x_n on a `DeviceBSpline` for the fit's
knots: the per-state basis sums S and the weighted sums A (`SplineMoments`).  The fit's sample terms are linear in
the spline coefficients, so `_bspline_calculate_f`, `_bspline_calculate_g` and `_get_MC_loglikelihood` answer from
them (`pymbar_b200.fes.spline_objective` / `spline_gradient` / `spline_mc_loglikelihood`) with O(K nb) arithmetic
and the reference's quadratures, where the reference evaluates the spline on every sample at every step.  They do
so only for the very x_n and w_n arrays the moments were built from and for splines on the same knots and degree;
any other call (another x_n passed to `sample_parameter_distribution`, 2-D samples) runs the original method.  The
optimiser, the Hessian, the information criteria and `_get_fes_spline` stay the reference's.

`generate_fes(fes_type="spline", n_bootstraps >= 2)` with 1-D samples in block order fits b = 0 as above, then draws
the replicates as the reference does and gives every replicate's sample terms from one
`DeviceBSpline.replicate_sums` call over weights V_b built on the host (`pymbar_b200.fes_bootstrap.spline_replicates`;
"unbiasedstate" runs one weighted solve per replicate for its log denominators, the other weightings none).  Each
replicate is fitted by the reference's `_generate_fes_spline(b, x_nb, w_nb)`, whose objective and gradient answer
from that replicate's terms, and appended to `fes_functions`; `_get_fes_spline` takes its bootstrap std from them
as the reference does.  Samples out of block order, 2-D samples, an unknown spline_weights and device errors call
the original with numpy's generator and the spline_parameters restored (`STATS["fes_boot_spline_*"]`).

`generate_fes` with n_bootstraps >= 2 for fes_type="histogram" or "kde" draws the replicates from numpy's global
generator as fes.py:395-406 does (one MBAR seed draw after every block included) and keeps the generator's state
before each replicate instead of its indices (`pymbar_b200.fes_bootstrap`).  A histogram replicate is one weighted
solve on the resident problem and one bin pass with the replicate's multiplicities; `histogram_datas[b]` builds
`bin_n`, `sample_label` and `nonzero_bins` on first read.  A KDE replicate has no solve: the replicate weights go to
the DeviceKde once, `FES.kdes` fits replicate b only when read, and `_get_fes_kde(uncertainty_method="bootstrap")`
answers "from-lowest" and "from-specified" from one `log_sum_replicates` call; `_get_fes_histogram` takes the std
over the replicates as fes.py:1417-1422 does.  A replicate that empties a bin tuple of b = 0, a state without
samples, other reference points, and device errors call the original with numpy's generator restored to its state at
entry (`STATS["fes_boot_*"]`).

Bootstrap uncertainties of surfaces generated without device replicates, device errors and any call whose weights
leave the device's range contract go to the original methods.

`install_timeseries_on` rebinds `statistical_inefficiency`, `statistical_inefficiency_multiple`,
`normalized_fluctuation_correlation_function` and `detect_equilibration` of `pymbar.timeseries` to
`pymbar_b200.timeseries`, which answers from a `DeviceAcf`.  `subsample_correlated_data`,
`integrated_autocorrelation_time(Multiple)` and fes.py reach them through the module's globals.  fft=True, inputs
that are not 1-D float64 or integer arrays (float32 means differ in the reference), a constant input or sigma^2 = 0 in
`_multiple` (the reference returns NaN or runs on rounding noise) and device errors go to the original functions.
Where the module has them, `normalized_fluctuation_correlation_function_multiple`, `statistical_inefficiency_fft`
and `detect_equilibration_binary_search` are rebound too (`STATS["ts_correlation_multiple"]`, `["ts_fft"]`,
`["ts_binary_search"]`); they need no statsmodels.  `statistical_inefficiency(fft=True)` still calls the original,
which reaches the rebound `statistical_inefficiency_fft` through the module's globals.  Constant remaining series,
unsupported input and device errors call their originals, which without statsmodels raise as before.

`install_other_estimators_on` rebinds `bar`, `bar_zero`, `exp` and `exp_gauss` of `pymbar.other_estimators` to
`pymbar_b200.other_estimators`, which answers from a `DeviceWork`; `install()` rebinds the same names on the `pymbar`
package, which bound them at import.  `bar_overlap` stays the reference's and reaches the patched `bar` through the
module's globals.  Input that is not a 1-D float64 or signed integer ndarray (the reference fails on lists in `bar`,
and float32 changes its arithmetic), empty or non-finite input, `verbose=True`, an unknown `method` or
`uncertainty_method` (the original raises its own error) and device errors go to the original functions.
"""
from __future__ import annotations

import threading
from timeit import default_timer as _timer

import numpy as np

from . import estimators as est

_TLS = threading.local()
_SAVED = {}
STATS = {"tickets": 0, "redeemed": 0, "moments": 0, "expectations": 0, "expectations_fallbacks": 0, "log_weights": 0,
         "fes_histograms": 0, "fes_theta": 0, "fes_w_kn": 0, "fes_kde_fits": 0, "fes_kde_queries": 0,
         "fes_spline_moments": 0, "fes_spline_calls": 0, "ts_inefficiency": 0, "ts_multiple": 0, "ts_correlation": 0,
         "ts_equilibration": 0, "ts_fft": 0, "ts_binary_search": 0, "ts_correlation_multiple": 0, "ts_fallbacks": 0,
         "oe_bar": 0, "oe_bar_zero": 0, "oe_exp": 0, "oe_exp_gauss": 0,
         "oe_evaluations": 0, "oe_fallbacks": 0, "fes_boot_solves": 0, "fes_boot_passes": 0, "fes_boot_fallbacks": 0,
         "fes_boot_spline_solves": 0, "fes_boot_spline_sums": 0, "mbar_boot_solves": 0, "mbar_boot_fallbacks": 0,
         "expectations_boot": 0, "boot_rints_built": 0}


class LogWeightTicket:
    """Stands for `mbar_log_W_nk(u_kn, N_k, f_k)` until somebody needs the numbers."""

    __slots__ = ("u_kn", "N_k", "f_k")

    def __init__(self, u_kn, N_k, f_k):
        self.u_kn, self.N_k, self.f_k = u_kn, np.array(N_k), np.array(f_k, dtype=np.float64)
        STATS["tickets"] += 1

    def redeem(self):
        from . import mbar_solvers as ms

        STATS["redeemed"] += 1
        return ms.mbar_log_W_nk(self.u_kn, self.N_k, self.f_k)


def deferring():
    return getattr(_TLS, "defer", 0) > 0


def _moments(mbar):
    """(S_k, G = W^T W) of the converged weights, all K states, computed on the device once per MBAR object."""
    cached = mbar.__dict__.get("_b200_moments")
    if cached is not None and np.array_equal(cached[2], mbar.f_k):
        return cached[0], cached[1]
    from . import mbar_solvers as ms

    STATS["moments"] += 1
    with ms._borrow(mbar.u_kn, np.asarray(mbar.N_k, dtype=np.float64)) as p:
        S, G = p.weight_moments(np.asarray(mbar.f_k, dtype=np.float64))
    mbar.__dict__["_b200_moments"] = (S, G, np.array(mbar.f_k))
    return S, G


def _device_log_weights(mbar, u_n):
    """-u_n - L_n: the unnormalised log weights of the target state u_n (mbar.py:1919-1934)."""
    from . import mbar_solvers as ms

    STATS["log_weights"] += 1
    u_n = np.asarray(u_n, dtype=np.float64)
    with ms._borrow(mbar.u_kn, np.asarray(mbar.N_k, dtype=np.float64)) as p:
        L = p.log_denominator(np.asarray(mbar.f_k, dtype=np.float64))
    return -u_n - L


def _check_normalised(S, tolerance=1.0e-4):
    # utils.check_w_normalized (utils.py:340-388): column sums of W must be 1
    from . import utils as u

    bad = np.flatnonzero(np.abs(S - 1.0) > tolerance)
    if bad.size:
        raise u.ParameterError(f"Warning: Should have \\sum_n W_nk = 1.  Actual column sum for state "
                               f"{int(bad[0]):d} was {S[bad[0]]:f}. {bad.size:d} other columns have similar problems")


class RintsTicket:
    """Stands for MBAR.bootstrap_rints [B, N] (mbar.py:423-445) until somebody reads it: the generator state before
    each replicate's draws, from which the rows are regenerated bit for bit."""

    __slots__ = ("rng", "states", "N_k", "members")

    def __init__(self, rng, states, N_k, members):
        self.rng, self.states, self.N_k, self.members = rng, states, N_k, members

    def redeem(self):
        from . import bootstrap as bs

        STATS["boot_rints_built"] += 1
        out = np.zeros((len(self.states), int(np.sum(self.N_k))), int)
        for b, state in enumerate(self.states):
            out[b] = bs.replicate_rints(self.rng, state, self.N_k, self.members)
        return out


def _solver_module(mbar):
    """The solver module the MBAR class resolves its solves through (pymbar.mbar_solvers for pymbar.MBAR)."""
    import sys

    from . import mbar_solvers as ms

    own = getattr(type(mbar), "solvers", None)
    return own if own is not None else getattr(sys.modules.get(type(mbar).__module__), "mbar_solvers", ms)


def _bootstrap_protocol(mbar, prot):
    """The bootstrap_solver_protocol as mbar.py:370-411 resolves it (the original normalised the dicts in place)."""
    import sys

    from . import fes_bootstrap as fb

    mod = sys.modules.get(type(mbar).__module__)
    solvers = _solver_module(mbar)

    def const(name):
        v = getattr(mod, name, None)
        return v if v is not None else getattr(solvers, name)

    default = const("BOOTSTRAP_SOLVER_PROTOCOL")
    if prot is None or (isinstance(prot, str) and prot == "default"):
        prot = default
    elif isinstance(prot, str) and prot == "robust":
        prot = const("ROBUST_SOLVER_PROTOCOL")
    elif isinstance(prot, str) and prot == "jax":
        prot = const("JAX_SOLVER_PROTOCOL")
    elif any(not isinstance(st, dict) for st in prot):
        prot = default
    return fb.solver_protocol(prot)


def _mbar_bootstraps(mbar, n_bootstraps, members, arguments):
    """f_k_boots of mbar.py:417-449 after the original constructor ran with n_bootstraps=0.  The replicates are drawn
    from mbar.rng as the reference draws them; each is one weighted solve on the resident problem of mbar.u_kn
    (bootstrap.bootstrap_f_k), started at mbar.f_k or, under initialize="BAR", at BAR on the replicate's columns.  A
    replicate whose device solve raises is solved the original way, on the gathered u_kn[:, rints]."""
    import logging

    from . import _lib
    from . import bootstrap as bs
    from . import initialize as init
    from . import mbar_solvers as ms

    N_k = np.asarray(mbar.N_k, dtype=np.int64)
    protocol = _bootstrap_protocol(mbar, arguments.get("bootstrap_solver_protocol"))
    f_k = np.array(mbar.f_k, dtype=np.float64)
    bar = arguments.get("initialize") == "BAR"
    verbose = arguments.get("verbose")
    maxfrac = int(max((1, 0.1 * n_bootstraps)))
    log = logging.getLogger(type(mbar).__module__)
    boots = np.zeros((n_bootstraps, len(N_k)))
    with ms._borrow(mbar.u_kn, N_k.astype(np.float64)) as p:
        def solve(b, rints):
            start = init.initialize_with_bar(mbar.u_kn, N_k, mbar.x_kindices, f_k, columns=rints) if bar else f_k
            try:
                boots[b] = bs.bootstrap_f_k(p, start, N_k, rints=rints[None], solver_protocol=protocol)[0]
                STATS["mbar_boot_solves"] += 1
            except _lib.MbarB200Error:
                STATS["mbar_boot_fallbacks"] += 1
                boots[b] = _solver_module(mbar).solve_mbar_for_all_states(
                    mbar.u_kn[:, rints], mbar.N_k, np.array(start), np.flatnonzero(N_k > 0), protocol)
            if verbose and b % maxfrac == 0:
                log.info(f"Calculated {b + 1:d}/{n_bootstraps:d} bootstrap samples")

        states, counts = bs.draw_mbar_replicates(mbar.rng, N_k, members, n_bootstraps, solve)
    mbar.n_bootstraps = n_bootstraps
    mbar.f_k_boots = boots
    mbar.__dict__["_b200_rints"] = RintsTicket(mbar.rng, states, N_k, members)
    mbar.__dict__["_b200_boot_counts"] = counts


def _replicate_counts(mbar):
    """counts [B, N] of the replicates behind mbar.f_k_boots: the constructor's, or the multiplicities of whatever was
    assigned to bootstrap_rints; None when one exceeds 65535."""
    if "_b200_boot_counts" in mbar.__dict__:
        return mbar.__dict__["_b200_boot_counts"]
    rints = np.asarray(mbar.bootstrap_rints)
    counts = np.stack([np.bincount(r, minlength=int(mbar.N)) for r in rints])
    return counts if counts.max(initial=0) <= 65535 else None


def install_on(MBAR):
    """Patch the class object `MBAR` (pymbar.mbar.MBAR)."""
    if MBAR in _SAVED:
        return
    saved = {name: MBAR.__dict__.get(name) for name in
             ("__init__", "Log_W_nk", "compute_effective_sample_number", "compute_overlap",
              "compute_free_energy_differences", "compute_expectations_inner", "_initialize_with_bar",
              "_computeUnnormalizedLogWeights", "bootstrap_rints")}
    _SAVED[MBAR] = saved
    orig_init = saved["__init__"]
    orig_fed = saved["compute_free_energy_differences"]
    orig_inner = saved["compute_expectations_inner"]
    import inspect

    try:
        init_sig = inspect.signature(orig_init)
    except (TypeError, ValueError):
        init_sig = None

    def _bootstrap_request(self, args, kwargs):
        """(bound arguments, B, members) when the device draws and solves the replicates: n_bootstraps a positive
        int (not bool) and x_kindices a labelling for which the reference's draws are defined; else None."""
        from . import bootstrap as bs

        if init_sig is None or "n_bootstraps" not in init_sig.parameters:
            return None
        try:
            bound = init_sig.bind(self, *args, **kwargs)
        except TypeError:
            return None
        bound.apply_defaults()
        n = bound.arguments["n_bootstraps"]
        if not isinstance(n, (int, np.integer)) or isinstance(n, bool) or n <= 0:
            return None
        try:
            N_k = np.array(bound.arguments["N_k"], dtype=np.int64)
            x = bound.arguments.get("x_kindices")
            x = np.repeat(np.arange(len(N_k)), N_k) if x is None else x
            members = bs.state_members(N_k, x)
        except (TypeError, ValueError):
            return None
        return None if members is None else (bound, int(n), members)

    def __init__(self, *args, **kwargs):
        boot = _bootstrap_request(self, args, kwargs)
        if boot is not None:
            bound = boot[0]
            bound.arguments["n_bootstraps"] = 0
            args, kwargs = bound.args[1:], bound.kwargs
        _TLS.defer = getattr(_TLS, "defer", 0) + 1
        try:
            orig_init(self, *args, **kwargs)
        finally:
            _TLS.defer -= 1
        if boot is not None:
            _mbar_bootstraps(self, boot[1], boot[2], boot[0].arguments)

    def _get_rints(self):
        try:
            v = self.__dict__["_b200_rints"]
        except KeyError:
            raise AttributeError(f"{type(self).__name__!r} object has no attribute 'bootstrap_rints'") from None
        if isinstance(v, RintsTicket):
            v = v.redeem()
            self.__dict__["_b200_rints"] = v
        return v

    def _set_rints(self, value):
        self.__dict__["_b200_rints"] = value
        self.__dict__.pop("_b200_boot_counts", None)

    def _get_logw(self):
        v = self.__dict__.get("_b200_logw")
        if isinstance(v, LogWeightTicket):
            v = v.redeem()
            self.__dict__["_b200_logw"] = v
        return v

    def _set_logw(self, value):
        self.__dict__["_b200_logw"] = value

    def compute_effective_sample_number(self, verbose=False):
        _, G = _moments(self)
        n_eff = est.effective_sample_number(G)
        if verbose:
            import logging

            log = logging.getLogger("pymbar.mbar")
            for k in range(self.K):
                log.info("Effective number of sample in state {:d} is {:10.3f}".format(k, n_eff[k]))
                log.info("Efficiency for state {:d} is {:6f}/{:d} = {:10.4f}".format(k, n_eff[k], self.N,
                                                                                     n_eff[k] / self.N))
        return n_eff

    def compute_overlap(self):
        _, G = _moments(self)
        return est.overlap(G, self.N_k)

    def compute_free_energy_differences(self, compute_uncertainty=True, uncertainty_method=None,
                                        warning_cutoff=1.0e-10, return_theta=False):
        # bootstrap: the spread of the replicates' differences (mbar.py:706-714), Theta from the device's moments
        boot = uncertainty_method == "bootstrap" and getattr(self, "f_k_boots", None) is not None
        device_ok = uncertainty_method in (None, "svd-ew", "approximate") or boot
        if not device_ok and (compute_uncertainty or return_theta):
            return orig_fed(self, compute_uncertainty=compute_uncertainty, uncertainty_method=uncertainty_method,
                            warning_cutoff=warning_cutoff, return_theta=return_theta)
        Delta = np.array(self.f_k - np.vstack(self.f_k))
        self._zerosamestates(Delta)
        out = {"Delta_f": Delta}
        if boot and compute_uncertainty:
            F = np.asarray(self.f_k_boots)
            out["dDelta_f"] = np.std(F[:, None, :] - F[:, :, None], axis=0)
        if return_theta or (compute_uncertainty and not boot):
            S, G = _moments(self)
            _check_normalised(S)
            Theta = est.asymptotic_covariance(G, self.N_k, method=uncertainty_method)
            if compute_uncertainty and not boot:
                d = np.array(est.error_of_differences(Theta, warning_cutoff=warning_cutoff))
                self._zerosamestates(d)
                out["dDelta_f"] = d
            if return_theta:
                out["Theta"] = Theta
        return out

    def compute_expectations_inner(self, A_n, u_ln, state_map, uncertainty_method=None, warning_cutoff=1.0e-10,
                                   return_theta=False):
        boot = uncertainty_method == "bootstrap" and getattr(self, "f_k_boots", None) is not None
        if uncertainty_method not in (None, "svd-ew", "approximate") and not boot:
            return orig_inner(self, A_n, u_ln, state_map, uncertainty_method=uncertainty_method,
                              warning_cutoff=warning_cutoff, return_theta=return_theta)
        from . import _lib
        from . import expectations as ex
        from . import mbar_solvers as ms

        def fallback():
            STATS["expectations_fallbacks"] += 1
            return orig_inner(self, A_n, u_ln, state_map, uncertainty_method=uncertainty_method,
                              warning_cutoff=warning_cutoff, return_theta=return_theta)

        # the augmented problem holds K + one row per state of interest + one per (state, observable) pair; past
        # what a context takes, the original answers (checked up front: ERR_INVALID may also mean a bad argument)
        if ex.augmented_states(np.shape(self.u_kn)[0], state_map) > _lib.MAX_STATES:
            return fallback()
        if not boot:
            STATS["expectations"] += 1
            return ex.expectations_inner(self.u_kn, self.N_k, self.f_k, A_n, u_ln, state_map,
                                         uncertainty_method=uncertainty_method, return_theta=return_theta,
                                         device=ms._DEVICE)
        # bootstrap: every replicate's appended rows from one replicate_unsampled call (mbar.py:890-971)
        counts = _replicate_counts(self)
        if counts is None:
            return fallback()
        try:
            out = ex.expectations_inner(self.u_kn, self.N_k, self.f_k, A_n, u_ln, state_map,
                                        uncertainty_method=uncertainty_method, return_theta=return_theta,
                                        device=ms._DEVICE, replicates=(self.f_k_boots, counts))
        except _lib.MbarB200Error:
            return fallback()
        STATS["expectations_boot"] += 1
        return out

    def _initialize_with_bar(self, u_kn, f_k_init=None):
        from . import initialize as init

        return init.initialize_with_bar(u_kn, self.N_k, self.x_kindices, f_k_init)

    def _computeUnnormalizedLogWeights(self, u_n):
        return _device_log_weights(self, u_n)

    MBAR._computeUnnormalizedLogWeights = _computeUnnormalizedLogWeights
    MBAR._initialize_with_bar = _initialize_with_bar
    MBAR.__init__ = __init__
    MBAR.Log_W_nk = property(_get_logw, _set_logw, doc="log weights [N, K] (mbar.py:455), downloaded on first use")
    MBAR.bootstrap_rints = property(_get_rints, _set_rints,
                                    doc="bootstrap indices [B, N] (mbar.py:423-445), regenerated on first use")
    MBAR.compute_effective_sample_number = compute_effective_sample_number
    MBAR.compute_overlap = compute_overlap
    MBAR.compute_free_energy_differences = compute_free_energy_differences
    MBAR.compute_expectations_inner = compute_expectations_inner


class WeightMatrixTicket:
    """Stands for FES.w_kn = np.exp(mbar.Log_W_nk) (fes.py:416) until somebody reads it."""

    __slots__ = ("mbar",)

    def __init__(self, mbar):
        self.mbar = mbar

    def redeem(self):
        STATS["fes_w_kn"] += 1
        return np.exp(self.mbar.Log_W_nk)


def _out_of_range(err):
    from . import _lib

    return isinstance(err, _lib.MbarB200Error) and err.status == -6     # MBAR_B200_ERR_RANGE


def _drop_device_kde(fes):
    dev = fes.__dict__.pop("_b200_kde_dev", None)
    if dev is not None and hasattr(dev[0], "close"):
        dev[0].close()


def _device_kde(fes, x_n):
    """The KDE of fes.py:650-699 (b = 0) for the device: upload x_n and fes.w_n to a DeviceKde and leave FES.kde
    unfitted until something reads it.  False when the device does not serve these parameters or cannot take the
    samples; the caller then fits sklearn's tree as the reference does."""
    from . import _lib
    from . import fes as hist
    from . import mbar_solvers as ms

    if np.ndim(x_n) == 1 and not hasattr(x_n, "reshape"):
        return False                    # fes.py:677 reshapes 1-D samples with x_n.reshape: let the original raise
    x = np.asarray(x_n)
    if x.ndim == 1:
        x = x.reshape(-1, 1)
    kde = fes.__dict__.get("_b200_kde")
    if x.ndim != 2 or not hasattr(kde, "get_params"):
        return False
    settings = hist.kde_settings(kde.get_params(), x.shape[0], x.shape[1])
    if settings is None:
        return False
    w = fes.w_n
    try:
        dev = ms.DeviceKde(x, w, device=ms._DEVICE)
    except (_lib.MbarB200Error, ValueError, TypeError):
        return False
    fes.__dict__["_b200_kde_dev"] = (dev, settings, float(np.log(np.sum(w))))
    fes.__dict__["_b200_kde_fit"] = (x_n if np.ndim(x_n) != 1 else x, w)
    return True


class SplineMoments:
    """The basis sums of one spline fit: S [K, nb] (or None) and A [nb] (or None) of the samples x_n, weights w_n
    and state labels, for the knots t and degree k, with their sample terms v (fes.spline_sample_terms).  F_k, the
    per-state sums of the bias callables, is computed on first use by the MC likelihood."""

    __slots__ = ("x", "w", "labels", "t", "k", "weights", "S", "A", "N_k", "v", "F_k")

    def __init__(self, x, w, labels, t, k, weights, S, A, N):
        from . import fes as hist

        self.x, self.w, self.labels, self.t, self.k, self.weights, self.S, self.A = x, w, labels, t, k, weights, S, A
        self.N_k = None if S is None else np.bincount(labels, minlength=S.shape[0])
        self.v = hist.spline_sample_terms(S, A, weights, N, self.N_k)
        self.F_k = None

    def serves(self, x_n, w_n, t, k):
        return x_n is self.x and w_n is self.w and k == self.k and np.array_equal(t, self.t)


def _device_spline(fes, x_n):
    """One DeviceBSpline pass over x_n for the knots of fes.spline_data["bspline"] (after _setup_fes_spline and the
    device weights); the moments are kept in fes.__dict__["_b200_spline"].  Nothing is kept for 2-D samples, an
    unknown spline_weights or a device error (NaN samples, labels outside [0, K)): the fit then runs the original
    methods."""
    from . import _lib
    from . import fes as hist
    from . import mbar_solvers as ms

    weights = fes.spline_parameters.get("spline_weights")
    if np.ndim(x_n) != 1 or weights not in hist.SPLINE_WEIGHTS:
        return
    b = fes.spline_data["bspline"]
    t, k = np.array(b.t, dtype=np.float64), int(b.k)
    want_S = weights != "unbiasedstate"
    K = fes.mbar.K
    labels = np.asarray(fes.mbar.x_kindices) if want_S else None
    try:
        dev = ms.DeviceBSpline(np.asarray(x_n, dtype=np.float64), None if want_S else fes.w_n, labels,
                               K=K if want_S else None, device=ms._DEVICE)
        try:
            S, A = dev.moments(t, k, want_S=want_S, want_A=not want_S)
        finally:
            dev.close()
    except (_lib.MbarB200Error, ValueError, TypeError):
        return
    STATS["fes_spline_moments"] += 1
    fes.__dict__["_b200_spline"] = SplineMoments(x_n, fes.w_n, labels, t, k, weights, S, A, fes.N)


class ReplicateSplineTerms:
    """The sample terms v of one bootstrap replicate's spline fit, for the replicate's own x_nb and w_nb arrays (the
    ones passed to _generate_fes_spline) on the fit's knots t and degree k."""

    __slots__ = ("x", "w", "t", "k", "weights", "v")

    def __init__(self, x, w, t, k, weights, v):
        self.x, self.w, self.t, self.k, self.weights, self.v = x, w, t, k, weights, v

    def serves(self, x_n, w_n, t, k):
        return x_n is self.x and w_n is self.w and k == self.k and np.array_equal(t, self.t)


def _spline_moments_for(fes, x_n, w_n, t, k, weights, slot="_b200_spline"):
    m = fes.__dict__.get(slot)
    if m is None or weights != m.weights or not m.serves(x_n, w_n, t, k):
        return None
    return m


def _spline_boot_served(fes, x_n, spline_parameters):
    """True when the device serves the spline replicates: 1-D samples, a known spline_weights, and samples in block
    order (the reference labels replicate positions with b = 0's x_kindices, which are the replicate's samples' own
    labels only in block order)."""
    from . import fes as hist
    from . import fes_bootstrap as fb

    mbar = fes.mbar
    return (np.ndim(x_n) == 1 and isinstance(spline_parameters, dict)
            and spline_parameters.get("spline_weights") in hist.SPLINE_WEIGHTS
            and fb.in_block_order(mbar.x_kindices, mbar.N_k))


def _spline_bootstraps(fes, x_n, u_n, n_bootstraps):
    """fes.fes_functions for n_bootstraps spline replicates (fes.py:388-430, :971-1098).  The replicates are drawn as
    the reference draws them; "unbiasedstate" runs one weighted solve per replicate on the resident problem for its
    log denominators, the other weightings none.  One DeviceBSpline.replicate_sums call gives every replicate's sample
    terms, and each replicate is then fitted by fes._generate_fes_spline(b, x_nb, w_nb) with its objective and
    gradient answered from them.  False, with numpy's generator advanced, when the device refuses: the caller then
    restores the generator and runs the original."""
    from . import _lib
    from . import fes_bootstrap as fb
    from . import mbar_solvers as ms
    from .bootstrap import bootstrap_f_k

    mbar = fes.mbar
    N_k = np.asarray(mbar.N_k)
    weights = fes.spline_parameters["spline_weights"]
    spline = fes.spline_data["bspline"]
    t, k = np.array(spline.t, dtype=np.float64), int(spline.k)
    f_k = np.asarray(mbar.f_k, dtype=np.float64)
    times = {"solves": 0.0}
    try:
        start = _timer()
        with ms._borrow(mbar.u_kn, np.asarray(N_k, dtype=np.float64)) as p:
            if weights == "unbiasedstate" and not hasattr(p, "set_sample_weights"):
                return False                    # a backend without multiplicities (the tests' stand-in)
            protocol = fb.solver_protocol(ms.DEFAULT_SOLVER_PROTOCOL)

            def log_weights(idx):
                t0 = _timer()
                f_b = bootstrap_f_k(p, f_k, N_k, rints=idx[None], solver_protocol=protocol)[0]
                L = p.log_denominator(f_b)
                STATS["fes_boot_spline_solves"] += 1
                times["solves"] += _timer() - t0
                return -u_n - L

            states, V = fb.spline_replicates(N_k, n_bootstraps, weights, log_weights)
        times["draws"] = _timer() - start - times["solves"]
        start = _timer()
        dev = ms.DeviceBSpline(np.asarray(x_n, dtype=np.float64), device=ms._DEVICE)
        try:
            if not hasattr(dev, "replicate_sums"):
                return False                    # a backend without replicates (the tests' plain numpy stand-in)
            dev.set_replicates(V)
            R = dev.replicate_sums(t, k)
            times["sums_kernel_ms"] = dev.last_stats()["ms"] if hasattr(dev, "last_stats") else None
        finally:
            dev.close()
    except (_lib.MbarB200Error, ValueError, TypeError):
        return False
    STATS["fes_boot_spline_sums"] += 1
    times["sums"] = _timer() - start
    v = fes.N * R if weights == "unbiasedstate" else R
    start = _timer()
    try:
        for b, state in enumerate(states):
            x_nb, w_nb = fb.spline_replicate_samples(state, N_k, x_n, V[b], weights)
            fes.__dict__["_b200_spline_replicate"] = ReplicateSplineTerms(x_nb, w_nb, t, k, weights, v[b])
            fes._generate_fes_spline(b + 1, x_nb, w_nb)
    finally:
        fes.__dict__.pop("_b200_spline_replicate", None)
    times["fits"] = _timer() - start
    fes.__dict__["_b200_spline_boot_times"] = times
    return True


def _histogram_bootstraps(fes, u_n, n_bootstraps):
    """fes.histogram_datas for n_bootstraps replicates (fes.py:388-430), each one weighted solve and one bin pass on
    the resident problem.  False, with numpy's generator advanced, when a replicate empties a bin tuple of b = 0 or
    the device fails: the caller then restores the generator and runs the original."""
    from . import _lib
    from . import fes_bootstrap as fb
    from . import mbar_solvers as ms

    mbar = fes.mbar
    N_k = np.asarray(mbar.N_k)
    tuples, n_tuples = fb.tuple_index(fes.histogram_data["bin_n"])
    covered = []
    states = fb.draw_replicates(N_k, n_bootstraps,
                                lambda b, idx: covered.append(fb.covers_every_tuple(idx, tuples, n_tuples)))
    if not all(covered):
        return False
    protocol = fb.solver_protocol(ms.DEFAULT_SOLVER_PROTOCOL)

    def solved():
        STATS["fes_boot_solves"] += 1

    try:
        with ms._borrow(mbar.u_kn, np.asarray(N_k, dtype=np.float64)) as p:
            if not hasattr(p, "set_sample_weights"):      # a backend without multiplicities (the tests' stand-in)
                return False
            datas = fb.histogram_replicates(p, np.asarray(mbar.f_k, dtype=np.float64), N_k, u_n,
                                            fes.histogram_data, states, protocol, on_solve=solved)
    except _lib.MbarB200Error:
        return False
    fes.histogram_datas = datas
    return True


def _kde_bootstraps(fes, x_n, n_bootstraps):
    """The replicate weights V [B, N] of n_bootstraps KDE replicates (fes.py:388-430, :689-699) on fes's DeviceKde,
    and fes.kdes as a ReplicateKdes.  False, with numpy's generator advanced, when the device refuses them."""
    from . import _lib
    from . import fes_bootstrap as fb

    dev = fes.__dict__["_b200_kde_dev"][0]
    if not hasattr(dev, "set_replicates"):         # a KDE backend without replicates (the tests' numpy stand-in)
        return False
    N_k = np.asarray(fes.mbar.N_k)
    w = np.asarray(fes.w_n, dtype=np.float64)
    V = np.empty((int(n_bootstraps), len(w)))

    def weights(b, idx):
        V[b] = np.bincount(idx, weights=w, minlength=len(w))

    states = fb.draw_replicates(N_k, n_bootstraps, weights)
    try:
        dev.set_replicates(V)
    except (_lib.MbarB200Error, ValueError):
        return False

    def fitted():
        STATS["fes_kde_fits"] += 1

    fes.kdes = fb.ReplicateKdes(fes.__dict__["_b200_kde"].get_params(), x_n, fes.w_n, N_k, states, on_fit=fitted)
    return True


def install_fes_on(FES):
    """Patch the class object `FES` (pymbar.fes.FES)."""
    if FES in _SAVED:
        return
    saved = {name: FES.__dict__.get(name) for name in ("generate_fes", "_get_fes_histogram", "w_kn", "_get_fes_kde",
                                                         "kde", "_bspline_calculate_f", "_bspline_calculate_g",
                                                         "_get_MC_loglikelihood")}
    _SAVED[FES] = saved
    orig_generate = saved["generate_fes"]
    orig_get_hist = saved["_get_fes_histogram"]
    orig_get_kde = saved["_get_fes_kde"]
    # the class's own spline methods, or those it inherits
    orig_spline_f = FES._bspline_calculate_f if hasattr(FES, "_bspline_calculate_f") else None
    orig_spline_g = FES._bspline_calculate_g if hasattr(FES, "_bspline_calculate_g") else None
    orig_mc_ll = FES._get_MC_loglikelihood if hasattr(FES, "_get_MC_loglikelihood") else None

    def generate_fes(self, u_n, x_n, fes_type="histogram", histogram_parameters=None, kde_parameters=None,
                     spline_parameters=None, n_bootstraps=0, seed=-1):
        args = (u_n, x_n, fes_type, histogram_parameters, kde_parameters, spline_parameters, n_bootstraps, seed)
        # a DeviceKde, or spline moments, answer only for the surface the last generate_fes built
        _drop_device_kde(self)
        self.__dict__.pop("_b200_spline", None)
        self.__dict__.pop("_b200_spline_boot_times", None)
        counted = isinstance(n_bootstraps, (int, np.integer)) and not isinstance(n_bootstraps, bool)
        boot = counted and n_bootstraps >= 2
        if not (boot or (counted and n_bootstraps == 0)) or fes_type not in ("histogram", "kde", "spline"):
            return orig_generate(self, *args)
        entry = np.random.get_state() if boot else None
        restore = []

        def fallback():
            # the original from where the caller left numpy's generator (the same replicates, the same errors) and
            # with the spline_parameters it was given (_setup_fes_spline edits them in place)
            STATS["fes_boot_fallbacks"] += 1
            _drop_device_kde(self)
            self.__dict__.pop("_b200_spline", None)
            for undo in restore:
                undo()
            np.random.set_state(entry)
            return orig_generate(self, *args)

        # randint(0, 0) raises for an empty state, and the reference indexes x_n with the replicate's indices
        if boot and (not isinstance(x_n, np.ndarray) or np.any(np.asarray(self.mbar.N_k) < 1)):
            return fallback()
        if boot and fes_type == "spline":
            if not _spline_boot_served(self, x_n, spline_parameters):
                return fallback()
            given = {key: (dict(v) if isinstance(v, dict) else v) for key, v in spline_parameters.items()}

            def undo_setup():
                spline_parameters.clear()
                spline_parameters.update(given)

            restore.append(undo_setup)
        from . import fes as hist
        from . import mbar_solvers as ms
        from .utils import kn_to_n

        # fes.py:335-438 for the one, non-bootstrap, sample set
        result_vals = {}
        self.fes_type = fes_type
        if len(np.shape(u_n)) == 2:
            u_n = kn_to_n(u_n, N_k=self.N_k)
        self.u_n = u_n
        if seed >= 0:
            np.random.seed(seed)
        self.n_bootstraps = n_bootstraps
        timings = getattr(self, "timings", False)
        start = _timer() if timings else None
        self.fes_function = list()
        self.mc_data = None
        if fes_type == "histogram":
            self._setup_fes_histogram(histogram_parameters)
        elif fes_type == "kde":
            self._setup_fes_kde(kde_parameters)
        else:
            self._setup_fes_spline(spline_parameters)
        mbar = self.mbar
        f_k = np.asarray(mbar.f_k, dtype=np.float64)
        u = np.asarray(u_n, dtype=np.float64)
        try:
            log_w = _device_log_weights(mbar, u)
            if fes_type == "histogram":
                with ms._borrow(mbar.u_kn, np.asarray(mbar.N_k, dtype=np.float64)) as p:
                    data = hist.histogram_fes(p, f_k, u, x_n, self.histogram_parameters["bin_edges"])
                STATS["fes_histograms"] += 1
        except Exception as err:
            if _out_of_range(err):
                return fallback() if boot else orig_generate(self, *args)
            raise
        w_n = np.exp(log_w - np.max(log_w))
        self.w_n = w_n / np.sum(w_n)
        self.w_kn = WeightMatrixTicket(mbar)
        if fes_type == "histogram":
            self.histogram_data = data
            if boot and not _histogram_bootstraps(self, u, n_bootstraps):
                return fallback()
        elif fes_type == "kde":
            if not _device_kde(self, x_n):
                if boot:
                    return fallback()
                self._generate_fes_kde(0, x_n, self.w_n)
            elif boot and not _kde_bootstraps(self, x_n, n_bootstraps):
                return fallback()
        else:
            _device_spline(self, x_n)
            if boot and "_b200_spline" not in self.__dict__:
                return fallback()
            self._generate_fes_spline(0, x_n, self.w_n)
            if boot and not _spline_bootstraps(self, x_n, u, n_bootstraps):
                return fallback()
        if timings:
            result_vals["timing"] = _timer() - start
        return result_vals

    def _get_fes_histogram(self, x, reference_point="from-lowest", fes_reference=None, uncertainty_method=None):
        from . import fes_bootstrap as fb

        boot = uncertainty_method == "bootstrap"
        datas = getattr(self, "histogram_datas", None)
        served = boot and isinstance(datas, list) and len(datas) > 0 and \
            all(isinstance(h, fb.ReplicateHistogram) for h in datas)
        if (uncertainty_method not in (None, "analytical") and not served) or \
                reference_point not in ("from-lowest", "from-specified"):
            if boot:
                STATS["fes_boot_fallbacks"] += 1
            return orig_get_hist(self, x, reference_point=reference_point, fes_reference=fes_reference,
                                 uncertainty_method=uncertainty_method)
        from . import fes as hist
        from . import mbar_solvers as ms

        mbar = self.mbar
        K = mbar.K

        if boot:
            def df_fn(j):
                return fb.bootstrap_df(datas, j, len(self.histogram_data["f"]))

            return hist.query(self.histogram_data, x, reference_point, fes_reference, df_fn)

        def df_fn(j):
            STATS["fes_theta"] += 1
            with ms._borrow(mbar.u_kn, np.asarray(mbar.N_k, dtype=np.float64)) as p:
                Theta, S, _ = hist.histogram_theta(p, np.asarray(mbar.f_k, dtype=np.float64), mbar.N_k,
                                                   np.asarray(self.u_n, dtype=np.float64), self.histogram_data,
                                                   return_moments=True)
            _check_normalised(S)
            return hist.bin_uncertainties(Theta, K, j, len(self.histogram_data["f"]))

        try:
            return hist.query(self.histogram_data, x, reference_point, fes_reference,
                              df_fn if uncertainty_method == "analytical" else None)
        except Exception as err:
            if _out_of_range(err):
                return orig_get_hist(self, x, reference_point=reference_point, fes_reference=fes_reference,
                                     uncertainty_method=uncertainty_method)
            raise

    def _get_fes_kde(self, x, reference_point="from-normalization", fes_reference=None, uncertainty_method=None):
        dev = self.__dict__.get("_b200_kde_dev")
        if dev is not None and uncertainty_method is None:
            from . import _lib
            from . import fes as hist

            kde, settings, log_sum_w = dev
            try:
                out = hist.kde_query(kde, settings, x, reference_point, fes_reference, log_sum_w)
            except _lib.MbarB200Error:
                out = None
            if out is not None:
                STATS["fes_kde_queries"] += 1
                return out
        if uncertainty_method == "bootstrap":
            from . import _lib
            from . import fes_bootstrap as fb

            kdes = getattr(self, "kdes", None)
            if (dev is not None and reference_point in ("from-lowest", "from-specified")
                    and isinstance(kdes, fb.ReplicateKdes) and dev[0].B == len(kdes)):
                try:
                    out = fb.kde_bootstrap_query(dev[0], dev[1], x, reference_point, fes_reference, dev[2])
                except _lib.MbarB200Error:
                    out = None
                if out is not None:
                    STATS["fes_boot_passes"] += 1
                    return out
            STATS["fes_boot_fallbacks"] += 1
        return orig_get_kde(self, x, reference_point=reference_point, fes_reference=fes_reference,
                            uncertainty_method=uncertainty_method)

    def _fit_moments(self, x_n, w_n):
        # b = 0's moments, or the sample terms of the bootstrap replicate being fitted
        b = self.spline_data["bspline"]
        weights = self.spline_parameters.get("spline_weights")
        m = _spline_moments_for(self, x_n, w_n, b.t, b.k, weights)
        if m is None:
            m = _spline_moments_for(self, x_n, w_n, b.t, b.k, weights, slot="_b200_spline_replicate")
        return m

    def _bspline_calculate_f(self, xi, x_n, w_n):
        m = _fit_moments(self, x_n, w_n)
        if m is None:
            return orig_spline_f(self, xi, x_n, w_n)
        from . import fes as hist

        STATS["fes_spline_calls"] += 1
        return hist.spline_objective(self, xi, m.v)

    def _bspline_calculate_g(self, xi, x_n, w_n):
        m = _fit_moments(self, x_n, w_n)
        if m is None:
            return orig_spline_g(self, xi, x_n, w_n)
        from . import fes as hist

        STATS["fes_spline_calls"] += 1
        return hist.spline_gradient(self, xi, m.v)

    def _get_MC_loglikelihood(self, x_n, w_n, spline_weights, spline, xrange):
        m = _spline_moments_for(self, x_n, w_n, spline.t, spline.k, spline_weights)
        if m is None:
            return orig_mc_ll(self, x_n, w_n, spline_weights, spline, xrange)
        from . import fes as hist

        if m.S is not None and m.F_k is None:
            m.F_k = hist.state_bias_sums(self.spline_parameters["fkbias"], m.x, m.labels, m.S.shape[0])
        STATS["fes_spline_calls"] += 1
        return hist.spline_mc_loglikelihood(self, spline, spline_weights, xrange, m.S, m.A, m.F_k, m.N_k)

    def _get_kde(self):
        try:
            kde = self.__dict__["_b200_kde"]
        except KeyError:
            raise AttributeError(f"{type(self).__name__!r} object has no attribute 'kde'") from None
        pending = self.__dict__.pop("_b200_kde_fit", None)
        if pending is not None:
            STATS["fes_kde_fits"] += 1
            kde.fit(pending[0], sample_weight=pending[1])
        return kde

    def _set_kde(self, value):
        self.__dict__["_b200_kde"] = value
        self.__dict__.pop("_b200_kde_fit", None)

    def _get_w_kn(self):
        v = self.__dict__.get("_b200_w_kn")
        if isinstance(v, WeightMatrixTicket):
            v = v.redeem()
            self.__dict__["_b200_w_kn"] = v
        return v

    def _set_w_kn(self, value):
        self.__dict__["_b200_w_kn"] = value

    FES.generate_fes = generate_fes
    FES._get_fes_histogram = _get_fes_histogram
    FES._get_fes_kde = _get_fes_kde
    if orig_spline_f is not None:
        FES._bspline_calculate_f = _bspline_calculate_f
        FES._bspline_calculate_g = _bspline_calculate_g
    if orig_mc_ll is not None:
        FES._get_MC_loglikelihood = _get_MC_loglikelihood
    FES.kde = property(_get_kde, _set_kde, doc="the sklearn KernelDensity (fes.py:648), fitted on first use")
    FES.w_kn = property(_get_w_kn, _set_w_kn, doc="weights [N, K] of all states (fes.py:416), computed on first use")


def _ts_series(x, need_array=False):
    """x as the device takes it: a 1-D float64 or integer array (a list becomes one), else None."""
    if need_array and not isinstance(x, np.ndarray):
        return None
    a = np.asarray(x)
    if a.ndim != 1 or a.size == 0 or not (a.dtype == np.float64 or a.dtype.kind in "iu"):
        return None
    return a


def install_timeseries_on(module):
    """Patch the module object `module` (pymbar.timeseries)."""
    if module in _SAVED:
        return
    names = ("statistical_inefficiency", "statistical_inefficiency_multiple",
             "normalized_fluctuation_correlation_function", "detect_equilibration",
             "normalized_fluctuation_correlation_function_multiple", "statistical_inefficiency_fft",
             "detect_equilibration_binary_search")
    saved = {name: module.__dict__.get(name) for name in names}
    _SAVED[module] = saved
    orig_si, orig_multi, orig_corr, orig_eq, orig_corr_multi, orig_fft, orig_bs = (saved[n] for n in names)

    def _fallback(fn, *args, **kwargs):
        STATS["ts_fallbacks"] += 1
        return fn(*args, **kwargs)

    def statistical_inefficiency(A_n, B_n=None, fast=False, mintime=3, fft=False):
        args = (A_n, B_n, fast, mintime, fft)
        if fft or _ts_series(A_n) is None or (B_n is not None and _ts_series(B_n) is None):
            return _fallback(orig_si, *args)
        from . import _lib
        from . import timeseries as ts

        try:
            g = ts.statistical_inefficiency(A_n, B_n, fast=fast, mintime=mintime)
        except _lib.MbarB200Error:
            return _fallback(orig_si, *args)
        STATS["ts_inefficiency"] += 1
        return g

    def statistical_inefficiency_multiple(A_kn, fast=False, return_correlation_function=False):
        args = (A_kn, fast, return_correlation_function)
        from . import _lib
        from . import timeseries as ts
        from . import utils as u

        if isinstance(A_kn, np.ndarray):
            ok = A_kn.ndim in (1, 2) and _ts_series(A_kn.ravel()) is not None
        else:
            ok = all(_ts_series(x, need_array=True) is not None for x in A_kn) and len(A_kn) > 0
        if not ok:
            return _fallback(orig_multi, *args)
        try:
            out = ts.statistical_inefficiency_multiple(A_kn, fast=fast,
                                                       return_correlation_function=return_correlation_function)
        except (_lib.MbarB200Error, u.ParameterError):
            return _fallback(orig_multi, *args)
        STATS["ts_multiple"] += 1
        return out

    def normalized_fluctuation_correlation_function(A_n, B_n=None, N_max=None, norm=True):
        args = (A_n, B_n, N_max, norm)
        if _ts_series(A_n) is None or (B_n is not None and _ts_series(B_n) is None):
            return _fallback(orig_corr, *args)
        from . import _lib
        from . import timeseries as ts

        try:
            C = ts.normalized_fluctuation_correlation_function(A_n, B_n, N_max=N_max, norm=norm)
        except _lib.MbarB200Error:
            return _fallback(orig_corr, *args)
        STATS["ts_correlation"] += 1
        return C

    def detect_equilibration(A_t, fast=True, nskip=1):
        args = (A_t, fast, nskip)
        if _ts_series(A_t, need_array=True) is None or not isinstance(nskip, (int, np.integer)) or nskip < 1:
            return _fallback(orig_eq, *args)
        from . import _lib
        from . import timeseries as ts

        try:
            out = ts.detect_equilibration(A_t, fast=fast, nskip=nskip)
        except _lib.MbarB200Error:
            return _fallback(orig_eq, *args)
        STATS["ts_equilibration"] += 1
        return out

    # the three below: ts raises NotOnDevice where the reference's answer is not reproducible (constant remaining
    # series, unsupported input); the original then answers, or raises as it does without statsmodels
    def normalized_fluctuation_correlation_function_multiple(A_kn, B_kn=None, N_max=None, norm=True,
                                                             truncate=False):
        args = (A_kn, B_kn, N_max, norm, truncate)
        from . import _lib
        from . import timeseries as ts

        try:
            C = ts.normalized_fluctuation_correlation_function_multiple(A_kn, B_kn, N_max=N_max, norm=norm,
                                                                        truncate=truncate)
        except (_lib.MbarB200Error, ts.NotOnDevice):
            return _fallback(orig_corr_multi, *args)
        STATS["ts_correlation_multiple"] += 1
        return C

    def statistical_inefficiency_fft(A_n, mintime=3):
        args = (A_n, mintime)
        from . import _lib
        from . import timeseries as ts

        try:
            g = ts.statistical_inefficiency_fft(A_n, mintime=mintime)
        except (_lib.MbarB200Error, ts.NotOnDevice):
            return _fallback(orig_fft, *args)
        STATS["ts_fft"] += 1
        return g

    def detect_equilibration_binary_search(A_t, bs_nodes=10):
        args = (A_t, bs_nodes)
        from . import _lib
        from . import timeseries as ts

        try:
            out = ts.detect_equilibration_binary_search(A_t, bs_nodes=bs_nodes)
        except (_lib.MbarB200Error, ts.NotOnDevice):
            return _fallback(orig_bs, *args)
        STATS["ts_binary_search"] += 1
        return out

    for name, fn in zip(names, (statistical_inefficiency, statistical_inefficiency_multiple,
                                normalized_fluctuation_correlation_function, detect_equilibration,
                                normalized_fluctuation_correlation_function_multiple, statistical_inefficiency_fft,
                                detect_equilibration_binary_search)):
        if saved[name] is not None:
            fn.__doc__ = saved[name].__doc__
            setattr(module, name, fn)


OE_NAMES = ("bar", "bar_zero", "exp", "exp_gauss")


def _oe_work(x):
    """x if the device takes it as the reference computes it: a non-empty 1-D float64 ndarray, or a signed integer one
    (32 or 64 bit) whose values, and -w - max(-w), are exact in fp64; else None."""
    if not isinstance(x, np.ndarray) or x.ndim != 1 or x.size == 0:
        return None
    if x.dtype == np.float64:
        return x
    if x.dtype.kind == "i" and x.dtype.itemsize in (4, 8):
        lim = min(2 ** 52, 2 ** (8 * x.dtype.itemsize - 3))
        if int(x.min()) >= -lim and int(x.max()) <= lim:
            return x
    return None


def install_other_estimators_on(module):
    """Patch the module object `module` (pymbar.other_estimators): bar, bar_zero, exp and exp_gauss."""
    if module in _SAVED:
        return
    saved = {name: module.__dict__.get(name) for name in OE_NAMES}
    _SAVED[module] = saved
    orig_bar, orig_zero, orig_exp, orig_gauss = (saved[n] for n in OE_NAMES)

    def _fallback(fn, *args):
        STATS["oe_fallbacks"] += 1
        return fn(*args)

    def _device_call(counter, fn, *args, **kwargs):
        """fn on the device; None when the device refuses the input.  The reference's own exceptions are raised as the
        patched module's classes."""
        from . import _lib
        from . import other_estimators as oe
        from . import utils as u

        n0 = oe.EVALUATIONS[0]
        try:
            out = fn(*args, **kwargs)
        except _lib.MbarB200Error:
            return None
        except (u.ParameterError, u.ConvergenceError, u.BoundsError) as e:
            for name in ("ParameterError", "ConvergenceError", "BoundsError"):
                theirs = module.__dict__.get(name)
                if isinstance(e, getattr(u, name)) and isinstance(theirs, type) and not isinstance(e, theirs):
                    raise theirs(*e.args) from None
            raise
        finally:
            STATS["oe_evaluations"] += oe.EVALUATIONS[0] - n0
        STATS[counter] += 1
        return (out,)

    def bar(w_F, w_R, DeltaF=0.0, compute_uncertainty=True, uncertainty_method="BAR", maximum_iterations=500,
            relative_tolerance=1.0e-12, verbose=False, method="false-position", iterated_solution=True):
        from . import other_estimators as oe

        args = (w_F, w_R, DeltaF, compute_uncertainty, uncertainty_method, maximum_iterations, relative_tolerance,
                verbose, method, iterated_solution)
        solver = method if iterated_solution else "self-consistent-iteration"
        if (verbose or _oe_work(w_F) is None or _oe_work(w_R) is None or not isinstance(solver, str)
                or solver not in oe.METHODS or not isinstance(uncertainty_method, str)
                or uncertainty_method not in oe.UNCERTAINTY_METHODS):
            return _fallback(orig_bar, *args)
        r = _device_call("oe_bar", oe.bar, w_F, w_R, DeltaF=DeltaF, compute_uncertainty=compute_uncertainty,
                         uncertainty_method=uncertainty_method, maximum_iterations=maximum_iterations,
                         relative_tolerance=relative_tolerance, method=method, iterated_solution=iterated_solution)
        return _fallback(orig_bar, *args) if r is None else r[0]

    def bar_zero(w_F, w_R, DeltaF):
        from . import other_estimators as oe

        if _oe_work(w_F) is None or _oe_work(w_R) is None:
            return _fallback(orig_zero, w_F, w_R, DeltaF)
        r = _device_call("oe_bar_zero", oe.bar_zero, w_F, w_R, DeltaF)
        return _fallback(orig_zero, w_F, w_R, DeltaF) if r is None else r[0]

    def exp(w_F, compute_uncertainty=True, is_timeseries=False):
        from . import other_estimators as oe

        args = (w_F, compute_uncertainty, is_timeseries)
        if _oe_work(w_F) is None:
            return _fallback(orig_exp, *args)
        r = _device_call("oe_exp", oe.exp, *args)
        return _fallback(orig_exp, *args) if r is None else r[0]

    def exp_gauss(w_F, compute_uncertainty=True, is_timeseries=False):
        from . import other_estimators as oe

        args = (w_F, compute_uncertainty, is_timeseries)
        if _oe_work(w_F) is None:
            return _fallback(orig_gauss, *args)
        r = _device_call("oe_exp_gauss", oe.exp_gauss, *args)
        return _fallback(orig_gauss, *args) if r is None else r[0]

    for name, fn in zip(OE_NAMES, (bar, bar_zero, exp, exp_gauss)):
        if saved[name] is not None:
            fn.__doc__ = saved[name].__doc__
            setattr(module, name, fn)


def uninstall_from(MBAR):
    saved = _SAVED.pop(MBAR, None)
    if saved is None:
        return
    for name, value in saved.items():
        if value is None:
            if name in MBAR.__dict__:
                delattr(MBAR, name)
        else:
            setattr(MBAR, name, value)

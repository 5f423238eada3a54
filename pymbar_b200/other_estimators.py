"""The host side of pymbar.other_estimators (other_estimators.py:56-719) over the sums of a `DeviceWork`.

`bar_zero`, `bar`, `exp` and `exp_gauss` take the reference's arguments and return what it returns: the same keys,
np.float64 values and a plain 0.0 where the reference returns one.  The device evaluates every sum over the work
values in the reference's fp64 formulas (include/mbar_b200.h, DESIGN.md §3.5e); the host keeps the reference's scalar
arithmetic and control flow: the bracket from the two EXP estimates and its widening, false-position, bisection and
self-consistent iteration, the `FNew == 0` and `DeltaF == 0` exits, the relative-change test, `iterated_solution=False`,
`ConvergenceError` / `BoundsError` with the reference's messages and both uncertainty formulas.  Only the order of
the device's sums differs from numpy's, so a result agrees with the reference to a few ulps of each sum.

`bar` is written as a generator (`_bar_steps`) that yields the sums it needs next and receives them.  `bar_many`
runs the generators of many pairs in lockstep over one `DeviceWork`: one device call per iteration evaluates the
numerator and denominator sums of every active pair.  A pair's iterates depend only on its own sums, and a request's
sums do not depend on the other requests of a call, so each pair's result is the same bits as `bar` on that pair.
"""
from __future__ import annotations

import logging

import numpy as np

from . import utils as _u

logger = logging.getLogger(__name__)

DeviceWork = None          # the device class; resolved on first use (a test may put a stand-in here)

FERMI, FERMI_MOMENTS, EXP, GAUSS = 0, 1, 2, 3       # MBAR_B200_WORK_*
METHODS = ("self-consistent-iteration", "false-position", "bisection")
UNCERTAINTY_METHODS = ("BAR", "MBAR")
EVALUATIONS = [0]          # device calls made by the drivers (the facade reports them)


def _device(vectors):
    global DeviceWork
    from . import mbar_solvers as ms

    if DeviceWork is None:
        DeviceWork = ms.DeviceWork
    return DeviceWork(vectors, device=ms._DEVICE)


def _evaluate(dev, requests):
    """out rows for requests (vector, kind, c1, c2) in one device call."""
    EVALUATIONS[0] += 1
    v, k, a, b = zip(*requests)
    return dev.evaluate(np.array(v), np.array(k), np.array(a, dtype=np.float64), np.array(b, dtype=np.float64))


def _zero_requests(M, DeltaF):
    """bar_zero's numerator (forward vector 0) and denominator (reverse vector 1) sums at DeltaF.

    exp_arg_F = M + w_F - DeltaF = (w_F + M) + (-DeltaF), and exp_arg_R = -(M - w_R - DeltaF) = (w_R + (-M)) + DeltaF
    exactly (round-to-nearest is symmetric), so one kind with two constants serves both."""
    DeltaF = float(DeltaF)
    return [(0, FERMI, M, -DeltaF), (1, FERMI, -M, DeltaF)]


def _zero_steps(M, *DeltaFs):
    """bar_zero at each DeltaF (other_estimators.py:56-153), all in one device call."""
    reqs = []
    for DF in DeltaFs:
        reqs += _zero_requests(M, DF)
    rows = yield reqs
    np.seterr(over="warn")                       # bar_zero leaves numpy's overflow mode at "warn" (:97, :150)
    return [rows[2 * j][0] - rows[2 * j + 1][0] for j in range(len(DeltaFs))]


def _bar_steps(T_F, T_R, DeltaF=0.0, compute_uncertainty=True, uncertainty_method="BAR", maximum_iterations=500,
               relative_tolerance=1.0e-12, method="false-position", iterated_solution=True):
    """bar (other_estimators.py:235-531) for a forward vector 0 of T_F values and a reverse vector 1 of T_R values:
    yields lists of requests (vector, kind, c1, c2), receives their out rows, and returns the result dict."""
    result_vals = dict()
    if not iterated_solution:
        maximum_iterations = 1
        method = "self-consistent-iteration"
        DeltaF_initial = DeltaF

    if method not in ["self-consistent-iteration", "false-position", "bisection"]:
        raise _u.ParameterError("method {} is not defined for bar".format(method))

    if uncertainty_method not in ["BAR", "MBAR"]:
        raise _u.ParameterError("uncertainty_method {:d} is not defined for bar".format(uncertainty_method))

    T_F, T_R = float(T_F), float(T_R)
    M = np.log(T_F / T_R)

    if method == "self-consistent-iteration":
        nfunc = 0

    if method == "bisection" or method == "false-position":
        rows = yield [(0, EXP, 0.0, 0.0), (1, EXP, 0.0, 0.0)]
        UpperB = -(rows[0][0] - np.log(T_F))             # exp(w_F)["Delta_f"]
        LowerB = -(-(rows[1][0] - np.log(T_R)))          # -exp(w_R)["Delta_f"]

        FUpperB, FLowerB = yield from _zero_steps(M, UpperB, LowerB)
        nfunc = 2

        if np.isnan(FUpperB) or np.isnan(FLowerB):
            logger.warning(
                "BAR is likely to be inaccurate because of poor overlap. Improve the sampling, or decrease the spacing "
                "between states.  For now, guessing that the free energy difference is 0 with no uncertainty.")
            if compute_uncertainty:
                result_vals["Delta_f"] = 0.0
                result_vals["dDelta_f"] = 0.0
                return result_vals
            else:
                result_vals["Delta_f"] = 0.0
                return result_vals

        while FUpperB * FLowerB > 0:
            FAve = (UpperB + LowerB) / 2
            UpperB = UpperB - max(abs(UpperB - FAve), 0.1)
            LowerB = LowerB + max(abs(LowerB - FAve), 0.1)
            FUpperB, FLowerB = yield from _zero_steps(M, UpperB, LowerB)
            nfunc += 2

    for iteration in range(maximum_iterations + 1):
        DeltaF_old = DeltaF

        if method == "false-position":
            if (LowerB == 0.0) and (UpperB == 0.0):
                DeltaF = 0.0
                FNew = 0.0
            else:
                DeltaF = UpperB - FUpperB * (UpperB - LowerB) / (FUpperB - FLowerB)
                (FNew,) = yield from _zero_steps(M, DeltaF)
            nfunc += 1

            if FNew == 0:
                relative_change = 10 ** (-15)
                break

        if method == "bisection":
            DeltaF = (UpperB + LowerB) / 2
            (FNew,) = yield from _zero_steps(M, DeltaF)
            nfunc += 1

        if method == "self-consistent-iteration":
            (F,) = yield from _zero_steps(M, DeltaF)
            DeltaF = -F + DeltaF
            nfunc += 1

        if DeltaF == 0.0:
            break

        if iterated_solution:
            relative_change = abs((DeltaF - DeltaF_old) / DeltaF)
            if (iteration > 0) and (relative_change < relative_tolerance):
                break

        if method == "false-position" or method == "bisection":
            if FUpperB * FNew < 0:
                LowerB = DeltaF
                FLowerB = FNew
            elif FLowerB * FNew <= 0:
                UpperB = DeltaF
                FUpperB = FNew
            else:
                message = "WARNING: Cannot determine bound on free energy"
                raise _u.BoundsError(message)

    if iterated_solution:
        if not iteration < maximum_iterations:
            message = ("WARNING: Did not converge to within specified tolerance. max_delta = {:f}, TOLERANCE = {:f}, "
                       "MAX_ITS = {:d}".format(relative_change, relative_tolerance, maximum_iterations))
            raise _u.ConvergenceError(message)

    if compute_uncertainty:
        if iterated_solution:
            C = M - DeltaF
        else:
            C = M - DeltaF_initial
        # exp_arg_R = w_R - C = w_R + (-C)
        rows = yield [(0, FERMI_MOMENTS, C, 0.0), (1, FERMI_MOMENTS, -C, 0.0)]
        (lse_F, lse2_F, max_arg_F), (lse_R, lse2_R, max_arg_R) = rows[0], rows[1]
        afF = np.exp(lse_F - max_arg_F) / T_F
        afR = np.exp(lse_R - max_arg_R) / T_R
        afF2 = np.exp(lse2_F - 2 * max_arg_F) / T_F
        afR2 = np.exp(lse2_R - 2 * max_arg_R) / T_R

        nrat = (T_F + T_R) / (T_F * T_R)

        if uncertainty_method == "BAR":
            variance = (afF2 / afF**2) / T_F + (afR2 / afR**2) / T_R - nrat
            dDeltaF = np.sqrt(variance)
        else:
            vartemp = (afF - afF2) * T_F + (afR - afR2) * T_R
            dDeltaF = np.sqrt(1.0 / vartemp - nrat)
        result_vals["Delta_f"] = DeltaF
        result_vals["dDelta_f"] = dDeltaF
        return result_vals
    else:
        result_vals["Delta_f"] = DeltaF
        return result_vals


def _as_work(w):
    a = np.asarray(w)
    if a.ndim != 1:
        raise ValueError(f"work values must be one-dimensional, got shape {a.shape}")
    return a


def _send(gen, value):
    """Advance a pair's generator: ("wait", requests), ("done", result) or ("error", exception)."""
    try:
        return "wait", gen.send(value)
    except StopIteration as stop:
        return "done", stop.value
    except Exception as e:                     # the reference's own exceptions (ConvergenceError, BoundsError, ...)
        return "error", e


def bar_many(w_F_list, w_R_list, **bar_kwargs):
    """`bar` for every pair (w_F_list[p], w_R_list[p]): the list of dicts that calling bar on each pair returns.

    All pairs live in one DeviceWork and step in lockstep, one device call per iteration for every active pair.  Each
    pair's result is the same bits as `bar` on that pair alone.  If any pair fails, the exception of the lowest-index
    failing pair is raised."""
    if len(w_F_list) != len(w_R_list):
        raise ValueError("w_F_list and w_R_list must have the same length")
    P = len(w_F_list)
    if P == 0:
        return []
    vectors = []
    for wf, wr in zip(w_F_list, w_R_list):
        vectors += [_as_work(wf), _as_work(wr)]
    gens = [_bar_steps(vectors[2 * p].size, vectors[2 * p + 1].size, **bar_kwargs) for p in range(P)]
    results, errors, waiting = [None] * P, {}, {}

    def settle(p, state, value):
        if state == "wait":
            waiting[p] = value
        elif state == "done":
            results[p] = value
        else:
            errors[p] = value

    for p in range(P):
        settle(p, *_send(gens[p], None))
    if waiting:
        with _device(vectors) as dev:
            while waiting:
                if errors:                     # pairs after the lowest failing one can no longer decide the outcome
                    for p in [q for q in waiting if q > min(errors)]:
                        del waiting[p]
                    if not waiting:
                        break
                order = sorted(waiting)
                reqs, spans = [], []
                for p in order:
                    r = waiting[p]
                    spans.append((len(reqs), len(r)))
                    reqs += [(2 * p + side, kind, c1, c2) for side, kind, c1, c2 in r]
                out = _evaluate(dev, reqs)
                waiting = {}
                for p, (s, n) in zip(order, spans):
                    settle(p, *_send(gens[p], out[s:s + n]))
    if errors:
        raise errors[min(errors)]
    return results


def bar(w_F, w_R, DeltaF=0.0, compute_uncertainty=True, uncertainty_method="BAR", maximum_iterations=500,
        relative_tolerance=1.0e-12, verbose=False, method="false-position", iterated_solution=True):
    """bar (other_estimators.py:156-531) on the device; `verbose` is accepted and ignored (the facade sends verbose
    calls to the reference)."""
    return bar_many([w_F], [w_R], DeltaF=DeltaF, compute_uncertainty=compute_uncertainty,
                    uncertainty_method=uncertainty_method, maximum_iterations=maximum_iterations,
                    relative_tolerance=relative_tolerance, method=method, iterated_solution=iterated_solution)[0]


def bar_zero(w_F, w_R, DeltaF):
    """bar_zero (other_estimators.py:56-153): log numerator - log denominator of Bennett's equation at DeltaF."""
    w_F, w_R = _as_work(w_F), _as_work(w_R)
    M = np.log(float(w_F.size) / float(w_R.size))
    gen = _zero_steps(M, DeltaF)
    reqs = gen.send(None)
    with _device([w_F, w_R]) as dev:
        out = _evaluate(dev, reqs)
    _, value = _send(gen, out)
    return value[0]


def _statistical_inefficiency():
    # looked up at call time, as the reference does: the device's when pymbar_b200 is installed
    from pymbar import timeseries

    return timeseries.statistical_inefficiency


def exp(w_F, compute_uncertainty=True, is_timeseries=False):
    """exp (other_estimators.py:572-647): one device call for log sum exp(-w), sum x and sum (x - mean x)^2."""
    w_F = _as_work(w_F)
    result_vals = dict()
    T = float(np.size(w_F))
    with _device([w_F]) as dev:
        lse, Sx, Sxx = _evaluate(dev, [(0, EXP, 0.0, 0.0)])[0]
    DeltaF = -(lse - np.log(T))
    if compute_uncertainty:
        Ex = Sx / T
        g = 1.0
        if is_timeseries:
            max_arg = np.max(-w_F)
            x = np.exp(-w_F - max_arg)
            g = _statistical_inefficiency()(x, x)
        dx = np.sqrt(Sxx / T) / np.sqrt(T / g)
        dDeltaF = dx / Ex
        result_vals["Delta_f"] = DeltaF
        result_vals["dDelta_f"] = dDeltaF
    else:
        result_vals["Delta_f"] = DeltaF
    return result_vals


def exp_gauss(w_F, compute_uncertainty=True, is_timeseries=False):
    """exp_gauss (other_estimators.py:650-719): one device call for sum w and sum (w - mean w)^2."""
    w_F = _as_work(w_F)
    T = float(np.size(w_F))
    with _device([w_F]) as dev:
        Sw, Sww, _ = _evaluate(dev, [(0, GAUSS, 0.0, 0.0)])[0]
    var = Sww / T
    DeltaF = Sw / T - 0.5 * var

    result_vals = dict()
    if compute_uncertainty:
        g = 1.0
        T_eff = T
        if is_timeseries:
            g = _statistical_inefficiency()(w_F, w_F)
            T_eff = T / g
        dx2 = var / T_eff + 0.5 * var * var / (T_eff - 1)
        dDeltaF = np.sqrt(dx2)
        result_vals["Delta_f"] = DeltaF
        result_vals["dDelta_f"] = dDeltaF
    else:
        result_vals["Delta_f"] = DeltaF
    return result_vals

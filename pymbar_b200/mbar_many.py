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

Bootstraps (n_bootstraps = B > 0, DESIGN.md 3.5g').  Problem p's replicate b is the one
`pymbar.MBAR(u_kn_list[p], N_k_list[p], n_bootstraps=B, rseed=rseed[p])` draws (samples in block order), drawn on the
host by the functions of `bootstrap` and kept as uint16 multiplicities.  Every replicate of every problem with at most
64 states is a replicate slot of the same `DeviceMbarBatch`: slots are solved in lockstep from their problem's final
f_k with the adaptive stage of BOOTSTRAP_SOLVER_PROTOCOL, then one weighted all-rows moments call gives every slot's
all-state update, and f[0] = 0 fixes the gauge, as `bootstrap.bootstrap_f_k` does.  Slots go to the device in waves
whose device footprint stays under BOOT_WAVE_BYTES; a replicate's result is the same bits in any wave.  A replicate is
solved by `bootstrap.bootstrap_f_k` on one DeviceProblem per problem instead when its batched solve does not converge
or a sum of it is flagged, when its problem has more than 64 states, or when its problem's multiplicities overflow
uint16.  Each problem's dict then adds f_k_boots [B, K] and boot_single, the number of its replicates that took that
path.
"""
from __future__ import annotations

import contextlib
import numbers

import numpy as np

from . import bootstrap
from . import estimators
from . import mbar_solvers as ms
from .utils import ParameterError

DeviceMbarBatch = None     # the device classes; resolved on first use (a test may put stand-ins here)
DeviceProblem = None

MAX_BATCH_K = 64
UNCERTAINTY_METHODS = (None, "svd-ew", "approximate", "bootstrap")
DEFAULT_OPTIONS = dict(min_sc_iter=0, gamma=1.0, maxiter=10000)
BOOT_WAVE_BYTES = 2 << 30   # device footprint of one wave of replicate slots


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
    """The dict of one problem.  With uncertainty_method="bootstrap", dDelta_f comes later from the replicates and
    Theta is "svd-ew" (mbar.py:1796)."""
    out = dict(f_k=f, Delta_f=f - np.vstack(f), path=path, iterations=iterations, success=bool(success))
    analytic = compute_uncertainty and uncertainty_method != "bootstrap"
    if analytic or return_theta:
        d = estimators.free_energy_differences(f, G, N_k, uncertainty_method=uncertainty_method,
                                               return_theta=return_theta)
        if analytic:
            out["dDelta_f"] = d["dDelta_f"]
        if return_theta:
            out["Theta"] = d["Theta"]
    return out


def _bootstrap_std(f_k_boots):
    """dDelta_f of mbar.py:706-714: the standard deviation over replicates of f_b - f_b^T."""
    f = np.asarray(f_k_boots)
    return np.std(f[:, None, :] - f[:, :, None], axis=0)


def _chunk_tiles(nT, K):
    """Tiles per chunk of the batched pass (batch_chunk_tiles in batch.cu)."""
    return max(max(2048 // K, 4), -(-nT // 4096))


def slot_bytes(K, N):
    """Device bytes of one replicate slot in a wave: its counts, the chunk partials and packed outputs of its two
    candidates with their Gram, and their f."""
    nT = -(-int(N) // 32)
    nc = -(-nT // _chunk_tiles(nT, int(K)))
    part = 2 * K + 2 + K * (K + 1) // 2
    out = 2 * K + 2 + K * K
    return 2 * nT * 32 + 2 * 8 * (nc * part + out + K)


def _validate_boot(n_bootstraps, rseed, P):
    if isinstance(n_bootstraps, bool) or not isinstance(n_bootstraps, numbers.Integral) or n_bootstraps < 0:
        raise ParameterError(f"n_bootstraps must be a non-negative int, got {n_bootstraps!r}")
    if rseed is None:
        return None
    if np.ndim(rseed) != 1:
        raise ParameterError("rseed must be None or one seed per problem: a single seed would give every problem "
                             "with the same N_k identical replicates")
    if len(rseed) != P:
        raise ParameterError(f"rseed must hold one seed per problem ({P}), got {len(rseed)}")
    return list(rseed)


class _Draws:
    """Problem p's bootstrap draws, made as pymbar.MBAR(..., n_bootstraps=B, rseed=seed) makes them (mbar.py:273-297,
    :424-433) and handed out in order, a few replicates at a time: counts [n, N] uint16 (None if a multiplicity
    overflows uint16) and the generator state before each replicate, from which replicate_rints regenerates its
    indices."""

    def __init__(self, N_k, seed):
        self.N_k = np.asarray(N_k).astype(np.int64)
        N = int(self.N_k.sum())
        self.members = bootstrap.state_members(self.N_k, bootstrap.default_x_kindices(self.N_k))
        self.rng = np.random.default_rng(seed)
        self.rng.choice(np.arange(N), min(50, N))
        self.states = []

    def next(self, n):
        states, counts = bootstrap.draw_mbar_replicates(self.rng, self.N_k, self.members, n)
        self.states += states
        return counts

    def rints(self, b):
        return bootstrap.replicate_rints(self.rng, self.states[b], self.N_k, self.members)


def _single_replicates(u_kn, N_k, f_k, rints, protocol):
    """f_k_boots rows of the replicates `rints` on one DeviceProblem, uploaded once."""
    _, Prob = _classes()
    with Prob(u_kn, N_k, device=ms._DEVICE) as p:
        return bootstrap.bootstrap_f_k(p, f_k, np.asarray(N_k).astype(np.int64), rints=rints,
                                       solver_protocol=protocol)


def _bootstraps(dev, batch, probs, f_main, seeds, B, tol, opts):
    """(f_k_boots [P][B, K], boot_single [P]) of every problem; dev holds the problems `batch` (None if none)."""
    P = len(probs)
    draws = [_Draws(probs[p][1], seeds[p]) for p in range(P)]
    boots = [np.zeros((B, probs[p][0].shape[0])) for p in range(P)]
    single = [set() for _ in range(P)]          # replicates of each problem for the single path
    overflow = set()
    slot_of = {p: i for i, p in enumerate(batch)}
    for p in range(P):
        if p not in slot_of:
            draws[p].next(B)                    # the generator states of every replicate
            single[p] = set(range(B))
    # waves of (problem, replicate) pairs in problem-major order, each under BOOT_WAVE_BYTES on the device
    pairs = [(p, b) for p in batch for b in range(B)]
    i = 0
    while i < len(pairs):
        wave, used = [], 0
        while i < len(pairs):
            p = pairs[i][0]
            need = slot_bytes(*probs[p][0].shape)
            if wave and used + need > BOOT_WAVE_BYTES:
                break
            wave.append(pairs[i])
            used += need
            i += 1
        counts = {}
        for p in dict.fromkeys(p for p, _ in wave):
            n = sum(1 for q, _ in wave if q == p)
            c = draws[p].next(n)
            if c is None:
                overflow.add(p)
            else:
                counts[p] = c
        slots = [(p, b) for p, b in wave if p not in overflow]
        if not slots:
            continue
        first = {}
        for k, (p, b) in enumerate(wave):
            first.setdefault(p, k)
        dev.set_replicates([slot_of[p] for p, _ in slots], [counts[p][b - wave[first[p]][1]] for p, b in slots])
        f_list, status, _ = dev.solve_replicates([f_main[p] for p, _ in slots], tol=tol, maxiter=int(opts["maxiter"]),
                                                 min_sc_iter=int(opts["min_sc_iter"]), gamma=float(opts["gamma"]))
        ok = [s for s in range(len(slots)) if status[s] == 0]
        for s in range(len(slots)):
            if status[s] != 0:
                single[slots[s][0]].add(slots[s][1])
        if ok:
            sums = dev.moments([f_list[s] for s in ok], all_rows=True, slots=ok)
            for s, m in zip(ok, sums):
                p, b = slots[s]
                if m["flag"]:
                    single[p].add(b)
                    continue
                f = f_list[s] - m["log_S"]
                boots[p][b] = f - f[0]
    for p in overflow:
        single[p] = set(range(B))
    protocol = (dict(method="adaptive", tol=tol, options=dict(min_sc_iter=int(opts["min_sc_iter"]),
                                                                 gamma=float(opts["gamma"]),
                                                                 maxiter=int(opts["maxiter"]))),)
    for p in range(P):
        if single[p]:
            picked = sorted(single[p])
            rints = np.array([draws[p].rints(b) for b in picked])
            u, N_k, _ = probs[p]
            boots[p][picked] = _single_replicates(u, N_k, f_main[p], rints, protocol)
    return boots, [len(s) for s in single]


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
              return_theta=False, solver_tolerance=1.0e-12, options=None, n_bootstraps=0, rseed=None):
    """MBAR on every problem (u_kn_list[p], N_k_list[p]): one dict per problem, in input order, with f_k, Delta_f,
    dDelta_f (compute_uncertainty), Theta (return_theta), iterations (of the batched solve; None on the single path),
    success and path ("batch" or "single").

    f_k_init: None (zeros) or one starting vector per problem.  options update the adaptive solver's defaults
    (min_sc_iter=0, gamma=1, maxiter=10000).  uncertainty_method: None, "svd-ew", "approximate" or "bootstrap".  Every
    problem is validated before any device work; an invalid problem raises for the lowest failing index.

    n_bootstraps = B > 0 adds f_k_boots [B, K] (replicate b of problem p is the one pymbar.MBAR(u_kn_list[p],
    N_k_list[p], n_bootstraps=B, rseed=rseed[p]) draws) and boot_single (how many of them the single-problem path
    solved) to every dict.  rseed: one seed per problem, or None for one np.random.randint(2**31 - 1) per problem in
    problem order, as P constructions of MBAR would draw.  uncertainty_method="bootstrap" gives
    dDelta_f = std over b of f_b - f_b^T and needs B > 0; its Theta is "svd-ew"."""
    if uncertainty_method not in UNCERTAINTY_METHODS:
        raise ParameterError(f"uncertainty_method {uncertainty_method!r} is not supported by mbar_many "
                             f"(one of {UNCERTAINTY_METHODS})")
    if len(u_kn_list) != len(N_k_list):
        raise ValueError("u_kn_list and N_k_list must have the same length")
    P = len(u_kn_list)
    if f_k_init is not None and len(f_k_init) != P:
        raise ValueError("f_k_init must hold one vector per problem")
    seeds = _validate_boot(n_bootstraps, rseed, P)
    B = int(n_bootstraps)
    if uncertainty_method == "bootstrap" and B <= 0:
        raise ParameterError("Cannot request bootstrap sampling of free energy differences without any bootstraps.")
    opts = dict(DEFAULT_OPTIONS)
    opts.update(options or {})
    probs = [_validate(u_kn_list[p], N_k_list[p], None if f_k_init is None else f_k_init[p]) for p in range(P)]
    if B > 0 and seeds is None:
        seeds = [np.random.randint(np.iinfo(np.int32).max) for _ in range(P)]
    want_G = bool((compute_uncertainty and uncertainty_method != "bootstrap") or return_theta)
    results = [None] * P
    batch = [p for p in range(P) if probs[p][0].shape[0] <= MAX_BATCH_K]
    single = [p for p in range(P) if probs[p][0].shape[0] > MAX_BATCH_K]
    with contextlib.ExitStack() as stack:
        dev = None
        if batch:
            Batch, _ = _classes()
            dev = stack.enter_context(Batch([probs[p][0] for p in batch], [probs[p][1] for p in batch],
                                            device=ms._DEVICE))
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
        if B > 0:
            boots, nsingle = _bootstraps(dev, batch, probs, [r["f_k"] for r in results], seeds, B, solver_tolerance,
                                         opts)
            for r, fb, ns in zip(results, boots, nsingle):
                r["f_k_boots"] = fb
                r["boot_single"] = ns
                if compute_uncertainty and uncertainty_method == "bootstrap":
                    r["dDelta_f"] = _bootstrap_std(fb)
    return results

"""Bootstrap replicates of the MBAR solve without copying u_kn (SURVEY.md 8f, row N3).

pymbar resamples within every state's block of samples and solves again on the gathered array
``u_kn[:, rints]`` (mbar.py:417-449): one 8*K*N-byte copy and a fresh problem per replicate.  A replicate
is the same data with integer multiplicities ``w_n = #{i : rints[i] = n}``, so here the resident
problem is reused with ``DeviceProblem.set_sample_weights`` and only N doubles move per replicate.
"""
from __future__ import annotations

import numpy as np

from . import mbar_solvers as ms


def default_x_kindices(N_k):
    """mbar.py:264-268: samples in block order."""
    N_k = np.asarray(N_k, dtype=np.int64)
    return np.repeat(np.arange(len(N_k), dtype=np.int64), N_k)


def bootstrap_indices(N_k, n_bootstraps, rseed, x_kindices=None):
    """The `bootstrap_rints` MBAR.__init__ would draw for this rseed (mbar.py:273-275, :297, :428-433):
    the constructor's generator first spends one `choice` of min(50, N) indices on its duplicate-state
    check, then draws N_k[k] integers per state per replicate."""
    N_k = np.asarray(N_k, dtype=np.int64)
    N = int(N_k.sum())
    x = default_x_kindices(N_k) if x_kindices is None else np.asarray(x_kindices)
    rng = np.random.default_rng(rseed)
    rng.choice(np.arange(N), min(50, N))
    out = np.zeros((n_bootstraps, N), dtype=np.int64)
    for b in range(n_bootstraps):
        for k in range(len(N_k)):
            k_indices = np.where(x == k)[0]
            out[b, k_indices] = k_indices[rng.integers(int(N_k[k]), size=int(N_k[k]))]
    return out


def state_members(N_k, x_kindices):
    """[samples of state k for k < K], each in increasing order (np.where(x_kindices == k)[0] of mbar.py:430), from
    one stable argsort; None unless x_kindices labels every sample with a state in [0, K) and state k with exactly
    N_k[k] samples (the only labellings for which the reference's draws are well defined)."""
    N_k = np.asarray(N_k, dtype=np.int64)
    x = np.asarray(x_kindices)
    if x.shape != (int(N_k.sum()),) or not (x.dtype.kind in "iu" or x.size == 0):
        return None
    if x.size and (x.min() < 0 or x.max() >= len(N_k)):
        return None
    if not np.array_equal(np.bincount(x.astype(np.int64), minlength=len(N_k)), N_k):
        return None
    order = np.argsort(x, kind="stable")
    first = np.concatenate([[0], np.cumsum(N_k)])
    return [order[first[k]:first[k + 1]] for k in range(len(N_k))]


def _draw_rints(rng, N_k, members):
    N = int(np.sum(N_k))
    rints = np.zeros(N, int)
    for k, k_indices in enumerate(members):
        n = int(N_k[k])
        rints[k_indices] = k_indices[rng.integers(n, size=n)]
    return rints


def draw_mbar_replicates(rng, N_k, members, n_bootstraps, each=None):
    """(states, counts): MBAR.__init__'s bootstrap draws (mbar.py:424-433) from `rng` (MBAR.rng, advanced exactly as
    the reference advances it), as the generator state before each replicate and the multiplicities
    counts[b, n] = #{p : rints_b[p] = n} as uint16 [B, N] (2 B N bytes against the reference's 8 B N of int64
    bootstrap_rints).  counts is None if a multiplicity exceeds 65535.  each(b, rints), when given, sees every
    replicate's indices as they are drawn."""
    N = int(np.sum(N_k))
    states = []
    counts = np.zeros((int(n_bootstraps), N), dtype=np.uint16)
    fits = True
    for b in range(int(n_bootstraps)):
        states.append(rng.bit_generator.state)
        rints = _draw_rints(rng, N_k, members)
        c = np.bincount(rints, minlength=N)
        fits = fits and (c.max(initial=0) <= 65535)
        counts[b] = np.minimum(c, 65535)
        if each is not None:
            each(b, rints)
    return states, (counts if fits else None)


def replicate_rints(rng, state, N_k, members):
    """The reference's bootstrap_rints row of the replicate drawn from `state` (a bit-generator state of `rng`'s
    kind), regenerated on a private generator: `rng` is not advanced."""
    bg = type(rng.bit_generator)()
    bg.state = state
    return _draw_rints(np.random.Generator(bg), N_k, members)


def bootstrap_f_k(problem, f_k, N_k, rints=None, n_bootstraps=0, rseed=None, x_kindices=None,
                  solver_protocol=None):
    """f_k_boots[b, :] of mbar.py:421-443 on a resident problem.

    `rints` [n_bootstraps, N] may be given (e.g. MBAR.bootstrap_rints); otherwise it is drawn as the
    reference would for `rseed`.  Each replicate starts from f_k and runs BOOTSTRAP_SOLVER_PROTOCOL
    (mbar_solvers.py:117), then the all-state update and the f_0 gauge (:1012-1015)."""
    N_k = np.asarray(N_k, dtype=np.int64)
    N = int(N_k.sum())
    if rints is None:
        rints = bootstrap_indices(N_k, n_bootstraps, rseed, x_kindices)
    rints = np.atleast_2d(np.asarray(rints))
    protocol = ms.BOOTSTRAP_SOLVER_PROTOCOL if solver_protocol is None else solver_protocol
    sampled = np.flatnonzero(N_k > 0)
    out = np.zeros((rints.shape[0], len(N_k)))
    try:
        for b, r in enumerate(rints):
            problem.set_sample_weights(np.bincount(r, minlength=N).astype(np.float64))
            f = np.array(f_k, dtype=np.float64)
            if len(sampled) > 1:
                proto = tuple({k: (dict(v) if isinstance(v, dict) else v) for k, v in st.items()} for st in protocol)
                f, _ = ms._solve_protocol_on(problem, f, proto)
            else:
                f[sampled] = 0.0
            f = problem.self_consistent_update(f)
            out[b] = f - f[0]
    finally:
        problem.set_sample_weights(None)
    return out

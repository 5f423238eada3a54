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

`MbarMany` is the same solve kept resident: its estimators (expectations, perturbed free energies, entropy and
enthalpy, overlap, effective sample numbers) append each problem's extra rows to the batch it already holds and
evaluate every problem in one augmented moments pass (DESIGN.md 3.5g''), and with n_bootstraps > 0 every replicate of
every problem in one weighted augmented pass for uncertainty_method="bootstrap" (DESIGN.md 3.5g''').  `mbar_many` is
`MbarMany(...).results`.
"""
from __future__ import annotations

import contextlib
import numbers
import time

import numpy as np

from . import bootstrap
from . import estimators
from . import expectations as ex
from . import fes as hist
from . import fes_bootstrap as fb
from . import mbar_solvers as ms
from .utils import ParameterError

DeviceMbarBatch = None     # the device classes; resolved on first use (a test may put stand-ins here)
DeviceProblem = None
DeviceKdeMany = None

MAX_BATCH_K = 64
UNCERTAINTY_METHODS = (None, "svd-ew", "approximate", "bootstrap")
DEFAULT_OPTIONS = dict(min_sc_iter=0, gamma=1.0, maxiter=10000)
BOOT_WAVE_BYTES = 2 << 30   # device footprint of one wave of replicate slots
MAX_BATCH_ROWS = 192        # DeviceMbarBatch.MAX_ROWS: K_p plus appended rows of a batched estimator request
AUG_WAVE_BYTES = 2 << 30    # device footprint of one wave of appended rows
ESTIMATOR_METHODS = (None, "svd-ew", "approximate", "bootstrap")
FES_WAVE_BYTES = 2 << 30    # device footprint of one wave of histogram FES requests
FES_UNCERTAINTY_METHODS = (None, "analytical", "bootstrap")
FES_TYPES = ("histogram", "kde")
KDE_WAVE_BYTES = 1 << 30    # device footprint of the requests of one DeviceKdeMany.log_sum call
KDE_PART_BYTES = 64 << 20   # kde.cu: the chunk partials of one sub-batch of a DeviceKdeMany.log_sum call
KDE_PIECE_BYTES = 112       # kde.cu: sizeof(KdeManyPiece)


def _kde_class():
    global DeviceKdeMany
    if DeviceKdeMany is None:
        from .problem import DeviceKdeMany as K

        DeviceKdeMany = K
    return DeviceKdeMany


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
    return ex.std_of_differences(f_k_boots)


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


def augmented_bytes(K, N, M):
    """Device bytes of one problem's M appended rows in a wave: its appended tiles, L_n scratch, the pass and Gram
    partials and packed output of its augmented request, and its f (batch.cu's geometry)."""
    nT = -(-int(N) // 32)
    R = int(K) + int(M)
    nc = -(-nT // _chunk_tiles(nT, R))
    gct = max(512, -(-nT // 64))
    ngc = -(-nT // gct)
    nb = -(-R // 32)
    return 8 * (nT * 32 * (M + 1) + nc * (2 * R + 2) + nb * (nb + 1) // 2 * ngc * 1024 + 2 * R + 2 + R * R + R)


def boot_augmented_bytes(K, N, M):
    """Device bytes of one weighted appended slot in a wave: its counts, the pass partials and packed output of its
    request (no Gram) and its f (batch.cu's geometry).  The appended tiles are its problem's, counted by
    augmented_bytes."""
    nT = -(-int(N) // 32)
    R = int(K) + int(M)
    nc = -(-nT // _chunk_tiles(nT, R))
    return 2 * nT * 32 + 8 * (nc * (2 * R + 2) + 2 * R + 2 + R)


def _bin_geometry(nT, rows, nbins):
    """(bins per chunk, bin chunks, sample chunks) of one pass of a batched bin moments request (bin_geometry in
    batch.cu)."""
    BC = min(nbins, (108 * 1024 // 8) // rows)
    cap = max(1, (4 << 20) // (rows * nbins * 8))
    nsc = min(-(-nT // 64), 64, cap)
    ct = -(-nT // nsc)
    return BC, -(-nbins // BC), -(-nT // ct)


def bin_bytes(K, N, nbins, want_C):
    """Device bytes of one histogram request in a wave: its u_n, log w_n, L_n and bin slots, the per-bin arrays, the
    partials of its larger pass, C and D when asked for, its f and its request record (batch.cu's geometry)."""
    nT = -(-int(N) // 32)
    K, nbins = int(K), int(nbins)
    parts = _bin_geometry(nT, 1, nbins)[2] * nbins
    if want_C:
        parts = max(parts, _bin_geometry(nT, K + 1, nbins)[2] * (K + 1) * nbins)
    return 20 * nT * 32 + 40 * nbins + 8 * parts + (8 * (K + 1) * nbins if want_C else 0) + 8 * K + 164


def rep_bin_bytes(K, N, nbins):
    """Device bytes of one replicate histogram request in a wave, beyond its slot (slot_bytes): its log w_n, L_n and
    bin slots, the per-bin arrays, the partials of its bin-sum pass, its f and its request records (batch.cu's
    geometry), plus its target's u_n and bin index, counted with every slot as an upper bound."""
    nT = -(-int(N) // 32)
    K, nbins = int(K), int(nbins)
    return 32 * nT * 32 + 40 * nbins + 8 * _bin_geometry(nT, 1, nbins)[2] * nbins + 8 * K + 180


def log_weight_bytes(K, N):
    """Device bytes of one request of DeviceMbarBatch.log_weights in a wave: its u_n / log w_n slots, its f, its flag
    and its request record (batch.cu's geometry)."""
    nT = -(-int(N) // 32)
    return 8 * nT * 32 + 8 * int(K) + 4 + 164


def _kde_chunks(N):
    """Chunks of a sample set of N samples (kde_chunking in kde.cu)."""
    N = int(N)
    nPad = -(-N // 256) * 256
    nc = min(1024, max(1, -(-N // 4096)))
    chunk = -(-(-(-N // nc)) // 256) * 256
    return nPad, -(-nPad // chunk)


def kde_bytes(N, D, Q):
    """Device bytes of one DeviceKdeMany.log_sum request on a set of N samples in D dimensions with Q queries: its log
    weights (padded to 256), queries and outputs, and two records for each of its pieces of at most kde_query_cap
    queries (kde.cu).  The chunk partials of a call take at most KDE_PART_BYTES beyond these, or one piece's."""
    nPad, nc = _kde_chunks(N)
    cap = max(128, (KDE_PART_BYTES // (16 * nc)) // 128 * 128)
    pieces = -(-int(Q) // cap)
    return 8 * nPad + 8 * int(D) * int(Q) + 8 * int(Q) + 2 * KDE_PIECE_BYTES * pieces


def _waves(items, need, limit):
    """items split, in order, into waves whose need(item) sum stays under limit (one item at least per wave)."""
    waves, wave, used = [], [], 0
    for it in items:
        n = need(it)
        if wave and used + n > limit:
            waves.append(wave)
            wave, used = [], 0
        wave.append(it)
        used += n
    if wave:
        waves.append(wave)
    return waves


def _noted(err, p):
    """err with a note naming problem p, for errors of the single path."""
    err.add_note(f"raised for problem {p} (MbarMany histogram FES, single path)")
    return err


def _validate_fes_boot(n_bootstraps, seed, P):
    """The n_bootstraps rule of pymbar.FES.generate_fes (fes.py:357-360: an integer, 0 or >= 2; ValueError otherwise)
    and seed: None, or one entry per problem, each an int >= 0, -1 or None."""
    if not np.issubdtype(type(n_bootstraps), np.integer) or n_bootstraps == 1 or n_bootstraps < 0:
        raise ValueError(f"n_bootstraps must be an integer of 0 or >=2, it was set to {n_bootstraps}")
    if seed is None:
        return [None] * P
    if np.ndim(seed) != 1:
        raise ParameterError("seed must be None or one seed per problem: a single seed would give every problem "
                             "with the same N_k identical replicates")
    if len(seed) != P:
        raise ParameterError(f"seed must hold one entry per problem ({P}), got {len(seed)}")
    out = []
    for p, v in enumerate(seed):
        ok = v is None or (np.issubdtype(type(v), np.integer) and (v >= 0 or v == -1))
        if not ok:
            raise ParameterError(f"problem {p}: seed must be an int >= 0, -1 or None, got {v!r}")
        out.append(None if v is None or v < 0 else int(v))
    return out


def _kde_defaults():
    """KernelDensity().get_params(): the parameters pymbar.FES._setup_fes_kde fills kde_parameters into."""
    try:
        from sklearn.neighbors import KernelDensity
    except ImportError:
        raise ImportError("Cannot use 'kde' type FES without the scikit-learn module. Could not import sklearn")
    return KernelDensity().get_params()


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
        N = self.N = int(self.N_k.sum())
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

    def counts(self, b):
        """Replicate b's multiplicities [N] as uint16, regenerated from its generator state (they fit: problems whose
        draws overflow are kept out)."""
        return np.bincount(self.rints(b), minlength=self.N).astype(np.uint16)


def _single_replicates(u_kn, N_k, f_k, rints, protocol):
    """f_k_boots rows of the replicates `rints` on one DeviceProblem, uploaded once."""
    _, Prob = _classes()
    with Prob(u_kn, N_k, device=ms._DEVICE) as p:
        return bootstrap.bootstrap_f_k(p, f_k, np.asarray(N_k).astype(np.int64), rints=rints,
                                       solver_protocol=protocol)


def _solve_slots(dev, problems, counts, f_starts, tol, opts):
    """Replicate slots of a wave (slot s: problem problems[s] of the batch with multiplicities counts[s]) solved in
    lockstep from f_starts[s] with the adaptive stage, then one weighted all-rows moments call for the all-state update
    and the gauge f[0] = 0, as bootstrap.bootstrap_f_k does: {s: f [K]} for the slots whose solve converged and whose
    update is not flagged.  The slots stay resident for the caller's next request."""
    dev.set_replicates(problems, counts)
    f_list, status, _ = dev.solve_replicates(f_starts, tol=tol, maxiter=int(opts["maxiter"]),
                                             min_sc_iter=int(opts["min_sc_iter"]), gamma=float(opts["gamma"]))
    ok = [s for s in range(len(f_starts)) if status[s] == 0]
    out = {}
    if ok:
        sums = dev.moments([f_list[s] for s in ok], all_rows=True, slots=ok)
        for s, m in zip(ok, sums):
            if not m["flag"]:
                f = f_list[s] - m["log_S"]
                out[s] = f - f[0]
    return out


def _bootstraps(dev, batch, probs, f_main, seeds, B, tol, opts):
    """(f_k_boots [P][B, K], boot_single [P], draws [P], overflow) of every problem; dev holds the problems `batch`
    (None if none).  draws[p] keeps the generator state before each of problem p's replicates; overflow is the set of
    problems whose multiplicities overflow uint16."""
    P = len(probs)
    draws = [_Draws(probs[p][1], seeds[p]) for p in range(P)]
    boots = [np.zeros((B, probs[p][0].shape[0])) for p in range(P)]
    single = [set() for _ in range(P)]          # replicates of each problem for the single path
    overflow = set()
    slot_of = {p: i for i, p in enumerate(batch)}
    for p in range(P):
        if p not in slot_of:
            if draws[p].next(B) is None:        # the generator states of every replicate
                overflow.add(p)
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
        got = _solve_slots(dev, [slot_of[p] for p, _ in slots],
                           [counts[p][b - wave[first[p]][1]] for p, b in slots], [f_main[p] for p, _ in slots], tol,
                           opts)
        for s, (p, b) in enumerate(slots):
            if s in got:
                boots[p][b] = got[s]
            else:
                single[p].add(b)
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
    return boots, [len(s) for s in single], draws, overflow


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


class MbarMany:
    """MBAR on every problem (u_kn_list[p], N_k_list[p]), kept resident for the estimators that follow.

    The constructor solves as `mbar_many` does (same arguments) and `.results` is its list of dicts.  The batch of
    problems with at most 64 states stays on the device until `close()` (or the end of a `with` block), so that
    `compute_expectations`, `compute_perturbed_free_energies`, `compute_entropy_and_enthalpy`, `compute_overlap` and
    `compute_effective_sample_number` serve every problem without a new upload or a new solve (DESIGN.md 3.5g'').

    Each estimator takes one entry per problem, or None to skip a problem, and returns one dict per problem (None for
    a skipped one) with the keys of the pymbar.MBAR method of the same name and `path`, "batch" or "single".  Every
    request is validated before any device work; an invalid one raises ParameterError for the lowest failing index.
    uncertainty_method is None, "svd-ew", "approximate" or, with n_bootstraps > 0 at construction, "bootstrap"
    (compute_expectations, compute_perturbed_free_energies, compute_entropy_and_enthalpy; DESIGN.md 3.5g''').

    The appended rows of expectations.augmentation go on top of the resident problems in waves whose device footprint
    stays under AUG_WAVE_BYTES; a problem's result is the same bits in any wave.  Each wave takes one
    augmented_moments call at (f_k, 0), whose log S gives the appended rows' f = -log S (the self-consistent update
    of the single path), and, when a Theta is needed, one at the full f with the Gram.  A problem takes the single
    path (expectations.expectations_inner on a DeviceProblem of it) when it took the single path in the solve, when
    K_p plus its appended rows exceed MAX_BATCH_ROWS, or when either call flags it.

    Under bootstrap, every replicate b of a batched problem is a replicate slot with the problem's appended rows,
    asked at f = [f_k_boots[b], 0 ...] in sub-waves under BOOT_WAVE_BYTES, one weighted augmented_moments call each;
    the counts are regenerated from the construction's draws.  A flagged replicate sends its problem to the single
    path, expectations_inner(..., replicates=(f_k_boots, counts)).  A problem whose multiplicities overflow uint16
    raises ParameterError."""

    def __init__(self, u_kn_list, N_k_list, f_k_init=None, compute_uncertainty=True, uncertainty_method=None,
                 return_theta=False, solver_tolerance=1.0e-12, options=None, n_bootstraps=0, rseed=None):
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
            raise ParameterError("Cannot request bootstrap sampling of free energy differences without any "
                                 "bootstraps.")
        opts = dict(DEFAULT_OPTIONS)
        opts.update(options or {})
        probs = [_validate(u_kn_list[p], N_k_list[p], None if f_k_init is None else f_k_init[p]) for p in range(P)]
        if B > 0 and seeds is None:
            seeds = [np.random.randint(np.iinfo(np.int32).max) for _ in range(P)]
        self._probs = probs
        self._stack = contextlib.ExitStack()
        self._dev = None
        self._slot = {}              # problem -> its index in the device batch
        self._G = {}                 # problem -> W^T W at its final f, where the solve computed it
        self._B = B
        self._draws = []             # problem -> its _Draws (n_bootstraps > 0): replicate counts are regenerated
        self._overflow = set()       # problems whose replicate multiplicities overflow uint16
        self.histogram_datas = [None] * P    # problem -> the reference's histogram_data dict (generate_fes)
        self.replicate_histogram_datas = [None] * P  # problem -> its B ReplicateHistograms (generate_fes, B >= 2)
        self.fes_boot_single = [0] * P       # problem -> how many of those replicates took the single path
        self._tol, self._opts = solver_tolerance, opts
        self._fes = {}                       # problem -> its histogram request, path and cached Theta
        self.fes_types = [None] * P          # problem -> "histogram" or "kde": the surface the last generate_fes built
        self.kde_settings = [None] * P       # problem -> {"kernel", "h", "D"} of its KDE surface
        self._kde = {}                       # problem -> its KDE surface: sample set, weights, replicate weights, path
        self._closed = False
        self.device_stats = dict(ms=0.0, launches=0, calls=0, bytes_read=0)
        # host time spent regenerating replicate counts for the estimators, and drawing bootstrap surfaces' replicates
        self.host_stats = dict(counts_s=0.0, fes_draws_s=0.0)
        self.kde_stats = dict(ms=0.0, launches=0, calls=0, pairs=0, upload_bytes=0)   # DeviceKdeMany calls
        try:
            self.results = self._solve(probs, seeds, B, compute_uncertainty, uncertainty_method, return_theta,
                                       solver_tolerance, opts)
        except BaseException:
            self.close()
            raise

    def close(self):
        """Free the device batch and the KDE sample sets.  The results stay."""
        self._dev = None
        self._closed = True
        self._stack.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _solve(self, probs, seeds, B, compute_uncertainty, uncertainty_method, return_theta, solver_tolerance, opts):
        P = len(probs)
        want_G = bool((compute_uncertainty and uncertainty_method != "bootstrap") or return_theta)
        results = [None] * P
        batch = [p for p in range(P) if probs[p][0].shape[0] <= MAX_BATCH_K]
        single = [p for p in range(P) if probs[p][0].shape[0] > MAX_BATCH_K]
        dev = None
        if batch:
            Batch, _ = _classes()
            dev = self._stack.enter_context(Batch([probs[p][0] for p in batch], [probs[p][1] for p in batch],
                                                  device=ms._DEVICE))
            self._dev = dev
            self._slot = {p: i for i, p in enumerate(batch)}
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
                if i in G:
                    self._G[p] = G[i]
                results[p] = _result(f_final[i], G.get(i), probs[p][1], "batch", int(iters[i]), True,
                                     compute_uncertainty, uncertainty_method, return_theta)
        for p in sorted(single):
            u, N_k, f0 = probs[p]
            f, G = _single(u, N_k, f0, solver_tolerance, want_G)
            if G is not None:
                self._G[p] = G
            success = bool(np.all(np.isfinite(f)))
            results[p] = _result(f, G, N_k, "single", None, success, compute_uncertainty, uncertainty_method,
                                 return_theta)
        if B > 0:
            boots, nsingle, self._draws, self._overflow = _bootstraps(dev, batch, probs, [r["f_k"] for r in results],
                                                                      seeds, B, solver_tolerance, opts)
            for r, fb, ns in zip(results, boots, nsingle):
                r["f_k_boots"] = fb
                r["boot_single"] = ns
                if compute_uncertainty and uncertainty_method == "bootstrap":
                    r["dDelta_f"] = _bootstrap_std(fb)
        return results

    # ---- estimators on the resident problems ----
    def _entries(self, values, name):
        P = len(self._probs)
        if values is None:
            return [None] * P
        if len(values) != P:
            raise ValueError(f"{name} must hold one entry (or None) per problem ({P}), got {len(values)}")
        return list(values)

    def _rows(self, p, a, name, allow_1d=True):
        """a as float64 rows [L, N_p]; ParameterError for a shape that does not match N_p or for NaN."""
        N = self._probs[p][0].shape[1]
        a = np.asarray(a, dtype=np.float64)
        if a.ndim == 1 and allow_1d:
            a = a.reshape(1, -1)
        if a.ndim != 2 or a.shape[1] != N or a.shape[0] < 1:
            raise ParameterError(f"problem {p}: {name} has shape {a.shape}, the problem has N={N} samples")
        if np.isnan(a).any():
            raise ParameterError(f"problem {p}: {name} holds NaN")
        return a

    def _inner_many(self, requests, uncertainty_method, return_theta):
        """expectations_inner of every request (requests[p] = (A_n, u_ln, state_map) or None): ([inner or None] per
        problem, [path or None] per problem).  uncertainty_method="bootstrap" adds every replicate's keys
        ('bootstrapped_observables', 'bootstrapped_f')."""
        P = len(self._probs)
        boot = uncertainty_method == "bootstrap"
        if boot:
            for p, req in enumerate(requests):
                if req is not None and p in self._overflow:
                    raise ParameterError(f"problem {p}: a bootstrap multiplicity exceeds 65535, so its replicates "
                                         f"cannot be evaluated")
        plans = {p: ex.augmentation(self._probs[p][0].shape[0], *req) for p, req in enumerate(requests)
                 if req is not None}
        batched, single = [], []
        for p in sorted(plans):
            R = self._probs[p][0].shape[0] + plans[p]["extra"].shape[0]
            on_batch = self.results[p]["path"] == "batch" and p in self._slot
            (batched if on_batch and R <= MAX_BATCH_ROWS else single).append(p)
        inner = [None] * P
        path = [None] * P
        i = 0
        while i < len(batched):
            wave, used = [], 0
            while i < len(batched):
                p = batched[i]
                need = augmented_bytes(*self._probs[p][0].shape, plans[p]["extra"].shape[0])
                if wave and used + need > AUG_WAVE_BYTES:
                    break
                wave.append(p)
                used += need
                i += 1
            single += self._wave(wave, plans, uncertainty_method, return_theta, inner, path)
        if batched:
            self._dev.set_unsampled([], [])
            if boot:
                self._dev.set_replicates([], [])
        _, Prob = _classes()
        for p in sorted(single):
            u, N_k, _ = self._probs[p]
            reps = None
            if boot:
                reps = (self.results[p]["f_k_boots"], self._replicate_counts([(p, b) for b in range(self._B)]))
            with Prob(u, N_k, device=ms._DEVICE) as q:
                inner[p] = ex.expectations_inner(u, N_k, self.results[p]["f_k"], *requests[p],
                                                 uncertainty_method=uncertainty_method, return_theta=return_theta,
                                                 problem=q, replicates=reps)
            path[p] = "single"
        return inner, path

    def _replicate_counts(self, pairs):
        """The multiplicities [len(pairs), N] uint16 of the replicates (problem, b), regenerated from the draws."""
        t0 = time.perf_counter()
        out = [self._draws[p].counts(b) for p, b in pairs]
        self.host_stats["counts_s"] += time.perf_counter() - t0
        return out

    def _count(self):
        s = self._dev.last_stats()
        self.device_stats["ms"] += s["ms"]
        self.device_stats["launches"] += s["launches"]
        self.device_stats["calls"] += 1
        self.device_stats["bytes_read"] += s["bytes_read"]

    def _wave(self, wave, plans, uncertainty_method, return_theta, inner, path):
        """One wave of batched problems: fills inner and path, returns the problems the device flagged."""
        dev = self._dev
        ids = [self._slot[p] for p in wave]
        dev.set_unsampled(ids, [plans[p]["extra"] for p in wave])
        f0 = [np.concatenate([self.results[p]["f_k"], np.zeros(plans[p]["extra"].shape[0])]) for p in wave]
        sums = dev.augmented_moments(f0, problems=ids)
        self._count()
        flagged, ok, f_aug = [], [], {}
        for p, f, m in zip(wave, f0, sums):
            if m["flag"]:
                flagged.append(p)
                continue
            K = self._probs[p][0].shape[0]
            fa = f.copy()
            fa[K:] = (f - m["log_S"])[K:]          # appended rows: the self-consistent update from f = 0
            f_aug[p] = fa
            ok.append(p)
        G = {}
        if ok and return_theta:
            sums = dev.augmented_moments([f_aug[p] for p in ok], want_G=True, problems=[self._slot[p] for p in ok])
            self._count()
            for p, m in zip(ok, sums):
                if m["flag"]:
                    flagged.append(p)
                    continue
                G[p] = _gram_to_G(m["G"], self._N_aug(p, plans[p]))
        ok = [p for p in ok if not return_theta or p in G]
        F_aug = {}
        if ok and uncertainty_method == "bootstrap":
            F_aug = self._replicate_waves(ok, plans, f_aug)
            flagged += [p for p in ok if p not in F_aug]
            ok = [p for p in ok if p in F_aug]
        for p in ok:
            inner[p] = ex.finish(plans[p], f_aug[p], G.get(p), self._N_aug(p, plans[p]),
                                 uncertainty_method=uncertainty_method, return_theta=return_theta)
            if p in F_aug:
                inner[p].update(ex.bootstrap_keys(plans[p], F_aug[p]))
            path[p] = "batch"
        return flagged

    def _replicate_waves(self, wave, plans, f_aug):
        """Every replicate b of every problem p of `wave` (whose appended rows are resident) as a replicate slot at
        f = [f_k_boots[p][b], 0 ...], in sub-waves under BOOT_WAVE_BYTES, one weighted augmented_moments call each:
        {p: F_aug [B, R_p]} with F_aug[b, K:] = -log S[K:], for the problems none of whose replicates is flagged."""
        dev, B = self._dev, self._B
        F_aug = {}
        for p in wave:
            F_aug[p] = np.zeros((B, len(f_aug[p])))
            F_aug[p][:, :self._probs[p][0].shape[0]] = self.results[p]["f_k_boots"]
        bad = set()
        pairs = [(p, b) for p in wave for b in range(B)]
        i = 0
        while i < len(pairs):
            sub, used = [], 0
            while i < len(pairs):
                p = pairs[i][0]
                need = boot_augmented_bytes(*self._probs[p][0].shape, plans[p]["extra"].shape[0])
                if sub and used + need > BOOT_WAVE_BYTES:
                    break
                sub.append(pairs[i])
                used += need
                i += 1
            dev.set_replicates([self._slot[p] for p, _ in sub], self._replicate_counts(sub))
            f0 = [F_aug[p][b].copy() for p, b in sub]
            sums = dev.augmented_moments(f0, slots=list(range(len(sub))))
            self._count()
            for (p, b), f, m in zip(sub, f0, sums):
                if m["flag"]:
                    bad.add(p)
                    continue
                K = self._probs[p][0].shape[0]
                F_aug[p][b, K:] = (f - m["log_S"])[K:]      # appended rows: the replicate's update from f = 0
        return {p: F for p, F in F_aug.items() if p not in bad}

    def _N_aug(self, p, plan):
        return np.concatenate([np.asarray(self._probs[p][1], dtype=np.float64), np.zeros(plan["extra"].shape[0])])

    def _method(self, uncertainty_method):
        if uncertainty_method not in ESTIMATOR_METHODS:
            raise ParameterError(f"uncertainty_method {uncertainty_method!r} is not served by MbarMany's estimators "
                                 f"(one of {ESTIMATOR_METHODS}); 'svd' uncertainties are not served here")
        if uncertainty_method == "bootstrap" and self._B <= 0:
            raise ParameterError("Cannot request bootstrap sampling of expectations without any bootstraps.")
        return uncertainty_method == "bootstrap"

    @staticmethod
    def _with_boot(out, inner, keys):
        """out plus inner's bootstrap keys among `keys` (nothing without bootstrap)."""
        return dict(out, **{k: inner[k] for k in keys if k in inner})

    def compute_perturbed_free_energies(self, u_ln_list, compute_uncertainty=True, uncertainty_method=None,
                                        warning_cutoff=1.0e-10):
        """Delta_f, dDelta_f (compute_uncertainty) of the states u_ln_list[p] [L, N_p] of each problem
        (MBAR.compute_perturbed_free_energies).

        uncertainty_method="bootstrap" (n_bootstraps > 0 at construction): dDelta_f is the standard deviation over
        replicates of the perturbed free energies, a vector [L] as the reference returns it, not the [L, L] matrix of
        the analytic methods, and each dict adds bootstrapped_f [B, L]."""
        boot = self._method(uncertainty_method)
        reqs = []
        for p, u_ln in enumerate(self._entries(u_ln_list, "u_ln_list")):
            if u_ln is None:
                reqs.append(None)
                continue
            u_ln = self._rows(p, u_ln, "u_ln")
            reqs.append((np.array([0.0]), u_ln, np.arange(u_ln.shape[0])))
        inner, path = self._inner_many(reqs, uncertainty_method, bool(compute_uncertainty) and not boot)
        return [None if r is None else
                dict(self._with_boot(ex.perturbed_result(r, compute_uncertainty, warning_cutoff, uncertainty_method),
                                     r, ("bootstrapped_f",)), path=w)
                for r, w in zip(inner, path)]

    def compute_expectations(self, A_n_list, u_ln_list=None, output="averages", state_dependent=False,
                             compute_uncertainty=True, uncertainty_method=None, warning_cutoff=1.0e-10,
                             return_theta=False):
        """mu, sigma (compute_uncertainty) and Theta (return_theta) of the observables A_n_list[p] ([N_p], or [L, N_p]
        when state_dependent) at the states u_ln_list[p] [L, N_p] (the problem's own states when None)
        (MBAR.compute_expectations).

        uncertainty_method="bootstrap" (n_bootstraps > 0 at construction): sigma is the standard deviation over
        replicates of the observables ("averages") or of their differences A_b - A_b^T ("differences"), Theta is the
        "svd-ew" one of the problem's own samples, and each dict adds bootstrapped_observables [B, L] and
        bootstrapped_f [B, L]."""
        boot = self._method(uncertainty_method)
        if output not in ("averages", "differences"):
            raise ParameterError(f"output={output!r} must be 'averages' or 'differences'")
        u_lns = self._entries(u_ln_list, "u_ln_list")
        reqs, Ks = [], []
        for p, A_n in enumerate(self._entries(A_n_list, "A_n_list")):
            if A_n is None:
                reqs.append(None)
                Ks.append(0)
                continue
            u = self._probs[p][0] if u_lns[p] is None else self._rows(p, u_lns[p], "u_ln")
            A = self._rows(p, A_n, "A_n")
            if A.shape[0] != (u.shape[0] if state_dependent else 1):
                raise ParameterError(f"problem {p}: A_n has {A.shape[0]} rows for {u.shape[0]} states "
                                     f"(state_dependent={state_dependent})")
            reqs.append((A, u, ex.expectation_state_map(u.shape[0], state_dependent)))
            Ks.append(u.shape[0])
        theta = bool(return_theta or (compute_uncertainty and not boot))
        inner, path = self._inner_many(reqs, uncertainty_method, theta)
        keys = ("bootstrapped_observables", "bootstrapped_f")
        return [None if r is None else
                dict(self._with_boot(ex.expectations_result(r, Ks[p], output, compute_uncertainty, return_theta,
                                                            warning_cutoff, uncertainty_method), r, keys),
                     path=path[p])
                for p, r in enumerate(inner)]

    def compute_entropy_and_enthalpy(self, u_ln_list=None, uncertainty_method=None, warning_cutoff=1.0e-10):
        """Delta_f, dDelta_f, Delta_u, dDelta_u, Delta_s, dDelta_s of each problem at the states u_ln_list[p]
        [L, N_p] (every problem at its own states when u_ln_list is None; an entry None skips its problem)
        (MBAR.compute_entropy_and_enthalpy).  A problem's augmented rows number 3L; up to L = 64 they stay batched.

        uncertainty_method="bootstrap" (n_bootstraps > 0 at construction) follows the reference: dDelta_f from the
        problem's f_k_boots, dDelta_u from the bootstrapped observables and dDelta_s from their difference, and each
        dict adds bootstrapped_observables [B, L] and bootstrapped_f [B, L].  The reference pairs the bootstrapped
        observables with f_k_boots [B, K_p], so u_ln with L != K_p raises ParameterError."""
        boot = self._method(uncertainty_method)
        own = u_ln_list is None
        u_lns = [None] * len(self._probs) if own else self._entries(u_ln_list, "u_ln_list")
        reqs, Ls = [], []
        for p, u_ln in enumerate(u_lns):
            if u_ln is None and not own:
                reqs.append(None)
                Ls.append(0)
                continue
            u = self._probs[p][0] if own else self._rows(p, u_ln, "u_ln")
            L = u.shape[0]
            if boot and L != self._probs[p][0].shape[0]:
                raise ParameterError(f"problem {p}: bootstrap entropies and enthalpies pair u_ln's {L} states with the "
                                     f"problem's {self._probs[p][0].shape[0]} bootstrapped free energies")
            state_map = np.array([np.arange(L), np.arange(L)])
            reqs.append((u, u, state_map))
            Ls.append(L)
        inner, path = self._inner_many(reqs, uncertainty_method, not boot)
        keys = ("bootstrapped_observables", "bootstrapped_f")
        return [None if r is None else
                dict(self._with_boot(ex.entropy_enthalpy_result(r, Ls[p], warning_cutoff,
                                                                self.results[p]["f_k_boots"] if boot else None),
                                     r, keys), path=path[p])
                for p, r in enumerate(inner)]

    def _grams(self, problems=None):
        """W^T W at the final f of every problem (of `problems`): the solve's where it computed one, one batched
        moments call for the other batched problems, DeviceProblem.weight_moments for the rest."""
        P = len(self._probs)
        problems = range(P) if problems is None else problems
        need = [p for p in problems if p not in self._G]
        batched = [p for p in need if self.results[p]["path"] == "batch"]
        if batched:
            sums = self._dev.moments([self.results[p]["f_k"] for p in batched], want_G=True, all_rows=True,
                                     problems=[self._slot[p] for p in batched])
            self._count()
            for p, m in zip(batched, sums):
                if not m["flag"]:
                    self._G[p] = _gram_to_G(m["G"], self._probs[p][1])
        _, Prob = _classes()
        for p in need:
            if p not in self._G:
                u, N_k, _ = self._probs[p]
                with Prob(u, N_k, device=ms._DEVICE) as q:
                    _, self._G[p] = q.weight_moments(self.results[p]["f_k"])
        return [self._G[p] for p in problems]

    def compute_overlap(self):
        """scalar, eigenvalues, matrix of every problem (MBAR.compute_overlap), from W^T W at the final f.  A
        one-state problem has no second eigenvalue: its scalar is NaN, where the reference raises."""
        out = []
        for p, G in enumerate(self._grams()):
            N_k = self._probs[p][1]
            if len(N_k) > 1:
                d = estimators.overlap(G, N_k)
            else:
                O = np.asarray(N_k, dtype=np.float64) * np.asarray(G)
                d = {"scalar": np.nan, "eigenvalues": np.linalg.eigvals(O), "matrix": O}
            out.append(dict(d, path=self.results[p]["path"]))
        return out

    # ---- histogram free-energy surfaces (DESIGN.md 3.5h) ----
    def _per_problem(self, value, single):
        """value for every problem: one entry per problem (a list or tuple of P entries, each None or a valid
        single value for its problem) or one value for all; single(p, v) tells whether v is a single value."""
        P = len(self._probs)
        if isinstance(value, (list, tuple)) and len(value) == P and \
                all(v is None or single(p, v) for p, v in enumerate(value)):
            return list(value)
        return [value] * P

    def generate_fes(self, u_n_list, x_n_list, fes_type="histogram", histogram_parameters=None, n_bootstraps=0,
                     seed=None, kde_parameters=None):
        """The histogram FES of the target state u_n_list[p] [N_p] over the coordinates x_n_list[p] ([N_p] or
        [N_p, dims]) of every problem (pymbar.FES.generate_fes with fes_type="histogram"); an entry None skips its
        problem, whose earlier surface, if any, stays.  histogram_parameters: {"bin_edges": ...} for every problem,
        or one such dict per problem.  self.histogram_datas[p] becomes the reference's histogram_data dict.

        The batched problems' f comes from one bin_moments call per wave (waves under FES_WAVE_BYTES); a problem that
        took the single path in the solve, or whose request the batch flags, goes through fes.histogram_fes on a
        DeviceProblem.  Every argument is checked before any device work.

        n_bootstraps = B >= 2 (DESIGN.md 3.5h') also builds B bootstrap replicates of every requested surface:
        self.replicate_histogram_datas[p] becomes the reference's FES.histogram_datas, B ReplicateHistograms, and
        self.fes_boot_single[p] counts those that took the single path.  Replicate b of problem p is the one
        pymbar.FES(u_kn_p, N_k_p).generate_fes(..., n_bootstraps=B, seed=seed[p]) draws from numpy's global
        generator; problems draw in increasing order, and the generator ends where P such calls leave it.  seed: None
        (continue the global stream) or one entry per problem, an int >= 0 (np.random.seed before the problem's
        draws), -1 or None.  With B = 0 the generator is not touched and replicate_histogram_datas[p] becomes None.
        A problem with an empty state, or a replicate that draws no sample from a bin tuple of the surface, raises
        ParameterError; a call that raises restores the generator and changes no surface.

        fes_type="kde" (DESIGN.md 3.5h'') builds what pymbar.FES(u_kn_p, N_k_p).generate_fes(u_n_p, x_n_p,
        fes_type="kde", kde_parameters=..., n_bootstraps=B, seed=seed[p]) builds.  kde_parameters: one dict of
        KernelDensity parameters for every problem, or one per problem; an unknown key raises the reference's
        ParameterError, and so do parameters fes.kde_settings does not serve (another metric, metric_params, more
        than 4 dimensions, values sklearn's fit rejects) and None, where the reference raises TypeError.  b = 0's
        weights come from one log_weights call per wave on the batch (DeviceProblem.log_denominator for problems on
        the single path or flagged there; self._kde[p]["path"]), normalised as fes.py:411-414 does.  Replicate b puts
        weight V_bn = sum of w_m over the positions m with idx_b[m] = n on sample n (b = 0's weights by position,
        fes.py:689-699); the reference's K MBAR constructions per replicate change no KDE output and are not run, but
        their seed draws are made.  The call's coordinates are uploaded once into one DeviceKdeMany; the surfaces are
        scored at get_fes.  self.kde_settings[p] becomes {"kernel", "h", "D"} and self.fes_types[p] "kde"; a KDE surface
        clears the problem's histogram_datas and replicate_histogram_datas, and a histogram surface clears its KDE."""
        if fes_type not in FES_TYPES:
            raise ParameterError(f"fes_type {fes_type!r} is not served by MbarMany (one of {FES_TYPES})")
        P = len(self._probs)
        seeds = _validate_fes_boot(n_bootstraps, seed, P)
        B = int(n_bootstraps)
        for name, v in (("u_n_list", u_n_list), ("x_n_list", x_n_list)):
            if v is None or len(v) != P:
                raise ParameterError(f"{name} must hold one entry (or None) per problem ({P}), got "
                                     f"{'None' if v is None else len(v)}")
        if fes_type == "kde":
            return self._generate_kde(u_n_list, x_n_list, kde_parameters, B, seeds)
        params = self._per_problem(histogram_parameters, lambda p, v: isinstance(v, dict))
        reqs = {}
        for p in range(P):
            u, x = u_n_list[p], x_n_list[p]
            if u is None and x is None:
                continue
            if u is None or x is None:
                raise ParameterError(f"problem {p}: give both u_n and x_n, or neither")
            par = params[p]
            if not isinstance(par, dict) or "bin_edges" not in par:
                raise ParameterError(f"problem {p}: histogram_parameters must be a dict with 'bin_edges', got "
                                     f"{par!r}")
            N = self._probs[p][0].shape[1]
            u = np.asarray(u, dtype=np.float64)
            if u.shape != (N,):
                raise ParameterError(f"problem {p}: u_n has shape {u.shape}, the problem has N={N} samples")
            if np.isnan(u).any():
                raise ParameterError(f"problem {p}: u_n holds NaN")
            edges = par["bin_edges"]
            dims = len(hist._edges(edges))
            xs = np.shape(x)
            if not ((len(xs) == 1 and dims == 1 and xs[0] == N) or (len(xs) == 2 and xs == (N, dims))):
                raise ParameterError(f"problem {p}: x_n has shape {xs}, the problem has N={N} samples and the bins "
                                     f"{dims} dimension(s)")
            if B > 0 and np.any(np.asarray(self._probs[p][1]) == 0):
                raise ParameterError(f"problem {p}: a state without samples cannot be resampled for bootstrap "
                                     f"surfaces")
            data, dense, nb = hist.histogram_bins(x, edges)
            reqs[p] = dict(u_n=u, x_n=x, edges=edges, data=data, dense=dense, nb=nb)
        batched = [p for p in sorted(reqs) if self.results[p]["path"] == "batch" and p in self._slot]
        single = [p for p in sorted(reqs) if p not in batched]
        for wave in _waves(batched, lambda p: bin_bytes(*self._probs[p][0].shape, reqs[p]["nb"], False),
                           FES_WAVE_BYTES):
            out, flags = self._dev.bin_moments([self._slot[p] for p in wave], [self.results[p]["f_k"] for p in wave],
                                               [reqs[p]["u_n"] for p in wave], [reqs[p]["dense"] for p in wave],
                                               [reqs[p]["nb"] for p in wave], want_C=False)
            self._count()
            for p, (f_bin, _, _), flag in zip(wave, out, flags):
                if flag:
                    single.append(p)
                else:
                    reqs[p]["data"] = hist.with_bin_f(reqs[p]["data"], f_bin)
                    reqs[p]["path"] = "batch"
        _, Prob = _classes()
        for p in sorted(single):
            u_kn, N_k, _ = self._probs[p]
            r = reqs[p]
            try:
                with Prob(u_kn, N_k, device=ms._DEVICE) as q:
                    r["data"] = hist.histogram_fes(q, self.results[p]["f_k"], r["u_n"], r["x_n"], r["edges"])
            except Exception as err:
                raise _noted(err, p)
            r["path"] = "single"
        reps, nsingle = {}, {}
        if B > 0:
            state = np.random.get_state()
            try:
                reps, nsingle = self._fes_replicates(reqs, B, seeds)
            except BaseException:
                np.random.set_state(state)
                raise
        for p, r in reqs.items():
            self.histogram_datas[p] = r["data"]
            self._fes[p] = dict(u_n=r["u_n"], dense=r["dense"], nb=r["nb"], path=r["path"], theta=None)
            self.replicate_histogram_datas[p] = reps.get(p)
            self.fes_boot_single[p] = nsingle.get(p, 0)
            self.fes_types[p] = "histogram"
            self.kde_settings[p] = None
            self._kde.pop(p, None)

    def _generate_kde(self, u_n_list, x_n_list, kde_parameters, B, seeds):
        """generate_fes(..., fes_type="kde") (DESIGN.md 3.5h''): every argument checked, then the target weights, the
        replicate weights and one DeviceKdeMany upload of the call's coordinates; the surfaces are committed last."""
        P = len(self._probs)
        params = self._per_problem(kde_parameters, lambda p, v: isinstance(v, dict))
        reqs = {}
        defaults = None
        for p in range(P):
            u, x = u_n_list[p], x_n_list[p]
            if u is None and x is None:
                continue
            if u is None or x is None:
                raise ParameterError(f"problem {p}: give both u_n and x_n, or neither")
            par = params[p]
            if not isinstance(par, dict):
                raise ParameterError(f"problem {p}: fes_type 'kde' needs kde_parameters, a dict of KernelDensity "
                                     f"parameters, got {par!r}")
            if defaults is None:
                defaults = _kde_defaults()
            for k in par:
                if k not in defaults:
                    raise ParameterError(f"problem {p}: Warning: {k} is not a parameter in KernelDensity")
            N = self._probs[p][0].shape[1]
            u = np.asarray(u, dtype=np.float64)
            if u.shape != (N,):
                raise ParameterError(f"problem {p}: u_n has shape {u.shape}, the problem has N={N} samples")
            if np.isnan(u).any():
                raise ParameterError(f"problem {p}: u_n holds NaN")
            xa = np.asarray(x, dtype=np.float64)
            if xa.ndim == 1:
                xa = xa.reshape(-1, 1)
            if xa.ndim != 2 or xa.shape[0] != N:
                raise ParameterError(f"problem {p}: x_n has shape {np.shape(x)}, the problem has N={N} samples")
            if not np.all(np.isfinite(xa)):
                raise ParameterError(f"problem {p}: x_n holds NaN or infinite coordinates")
            settings = hist.kde_settings(dict(defaults, **par), N, xa.shape[1])
            if settings is None:
                raise ParameterError(f"problem {p}: kde_parameters {par!r} in {xa.shape[1]} dimension(s) are not served "
                                     f"by MbarMany (euclidean metric, no metric_params, 1 to 4 dimensions, and values "
                                     f"KernelDensity.fit accepts)")
            if B > 0 and np.any(np.asarray(self._probs[p][1]) == 0):
                raise ParameterError(f"problem {p}: a state without samples cannot be resampled for bootstrap "
                                     f"surfaces")
            reqs[p] = dict(u_n=u, x=np.ascontiguousarray(xa), settings=settings)
        if not reqs:
            return
        # b = 0: log w_n = -u_n - L_n, one log_weights call per wave on the batch; the single path otherwise
        log_w = {}
        batched = [p for p in sorted(reqs) if self.results[p]["path"] == "batch" and p in self._slot]
        single = [p for p in sorted(reqs) if p not in batched]
        for wave in _waves(batched, lambda p: log_weight_bytes(*self._probs[p][0].shape), FES_WAVE_BYTES):
            out, flags = self._dev.log_weights([self._slot[p] for p in wave], [self.results[p]["f_k"] for p in wave],
                                               [reqs[p]["u_n"] for p in wave])
            self._count()
            for p, lw, flag in zip(wave, out, flags):
                if flag:
                    single.append(p)
                else:
                    log_w[p] = lw
                    reqs[p]["path"] = "batch"
        _, Prob = _classes()
        for p in sorted(single):
            u_kn, N_k, _ = self._probs[p]
            with Prob(u_kn, N_k, device=ms._DEVICE) as q:
                L = q.log_denominator(np.asarray(self.results[p]["f_k"], dtype=np.float64))
            log_w[p] = -reqs[p]["u_n"] - L            # facade._device_log_weights
            reqs[p]["path"] = "single"
        for p in sorted(reqs):
            lw = log_w[p]
            with np.errstate(invalid="ignore", over="ignore"):
                w = np.exp(lw - np.max(lw))           # fes.py:411-414
                w = w / np.sum(w)
            if not np.all(np.isfinite(w)):
                raise ParameterError(f"problem {p}: the target state's weights are not finite (log w_n holds NaN, or "
                                     f"every sample has weight 0)")
            reqs[p]["w"] = w
            reqs[p]["log_sum_w"] = float(np.log(np.sum(w)))
        order = sorted(reqs)
        Kde = _kde_class()
        dev = Kde([reqs[p]["x"] for p in order], device=ms._DEVICE)
        try:
            if B > 0:
                state = np.random.get_state()
                try:
                    for p in order:
                        reqs[p]["V"] = self._kde_replicates(p, reqs[p]["w"], B, seeds[p])
                except BaseException:
                    np.random.set_state(state)
                    raise
        except BaseException:
            dev.close()
            raise
        self._stack.enter_context(dev)
        self.kde_stats["upload_bytes"] += int(sum(reqs[p]["x"].nbytes for p in order))
        for i, p in enumerate(order):
            r = reqs[p]
            self._kde[p] = dict(dev=dev, set=i, w=r["w"], log_sum_w=r["log_sum_w"], V=r.get("V"),
                                settings=r["settings"], path=r["path"])
            self.kde_settings[p] = r["settings"]
            self.fes_types[p] = "kde"
            self.histogram_datas[p] = None
            self.replicate_histogram_datas[p] = None
            self.fes_boot_single[p] = 0
            self._fes.pop(p, None)

    def _kde_replicates(self, p, w, B, seed):
        """V [B, N_p]: the weight of every sample in each of problem p's B bootstrap replicates, V_bn = sum of w_m over
        the positions m with idx_b[m] = n (the reference fits replicate b to x_n[idx_b] with b = 0's weights by
        position, fes.py:689-699), drawn from numpy's global generator as the reference draws them."""
        t0 = time.perf_counter()
        N_k = np.asarray(self._probs[p][1]).astype(np.int64)
        V = np.empty((B, len(w)))

        def each(b, idx):
            V[b] = np.bincount(idx, weights=w, minlength=len(w))

        if seed is not None:
            np.random.seed(seed)
        fb.draw_replicates(N_k, B, each)
        self.host_stats["fes_draws_s"] += time.perf_counter() - t0
        return V

    def _fes_replicates(self, reqs, B, seeds):
        """({p: [B ReplicateHistogram]}, {p: replicates on the single path}) of every request of generate_fes, drawn
        from numpy's global generator in problem order.  The (problem, replicate) pairs of problems whose b = 0
        request took the batch path are drawn and evaluated one wave at a time under BOOT_WAVE_BYTES: _solve_slots,
        then one replicate_bin_moments call on the same resident slots, each problem's target uploaded once.  The
        others, and replicates the batch does not serve, go through fes_bootstrap.histogram_replicates."""
        probs, dev = self._probs, self._dev
        reps = {p: [None] * B for p in reqs}
        states = {p: [None] * B for p in reqs}
        single = {p: set() for p in reqs}
        overflow = set()
        wave, used = [], 0

        def flush():
            nonlocal wave, used
            if wave:
                self._fes_wave(wave, reqs, reps, single)
            wave, used = [], 0

        for p in sorted(reqs):
            r = reqs[p]
            N_k = np.asarray(probs[p][1]).astype(np.int64)
            N = int(N_k.sum())
            tuples, n_tuples = fb.tuple_index(r["data"]["bin_n"])
            batched = r["path"] == "batch"
            need = slot_bytes(*probs[p][0].shape) + rep_bin_bytes(*probs[p][0].shape, r["nb"])
            if seeds[p] is not None:
                np.random.seed(seeds[p])
            for b in range(B):
                t0 = time.perf_counter()
                drawn = []
                states[p][b] = fb.draw_replicates(N_k, 1, lambda _, idx: drawn.append(idx))[0]
                idx = drawn[0]
                covered = fb.covers_every_tuple(idx, tuples, n_tuples)
                c = np.bincount(idx, minlength=N) if batched and p not in overflow else None
                self.host_stats["fes_draws_s"] += time.perf_counter() - t0
                if not covered:
                    raise ParameterError(f"problem {p}: bootstrap replicate {b} draws no sample from a bin of the "
                                         f"surface, so its histogram has fewer bins than the surface")
                if c is None:
                    continue
                if c.max() > 65535:
                    overflow.add(p)
                    continue
                if wave and used + need > BOOT_WAVE_BYTES:
                    flush()
                wave.append((p, b, c.astype(np.uint16), states[p][b]))
                used += need
        flush()
        if any(r["path"] == "batch" for r in reqs.values()):
            dev.set_replicates([], [])
        _, Prob = _classes()
        protocol = tuple(dict(st, tol=self._tol) for st in fb.solver_protocol(ms.DEFAULT_SOLVER_PROTOCOL))
        for p in sorted(reqs):
            r = reqs[p]
            picked = list(range(B)) if r["path"] != "batch" or p in overflow else sorted(single[p])
            if not picked:
                continue
            u_kn, N_k, _ = probs[p]
            try:
                with Prob(u_kn, N_k, device=ms._DEVICE) as q:
                    got = fb.histogram_replicates(q, self.results[p]["f_k"], np.asarray(N_k).astype(np.int64),
                                                  r["u_n"], r["data"], [states[p][b] for b in picked], protocol)
            except Exception as err:
                raise _noted(err, p)
            for b, h in zip(picked, got):
                reps[p][b] = h
            single[p] = set(picked)
        return reps, {p: len(single[p]) for p in reqs}

    def _fes_wave(self, wave, reqs, reps, single):
        """One wave of (problem, replicate, counts, generator state): the replicates solved on resident slots
        (_solve_slots) and binned by one replicate_bin_moments call on those slots; replicates either step does not
        serve go to single."""
        dev = self._dev
        got = _solve_slots(dev, [self._slot[p] for p, _, _, _ in wave], [c for _, _, c, _ in wave],
                           [self.results[p]["f_k"] for p, _, _, _ in wave], self._tol, self._opts)
        ok = [s for s in range(len(wave)) if s in got]
        for s in range(len(wave)):
            if s not in got:
                single[wave[s][0]].add(wave[s][1])
        if not ok:
            return
        targets = list(dict.fromkeys(wave[s][0] for s in ok))
        tix = {p: t for t, p in enumerate(targets)}
        f_bins, flags = dev.replicate_bin_moments([self._slot[p] for p in targets], [reqs[p]["u_n"] for p in targets],
                                                  [reqs[p]["dense"] for p in targets],
                                                  [reqs[p]["nb"] for p in targets], ok,
                                                  [tix[wave[s][0]] for s in ok], [got[s] for s in ok])
        self._count()
        for s, f_bin, flag in zip(ok, f_bins, flags):
            p, b, _, state = wave[s]
            if flag:
                single[p].add(b)
                continue
            base = reqs[p]["data"]
            f = np.zeros(len(base["f"]))
            f[:reqs[p]["nb"]] = f_bin
            reps[p][b] = fb.ReplicateHistogram(f, base, state, np.asarray(self._probs[p][1]).astype(np.int64))

    def _thetas(self, problems):
        """Theta of the augmented problem ("svd-ew", fes.py:1382-1406) of every problem of `problems` that lacks
        one: one bin_moments call for C and D per wave of the batched ones, G from _grams; the single path
        (fes.histogram_theta) for the rest and for flagged requests."""
        need = [p for p in problems if self._fes[p]["theta"] is None]
        batched = [p for p in need if self._fes[p]["path"] == "batch"]
        single = [p for p in need if p not in batched]
        if batched:
            G = dict(zip(batched, self._grams(batched)))
        for wave in _waves(batched, lambda p: bin_bytes(*self._probs[p][0].shape, self._fes[p]["nb"], True),
                           FES_WAVE_BYTES):
            st = [self._fes[p] for p in wave]
            out, flags = self._dev.bin_moments([self._slot[p] for p in wave], [self.results[p]["f_k"] for p in wave],
                                               [s["u_n"] for s in st], [s["dense"] for s in st],
                                               [s["nb"] for s in st], want_C=True)
            self._count()
            for p, (_, C, D), flag in zip(wave, out, flags):
                if flag:
                    single.append(p)
                else:
                    self._fes[p]["theta"], _ = hist.augmented_theta(G[p], C, D, self._probs[p][1])
        _, Prob = _classes()
        for p in sorted(single):
            u_kn, N_k, _ = self._probs[p]
            s = self._fes[p]
            try:
                with Prob(u_kn, N_k, device=ms._DEVICE) as q:
                    s["theta"] = hist.histogram_theta(q, self.results[p]["f_k"], N_k, s["u_n"],
                                                      self.histogram_datas[p])
            except Exception as err:
                raise _noted(err, p)
            s["path"] = "single"

    def get_fes(self, x_list, reference_point="from-lowest", fes_reference=None, uncertainty_method=None):
        """f_i (and df_i with uncertainty_method="analytical" or "bootstrap") of every problem's surface at the points
        x_list[p] (pymbar.FES.get_fes), plus `path`, "batch" or "single"; an entry None skips its problem.
        fes_reference: one point for every problem, or one per problem.

        Histogram surfaces: reference points and their errors are those of the reference ("from-lowest",
        "from-specified"; "all-differences" and "from-normalization" raise what it raises).  The first "analytical"
        query computes Theta for every problem of the call that lacks one (one bin_moments call per wave) and keeps
        it.  "bootstrap" takes df_i from the replicates of generate_fes(..., n_bootstraps=B) (fes.py:1417-1422), with
        no device work.

        KDE surfaces (DESIGN.md 3.5h''): f_i = -score_samples(x) of the reference's KernelDensity, relative to
        "from-lowest", "from-specified" or "from-normalization", and df_i None without uncertainties, as
        _get_fes_kde (fes.py:1523-1609) returns them.  Every KDE problem of the call is answered by one
        DeviceKdeMany.log_sum call per uploaded sample-set object and wave (waves under KDE_WAVE_BYTES): a request
        holds a problem's queries and its "from-specified" point and, with "bootstrap", one request per replicate
        holds its queries under the replicate's weights.  df_i is then np.std over the replicates of
        -score_b - fmin, every replicate sharing b = 0's weight sum (fes.py:1590-1601).  As in the reference, the
        gaussian and tophat kernels draw from numpy's global generator at every query (KernelDensity.sample) and the
        other kernels raise NotImplementedError, and a dimension mismatch raises DataError.  "analytical" raises the
        reference's ParameterError; "bootstrap" with "from-normalization" raises ParameterError, where the reference
        fails with UnboundLocalError.  Problems are taken in increasing order; a call that raises, raises for the
        lowest failing problem and restores numpy's generator.  After close(), a KDE query raises ParameterError."""
        if uncertainty_method not in FES_UNCERTAINTY_METHODS:
            raise ParameterError(f"uncertainty_method {uncertainty_method!r} is not served by MbarMany's FES "
                                 f"(one of {FES_UNCERTAINTY_METHODS})")
        P = len(self._probs)
        if x_list is None or len(x_list) != P:
            raise ParameterError(f"x_list must hold one entry (or None) per problem ({P}), got "
                                 f"{'None' if x_list is None else len(x_list)}")
        asked = [p for p in range(P) if x_list[p] is not None]
        for p in asked:
            if self.fes_types[p] is None:
                raise ParameterError(f"problem {p}: get_fes before generate_fes built its surface")
            if self.fes_types[p] == "histogram" and uncertainty_method == "bootstrap" and \
                    self.replicate_histogram_datas[p] is None:
                raise ParameterError(f"problem {p}: Can't calculate uncertainties via bootstrap if bootstrapping was "
                                     f"not performed when running get_fes")
        kde_asked = [p for p in asked if self.fes_types[p] == "kde"]
        hist_asked = [p for p in asked if self.fes_types[p] == "histogram"]

        def single_ref(p, v):
            if self.fes_types[p] == "kde":
                dims = self.kde_settings[p]["D"]
            else:
                dims = self.histogram_datas[p]["dims"] if p in self._fes else 1
            return np.ndim(v) == 0 if dims == 1 else (np.shape(v) == (dims,))

        refs = self._per_problem(fes_reference, single_ref)
        out = [None] * P
        if kde_asked:
            got = self._kde_get_fes(kde_asked, x_list, reference_point, refs, uncertainty_method)
            for p in kde_asked:
                out[p] = got[p]
        analytical = uncertainty_method == "analytical"
        for p in hist_asked:
            data = self.histogram_datas[p]
            K = self._probs[p][0].shape[0]

            def df_fn(j, p=p, data=data, K=K):
                self._thetas(hist_asked)
                return hist.bin_uncertainties(self._fes[p]["theta"], K, j, len(data["f"]))

            def boot_fn(j, p=p, data=data):
                return fb.bootstrap_df(self.replicate_histogram_datas[p], j, len(data["f"]))

            fn = df_fn if analytical else (boot_fn if uncertainty_method == "bootstrap" else None)
            r = hist.query(data, x_list[p], reference_point, refs[p], fn)
            out[p] = dict(r, path=self._fes[p]["path"])
        return out

    def _kde_get_fes(self, problems, x_list, reference_point, refs, uncertainty_method):
        """{p: get_fes dict} of the KDE problems `problems` (increasing): kde_query_prepare for each, the device sums of
        every request in waves, then kde_query_finish (and kde_bootstrap_finish).  numpy's generator is restored when
        anything raises."""
        boot = uncertainty_method == "bootstrap"
        state = np.random.get_state()
        try:
            prep = {}
            for p in problems:
                if self._closed:
                    raise ParameterError(f"problem {p}: the KDE surface's samples were freed by close()")
                k = self._kde[p]
                x = np.array(x_list[p])
                if np.ndim(x) <= 1:
                    x = x.reshape(-1, 1)              # FES.get_fes
                y, Q = hist.kde_query_prepare(k["settings"], x, reference_point, refs[p])
                if reference_point not in ("from-lowest", "from-specified", "from-normalization"):
                    raise hist._kde_errors()[1](f"reference point choice {reference_point} for kde is unavailable")
                if uncertainty_method == "analytical":
                    raise ParameterError(f"problem {p}: Uncertainty method {uncertainty_method} for kde is not "
                                         f"implemented")
                if boot and k["V"] is None:
                    raise ParameterError(f"problem {p}: Cannot calculate bootstrap error of bootstrap KDE's not "
                                         f"determined")
                if boot and reference_point == "from-normalization":
                    raise ParameterError(f"problem {p}: bootstrap uncertainties of a KDE surface need a reference "
                                         f"point: 'from-normalization' has none (the reference fails there)")
                prep[p] = (y, Q)
            # requests: (problem, -1) for b = 0 (queries and the reference point), (problem, b) per replicate
            sums = {}
            by_dev = {}
            for p in problems:
                by_dev.setdefault(id(self._kde[p]["dev"]), []).append(p)
            for ps in by_dev.values():
                dev = self._kde[ps[0]]["dev"]
                items = [(p, -1) for p in ps]
                if boot:
                    items += [(p, b) for p in ps for b in range(self._kde[p]["V"].shape[0])]

                def need(it):
                    p, b = it
                    k = self._kde[p]
                    n = prep[p][0].shape[0] if b < 0 else prep[p][1]
                    return kde_bytes(len(k["w"]), k["settings"]["D"], n)

                for wave in _waves(items, need, KDE_WAVE_BYTES - KDE_PART_BYTES):
                    reqs = [(p, b) for p, b in wave]
                    ks = [self._kde[p] for p, _ in reqs]
                    got = dev.log_sum([k["set"] for k in ks], [k["settings"]["kernel"] for k in ks],
                                      [k["settings"]["h"] for k in ks],
                                      [k["w"] if b < 0 else k["V"][b] for (p, b), k in zip(reqs, ks)],
                                      [prep[p][0] if b < 0 else prep[p][0][:prep[p][1]] for p, b in reqs])
                    self._count_kde(dev)
                    for it, l in zip(reqs, got):
                        sums[it] = l
            out = {}
            for p in problems:
                k = self._kde[p]
                y, Q = prep[p]
                r, fmin = hist.kde_query_finish(k["settings"], sums[(p, -1)], Q, reference_point, k["log_sum_w"],
                                                with_fmin=True)
                if boot:
                    reps = np.array([sums[(p, b)] for b in range(k["V"].shape[0])])
                    r = fb.kde_bootstrap_finish(k["settings"], r, fmin, reps, k["log_sum_w"])
                out[p] = dict(r, path=k["path"])
            return out
        except BaseException:
            np.random.set_state(state)
            raise

    def _count_kde(self, dev):
        s = dev.last_stats()
        self.kde_stats["ms"] += s["ms"]
        self.kde_stats["launches"] += s["launches"]
        self.kde_stats["calls"] += 1
        self.kde_stats["pairs"] += s["pairs"]

    def compute_effective_sample_number(self):
        """N_eff [K_p] of every problem (MBAR.compute_effective_sample_number), from W^T W at the final f."""
        return [dict(N_eff=estimators.effective_sample_number(G), path=self.results[p]["path"])
                for p, G in enumerate(self._grams())]


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
    with MbarMany(u_kn_list, N_k_list, f_k_init=f_k_init, compute_uncertainty=compute_uncertainty,
                  uncertainty_method=uncertainty_method, return_theta=return_theta, solver_tolerance=solver_tolerance,
                  options=options, n_bootstraps=n_bootstraps, rseed=rseed) as m:
        return m.results

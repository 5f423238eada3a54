"""Edge cases of the batched MBAR pass (batch.cu, DESIGN.md 3.5g), an extended-precision restatement of one request,
the rule for when the device must flag a request, and the tolerances the outputs are held to.

A request is (u [K, N], N_k, f), optionally with replicate counts c_n (a weighted slot).  `restate` computes in long
double, on the array actually passed, what the device returns:

    L_n = log sum_{j sampled} N_j e^{f_j - u_jn},   a_kn = f_k - u_kn - L_n,
    S_k = sum_n c_n e^{a_kn},   Ghat_ij = sum_n c_n w_in w_jn,   sum L = sum_n c_n L_n,

with w_kn = N_k e^{a_kn} on sampled rows, e^{a_kn} on unsampled rows when all rows are asked for, 0 otherwise, and
c_n = 1 without counts.  Only drawn samples (c_n > 0) enter, as in the reference's gathered array.  Sums are kept in
the log domain too, so the rule can be judged where fp64 over- or underflows.

`predict_flag` restates the flag of batch_finalize_kernel.  A request is flagged when
  * a NaN reaches a sum: a drawn sample whose sampled-state energies are all +inf has no L_n;
  * a sampled S_k lies outside (1e-280, 1e300);
  * all rows are asked for and an unsampled S_k exceeds DBL_MAX;
  * the Gram is asked for and an entry of Ghat exceeds DBL_MAX (the diagonal holds the largest entry).
It returns the flag and its margin: the log-domain distance of the deciding quantity from its threshold.  Tests
assert the flag only where the margin is clear (> CLEAR), as `tests/_edges.bands` does.

`tiled` builds large-N problems from a block of 97 distinct columns (97 is not a multiple of 32, so the block never
lines up with tiles); the reference is computed once per distinct column with that column's multiplicity.
"""
import numpy as np

from tests import _edges as E
from tests import _moments as M

LD = np.longdouble
EPS = 2.0 ** -53
DBL_MAX = float(np.finfo(np.float64).max)
LOG_DBL_MAX = float(np.log(DBL_MAX))          # 709.78
LOG_S_LO, LOG_S_HI = float(np.log(1e-280)), float(np.log(1e300))
CLEAR = 0.05                                  # log-domain margin beyond which the flag is asserted
BLOCK = 97                                    # distinct columns of a tiled problem
UINT16_MAX = 65535


# ---- chunk geometry (batch_chunk_tiles in batch.cu) --------------------------------------------------------------
def chunk_tiles(nT, K):
    return max(max(2048 // K, 4), -(-nT // 4096))


def geometry(N, K):
    """(nT, tiles per chunk, chunks, tiles of the last chunk)."""
    nT = -(-int(N) // 32)
    ct = chunk_tiles(nT, K)
    nc = -(-nT // ct)
    return nT, ct, nc, nT - (nc - 1) * ct


# ---- the long-double restatement ----------------------------------------------------------------------------------
def _lse(x, axis):
    top = np.max(x, axis=axis, keepdims=True)
    top = np.where(np.isfinite(top), top, 0)
    with np.errstate(divide="ignore"):
        return (np.log(np.exp(x - top).sum(axis=axis, keepdims=True)) + top).squeeze(axis)


def restate(u, N_k, f, all_rows, mult=None, want_G=True):
    """Long-double sums of one request (see the module docstring).  mult: per-column multiplicities (counts, or the
    number of copies of a distinct column).  Returns dict with logS, S, G (None when it would not be finite),
    logG (log of the largest Ghat entry), sumL, nan (a drawn sample has no L_n), A (per row: a bound on the
    magnitudes the device's exp arguments are formed from), absL = sum c (|L'_n| + 4 max_k (|c_k| + |u'_kn|)) (the
    scale of L'_n and of its rounding), absx = sum c |x_n|."""
    u = np.asarray(u, np.float64)
    N_k = np.asarray(N_k, np.float64)
    K, N = u.shape
    m = np.ones(N) if mult is None else np.asarray(mult, np.float64)
    on = m > 0
    u, m = u[:, on], m[on]
    s = N_k > 0
    rows = np.ones(K, bool) if all_rows else s
    # the per-sample shift x_n = min over sampled states (0 where all are +inf), as the device uploads it; in long
    # double u - x is exact wherever it cancels, so energies offset by 1e8 cost the reference no precision
    xs = np.where(np.isfinite(u[s]), u[s], np.inf).min(axis=0)
    x = np.where(np.isfinite(xs), xs, 0.0)
    fL = np.asarray(f, np.float64).astype(LD)
    uL = u.astype(LD) - x.astype(LD)[None, :]
    logN = np.zeros(K, LD)
    logN[s] = np.log(N_k[s].astype(LD))
    with np.errstate(invalid="ignore"):
        L = _lse((fL[s] + logN[s])[:, None] - uL[s], axis=0)                # L'_n
    has = np.isfinite(u[s]).any(axis=0)
    nan = bool(np.any(~has)) if u.shape[1] else False
    Lf = np.where(has, L, 0)
    with np.errstate(invalid="ignore"):
        arg = fL[:, None] - uL - Lf[None, :]                              # -inf for +inf energies
    arg[~rows] = -np.inf
    logm = np.log(m.astype(LD))
    logS = _lse(arg + logm[None, :], axis=1) if arg.shape[1] else np.full(K, -np.inf, LD)
    logw = arg + np.where(s, logN, 0)[:, None]
    logGd = _lse(2 * logw + logm[None, :], axis=1) if arg.shape[1] else np.full(K, -np.inf, LD)
    logGd[~rows] = -np.inf
    logG = float(logGd.max())
    G = None
    if want_G and logG < 11000:
        w = np.exp(logw) * np.sqrt(m.astype(LD))[None, :]
        w[~rows] = 0
        G = w @ w.T
    # error bounds: the rounding of a_kn is a few eps times |f_k| + |u'_kn| + |L'_n| (+ |c| inside L'), counted over
    # the entries whose weight is in the normal range (floored ones are covered by entry_tol's absolute term); each
    # L'_n carries a few eps of |c_k| + |u'_kn| over its sampled entries
    Lp = Lf.astype(np.float64)
    up = np.abs(uL.astype(np.float64))
    with np.errstate(invalid="ignore"):
        mag = np.abs(np.asarray(f, np.float64))[:, None] + up + np.abs(Lp)[None, :]
    normal = np.isfinite(arg) & (arg + np.where(s, logN, 0)[:, None] >= M.LOG_NORMAL) & np.isfinite(mag)
    c = np.asarray(f, np.float64)[s] + np.log(N_k[s])
    cmax = float(np.max(np.abs(c)))
    A = np.where(normal, mag, 0).max(axis=1).astype(np.float64) + cmax if mag.size else np.full(K, cmax)
    with np.errstate(invalid="ignore"):
        lmag = np.abs(c)[:, None] + up[s]
    lmag = np.where(np.isfinite(lmag), lmag, 0).max(axis=0) if lmag.size else np.zeros(0)
    return dict(logS=logS, S=np.exp(logS), G=G, logG=logG, logGd=logGd,
                sumL=(m.astype(LD) * (L - x.astype(LD))).sum(), nan=nan, A=A,
                absL=float((m * (np.abs(Lp) + 4 * lmag)).sum()), absx=float((m * np.abs(x)).sum()),
                N=int(m.sum()) if mult is not None else N)


def predict_flag(u, N_k, f, all_rows, want_G, counts=None, ref=None):
    """(flag, margin) of one request: whether batch_finalize_kernel must flag it and the log-domain distance of the
    deciding quantity from its threshold (inf for a NaN, which is not a matter of degree)."""
    N_k = np.asarray(N_k, np.float64)
    r = restate(u, N_k, f, all_rows, mult=counts, want_G=False) if ref is None else ref
    if r["nan"]:
        return True, np.inf
    s = N_k > 0
    d = []                                            # > 0: on the flagged side
    ls = r["logS"].astype(np.float64)
    for k in np.flatnonzero(s):
        d.append(max(LOG_S_LO - ls[k], ls[k] - LOG_S_HI))
    if all_rows:
        d += [ls[k] - LOG_DBL_MAX for k in np.flatnonzero(~s)]
    if want_G:
        d.append(r["logG"] - LOG_DBL_MAX)
    top = max(d)
    return bool(top > 0), abs(top)


def is_clear(margin):
    return margin > CLEAR


# ---- tolerances --------------------------------------------------------------------------------------------------
def s_tol(S, A, N):
    """The Stol of the mbar_many tests, with A the magnitude bound of `restate`."""
    return 8 * EPS * (np.abs(A) + np.sqrt(N) + 8) * np.abs(np.asarray(S, np.float64)) + 1e-300


def log_s_tol(A, N, K):
    """Absolute bound on log S_k of an unsampled row.  The row is a running (max, sum) pair: each term e^{a - max}
    carries the rounding of its argument (a few eps times the magnitudes it is formed from, A_k) and of exp; the sum
    of positive terms then has a relative error of at most a few eps per combination: a 5-level warp butterfly, one
    merge per round of a warp (ceil(ct / 4)), three across the warps, one per chunk.  16 eps (A_k + log N + 8)
    covers the arguments and the butterfly; 4 eps per merge covers the rest (three roundings each)."""
    _, ct, nc, _ = geometry(N, K)
    return 16 * EPS * (np.abs(A) + np.log(N) + 8) + 4 * EPS * (-(-ct // 4) + 3 + nc)


def sum_l_tol(ref, N, K):
    """sum L = sum_n c_n L'_n - sum_n c_n x_n.  Each L'_n has an error of a few eps (|L'_n| + |c_k| + |u'_kn|)
    over its sampled entries (restate's absL holds that scale); the device adds
    them in a thread's rounds, a 128-thread tree and the chunk partials in order, and sum c x in strided runs of
    N / 256 and a 256-thread tree, each addition rounding relative to the running |sum| <= the sum of |terms|.  The
    cancellation in sum L' - sum x then leaves eps * sum |x_n|, which with energies offset by 1e8 dominates."""
    _, ct, nc, _ = geometry(N, K)
    depth_L = -(-ct // 4) + 7 + nc + 8
    depth_x = -(-int(N) // 256) + 9
    return EPS * (depth_L * ref["absL"] + depth_x * ref["absx"] + 8 * ref["N"]) + 1e-300


def check_request(d, ref, N_k, all_rows, N, wmax=1.0, what=""):
    """Hold one unflagged request's outputs to its restatement `ref`: S (rows asked for), log S of unsampled rows,
    Ghat and sum L, N samples, counts at most wmax.  Every returned number must be finite (S may be 0 and log S
    -inf for a row of +inf only)."""
    N_k = np.asarray(N_k, np.float64)
    K = len(N_k)
    r = ref
    s = N_k > 0
    rows = np.ones(K, bool) if all_rows else s
    S = r["S"]
    assert np.all(np.isfinite(d["S"][rows])), what
    assert np.all(np.isfinite(d["log_S"][rows]) | (d["S"][rows] == 0)), what
    assert M.excess(d["S"][rows], S[rows], s_tol(S, r["A"], N)[rows]) <= 1.0, (what, "S")
    uns = rows & ~s
    if uns.any():
        ls = r["logS"][uns]
        fin = np.isfinite(ls)
        assert np.array_equal(np.isfinite(d["log_S"][uns]), fin), (what, "log_S support")
        err = np.abs(d["log_S"][uns][fin].astype(LD) - ls[fin])
        # the row's largest term has an argument near log S_k, whatever range its weights are in
        tol = log_s_tol(np.maximum(r["A"][uns][fin], np.abs(ls[fin].astype(np.float64))), N, K)
        assert np.all(err <= tol), (what, "log_S", float(np.max(err / tol)))
    if "G" in d:
        assert np.all(np.isfinite(d["G"])), (what, "G finite")
        tolG = M.entry_tol(r["G"], r["A"], N, wmax)
        assert M.excess(d["G"], r["G"], tolG) <= 1.0, (what, "G")
    err = abs(LD(d["sum_L"]) - r["sumL"])
    assert err <= sum_l_tol(r, N, K), (what, "sum_L", float(err), sum_l_tol(r, N, K))


# ---- replicate counts --------------------------------------------------------------------------------------------
def multinomial_counts(N, seed, zero=()):
    """Counts over N samples that sum to N (as set_replicates requires), multinomial with equal probabilities.
    `zero`: (start, stop) ranges of samples that get no count (their share goes to the other samples)."""
    rng = np.random.RandomState(seed)
    p = np.ones(N)
    for a, b in zero:
        p[a:b] = 0
    return rng.multinomial(N, p / p.sum()).astype(np.int64)


def all_on_one(N, n):
    """Every count on sample n: N <= 65535 fits one uint16."""
    assert N <= UINT16_MAX
    c = np.zeros(N, np.int64)
    c[n] = N
    return c


def slot_counts(N, K, seed):
    """The weighted slot of a problem: multinomial counts, with one whole chunk of zeros when there are at least
    three chunks."""
    nT, ct, nc, _ = geometry(N, K)
    zero = ((ct * 32, 2 * ct * 32),) if nc >= 3 else ()
    return multinomial_counts(N, seed, zero)


# ---- cases -------------------------------------------------------------------------------------------------------
LADDERS = ("ladder_K2", "ladder_K5", "ladder_K16", "ladder_K17", "ladder_K33", "ladder_K63", "ladder_K64",
           "ladder_K5_tiny")


def ladder_case(name):
    c = M.build(name)
    return dict(name=name, u=c["u"], N=c["N"], f=c["f"])


def family_cases():
    """The exponent families at their known f: offset pairs, an empty state below and above the samples (past 1e6
    too) and 64 offset copies.  At that f every S_k is 1 (log S_k = 0), unsampled rows included."""
    out = []
    for d in E.A_DELTAS:
        c = E.offset_pair(d)
        out.append(dict(name=f"pair_{d:g}", u=c["u"], N=c["N"], f=c["f_true"]))
    for sign, deltas in ((-1.0, E.B_BELOW + (2e6, 1e8)), (1.0, E.B_ABOVE + (2e6, 1e8))):
        for d in deltas:
            c = E.with_unsampled(d, sign=sign)
            out.append(dict(name=f"unsampled_{'below' if sign < 0 else 'above'}_{d:g}", u=c["u"], N=c["N"],
                            f=c["f_true"]))
    for d in (650.0, 1100.0):
        c = E.offset_copies(64, d)
        out.append(dict(name=f"copies64_{d:g}", u=c["u"], N=c["N"], f=c["f_true"]))
    return out


def unsampled_shift_for(u, N_k, f, k, target, quantity, counts=None):
    """f with f_k (an unsampled row) shifted so that `quantity` ("logS": log S_k, "logG": log Ghat_kk) equals
    `target`.  Both are linear in f_k: log S_k by 1, log Ghat_kk by 2."""
    r = restate(u, N_k, f, True, mult=counts, want_G=False)
    now = float(r["logS"][k]) if quantity == "logS" else float(r["logGd"][k])
    g = np.array(f, np.float64)
    g[k] += (target - now) / (1.0 if quantity == "logS" else 2.0)
    return g


def sampled_shift_for(u, N_k, f, k, target, counts=None):
    """f with f_k (a sampled row) lowered until log S_k = target (a few fixed-point steps: for S_k << 1, log S_k
    moves with f_k one for one)."""
    g = np.array(f, np.float64)
    for _ in range(6):
        r = restate(u, N_k, g, False, mult=counts, want_G=False)
        g[k] += target - float(r["logS"][k])
    return g


def threshold_cases():
    """(name, u, N_k, f) of requests at +-0.5 in the log domain around each flag threshold, and the row of +inf
    only.  The placements are made for the plain request; a weighted slot shifts them by its counts' log S."""
    out = []
    pair = E.offset_pair(30.0)
    below = E.with_unsampled(60.0, sign=-1.0)
    for side in (-0.5, 0.5):
        f = sampled_shift_for(pair["u"], pair["N"], pair["f_true"], 1, LOG_S_LO + side)
        out.append((f"sampled_S_1e-280{side:+g}", pair["u"], pair["N"], f))
        f = unsampled_shift_for(below["u"], below["N"], below["f_true"], 2, LOG_DBL_MAX + side, "logS")
        out.append((f"unsampled_S_DBL_MAX{side:+g}", below["u"], below["N"], f))
        f = unsampled_shift_for(below["u"], below["N"], below["f_true"], 2, LOG_DBL_MAX + side, "logG")
        out.append((f"gram_DBL_MAX{side:+g}", below["u"], below["N"], f))
    # the example of the Gram rule: an empty state 400 kT below the samples, at f = 0
    c = E.with_unsampled(400.0, sign=-1.0)
    out.append(("gram_400kT_below_f0", c["u"], c["N"], np.array([0.0, 5.0, 0.0])))
    # an unsampled row of +inf only: S = 0, log S = -inf, no flag
    c = E.with_unsampled(10.0, sign=-1.0)
    u = c["u"].copy()
    u[2] = np.inf
    out.append(("unsampled_all_inf", u, c["N"], np.array([0.0, 5.0, 3.0])))
    return out


def nan_case():
    """A problem one of whose samples has +inf energy in every sampled state: no L_n, a NaN reaches the sums."""
    c = E.with_unsampled(10.0, sign=-1.0)
    u = c["u"].copy()
    u[:2, 7] = np.inf
    return u, c["N"], c["f_true"]


def undrawn_nan_case():
    """The problem of nan_case with counts that never draw the sample without L_n: the replicate's sums exist."""
    u, N_k, f = nan_case()
    N = u.shape[1]
    c = multinomial_counts(N, 3, zero=((7, 8),))
    return u, N_k, f, c


def offset_energies(u, scale, seed):
    """u_kn + o_n with per-sample offsets of magnitude `scale` and random sign, as the reduced potentials of a
    solvated system carry (the rounding of the sum is part of the array passed)."""
    rng = np.random.RandomState(seed)
    o = scale * rng.choice([-1.0, 1.0], size=u.shape[1]) * (1.0 + 0.25 * rng.uniform(size=u.shape[1]))
    return u + o[None, :]


# ---- large N: a tiled block of distinct columns ----------------------------------------------------------------
def tiled_block(K=64, seed=64):
    """(block [K, 97], f): columns of a well-overlapping ladder with empty states first, in the middle and last and
    a few +inf entries in sampled rows."""
    c = M.ladder(K, max(2, -(-130 // (K - 3))), gaps=(1.5,), unsampled=(0, K // 2, K - 1), n_inf=12, seed=seed)
    rng = np.random.RandomState(seed)
    cols = np.sort(rng.choice(c["u"].shape[1], BLOCK, replace=False))
    return c["u"][:, cols].copy(), c["f"]


def tiled_N_k(K, N):
    """N samples spread over the sampled states of tiled_block (every state but 0, K/2 and K - 1)."""
    N_k = np.zeros(K)
    s = np.setdiff1d(np.arange(K), [0, K // 2, K - 1])
    N_k[s] = N // len(s)
    N_k[s[: N - int(N_k.sum())]] += 1
    return N_k


def tiled(block, N):
    """u [K, N] with column n = block[:, n % 97]."""
    return block[:, np.arange(N) % block.shape[1]]


def column_mult(N, counts=None, width=BLOCK):
    """Multiplicity of each distinct column: its copies, or the sum of its copies' counts."""
    n = np.arange(N) % width
    return np.bincount(n, weights=None if counts is None else counts, minlength=width).astype(np.float64)

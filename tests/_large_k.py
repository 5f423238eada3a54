"""Above 2048 states: the generic pass's launch plan, permuted ladders, and a sparse extended-precision reference of
the pass and of the second moments, with the tolerances the device is held to.

Above K = 2048 every pass is `pass_generic_kernel` and every Hessian is `weights_kernel` + `hessian_big_kernel` in
launches of at most 128 block pairs.  The generic kernel is sized from K alone (`launch_pass_generic`): W warps per
CTA, each with a 32 x 33 transposition tile and a [K][2] accumulator in shared memory.  `generic_plan` restates that
sizing, so a test can name the configuration it covers and assert it against `last_kernels()`.

A dense long-double reference needs 16 bytes per entry of u_kn (about 6 GB at K = 8192 and a few tiles per warp), so
`sparse_moments_ld` keeps, per sample, only the entries whose exponent lies within `cut` of the sample's largest one,
or within `cut` of the largest exponent of their own row (relative to its sample's maximum), so that no row is cut away
whole.  Every weight it drops is below e^-cut (module docstring of _moments: w_kn <= 1) and below e^-cut times its
row's largest weight, so the dropped part of N_k S_k and of every Ghat_ij is at most M e^-cut with M the sum of the
multiplicities (and at most N max(m) e^-cut relative for a row), and the dropped part of a denominator D_n at most
K e^-cut relative.  At the default cut of 1500 that is far below anything fp64 represents.
"""
import numpy as np

from tests import _moments as M

LD = M.LD
EPS = M.EPS
CUT = 1500.0

# ---- the generic pass's launch plan (pass_generic.cu, launch_pass_generic) ---------------------------------------
SMEM_BUDGET = 200 * 1024 - 256      # dynamic shared memory the kernel may take, less the 32-entry exp table
TILE_BYTES = 32 * 33 * 8            # one warp's transposition tile
MAX_GRID = 132 * 4                  # internal.cuh MAX_GRID: rows of the per-CTA partials buffer
K_MAX = 8192                        # MBAR_B200_MAX_STATES
FUSED_K_MAX = 2048                  # above this the fused pass never runs


def generic_plan(K, N, sm_count=132):
    """W (warps per CTA), smem (bytes), ctas_per_sm, grid, n_tiles and tiles_per_warp of one generic pass."""
    per_warp = TILE_BYTES + 16 * K
    W = min(8, SMEM_BUDGET // per_warp)
    smem = 256 + W * per_warp
    ctas_per_sm = 1 if smem > 100 * 1024 else 2
    n_tiles = -(-int(N) // 32)
    grid = min(-(-n_tiles // W), sm_count * ctas_per_sm, MAX_GRID)
    return dict(K=K, N=int(N), W=W, smem=smem, ctas_per_sm=ctas_per_sm, grid=grid, n_tiles=n_tiles,
                tiles_per_warp=-(-n_tiles // (grid * W)), max_grid=min(sm_count * ctas_per_sm, MAX_GRID))


def w_bands():
    """[(W, K_first, K_last)] over 1 <= K <= K_MAX, from the sizing formula."""
    bands = []
    for K in range(1, K_MAX + 1):
        W = generic_plan(K, 32)["W"]
        if bands and bands[-1][0] == W:
            bands[-1][2] = K
        else:
            bands.append([W, K, K])
    return [tuple(b) for b in bands]


def generic_ks():
    """Both sides of every change of W, K_MAX, and one K whose plan puts two CTAs on an SM."""
    ks = {K_MAX}
    for W, first, last in w_bands():
        if first > 1:
            ks.update((first - 1, first))
    two = max(K for K in range(1, 400) if generic_plan(K, 32)["ctas_per_sm"] == 2)
    ks.add(two - 70)
    return sorted(ks)


REGIMES = ("few", "one", "several")


def regime_n(K, regime, sm_count=132):
    """A sample count N (never a multiple of 32) for which the plan gives fewer tiles than warps in one CTA ('few';
    one tile, N < 32, when W <= 2), about one tile per warp ('one') or three tiles per warp ('several')."""
    p = generic_plan(K, 32, sm_count)
    W, g = p["W"], p["max_grid"]
    if regime == "few":
        return max(32 * (W - 2) + 5, 17)
    tiles = g * W if regime == "one" else 3 * g * W
    return 32 * tiles - 11


# ---- cases ---------------------------------------------------------------------------------------------------------
def _counts(n_sampled, n_per):
    """Bresenham spread of n_per (may be fractional) samples per state over n_sampled states."""
    edges = np.floor(np.arange(n_sampled + 1) * float(n_per) + 0.5).astype(int)
    return np.diff(edges).astype(np.float64)


def permutation(K, seed):
    return np.random.RandomState(10_000 + seed).permutation(K)


def permuted_ladder(K, n_per, seed, unsampled=(), n_inf=0, gaps=M.GAPS, f_noise=0.05):
    """_moments.ladder's energies with the state order permuted by a fixed permutation, so that neighbours on the
    ladder sit in arbitrary 128 x 128 block pairs.  `n_per` samples per sampled state (fractional: spread evenly);
    `unsampled` are indices AFTER the permutation.  Same dict as _moments.ladder; N is never a multiple of 32."""
    rng = np.random.RandomState(seed)
    perm = permutation(K, seed)                       # new state i is ladder state perm[i]
    centres = np.concatenate([[0.0], np.cumsum([gaps[k % len(gaps)] for k in range(K - 1)])])[perm]
    sampled = np.ones(K, bool)
    sampled[list(unsampled)] = False
    N_k = np.zeros(K)
    N_k[sampled] = _counts(int(sampled.sum()), n_per)
    if N_k.sum() == 0:
        N_k[np.flatnonzero(sampled)[0]] = 1
    if int(N_k.sum()) % 32 == 0:
        N_k[np.flatnonzero(sampled)[-1]] += 1
    owner = np.repeat(np.arange(K), N_k.astype(int))
    x = centres[owner] + rng.normal(size=owner.size)
    u = 0.5 * (x[None, :] - centres[:, None]) ** 2
    if n_inf:
        n = rng.randint(0, owner.size, size=n_inf)
        k = (owner[n] + 1 + rng.randint(0, K - 1, size=n_inf)) % K
        u[k, n] = np.inf
    f = rng.normal(scale=f_noise, size=K)
    f -= f[0]
    mult = rng.poisson(1.0, size=owner.size).astype(np.float64)
    return dict(u=u, N=N_k, f=f, mult=mult)


def few_sampled(K, N, seed):
    """unsampled indices leaving about N / 1.5 evenly spread sampled states (for N well below K)."""
    n_s = max(1, min(K, int(N / 1.5)))
    keep = np.unique(np.linspace(0, K - 1, n_s).astype(int))
    return tuple(np.setdiff1d(np.arange(K), keep))


# ---- tolerances ----------------------------------------------------------------------------------------------------
# Per entry of the pass, the device computes a' = c_k - u'_kn - L'_n in the frame shifted by x_n (u' = u - x_n, L' =
# L + x_n) and then exp(a') with its own exp.
EXP_REL = 2 * EPS                   # test_device_exp: |exp_fast(a) - e^a| <= (2 eps + 3.35e-17 |a|) e^a
EXP_ARG = 3.35e-17
ARG_ROUND = 3 * EPS                 # the shift u - x_n and the two subtractions of a', each rounding on |c|+|u'|+|L'|
LOG_MERGE = 4 * EPS                 # one (max, sum) merge of the log-domain rows: exp of a difference, a product, a sum


def exp_rel(a):
    return EXP_REL + EXP_ARG * np.abs(np.asarray(a, np.float64))


def reduction_depth(plan):
    """Additions a summand of S_k passes through: the plan's own `depth` where it states one (tests/_fused.py), else
    the generic pass's: 32 samples of a tile summed by one lane, the tiles of a warp, the W warps of a CTA, then the
    CTAs in index order.  Sequential sums of positive terms: relative error <= depth eps."""
    if "depth" in plan:
        return plan["depth"]
    return 32 + plan["tiles_per_warp"] + plan["W"] + plan["grid"]


def sparse_moments_ld(u, N_k, f, mult=None, all_rows=False, cut=CUT, want_G=False, chunk=None, c_abs=None):
    """The pass and the second moments in long double from the dense u [K, N], column chunk by column chunk, keeping
    the entries within `cut` of each sample's largest exponent.

    Returns a dict with L [N] (L_n = log sum_{j sampled} N_j e^(f_j - u_jn)), sumL, S [K] (sum_n m_n W_nk, all rows),
    logS [K], x [N] (the device's shift), A [K] (largest |exponent| of a normal-range weight, as _moments.moments_ld),
    drop (bound on the dropped part of any N_k S_k or Ghat_ij), and the error budget of the device's pass:
    dL [N] (absolute, of L_n), eS [K] (sum_n m_n W_nk e_kn / S_k, the first-order relative error of S_k from its
    entries) and eLogW [K] (the same for the log-domain rows).  With want_G: Gi, Gj, Gv, the support of Ghat
    (i >= j) in long double.  `c_abs` [K]: the magnitude of the state constant the device puts into each row's exp
    arguments where it is not |f_k + log N_k| (the fused pass centres the constants on a midpoint and gives unsampled
    rows log N = -80 in an all-state pass); the error budget then rounds on the larger of the two."""
    u = np.asarray(u, np.float64)
    K, N = u.shape
    N_k = np.asarray(N_k, np.float64)
    s = N_k > 0
    fL = np.asarray(f, np.float64).astype(LD)
    logN = np.zeros(K, LD)
    logN[s] = np.log(N_k[s].astype(LD))
    c = fL + logN                                   # unsampled rows: c = f (log N = 0)
    c64 = c.astype(np.float64)
    cab = np.abs(c64) if c_abs is None else np.maximum(np.abs(c64), np.asarray(c_abs, np.float64))
    m = np.ones(N) if mult is None else np.asarray(mult, np.float64)
    rows = np.ones(K, bool) if all_rows else s
    chunk = chunk or max(32, (1 << 23) // K)
    out = dict(L=np.empty(N, LD), x=np.empty(N), dL=np.empty(N), S=np.zeros(K, LD), eS=np.zeros(K, LD),
               eLogW=np.zeros(K, LD), A=np.zeros(K))
    Gi, Gj, Gv = [], [], []
    with np.errstate(invalid="ignore", over="ignore"):
        # first sweep: each row's largest exponent relative to its sample's maximum, so that no row is cut away whole
        best = np.full(K, -np.inf)
        for n0 in range(0, N, chunk):
            a64 = c64[:, None] - u[:, n0:min(N, n0 + chunk)]
            top = np.where(s[:, None], a64, -np.inf).max(axis=0)
            live = m[n0:min(N, n0 + chunk)] > 0           # a weight of multiplicity 0 adds nothing to its row
            best = np.maximum(best, np.where(live[None, :], a64 - top[None, :], -np.inf).max(axis=1))
        shift = np.where(np.isfinite(best), best, 0.0).astype(LD) - logN
        for n0 in range(0, N, chunk):
            n1 = min(N, n0 + chunk)
            uc = u[:, n0:n1]
            x = np.where(np.isfinite(uc[s]), uc[s], np.inf).min(axis=0)
            a64 = c64[:, None] - uc
            top = np.where(s[:, None], a64, -np.inf).max(axis=0)
            rel = a64 - top[None, :]
            kk, nn = np.nonzero((rel >= -cut) | (rel >= best[:, None] - cut))
            aL = c[kk] - uc[kk, nn].astype(LD)
            # denominators over the kept sampled entries
            sk = s[kk]
            D = np.zeros(n1 - n0, LD)
            np.add.at(D, nn[sk], np.exp(aL[sk] - top[nn[sk]].astype(LD)))
            L = top.astype(LD) + np.log(D)
            out["L"][n0:n1] = L
            out["x"][n0:n1] = x
            # error budget of L'_n: the K-term sequential sum of D_n, each term's argument and exp, the log
            up = np.abs(uc[kk, nn] - x[nn])
            mprime = np.abs(top + x)
            Lp = np.abs(L.astype(np.float64) + x)
            term = ARG_ROUND * (cab[kk] + up + mprime[nn]) + exp_rel(aL.astype(np.float64) - top[nn])
            wD = np.exp((aL - top[nn].astype(LD)).astype(np.float64))
            num = np.zeros(n1 - n0)
            np.add.at(num, nn[sk], (wD * term)[sk])
            dL = (K + 2) * EPS + num / D.astype(np.float64) + 2 * EPS * (mprime + Lp)
            out["dL"][n0:n1] = dL
            # weights of every kept entry: W_nk = e^(f_k - u_kn - L_n), w_kn = N_k W_nk (c carries log N_k)
            arg = aL - L[nn]
            # row sums scaled by e^-shift_k: a row far from every sample (e^-14000) underflows even long double
            mc = m[n0:n1]
            mm = mc[nn].astype(LD)
            # (a weight of multiplicity 0 may lie far above its row's live ones: it must not overflow into 0 * inf)
            Wk = np.where(mm > 0, np.exp(np.where(mm > 0, fL[kk] - uc[kk, nn].astype(LD) - L[nn] - shift[kk], 0)), 0)
            np.add.at(out["S"], kk, mm * Wk)
            e = dL[nn] + ARG_ROUND * (cab[kk] + up + Lp[nn]) + exp_rel(arg.astype(np.float64)) + 2 * EPS
            np.add.at(out["eS"], kk, mm * Wk * e.astype(LD))
            elog = e + EPS * np.abs(np.log(np.where(mc[nn] > 0, mc[nn], 1.0)))
            np.add.at(out["eLogW"], kk, mm * Wk * elog.astype(LD))
            a64n = arg.astype(np.float64)
            normal = rows[kk] & (a64n >= M.LOG_NORMAL)
            if normal.any():
                np.maximum.at(out["A"], kk[normal], np.abs(a64n[normal]))
            if want_G:
                keep = rows[kk] & (mc[nn] > 0)
                k2, n2, w2 = kk[keep], nn[keep], np.exp(arg[keep]) * np.sqrt(mm[keep])
                order = np.argsort(n2, kind="stable")
                k2, n2, w2 = k2[order], n2[order], w2[order]
                # every pair of kept entries of one sample: the entries of a sample are contiguous after the sort,
                # so the pairs lie d = 0, 1, ... positions apart (d = 0: the diagonal)
                d = 0
                while d < n2.size:
                    a = np.flatnonzero(n2[:n2.size - d] == n2[d:])
                    if a.size == 0:
                        break
                    ka, kb = k2[a], k2[a + d]
                    Gi.append(np.maximum(ka, kb))
                    Gj.append(np.minimum(ka, kb))
                    Gv.append(w2[a] * w2[a + d])
                    d += 1
    out["sumL"] = (m.astype(LD) * out["L"]).sum()
    with np.errstate(divide="ignore", invalid="ignore"):
        Ssh = out["S"]
        out["logS"] = np.log(Ssh) + shift
        out["eS"] = np.where(Ssh > 0, out["eS"] / Ssh, 0)          # relative budgets: the scale cancels
        out["eLogW"] = np.where(Ssh > 0, out["eLogW"] / Ssh, 0)
        out["S"] = Ssh * np.exp(shift)
    out["drop"] = LD(m.sum()) * np.exp(-LD(cut))        # long double: e^-1500 is 0 in fp64
    if want_G:
        gi, gj, gv = (np.concatenate(v) if v else np.zeros(0) for v in (Gi, Gj, Gv))
        key = gi.astype(np.int64) * K + gj
        uk, inv = np.unique(key, return_inverse=True)
        val = np.zeros(uk.size, LD)
        np.add.at(val, inv, gv.astype(LD))
        out["Gi"], out["Gj"], out["Gv"] = (uk // K).astype(np.int64), (uk % K).astype(np.int64), val
    return out


def pass_tolerances(ref, N_k, plan, mult=None, floor=None):
    """Absolute tolerances of S (sampled rows, linear sums), of log S (log-domain rows, every row) and of L_n.
    Either form may answer a sampled row (log-domain after an underflow), so tolS covers both.  `floor` [K] replaces
    the absolute term of weights on the exp floor, N max(m) 2^-1020 / N_k, where a pass divides floored entries by
    a denominator (the fused pass: per row sum_n m_n 2^-1020 max(1, e^(c_k - mid)) / (D_n N_k))."""
    N_k = np.asarray(N_k, np.float64)
    s = N_k > 0
    h = reduction_depth(plan)
    Nd = np.where(s, N_k, 1.0)
    S = ref["S"].astype(np.float64)
    M_ = float(plan["N"] if mult is None else np.sum(mult))
    mmax = 1.0 if mult is None else float(np.max(mult))
    floor_abs = plan["N"] * mmax * M.FLOOR / Nd if floor is None else np.asarray(floor, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        rel_lin = ref["eS"].astype(np.float64) + (h + 2) * EPS
        # log-domain rows: per-lane (max, sum) over 32 samples, merged over tiles, warps and CTAs
        tol_log = (ref["eLogW"].astype(np.float64) + (h + 2) * EPS + 4 * LOG_MERGE
                   + 2 * EPS * np.abs(ref["logS"].astype(np.float64)) + plan["N"] * mmax * float(np.exp(-LD(CUT))))
        if floor is not None:           # linear sums of every row (the fused all-state pass): the floor, relative
            tol_log = tol_log + np.where(S > 0, floor * Nd / np.where(S > 0, S * Nd, 1.0), 0.0)
        # a row whose every kept weight has multiplicity 0 sums to exactly 0 on both sides
        tolS = np.where(s, np.where(S > 0, np.maximum(S * rel_lin, S * np.expm1(np.minimum(tol_log, 1.0))), 0.0)
                        + floor_abs + float(ref["drop"]) / Nd, 0.0)
    tolL = ref["dL"] + 2 * EPS * (np.abs(ref["L"].astype(np.float64)) + np.abs(ref["x"])) + K_MAX * np.exp(-CUT)
    return dict(S=tolS, logS=tol_log, L=tolL, M=M_)


def sumL_tolerance(ref, plan, mult=None, mid=0.0):
    """sum_n m_n L'_n (warp butterfly, the tiles of a thread, warps, CTAs) less sum_n m_n x_n (host, N terms).  A
    plan may state its own `sumL_depth`; one with `logprod` sums log(D_n) = L'_n - mid as a product of mantissas
    (one rounding per sample, absolute in the log) and adds sum_n m_n mid at the end."""
    m = np.ones(plan["N"]) if mult is None else np.asarray(mult, np.float64)
    Lp = np.abs(ref["L"].astype(np.float64) + ref["x"]) + abs(mid)
    depth = plan.get("sumL_depth", 5 + plan.get("tiles_per_warp", 0) + plan.get("W", 0) + plan["grid"] + 2)
    prod = 2 * EPS * float(np.sum(m)) if plan.get("logprod") else 0.0
    return float(np.sum(m * ref["dL"]) + depth * EPS * np.sum(m * Lp) + plan["N"] * EPS * np.sum(m * np.abs(ref["x"]))
                 + prod)


def dense_G(ref, K):
    """The support of Ghat as a dense symmetric long-double matrix (tests at small K only)."""
    G = np.zeros((K, K), LD)
    G[ref["Gi"], ref["Gj"]] = ref["Gv"]
    G[ref["Gj"], ref["Gi"]] = ref["Gv"]
    return G

"""Extended-precision second moments of the MBAR weights, the per-entry tolerance the Hessian kernels are held to,
and the cases they are checked on.

With w_kn = exp(c_k - u_kn - L_n), c_k = f_k + log N_k (sampled states; f_k for unsampled states when all rows are
wanted) and L_n = log sum_{j sampled} N_j exp(f_j - u_jn):

    S_k = sum_n m_n W_nk,   Ghat_ij = sum_n m_n w_in w_jn,

where m_n are the per-sample multiplicities (1 when none are set) and W_nk = exp(f_k - u_kn - L_n).  Ghat is a sum
of non-negative products, so nothing cancels: every entry, however small, has a well-defined relative error, and
the device must reproduce each one to a small relative error plus the absolute floor of its exp.

np.longdouble carries a 64-bit mantissa and an exponent range down to about 1e-4932 here, so the reference never
underflows where fp64 does.  A platform whose long double is plain fp64 cannot serve as the reference: the module
refuses to import there rather than quietly check the device against itself.
"""
import numpy as np

from oracle import testsystems as ots

LD = np.longdouble
if np.finfo(LD).nmant < 63:
    raise ImportError(f"tests/_moments.py needs an 80-bit long double (nmant >= 63), got nmant={np.finfo(LD).nmant}")

EPS = 2.0 ** -53
FLOOR = 2.0 ** -1020              # the device's exp returns [0, 2^-1020] below the normal range (DESIGN 3.1)
LOG_NORMAL = np.log(2.0 ** -1022)  # arguments below this give floored weights: covered by the absolute term


def moments_ld(u, N_k, f, mult=None, all_rows=False, chunk=128):
    """(S, Ghat, A) in long double.  `+inf` energies give weight 0.  A_k is the largest |exp argument| of state k
    among the weights in the normal range (the floored ones are accounted for by entry_tol's absolute term)."""
    u = np.asarray(u, np.float64)
    N_k = np.asarray(N_k, np.float64)
    K, N = u.shape
    s = N_k > 0
    uL = u.astype(LD)
    fL = np.asarray(f, np.float64).astype(LD)
    logN = np.zeros(K, LD)
    logN[s] = np.log(N_k[s].astype(LD))
    a_s = (fL[s] + logN[s])[:, None] - uL[s]                      # [K_s, N], -inf for +inf energies
    top = a_s.max(axis=0)
    L = top + np.log(np.exp(a_s - top).sum(axis=0))
    rows = np.ones(K, bool) if all_rows else s
    c = fL + logN                                                  # unsampled rows: c = f (log N = 0 there)
    with np.errstate(invalid="ignore"):
        arg = c[:, None] - uL - L[None, :]
    arg[~rows] = -np.inf
    w = np.exp(arg)
    m = np.ones(N, LD) if mult is None else np.asarray(mult, np.float64).astype(LD)
    S = (np.exp(fL[:, None] - uL - L[None, :]) * m).sum(axis=1)
    normal = np.isfinite(arg) & (arg >= LOG_NORMAL)
    A = np.where(normal, np.abs(arg), 0).max(axis=1).astype(np.float64)
    G = np.zeros((K, K), LD)
    ws = w * np.sqrt(m)
    for n0 in range(0, N, chunk):
        blk = ws[:, n0:n0 + chunk]
        nz = np.flatnonzero((blk > 0).any(axis=1))                 # ladders: each chunk touches few states
        if nz.size:
            b = blk[nz]
            G[np.ix_(nz, nz)] += b @ b.T
    return S, G, A


def entry_tol(Ghat, A, N, wmax):
    """tol_ij = rho_ij Ghat_ij + alpha with rho_ij = 8 eps (A_i + A_j) + 8 eps sqrt(N) + 64 eps and
    alpha = 4 N 2^-1020 max(1, wmax).  A: rounding of the exp argument and the reduction term of the device exp
    (DESIGN 3.1); sqrt(N): the fp64 accumulation chains of the DMMA; alpha: weights on the exp floor, including
    subnormal products should the DMMA flush them.  A may be a scalar bound."""
    A = np.broadcast_to(np.asarray(A, np.float64), (Ghat.shape[0],))
    rho = 8 * EPS * (A[:, None] + A[None, :]) + 8 * EPS * np.sqrt(float(N)) + 64 * EPS
    alpha = 4.0 * N * FLOOR * max(1.0, float(wmax))
    return rho * np.asarray(Ghat, LD) + alpha


def excess(Gdev, Ghat, tol, mask=None):
    """max |Gdev - Ghat| / tol over the entries of `mask` (all entries when None); <= 1 passes."""
    r = np.abs(np.asarray(Gdev, np.float64).astype(LD) - Ghat) / tol
    if mask is not None:
        r = r[mask]
    return float(r.max()) if r.size else 0.0


# ---- cases -------------------------------------------------------------------------------------------------------
# Harmonic states of unit width whose centres are GAPS[k % len] standard deviations apart.  Neighbours 39 or 40
# apart couple at about e^-700 (Ghat spans more than 300 decades) and put weights on both sides of e^-707 (the
# exp floor); two gaps of 27 around a state make the products of the outer pair subnormal (about e^-729); the
# others give couplings at intermediate scales.
GAPS = (39.0, 27.0, 27.0, 15.0, 40.0, 22.0, 33.0, 10.0)
SHAPES = (2, 5, 16, 17, 33, 63, 64, 65, 127, 128, 129, 200, 255, 256, 257, 384, 513)


def ladder(K, n_per, gaps=GAPS, unsampled=(), n_inf=0, seed=0, f_noise=0.05):
    """u_kn [K, N], N_k, f and multiplicities (Poisson(1), so some are zero) of one ladder.  N_k varies by one
    sample between states; N is never a multiple of 32.  `n_inf` random entries of other states become +inf."""
    rng = np.random.RandomState(seed)
    centres = np.concatenate([[0.0], np.cumsum([gaps[k % len(gaps)] for k in range(K - 1)])])
    N_k = np.array([n_per + (k % 2) for k in range(K)], np.float64)
    N_k[list(unsampled)] = 0.0
    if int(N_k.sum()) % 32 == 0:
        N_k[np.flatnonzero(N_k)[-1]] += 1
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


def cases():
    """name -> builder arguments.  Unsampled states first, in the middle and last; +inf energies; N from 11 (one
    tile: most warp pairs of the small kernel get no tile) to 4200; K = 2100 needs two block-pair launches."""
    out = {}
    for K in SHAPES:
        n_per = 5 if K < 100 else 3
        kw = dict(K=K, n_per=n_per, seed=K)
        if K in (17, 257):
            kw["unsampled"] = (0,) if K == 17 else (0, K // 2, K - 1)
        if K == 65:
            kw["unsampled"] = (K // 2,)
        if K == 129:
            kw["unsampled"] = (K - 1,)
        if K in (33, 200):
            kw["n_inf"] = 2 * K
        out[f"ladder_K{K}"] = kw
    out["ladder_K5_tiny"] = dict(K=5, n_per=2, seed=55, unsampled=(2,))
    out["ladder_K2100"] = dict(K=2100, n_per=2, seed=2100, unsampled=(7, 1500))
    return out


def build(name):
    return ladder(**cases()[name])


def solve_ladder(K, seed):
    """A well-overlapping ladder (gaps of 1.5) for the solvers: f is known to statistical accuracy only."""
    return ladder(K, 30, gaps=(1.5,), seed=seed)


def reference(case, path):
    """(S, Ghat, A, rows) of the path's contract: P1 / P2 sampled rows, P3 all rows, P4 sampled rows with the
    multiplicities."""
    all_rows = path == "P3"
    mult = case["mult"] if path == "P4" else None
    S, G, A = moments_ld(case["u"], case["N"], case["f"], mult=mult, all_rows=all_rows)
    rows = np.ones(len(case["N"]), bool) if all_rows else case["N"] > 0
    return S, G, A, rows


def row_scale(N_k, path):
    """s_i with Ghat_ij = s_i s_j G_ij for the G the API returns (N_i; 1 for unsampled rows of weight_moments)."""
    N_k = np.asarray(N_k, np.float64)
    return np.where(N_k > 0, N_k, 1.0 if path == "P3" else 0.0)


def fused_stores_weights(case, path):
    """Whether the fused pass answers and stores the weights.  With multiplicities, a sampled state whose own samples
    all have multiplicity zero and whose neighbours are far away can have S_k below 1e-280, which the library
    treats as underflow: the generic pass answers."""
    K = len(case["N"])
    if path not in ("P1", "P4") or K > 2048:
        return False
    if path == "P4":
        S, _, _ = moments_ld(case["u"], case["N"], case["f"], mult=case["mult"])
        return bool(np.all(S[case["N"] > 0].astype(np.float64) > 1e-280))
    return True


def expected_kernel(case, path, inplace=False):
    """Substring of last_kernels()["hessian_kernel"] that the path must report."""
    if inplace:
        return "hessian_inplace_kernel"
    K = len(case["N"])
    wst = fused_stores_weights(case, path)
    if K <= 64:
        KT = 2 if K <= 16 else 4 if K <= 32 else 8
        how = "weights stored by the fused pass (WST)" if wst else "in-register conversion"
        return f"hessian_small_kernel<KT={KT}, {how}>"
    if wst:
        return "weights stored by the fused pass (WST) + hessian_big_kernel"
    return "weights_kernel + hessian_big_kernel"


PATHS = ("P1", "P2", "P3", "P4")


def device_moments(p, case, path):
    """Run one path twice on DeviceProblem `p`: P1 streaming_pass(want_G) after the fused pass (weights stored),
    P2 the same with the generic pass, P3 weight_moments, P4 streaming_pass(want_G) with the multiplicities.  P1
    and P2 also take hessian(f) twice.  Returns numpy arrays and kernel names."""
    f = case["f"]
    out = {}
    if path == "P2":
        p.set_kernel("generic")
    if path == "P4":
        p.set_sample_weights(case["mult"])
    try:
        for i in range(2):
            if path == "P3":
                S, G = p.weight_moments(f)
            else:
                S, _, G = p.streaming_pass(f, want_G=True)
            out[f"S{i}"], out[f"G{i}"] = S, G
            out[f"name{i}"] = p.last_kernels()["hessian_kernel"]
        if path in ("P1", "P2"):
            out["H0"], out["H1"] = p.hessian(f), p.hessian(f)
            out["hname"] = p.last_kernels()["hessian_kernel"]
    finally:
        p.set_kernel("auto")
        p.set_sample_weights(None)
    return out


def harmonic_c5(K=512):
    """Centres and spring constants of the synthesized C5 problem (test_gpu_fullsize's family)."""
    return np.linspace(1, 5, K), np.linspace(1, 3, K)


def analytic_f(kk):
    return ots.harmonic_analytical_f_k(kk)

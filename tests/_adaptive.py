"""One iteration of the adaptive solver, restated in extended precision, with the bounds a device step is held to,
and a numpy model of the device's Newton kernel.

`iteration` follows the reference's adaptive() (mbar_solvers.py:575-640) on the sampled states, with the gauge on the
first sampled state g0 (as the device loop keeps it, loops.cu): the pass at f gives S, Ghat and the gradient
g_k = N_k (S_k - 1); the self-consistent candidate is f_k - log S_k less the same at g0; the Newton step x solves
A x = g over the sampled states other than g0, A = H[1:,1:] with H_ij = delta_ij N_i S_i - Ghat_ij, and the Newton
candidate is f - gamma x there.  Both candidates get one more pass for their squared gradient norms, the smaller
one wins (unless the first `min_sc_iter` steps must be self-consistent), and the stop rule of :627-640 reads the
relative change of the chosen candidate and the largest relative difference of the two.

In long double the sums come from `_large_k.sparse_moments_ld` (every weight within `cut` of its sample's largest
one; what is dropped enters the bounds), A is factorised in fp64 by scipy and x refined with long-double residuals.
In fp64 the same step is computed densely the way the oracle computes it, so the restatement can be checked against
`oracle.mbar_oracle.adaptive` itself.

The bounds of a device step:
  S_k           `_large_k.pass_tolerances` of the fused pass (absolute), with a reduction depth that bounds every
                fused plan;
  Ghat_ij       `_moments.entry_tol` on the kept support, plus its absolute term and the dropped mass elsewhere;
  f_sci, g, gn  propagated from those, with the candidate's own error through the Hessian (|H| row sums are at
                most 2 N_i S_i) for the norms of the candidates;
  Newton step   a backward error that does not depend on the condition of A: with x_dev = (f - f_nr) / gamma
                recovered in long double,
                  ||A x_dev - g||_inf <= C (n eps max(|A||x_dev|) + ||dA||_inf ||x_dev||_inf + ||dg||_inf
                                            + ||A||_inf eps (||f|| + ||f_nr||) / gamma),
                and the forward error it implies, ||A^-1||_inf times that bound.
"""
import numpy as np
import scipy.linalg
import scipy.sparse
import scipy.sparse.linalg

from tests import _large_k as LK
from tests import _moments as M

LD = M.LD
EPS = M.EPS
CUT = 60.0           # e^-60 of a sample's largest weight is far below fp64 resolution; the drop is in the bounds
BACKWARD_C = 4.0     # the constant C of the backward-error bound


# ---- the pass -----------------------------------------------------------------------------------------------------
def fused_depth_bound(N):
    """A reduction depth no fused plan exceeds: every tile of one lane, the butterfly, 8 groups, 132 CTA groups."""
    return -(-int(N) // 32) + 5 + 8 + 132


def pass_ld(u, N_k, f, want_G, cut=CUT, mult=None):
    """The sums of one pass at f in long double and their device tolerances (fused pass, sampled rows, optional
    per-sample multiplicities)."""
    u = np.asarray(u, np.float64)
    N_k = np.asarray(N_k, np.float64)
    s = N_k > 0
    c = np.where(s, np.asarray(f, np.float64) + np.log(np.where(s, N_k, 1.0)), 0.0)
    spread = float(c[s].max() - c[s].min())
    ref = LK.sparse_moments_ld(u, N_k, f, mult=mult, want_G=want_G, cut=cut, c_abs=np.full(len(N_k), spread))
    plan = dict(N=u.shape[1], depth=fused_depth_bound(u.shape[1]))
    tol = LK.pass_tolerances(ref, N_k, plan, mult=mult)
    return ref, tol["S"]


def pass_fp64(u, N_k, f, want_G):
    """S and Ghat in fp64, the way the oracle computes them (dense log-sum-exp)."""
    s = N_k > 0
    logN = np.log(N_k[s])
    a = (f[s] + logN)[:, None] - u[s]
    top = a.max(axis=0)
    L = top + np.log(np.exp(a - top).sum(axis=0))
    W = np.exp(f[:, None] - u - L[None, :])             # [K, N]
    S = W.sum(axis=1)
    out = dict(S=S)
    if want_G:
        w = W * np.where(s, N_k, 0.0)[:, None]
        out["G"] = w @ w.T
    return out


# ---- the Newton system over the sampled states other than the gauge state ----------------------------------------
def newton_matrix(ref, N_k, S, active, dense):
    """A = diag(N_i S_i) - Ghat over active[1:], as a long-double dense matrix or a (rows, cols, vals) triplet."""
    K = len(N_k)
    free = np.asarray(active[1:])
    n = free.size
    pos = np.full(K, -1)
    pos[free] = np.arange(n)
    if "Gi" in ref:
        gi, gj, gv = ref["Gi"], ref["Gj"], ref["Gv"]
        both = np.concatenate([np.stack([gi, gj]), np.stack([gj, gi])[:, gi != gj]], axis=1)
        vals = np.concatenate([gv, gv[gi != gj]])
        a, b = pos[both[0]], pos[both[1]]
        keep = (a >= 0) & (b >= 0)
        rows, cols, vals = a[keep], b[keep], -vals[keep]
    else:
        G = np.asarray(ref["G"])
        rows, cols = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
        rows, cols = rows.ravel(), cols.ravel()
        vals = -G[np.ix_(free, free)].ravel()
    diag = (np.asarray(N_k)[free].astype(S.dtype) * S[free])
    rows = np.concatenate([rows, np.arange(n)])
    cols = np.concatenate([cols, np.arange(n)])
    vals = np.concatenate([vals.astype(S.dtype), diag])
    if dense:
        A = np.zeros((n, n), S.dtype)
        np.add.at(A, (rows, cols), vals)
        return A
    return rows, cols, vals, n


def matvec(T, x):
    """A x in the precision of x for a triplet A (long double: no BLAS, no rounding below 64 bits)."""
    rows, cols, vals, n = T
    y = np.zeros(n, np.result_type(vals.dtype, x.dtype))
    np.add.at(y, rows, vals * x[cols])
    return y


def abs_matvec(T, x):
    rows, cols, vals, n = T
    y = np.zeros(n, LD)
    np.add.at(y, rows, np.abs(vals).astype(LD) * np.abs(x[cols]).astype(LD))
    return y


def row_abs_sums(T):
    rows, cols, vals, n = T
    y = np.zeros(n, LD)
    np.add.at(y, rows, np.abs(vals).astype(LD))
    return y


def solve_refined(T, b, sweeps=3):
    """x with A x = b: fp64 sparse LU of A, then refinement with long-double residuals."""
    rows, cols, vals, n = T
    A64 = scipy.sparse.csc_matrix((vals.astype(np.float64), (rows, cols)), shape=(n, n))
    lu = scipy.sparse.linalg.splu(A64)
    x = lu.solve(b.astype(np.float64)).astype(LD)
    for _ in range(sweeps):
        r = b.astype(LD) - matvec(T, x)
        x = x + lu.solve(r.astype(np.float64)).astype(LD)
    return x, lu


def inverse_norm(lu, n):
    """||A^-1||_inf from the fp64 factorisation (columns of the inverse in blocks)."""
    best = np.zeros(n)
    for j0 in range(0, n, 512):
        E = np.zeros((n, min(512, n - j0)))
        E[np.arange(j0, j0 + E.shape[1]), np.arange(E.shape[1])] = 1.0
        best += np.abs(lu.solve(E)).sum(axis=1)
    return float(best.max()) * (1 + 1e-6)


# ---- one iteration ------------------------------------------------------------------------------------------------
def rel_change(new, old, thr):
    """|new - old| / |new| with |new| below thr counted as 1 (mbar_solvers.py:627-631)."""
    div = np.abs(new)
    div = np.where(div < thr, 1.0, div)
    return np.abs(new - old) / div


def _gnorm(N_k, S, s):
    g = np.where(s, N_k * (S - 1), 0).astype(S.dtype)
    return g, (g * g).sum()


def iteration(u, N_k, f, gamma=1.0, tol=1e-12, min_sc_iter=0, sci_done=0, precision="ld", cut=CUT, mult=None):
    """One adaptive iteration from f (gauge f[g0] = 0).  precision 'ld': long-double sums with device bounds;
    'fp64': the oracle's arithmetic (no bounds).  Returns a dict with f_sci, f_nr (None without a Newton candidate),
    gn_sci, gn_nr, choice ('sci' / 'nr'), f_new, max_delta, max_diff, stop, and (ld) the bound entries."""
    u = np.asarray(u, np.float64)
    N_k = np.asarray(N_k, np.float64)
    f = np.asarray(f, np.float64)
    K = len(N_k)
    s = N_k > 0
    active = np.flatnonzero(s)
    g0, free = active[0], active[1:]
    n = free.size
    ld = precision == "ld"
    if ld:
        ref, tolS = pass_ld(u, N_k, f, want_G=True, cut=cut, mult=mult)
        S = ref["S"]
        logS = ref["logS"]
        fW = f.astype(LD)
    else:
        ref = pass_fp64(u, N_k, f, want_G=True)
        S = ref["S"]
        logS = np.log(S)
        fW = f
    g, gn0 = _gnorm(N_k, S, s)
    f_sci = fW.copy()
    f_sci[active] = fW[active] - logS[active] - (fW[g0] - logS[g0])
    out = dict(active=active, S=S, g=g, f_sci=f_sci, n=n)
    # Newton step
    if ld:
        T = newton_matrix(ref, N_k, S, active, dense=False)
        x, lu = solve_refined(T, g[free])
    else:
        A = newton_matrix(ref, N_k, S, active, dense=True)
        x = scipy.linalg.solve(A, g[free], assume_a="pos")
    f_nr = fW.copy()
    f_nr[free] = fW[free] - gamma * x
    have_nr = bool(np.all(np.isfinite(f_nr[free].astype(np.float64)))
                   and np.all(np.abs(f_nr[free].astype(np.float64)) < 0.5e6))
    out.update(x=x, f_nr=f_nr if have_nr else None)
    # both candidates' gradient norms
    cand = dict(sci=f_sci, nr=f_nr)
    for name, fc in cand.items():
        if name == "nr" and not have_nr:
            out["gn_nr"], out["S_nr"] = np.inf, None
            continue
        if ld:
            r2, tol2 = pass_ld(u, N_k, fc.astype(np.float64), want_G=False, cut=cut, mult=mult)
            Sc = r2["S"]
            out[f"tolS_{name}"] = tol2
        else:
            Sc = pass_fp64(u, N_k, fc, want_G=False)["S"]
        out[f"gn_{name}"] = _gnorm(N_k, Sc, s)[1]
        out[f"S_{name}"] = Sc
    take_sci = out["gn_sci"] < out["gn_nr"] or sci_done < min_sc_iter
    out["choice"] = "sci" if take_sci else "nr"
    f_new = f_sci if take_sci else f_nr
    fnr = f_nr if have_nr else f_sci
    thr = min(1e-8, tol)
    out["f_new"] = f_new
    out["max_delta"] = rel_change(f_new[free], fW[free], thr).max() if n else 0.0
    # max |f_sci - f_nr| / |f_new| (mbar_solvers.py:632)
    div = np.where(np.abs(f_new[free]) < thr, 1.0, np.abs(f_new[free]))
    out["max_diff"] = (np.abs(f_sci[free] - fnr[free]) / div).max() if n else 0.0
    out["stop"] = bool(np.isnan(float(out["max_delta"])) or (out["max_delta"] < tol and out["max_diff"] < np.sqrt(tol)))
    if ld:
        out["T"] = T
        out.update(_bounds(u, N_k, f, ref, tolS, T, lu, out, gamma, mult))
    return out


def _bounds(u, N_k, f, ref, tolS, T, lu, it, gamma, mult):
    """The tolerances of the device's quantities at this iteration (see the module docstring)."""
    N = u.shape[1]
    s = N_k > 0
    active = it["active"]
    g0, free = active[0], active[1:]
    n = free.size
    S = ref["S"].astype(np.float64)
    Nd = np.where(s, N_k, 0.0)
    rho = np.where(s & (S > 0), tolS / np.where(S > 0, S, 1.0), 0.0)
    logS = np.abs(ref["logS"].astype(np.float64))
    fa = np.abs(f)
    # f_sci_k = f_k - log S_k - (f_g0 - log S_g0): the two logs, four roundings
    tol_fsci = np.zeros(len(N_k))
    tol_fsci[active] = (1.01 * (rho[active] + rho[g0]) + 4 * EPS * (fa[active] + logS[active] + fa[g0] + logS[g0])
                        + EPS * np.abs(it["f_sci"][active].astype(np.float64)))
    # g_k = N_k (S_k - 1)
    dg = Nd * (tolS + EPS * (S + 1)) + EPS * np.abs(it["g"].astype(np.float64))
    # A: the diagonal's S, every Ghat entry's entry_tol (kept support), the absolute floor and drop elsewhere
    Ahat = ref["A"]
    wmax = 1.0 if mult is None else float(np.max(mult))
    rho_g = lambda i, j: 8 * EPS * (Ahat[i] + Ahat[j]) + 8 * EPS * np.sqrt(float(N)) + 64 * EPS
    alpha = 4.0 * N * M.FLOOR * wmax + float(ref["drop"])
    pos = np.full(len(N_k), -1)
    pos[free] = np.arange(n)
    gi, gj, gv = ref["Gi"], ref["Gj"], ref["Gv"].astype(np.float64)
    dG = rho_g(gi, gj) * gv
    dA_rows = np.zeros(n)
    for a, b in ((gi, gj), (gj, gi)):
        m = (pos[a] >= 0) & (pos[b] >= 0) & ((a != b) | (a is gi))
        np.add.at(dA_rows, pos[a][m], dG[m])
    dA_rows += n * alpha + Nd[free] * (tolS[free] + EPS * S[free]) + 2 * EPS * (Nd[free] * S[free])
    dA = float(dA_rows.max()) if n else 0.0
    normA = float(row_abs_sums(T).max()) if n else 0.0
    dg_free = float(dg[free].max()) if n else 0.0
    # the candidates' gradient norms: the pass at the candidate, and the candidate's own error through the Hessian
    out = dict(tol_fsci=tol_fsci, dg=dg, dA=dA, normA=normA, dg_free=dg_free)
    out["inv_norm"] = inverse_norm(lu, n) if n else 0.0
    return out


def recover_step(f, f_nr, free, gamma):
    """x_dev = (f - f_nr) / gamma on the free states, in long double (exact up to the device's rounding of f_nr)."""
    return (np.asarray(f, np.float64)[free].astype(LD) - np.asarray(f_nr, np.float64)[free].astype(LD)) / LD(gamma)


def newton_backward(it, f, f_nr, gamma):
    """(ratio, residual, bound) of a device Newton candidate f_nr from f against this iteration's long-double A and
    g, with the device's errors of A and g in the bound: ratio <= 1 passes."""
    free = it["active"][1:]
    x_dev = recover_step(f, f_nr, free, gamma)
    return backward_ratio(it["T"], it["g"][free], x_dev, f, f_nr, gamma, dA=it["dA"], dg=it["dg_free"])


def forward_bound(it, f, f_nr, gamma):
    """||x_dev - x||_inf may reach ||A^-1||_inf times the backward bound (long-double x of this iteration)."""
    return it["inv_norm"] * newton_backward(it, f, f_nr, gamma)[2]


def backward_bound(n, absAx, dA, dg, normA, x_inf, f_inf, fnr_inf, gamma):
    return BACKWARD_C * (n * EPS * absAx + dA * x_inf + dg + normA * EPS * (f_inf + fnr_inf) / gamma)


def backward_ratio(T, g, x_dev, f, f_nr, gamma, dA=0.0, dg=0.0):
    """||A x_dev - g||_inf over its bound, for a triplet A in long double."""
    n = T[3]
    r = matvec(T, x_dev.astype(LD)) - g.astype(LD)
    res = float(np.abs(r).max())
    absAx = float(abs_matvec(T, x_dev).max())
    normA = float(row_abs_sums(T).max())
    b = backward_bound(n, absAx, dA, dg, normA, float(np.abs(x_dev).max()), float(np.abs(f).max()),
                       float(np.abs(f_nr).max()), gamma)
    return res / b, res, b


def gn_tolerance(N_k, S_c, tolS_c, gn, df, S_at_f, dgn_pass=True):
    """Bound on the device's squared gradient norm at a candidate: the pass at the candidate (tolS_c), the candidate's
    own error df (inf-norm) through the Hessian (|dg_k| <= 2 N_k S_k df), and the norm's rounding."""
    s = N_k > 0
    Sc = S_c.astype(np.float64)
    g = np.where(s, N_k * (Sc - 1), 0.0)
    dg = np.where(s, N_k * (tolS_c + EPS * (Sc + 1)) + EPS * np.abs(g) + 2.0 * N_k * np.maximum(Sc, S_at_f) * df
                  * (1 + 4 * df), 0.0)
    ng = float(np.sqrt(gn))
    ndg = float(np.sqrt((dg * dg).sum()))
    return 2 * ng * ndg + ndg * ndg + (len(N_k) + 64) * EPS * gn


# ---- a numpy model of newton_kernel (loops.cu) --------------------------------------------------------------------
FAULTS = ("skip_last_k", "skip_odd_remainder", "stale_row", "active_off_by_one")


def newton_model(A, g, active, f, gamma, fault=None):
    """newton_kernel's arithmetic on the n x n matrix A (fp64): left-looking Cholesky by columns, each row's dot
    product split over four lanes (k = ks, ks + 4, ... into two accumulators, the odd remainder into the first, then
    the butterfly (t0 + t1) + (t2 + t3)), the two triangular solves in the kernel's order, and f_nr = f - gamma x on
    active[1:].  `fault` injects one of FAULTS.  Returns f_nr, or None when a pivot is not positive."""
    A = np.array(A, np.float64)
    n = A.shape[0]
    M_ = A.T.copy()           # M_[j, i] = column j, row i (the kernel's column-major storage)
    prev_row = np.zeros(n)
    for j in range(n):
        row = M_[:j, j].copy()                         # row[k] = L[j, k], k < j
        if fault == "stale_row" and j >= 2:
            row[:j - 1] = prev_row[:j - 1]
        prev_row = np.concatenate([M_[:j, j], [0.0]]) if j else np.zeros(1)
        prev_row = np.pad(prev_row, (0, n - prev_row.size))
        if j:
            rows = np.arange(j, n)
            Lc = M_[:j, j:]                            # Lc[k, i - j] = L[i, k]
            P = Lc * row[:, None]
            if fault == "skip_last_k":
                P[j - 1] = 0.0
            lanes = np.zeros((4, rows.size))
            for ks in range(4):
                # k = ks, ks + 8, ... while k + 4 < j into s0, k + 4 into s1; then the odd remainder k < j into s0
                m = len(range(ks, j - 4, 8))
                k0 = np.arange(ks, ks + 8 * m, 8)
                s0 = -np.cumsum(P[k0], axis=0)[-1] if m else np.zeros(rows.size)
                s1 = -np.cumsum(P[k0 + 4], axis=0)[-1] if m else np.zeros(rows.size)
                k = ks + 8 * m
                if k < j and fault != "skip_odd_remainder":
                    s0 = s0 - P[k]
                lanes[ks] = s0 + s1
            t = (lanes[0] + lanes[1]) + (lanes[2] + lanes[3])
            M_[j, j:] = M_[j, j:] + t
        d = M_[j, j]
        if not (d > 0.0) or not (d < 1e300):
            return None
        sq = np.sqrt(d)
        M_[j, j + 1:] = M_[j, j + 1:] * (1.0 / sq)
        M_[j, j] = sq
    src = active[:-1] if fault == "active_off_by_one" else active[1:]
    b = np.array(g, np.float64)[src]
    for j in range(n):                                 # L y = g
        b[j] = b[j] / M_[j, j]
        b[j + 1:] = b[j + 1:] - M_[j, j + 1:] * b[j]
    for j in range(n - 1, -1, -1):                     # L^T x = y
        b[j] = b[j] / M_[j, j]
        b[:j] = b[:j] - M_[:j, j] * b[j]
    f_nr = np.array(f, np.float64)
    f_nr[active[1:]] = f_nr[active[1:]] - gamma * b
    return f_nr


def synthetic_system(n, seed, band=6, n_per=3):
    """A = H[1:,1:] of an MBAR-like Hessian: weights w [N, n + 1] of a ladder (each sample spread over its `band`
    neighbours on each side, rows summing to one), H = diag(sum_n w) - w^T w, and a gradient g summing to zero.
    Returns the long-double triplet of A, the fp64 dense A, g over n + 1 states and the active map."""
    rng = np.random.RandomState(seed)
    K = n + 1
    owner = np.repeat(np.arange(K), n_per)
    ns = owner.size
    raw = owner[:, None] + np.arange(-band, band + 1)[None, :]
    inside = (raw >= 0) & (raw < K)
    cols = np.clip(raw, 0, K - 1)
    vals = np.exp(-0.5 * ((raw - owner[:, None]) / (0.5 * band)) ** 2) * rng.uniform(0.5, 1.5, raw.shape) * inside
    wv = vals.astype(LD) / vals.sum(axis=1, keepdims=True).astype(LD)
    nb = cols.shape[1]
    H = np.zeros((K, K), LD)
    np.add.at(H, (np.repeat(cols, nb, axis=1).ravel(), np.tile(cols, (1, nb)).ravel()),
              -(wv[:, :, None] * wv[:, None, :]).ravel())
    np.add.at(H, (cols.ravel(), cols.ravel()), wv.ravel())
    A_ld = H[1:, 1:]
    g = rng.normal(size=K)
    g -= g.mean()
    r, c = np.nonzero(A_ld != 0)
    return (r, c, A_ld[r, c], n), A_ld.astype(np.float64), g, np.arange(K)

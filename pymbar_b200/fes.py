"""Free-energy surfaces from the resident MBAR problem: pymbar.FES with fes_type="histogram", "kde" and "spline".

pymbar's FES builds a histogram PMF from the log weights of one target state, log w_n = -u_n - L_n (mbar.py:1919-1934),
and its analytical uncertainty from the augmented weight matrix W_aug = [W | B] with B_ni = w^_n [bin(n) = i] and
w^_n = exp(log w_n + f_i): the bins are extra states with N = 0 (fes.py:1382-1415).  Both go through N x K and
N x (K + nbins) host arrays there.  Each sample lies in exactly one bin, so

    W_aug^T W_aug = [[ G    C       ]      G   = W^T W                       (DeviceProblem.weight_moments)
                     [ C^T  diag(D) ]]     C_ki = sum_{n in i} W_nk w^_n     (DeviceProblem.bin_moments)
                                           D_i  = sum_{n in i} w^_n^2

and everything comes from the resident u_kn plus two O(N) vectors (u_n and a dense bin index).  The bin labels are a
vectorised restatement of fes.py:513-573, quirks included: samples below the grid share the label -1, samples above
the top edge of a dimension get that dimension's bin count, and both pseudo-bins are bins in their own right.
The (K + nbins)^2 covariance algebra is the reference's own (estimators.asymptotic_covariance, "svd-ew").

A KDE surface is -score_samples of an sklearn KernelDensity fitted to x_n with the target state's weights w_n
(fes.py:650-699, :1566).  The N x Q part, l_q = log sum_n w_n k(|y_q - x_n| / h), is DeviceKde.log_sum; this module
holds sklearn's host algebra around it: the kernel and bandwidth (kde_settings), the kernel normalisation
(kde_log_norm) and the reference points of _get_fes_kde (kde_query).

A spline surface is fitted by minimising an objective whose sample term is linear in the B-spline coefficients c
(fes.py:2102-2306): c . A with A_i = sum_n w_n B_i(x_n), or c . S_k per state with S_ki = sum_{n in k} B_i(x_n).
DeviceBSpline.moments computes S and A in one pass; spline_sample_terms turns them into the term of each weighting,
and spline_objective / spline_gradient / spline_mc_loglikelihood restate the reference's objective, gradient and MC
log-likelihood around it with the reference's own quadratures, so that the fit costs O(K nb) arithmetic per step
instead of a spline evaluation on every sample.
"""
from __future__ import annotations

import math

import numpy as np

from . import estimators as est


def _edges(bin_edges):
    # fes.py:465-466: a single 1-D array of edges stands for [edges]
    if len(np.shape(bin_edges)) == 1:
        return [bin_edges]
    return bin_edges


def _first_rows(bin_n):
    """Index of the first sample of each distinct row of bin_n, in order of first appearance."""
    _, first = np.unique(bin_n, axis=0, return_index=True)
    return np.sort(first)


def histogram_labels(x_n, bin_edges):
    """Bin every sample as fes.py:513-573 does, without a Python loop over samples.

    Returns (bin_n [N, dims], sample_label [N], nonzero_bins, bin_label, bin_order): the per-dimension bin index
    (np.digitize - 1), the integer label sum_d bin_n[:, d] * len(bin_edges[d])**d (-1 for a sample below the grid in
    any dimension), the distinct bin tuples in order of first appearance, the label of each tuple, and the position
    of each distinct label in order of first appearance."""
    bins = _edges(bin_edges)
    dims = len(bins)
    x = np.asarray(x_n)
    if x.ndim == 1:
        x = x.reshape(-1, 1)
    bin_n = np.zeros(x.shape, int)
    for d in range(dims):
        bin_n[:, d] = np.digitize(x[:, d], bins[d]) - 1
    sample_label = np.zeros(len(x), int)
    for d in range(dims):
        sample_label += bin_n[:, d] * len(bins[d]) ** d
    sample_label[np.any(bin_n < 0, axis=1)] = -1
    first = _first_rows(bin_n)
    nonzero_bins = [tuple(int(v) for v in bin_n[n]) for n in first]
    bin_label = {t: int(sample_label[n]) for t, n in zip(nonzero_bins, first)}
    bin_order = {}
    for label in bin_label.values():
        if label not in bin_order:
            bin_order[label] = len(bin_order)
    return bin_n, sample_label, nonzero_bins, bin_label, bin_order


def dense_bins(sample_label, bin_order):
    """Per-sample index into f (bin_order[sample_label[n]]) as int32: the bin index the device kernel takes."""
    labels = np.fromiter(bin_order.keys(), dtype=np.int64, count=len(bin_order))
    order = np.fromiter(bin_order.values(), dtype=np.int64, count=len(bin_order))
    srt = np.argsort(labels)
    pos = np.searchsorted(labels[srt], sample_label)
    return order[srt][pos].astype(np.int32)


def histogram_bins(x_n, bin_edges):
    """(histogram_data without "f", dense bin index [N] int32, number of dense bins) of fes.py:476-578."""
    bins = _edges(bin_edges)
    bin_n, sample_label, nonzero_bins, bin_label, bin_order = histogram_labels(x_n, bins)
    dense = dense_bins(sample_label, bin_order)
    data = {"dims": len(bins), "bins": bins, "bin_n": bin_n, "nonzero_bins": nonzero_bins,
            "sample_label": sample_label, "bin_order": bin_order, "bin_label": bin_label}
    return data, dense, len(bin_order)


def with_bin_f(data, f_bin):
    """histogram_data["f"] from the dense bins' free energies f_bin.  fes.py:579 sizes f by the distinct bin TUPLES:
    when several out-of-grid tuples share the label -1 the trailing entries stay 0, and "from-lowest" can pick one of
    them, as in the reference."""
    f = np.zeros(len(data["bin_label"]))
    f[:len(data["bin_order"])] = f_bin
    data["f"] = f
    return data


def histogram_fes(problem, f_k, u_n, x_n, bin_edges):
    """The histogram_data dict of fes.py:476-600 for the target state u_n, with f from the device.

    `problem` is the DeviceProblem holding (u_kn, N_k); f_k its converged free energies.  The dict has the
    reference's keys and types, so the reference's get_fes code reads it unchanged."""
    data, dense, nb = histogram_bins(x_n, bin_edges)
    f_bin, _, _ = problem.bin_moments(f_k, u_n, dense, nb, want_C=False)
    return with_bin_f(data, f_bin)


def augmented_moments(G, C, D):
    """W_aug^T W_aug from its blocks: [[G, C], [C^T, diag(D)]]."""
    K, nb = np.shape(C)
    G_aug = np.zeros((K + nb, K + nb))
    G_aug[:K, :K] = G
    G_aug[:K, K:] = C
    G_aug[K:, :K] = np.transpose(C)
    G_aug[np.arange(K, K + nb), np.arange(K, K + nb)] = D
    return G_aug


def histogram_theta(problem, f_k, N_k, u_n, histogram_data, return_moments=False):
    """Theta of the augmented problem (fes.py:1382-1406) from the device's G, C and D, "svd-ew".

    Returns Theta [(K + nbins)^2]; with return_moments also (S_k, G_aug)."""
    dense = dense_bins(histogram_data["sample_label"], histogram_data["bin_order"])
    nb = len(histogram_data["bin_order"])
    _, C, D = problem.bin_moments(f_k, u_n, dense, nb)
    S, G = problem.weight_moments(f_k)
    Theta, G_aug = augmented_theta(G, C, D, N_k)
    return (Theta, S, G_aug) if return_moments else Theta


def augmented_theta(G, C, D, N_k):
    """(Theta, G_aug) of the augmented problem, "svd-ew" (fes.py:1402-1406): the bins are states with N = 0."""
    G_aug = augmented_moments(G, C, D)
    N_aug = np.concatenate([np.asarray(N_k, dtype=np.float64), np.zeros(np.shape(C)[1])])
    return est.asymptotic_covariance(G_aug, N_aug, method="svd-ew"), G_aug


def bin_uncertainties(Theta, K, j, n_out=None):
    """df_i = sqrt(Theta_ii + Theta_jj - 2 Theta_ij) over the bin block, relative to bin j (fes.py:1410-1415),
    zero-padded to n_out entries (the length of histogram_data["f"])."""
    nb = Theta.shape[0] - K
    df = np.zeros(nb if n_out is None else n_out)
    for i in range(nb):
        df[i] = math.sqrt(Theta[K + i, K + i] + Theta[K + j, K + j] - 2.0 * Theta[K + i, K + j])
    return df


def query(histogram_data, x, reference_point, fes_reference, df_fn=None):
    """f_i (and df_i) at the query points x, as _get_fes_histogram (fes.py:1263-1521) reports them.

    `df_fn(j)` returns the per-bin uncertainties relative to bin j (None: no uncertainty).  Raises what the
    reference raises; its ParameterError / DataError classes are looked up in pymbar when it is importable."""
    try:
        from pymbar.utils import DataError, ParameterError
    except ImportError:
        from .utils import ParameterError

        DataError = ParameterError
    x = np.array(x)
    if np.ndim(x) <= 1:
        x = x.reshape(-1, 1)
    bins = histogram_data["bins"]
    dims = histogram_data["dims"]
    bin_order = histogram_data["bin_order"]
    f = histogram_data["f"]
    if np.shape(x)[1] != dims:
        raise DataError("query coordinates have inconsistent dimension with the data the FES is fit to.")
    loc = np.zeros((len(x), dims), dtype=int)
    for d in range(dims):
        loc[:, d] = np.digitize(x[:, d], bins[d]) - 1
    if reference_point == "from-specified":
        if fes_reference is None:
            raise ParameterError("Specified reference point for FES not given")
        ref = [fes_reference] if dims == 1 else fes_reference
        ref_grid = np.zeros(dims, dtype=int)
        for d in range(dims):
            ref_grid[d] = np.digitize(ref[d], bins[d]) - 1
            if ref_grid[d] == -1 or ref_grid[d] == len(bins[d]):
                raise ParameterError(
                    "Specified reference point coordinate {:f} in dim {:d} grid point is out of the FES region "
                    "[{:f},{:f}]".format(ref_grid[d], d, np.min(bins[d]), np.max(bins[d])))
        j = bin_order[histogram_data["bin_label"][tuple(ref_grid)]]
    elif reference_point == "from-lowest":
        j = f.argmin()
    elif reference_point == "all-differences":
        raise ParameterError("reference point method of 'all-differences' is not yet supported for histogram "
                             "FES types (not implemented)")
    elif reference_point == "from-normalization":
        raise ParameterError("uncertainty_method 'from-normalization' is not currently supported for histograms")
    else:
        raise ParameterError(f"reference point {reference_point} is not supported")
    f_i = f - f[j]
    df_i = df_fn(j) if df_fn is not None else np.zeros(len(f))
    fx = np.full(len(x), np.nan)
    dfx = np.full(len(x), np.nan)
    top = np.array([len(b) for b in bins]) - 1
    inside = np.all(loc >= 0, axis=1) & np.all(loc < top, axis=1)
    for i in np.flatnonzero(inside):
        label = histogram_data["bin_label"][tuple(loc[i])]
        if label >= 0:
            fx[i] = f_i[bin_order[label]]
            dfx[i] = df_i[bin_order[label]]
    out = {"f_i": fx}
    if df_fn is not None:
        out["df_i"] = dfx
    return out


KDE_KERNELS = ("gaussian", "tophat", "epanechnikov", "exponential", "linear", "cosine")
_LOG_PI = math.log(math.pi)
_LOG_2PI = math.log(2 * math.pi)


def _log_vn(n):
    # log volume of the unit n-ball
    return 0.5 * n * _LOG_PI - math.lgamma(0.5 * n + 1)


def _log_sn(n):
    # log surface of the unit n-sphere
    return _LOG_2PI + _log_vn(n - 1)


def kde_log_norm(kernel, D, h):
    """log of the normalisation sklearn multiplies its unnormalised kernel sum by (its _log_kernel_norm), for one of
    KDE_KERNELS in D dimensions at bandwidth h."""
    if kernel == "gaussian":
        factor = 0.5 * D * _LOG_2PI
    elif kernel == "tophat":
        factor = _log_vn(D)
    elif kernel == "epanechnikov":
        factor = _log_vn(D) + math.log(2.0 / (D + 2.0))
    elif kernel == "exponential":
        factor = _log_sn(D - 1) + math.lgamma(D)
    elif kernel == "linear":
        factor = _log_vn(D) - math.log(D + 1.0)
    elif kernel == "cosine":
        factor = 0.0
        tmp = 2.0 / math.pi
        for k in range(1, D + 1, 2):
            factor += tmp
            tmp *= -(D - k) * (D - k - 1) * (2.0 / math.pi) ** 2
        # negative for D = 4: sklearn's log then gives NaN, and so does this
        factor = (math.log(factor) if factor > 0 else math.nan) + _log_sn(D - 1)
    else:
        raise ValueError(f"kernel {kernel!r} not recognized")
    return -factor - D * math.log(h)


def _nonnegative_real(v):
    return isinstance(v, (int, float, np.integer, np.floating)) and not isinstance(v, bool) and v >= 0


def kde_settings(params, N, D):
    """What the device needs of a KernelDensity with parameters `params` (its get_params()) fitted to N samples in
    D dimensions: {"kernel", "h", "D"}, or None when the device does not serve it (a metric other than euclidean,
    metric_params, D outside 1..4, or any parameter sklearn's fit would reject, so that the caller's fall-back
    raises sklearn's own error).  The bandwidth of "scott" / "silverman" is sklearn's, from N and D.

    atol, rtol, algorithm, leaf_size and breadth_first only choose how sklearn's tree approximates the sum: the
    device sums every pair, an exact answer that lies within the tolerance of any such setting."""
    kernel = params.get("kernel")
    bw = params.get("bandwidth")
    if kernel not in KDE_KERNELS or params.get("metric") != "euclidean" or params.get("metric_params") is not None:
        return None
    if not 1 <= D <= 4 or N < 1:
        return None
    if not (_nonnegative_real(params.get("atol")) and _nonnegative_real(params.get("rtol"))):
        return None
    leaf = params.get("leaf_size")
    if params.get("algorithm") not in ("auto", "kd_tree", "ball_tree"):
        return None
    if not isinstance(params.get("breadth_first"), (bool, np.bool_)):
        return None
    if not isinstance(leaf, (int, np.integer)) or isinstance(leaf, bool) or leaf < 1:
        return None
    # sklearn KernelDensity.fit: N = X.shape[0] counts every sample, zero weights included
    if isinstance(bw, str):
        if bw == "scott":
            h = N ** (-1 / (D + 4))
        elif bw == "silverman":
            h = (N * (D + 2) / 4) ** (-1 / (D + 4))
        else:
            return None
    elif isinstance(bw, (int, float, np.integer, np.floating)) and not isinstance(bw, bool):
        h = float(bw)
        if not (math.isfinite(h) and h > 0):
            return None
    else:
        return None
    return {"kernel": kernel, "h": float(h), "D": int(D)}


def _draw_as_sample(kernel, D):
    """What KernelDensity.sample() does to its caller, without the sample: _get_fes_kde calls it only for its shape
    (fes.py:1560).  Other kernels than gaussian and tophat raise NotImplementedError there; those two take one
    uniform and D normals from numpy's global generator."""
    if kernel not in ("gaussian", "tophat"):
        raise NotImplementedError()
    rng = np.random.mtrand._rand
    rng.uniform(0, 1, size=1)
    rng.normal(size=(1, D))


def _kde_errors():
    try:
        from pymbar.utils import DataError, ParameterError
    except ImportError:
        from .utils import ParameterError

        DataError = ParameterError
    return DataError, ParameterError


def kde_query_prepare(settings, x, reference_point, fes_reference):
    """The host steps of kde_query before the device sums: (y [Q, D], or [Q + 1, D] with the "from-specified" point
    last, and Q).  Draws what KernelDensity.sample() draws and raises what the reference raises before its scoring."""
    DataError, _ = _kde_errors()
    kernel, D = settings["kernel"], settings["D"]
    dims = np.shape(x)[1]
    _draw_as_sample(kernel, D)
    if dims != D:
        raise DataError("query coordinates have inconsistent dimension with the data the FES is fit to.")
    y = np.asarray(x, dtype=np.float64).reshape(-1, D)
    Q = len(y)
    if reference_point == "from-specified":
        ref = np.asarray(fes_reference, dtype=np.float64).reshape(1, -1)
        if ref.shape[1] != D:
            raise ValueError(f"X has {ref.shape[1]} features, but KernelDensity is expecting {D} features as input.")
        y = np.vstack([y, ref])
    return y, Q


def kde_query_finish(settings, log_sums, Q, reference_point, log_sum_w, with_fmin=False):
    """kde_query from the device's log sums of kde_query_prepare's points."""
    _, ParameterError = _kde_errors()
    kernel, h, D = settings["kernel"], settings["h"], settings["D"]
    # sklearn: the tree's log sum, += the kernel's normalisation, -= log of the weight sum
    score = np.array(log_sums, dtype=np.float64)
    score += kde_log_norm(kernel, D, h)
    score -= log_sum_w
    f_i = -score[:Q]
    fmin = None
    if reference_point == "from-lowest":
        fmin = np.min(f_i)
        f_i = f_i - fmin
    elif reference_point == "from-specified":
        fmin = -score[Q:]
        f_i = f_i - fmin
    elif reference_point == "from-normalization":
        pass
    else:
        raise ParameterError(f"reference point choice {reference_point} for kde is unavailable")
    out = {"f_i": f_i, "df_i": None}
    return (out, fmin) if with_fmin else out


def kde_query(kde, settings, x, reference_point, fes_reference, log_sum_w, with_fmin=False):
    """_get_fes_kde (fes.py:1523-1609) without uncertainties, from kde.log_sum (a DeviceKde): {"f_i", "df_i": None}
    with f_i = -score_samples(x) relative to the reference point, log_sum_w = log sum_n w_n of the fitted weights.
    with_fmin=True also returns the reference's fmin, the -score_samples subtracted for "from-lowest" and
    "from-specified" (None for "from-normalization"): (out, fmin).

    "from-specified" evaluates its reference point in the same call as the queries (a query's result does not
    depend on the others).  Raises what the reference raises: IndexError for 1-D x, NotImplementedError for kernels
    sklearn cannot sample from, DataError on a dimension mismatch, ParameterError for another reference point.
    kde_query_prepare and kde_query_finish are its two host halves, for callers that batch the device sums."""
    y, Q = kde_query_prepare(settings, x, reference_point, fes_reference)
    log_sums = kde.log_sum(settings["kernel"], settings["h"], y)
    return kde_query_finish(settings, log_sums, Q, reference_point, log_sum_w, with_fmin)


SPLINE_WEIGHTS = ("unbiasedstate", "biasedstates", "simplesum")


def spline_sample_terms(S, A, spline_weights, N, N_k):
    """v [nb] such that the sample term of the spline fit's objective (fes.py:2135-2167) is c . v, with c the full
    coefficient vector, and that of its gradient (:2242-2249) is v[1:].

    S [K, nb] and A [nb] are DeviceBSpline.moments of the fit's knots (S_ki = sum over state k's samples of B_i,
    A_i = sum_n w_n B_i); N_k [K] counts the samples of each state.  A state without samples makes "simplesum"
    NaN, as np.mean of an empty array does in the reference."""
    if spline_weights == "unbiasedstate":
        return N * np.asarray(A, np.float64)
    S = np.asarray(S, np.float64)
    if spline_weights == "biasedstates":
        return S.sum(axis=0)
    if spline_weights == "simplesum":
        K = S.shape[0]
        with np.errstate(invalid="ignore", divide="ignore"):
            return ((N / K) * (S / np.asarray(N_k, np.float64)[:, None])).sum(axis=0)
    raise ValueError(f"spline_weights {spline_weights!r} is not one of {SPLINE_WEIGHTS}")


def _spline_setup(fes):
    p = fes.spline_parameters
    K = fes.mbar.K
    N = fes.N
    weights = p["spline_weights"]
    scaling = (N / K) * np.ones(K) if weights == "simplesum" else fes.mbar.N_k
    return p, K, N, weights, scaling


def spline_objective(fes, xi, v):
    """The spline fit's objective at the coefficients xi (the last nspline - 1; fes.py:2102-2186) from the sample
    terms v of spline_sample_terms.  The partition functions are the reference's quadratures of the same integrands
    in the same order, stored in fes.spline_data["bspline_expf"] / ["bspline_pF"] as the reference stores them, so
    that the unpatched Hessian reads what it expects."""
    p, K, N, weights, scaling = _spline_setup(fes)
    xrange, fkbias = p["xrange"], p["fkbias"]
    bloc = fes._val_to_spline(xi)
    f = np.dot(bloc.c, v)
    if weights == "unbiasedstate":
        def expf(x):
            return np.exp(-bloc(x))

        pF = fes._integrate(expf, xrange[0], xrange[1])
        f += N * np.log(pF)
    else:
        pF = np.zeros(K)
        expf = []
        for k in range(K):
            def expfk(x, kf=k):
                return np.exp(-bloc(x) - fkbias[kf](x))

            pF[k] = fes._integrate(expfk, xrange[0], xrange[1], args=(k,))
            expf.append(expfk)
        f += np.dot(scaling, np.log(pF))
    fes.spline_data["bspline_expf"] = expf
    fes.spline_data["bspline_pF"] = pF
    logprior = p["map_data"]["logprior"]
    if logprior is not None:
        f -= logprior(np.concatenate([[0], xi], axis=None))
    return f


def spline_gradient(fes, xi, v):
    """The gradient of spline_objective (fes.py:2188-2306) from the sample terms v: v[1:] minus the Boltzmann-weighted
    basis integrals, computed and stored (spline_data["bspline_gkquad"] / ["bspline_pE"]) as the reference does."""
    p, K, N, weights, scaling = _spline_setup(fes)
    xrange, fkbias = p["xrange"], p["fkbias"]
    nspline = p["nspline"]
    db_c = fes.spline_data["bspline_derivatives"]
    xrangei = fes.spline_data["xrangei"]
    bloc = fes._val_to_spline(xi)
    g = np.array(v[1:], dtype=np.float64)
    if weights == "unbiasedstate":
        gkquad = 0

        def expf(x):
            return np.exp(-bloc(x))

        pF = fes._integrate(expf, xrange[0], xrange[1])
        pE = np.zeros(nspline - 1)

        def dexpf(x, index):
            return db_c[index + 1](x) * expf(x)

        for i in range(nspline - 1):
            pE[i] = fes._integrate(dexpf, xrangei[i + 1, 0], xrangei[i + 1, 1], args=(i,))
            pE[i] /= pF
        g -= N * pE
    else:
        pF = np.zeros(K)
        gkquad = np.zeros([nspline - 1, K])

        def expf(x, k):
            return np.exp(-bloc(x) - fkbias[k](x))

        pE = None
        for k in range(K):
            pF[k] = fes._integrate(expf, xrange[0], xrange[1], args=(k,))
            for i in range(nspline - 1):
                def dexpf(x, k, i=i):
                    return db_c[i + 1](x) * expf(x, k)

                # the reference keeps the last of these scalars in spline_data["bspline_pE"]
                pE = fes._integrate(dexpf, xrangei[i + 1, 0], xrangei[i + 1, 1], args=(k,))
                gkquad[i, k] = pE / pF[k]
        g -= np.dot(gkquad, scaling)
    dlogprior = p["map_data"]["dlogprior"]
    if dlogprior is not None:
        g -= dlogprior(np.concatenate([[0], xi], axis=None))
    fes.spline_data["bspline_gkquad"] = gkquad
    fes.spline_data["bspline_pE"] = pE
    return g


def state_bias_sums(fkbias, x_n, state_n, K):
    """F_k = sum over state k's samples of fkbias[k](x_n): one pass of the user's bias callables over the samples."""
    x = np.asarray(x_n)
    s = np.asarray(state_n)
    order = np.argsort(s, kind="stable")
    bounds = np.concatenate([[0], np.cumsum(np.bincount(s, minlength=K))])
    xs = x[order]
    return np.array([np.sum(fkbias[k](xs[bounds[k]:bounds[k + 1]])) for k in range(K)], dtype=np.float64)


def spline_mc_loglikelihood(fes, spline, spline_weights, xrange, S, A, F_k, N_k):
    """The MC chain's log-likelihood of `spline` (a BSpline on the fit's knots; fes.py:1954-2010) from the moments
    S, A, the per-state bias sums F_k (state_bias_sums) and the per-state sample counts N_k.  The per-state
    normalisations are the reference's quadratures."""
    N, K = fes.N, fes.K
    c = spline.c
    if spline_weights == "unbiasedstate":
        return N * np.dot(c, A)
    fkbias = fes.spline_parameters["fkbias"]

    def splinek(x, kf):
        return spline(x) + fkbias[kf](x)

    def expk(x, kf):
        return np.exp(-splinek(x, kf))

    loglikelihood = 0
    for k in range(K):
        normalize = np.log(fes._integrate(expk, xrange[0], xrange[1], args=(k,)))
        total = np.dot(S[k], c) + F_k[k]
        if spline_weights == "simplesum":
            with np.errstate(invalid="ignore", divide="ignore"):
                loglikelihood += (N / K) * (total / N_k[k])
            loglikelihood += (N / K) * normalize
        else:
            loglikelihood += total
            loglikelihood += fes.N_k[k] * normalize
    return loglikelihood

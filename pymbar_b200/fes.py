"""Histogram free-energy surfaces from the resident MBAR problem (pymbar.FES with fes_type="histogram").

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
    _, first = np.unique(bin_n, axis=0, return_index=True)
    first = np.sort(first)
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


def histogram_fes(problem, f_k, u_n, x_n, bin_edges):
    """The histogram_data dict of fes.py:476-600 for the target state u_n, with f from the device.

    `problem` is the DeviceProblem holding (u_kn, N_k); f_k its converged free energies.  The dict has the
    reference's keys and types, so the reference's get_fes code reads it unchanged."""
    bins = _edges(bin_edges)
    bin_n, sample_label, nonzero_bins, bin_label, bin_order = histogram_labels(x_n, bins)
    dense = dense_bins(sample_label, bin_order)
    f_bin, _, _ = problem.bin_moments(f_k, u_n, dense, len(bin_order), want_C=False)
    # fes.py:579 sizes f by the distinct bin TUPLES: when several out-of-grid tuples share the label -1 the trailing
    # entries stay 0, and "from-lowest" can pick one of them, as in the reference
    f = np.zeros(len(bin_label))
    f[:len(bin_order)] = f_bin
    return {"dims": len(bins), "bins": bins, "bin_n": bin_n, "nonzero_bins": nonzero_bins,
            "sample_label": sample_label, "bin_order": bin_order, "bin_label": bin_label, "f": f}


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
    G_aug = augmented_moments(G, C, D)
    N_aug = np.concatenate([np.asarray(N_k, dtype=np.float64), np.zeros(nb)])
    Theta = est.asymptotic_covariance(G_aug, N_aug, method="svd-ew")
    return (Theta, S, G_aug) if return_moments else Theta


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

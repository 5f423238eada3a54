"""Histogram FES test infrastructure: numpy / long-double restatements of bin_moments, the fixtures made by
tools/make_fes_golden.py from the unmodified reference FES, a DeviceProblem stand-in that answers bin_moments with
numpy, and an FES-shaped stand-in class for the facade."""
import os

import numpy as np
from scipy.special import logsumexp

from oracle import mbar_oracle as orc
from tests.test_driver_logic_cpu import OracleProblem

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURES = ("fes_hist_1d", "fes_hist_2d", "fes_hist_empty")


def umbrella_energies(x_n, centres, K0, Ku):
    """(u_kn, u_n) of umbrella sampling on u0(x) = K0/2 |x|^2 with biases Ku/2 |x - c_k|^2: the energies of the
    fixtures, regenerated from the stored samples (tools/make_fes_golden.py computes them with this function)."""
    x = np.asarray(x_n, np.float64).reshape(len(x_n), -1)
    centres = np.asarray(centres, np.float64)
    u0 = 0.5 * K0 * np.sum(x ** 2, axis=1)
    u_kn = np.stack([u0 + 0.5 * Ku * np.sum((x - centres[k]) ** 2, axis=1) for k in range(len(centres))])
    return u_kn, u0


def load(name):
    z = dict(np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False))
    dims = int(z["dims"])
    z["bin_edges"] = [z[f"edges_{d}"] for d in range(dims)]
    z["bin_order"] = dict(zip(z["bin_order_labels"].tolist(), z["bin_order_index"].tolist()))
    z["u_kn"], z["u_n"] = umbrella_energies(z["x_n"], z["centres"], float(z["K0"]), float(z["Ku"]))
    return z


def bin_moments(u_kn, N_k, f_k, u_n, bin_n, nbins, mult=None):
    """(f_bin, C, D) of mbar_b200_bin_moments in numpy fp64: W_nk over all K states, w^_n = exp(log w_n + f_i)."""
    u_kn = np.asarray(u_kn, np.float64)
    N_k = np.asarray(N_k, np.float64)
    f_k = np.asarray(f_k, np.float64)
    s = N_k > 0
    W = orc.mbar_W_nk(u_kn, N_k, f_k)
    lw = -np.asarray(u_n, np.float64) - orc.log_denominator_n(u_kn[s], N_k[s], f_k[s])
    c = np.ones(len(lw)) if mult is None else np.asarray(mult, np.float64)
    f_bin = np.array([-logsumexp(lw[bin_n == i], b=c[bin_n == i]) for i in range(nbins)])
    what = np.exp(lw + f_bin[bin_n])
    C = np.zeros((len(N_k), nbins))
    np.add.at(C.T, bin_n, W * (c * what)[:, None])
    D = np.bincount(bin_n, weights=c * what ** 2, minlength=nbins)
    return f_bin, C, D


def bin_moments_ld(u_kn, N_k, f_k, u_n, bin_n, nbins, mult=None):
    """The same in long double.  Returns (f_bin, C, D, A_C, A_D): A bounds |exp argument| of the factors of each C
    row / of D among weights in the normal range (the per-entry tolerance of tests/_moments.py)."""
    from tests._moments import LD, LOG_NORMAL

    u = np.asarray(u_kn, np.float64).astype(LD)
    N_k = np.asarray(N_k, np.float64)
    s = N_k > 0
    f = np.asarray(f_k, np.float64).astype(LD)
    a_s = (f[s] + np.log(N_k[s].astype(LD)))[:, None] - u[s]
    top = a_s.max(axis=0)
    L = top + np.log(np.exp(a_s - top).sum(axis=0))
    arg = f[:, None] - u - L[None, :]
    lw = -np.asarray(u_n, np.float64).astype(LD) - L
    c = np.ones(len(lw), LD) if mult is None else np.asarray(mult, np.float64).astype(LD)
    order = np.argsort(bin_n, kind="stable")
    b_sorted = bin_n[order]
    starts = np.searchsorted(b_sorted, np.arange(nbins))
    f_bin = np.zeros(nbins, LD)
    for i in range(nbins):
        idx = order[starts[i]:(starts[i + 1] if i + 1 < nbins else len(order))]
        idx = idx[c[idx] > 0]
        m = lw[idx].max()
        f_bin[i] = -(m + np.log((c[idx] * np.exp(lw[idx] - m)).sum()))
    wa = lw + f_bin[bin_n]
    what = np.exp(wa)
    right = (c * what)[order]
    C = np.add.reduceat(np.exp(arg)[:, order] * right[None, :], starts, axis=1)
    D = np.add.reduceat(right * what[order], starts)
    normal = np.isfinite(arg) & (arg >= LOG_NORMAL)
    A_C = np.where(normal, np.abs(arg), 0).max(axis=1).astype(np.float64)
    A_D = float(np.abs(wa[np.isfinite(wa) & (wa >= LOG_NORMAL)]).max())
    return f_bin, C, D, A_C, A_D


def moment_tol(ref, A_row, A_col, N):
    """Per-entry tolerance of tests/_moments.py:
    (8 eps (A_row + A_col) + 8 eps sqrt(N) + 64 eps) |ref| + 4 N 2^-1020."""
    from tests._moments import EPS, FLOOR, LD

    A_row = np.asarray(A_row, np.float64).reshape(-1, 1) if np.ndim(ref) == 2 else np.asarray(A_row, np.float64)
    rho = 8 * EPS * (A_row + A_col) + 8 * EPS * np.sqrt(float(N)) + 64 * EPS
    return rho * np.abs(np.asarray(ref, LD)) + 4.0 * N * FLOOR


class OracleFESProblem(OracleProblem):
    """OracleProblem with bin_moments answered by the numpy restatement above."""

    def bin_moments(self, f_k, u_n, bin_n, nbins, want_C=True):
        f_bin, C, D = bin_moments(self.u, self.N_k, f_k, u_n, np.asarray(bin_n), int(nbins))
        return (f_bin, C, D) if want_C else (f_bin, None, None)


class StandInFES:
    """The part of pymbar.FES (fes.py) that the facade reads or replaces, written for the tests: the MBAR object,
    the histogram set-up and the get_fes dispatch.  The methods the facade replaces raise if they are reached."""

    mbar_class = None

    def __init__(self, u_kn, N_k):
        self.u_kn = np.array(u_kn, dtype=np.float64)
        self.N_k = np.asarray(N_k, dtype=np.int64)
        self.K, self.N = self.u_kn.shape
        self.timings = True
        self.mbar = type(self).mbar_class(self.u_kn, self.N_k)

    def _setup_fes_histogram(self, histogram_parameters):
        if len(np.shape(histogram_parameters["bin_edges"])) == 1:
            histogram_parameters["bin_edges"] = [histogram_parameters["bin_edges"]]
        self.histogram_parameters = histogram_parameters
        self.histogram_data = None
        self.histogram_datas = None

    def get_fes(self, x, reference_point="from-lowest", fes_reference=None, uncertainty_method=None):
        x = np.array(x)
        if len(np.shape(x)) <= 1:
            x = x.reshape(-1, 1)
        return self._get_fes_histogram(x, reference_point, fes_reference, uncertainty_method)

    def _replaced(self, *args, **kwargs):
        raise AssertionError("reached a method the facade replaces")

    generate_fes = _get_fes_histogram = _replaced


def check_fes_facade(fes_cls, z, rtol_df=1e-5, atol_f=1e-8):
    """generate_fes / get_fes through the facade against the reference's outputs, with no Log_W_nk download."""
    from pymbar_b200 import facade

    s0 = dict(facade.STATS)
    fes = fes_cls(z["u_kn"], z["N_k"])
    edges = z["bin_edges"][0] if len(z["bin_edges"]) == 1 else z["bin_edges"]
    out = fes.generate_fes(z["u_n"], z["x_n"], fes_type="histogram", histogram_parameters={"bin_edges": edges})
    assert "timing" in out
    hd = fes.histogram_data
    np.testing.assert_array_equal(hd["sample_label"], z["sample_label"])
    assert hd["bin_order"] == z["bin_order"]
    np.testing.assert_allclose(hd["f"], z["f"], rtol=0, atol=atol_f)
    for tag, ref in (("lowest", "from-lowest"), ("specified", "from-specified")):
        r = fes.get_fes(z["queries"], reference_point=ref, fes_reference=z["fes_reference"].tolist() if
                        z["fes_reference"].ndim else float(z["fes_reference"]), uncertainty_method="analytical")
        np.testing.assert_array_equal(np.isnan(r["f_i"]), np.isnan(z[f"f_i_{tag}"]))
        np.testing.assert_allclose(r["f_i"], z[f"f_i_{tag}"], rtol=0, atol=atol_f)
        np.testing.assert_allclose(r["df_i"], z[f"df_i_{tag}"], rtol=rtol_df, atol=1e-12)
    assert facade.STATS["redeemed"] == s0["redeemed"] and facade.STATS["fes_w_kn"] == s0["fes_w_kn"]
    assert facade.STATS["fes_histograms"] == s0["fes_histograms"] + 1
    assert facade.STATS["fes_theta"] == s0["fes_theta"] + 2
    # FES.w_kn is lazy: the first read downloads the weights of every state
    w_kn = fes.w_kn
    assert w_kn.shape == (z["u_kn"].shape[1], len(z["N_k"])) and facade.STATS["redeemed"] == s0["redeemed"] + 1
    np.testing.assert_allclose(w_kn @ z["N_k"], 1.0, atol=1e-9)
    assert abs(fes.w_n.sum() - 1.0) < 1e-12
    return fes

"""Histogram FES on the CPU: the bin labels, the augmented-covariance assembly and the facade on an FES-shaped class,
against the outputs of the unmodified reference FES (tests/golden/fes_hist_*.npz, tools/make_fes_golden.py)."""
import numpy as np
import pytest

from pymbar_b200 import estimators as est
from pymbar_b200 import fes as hist
from tests import _fes
from tests.test_driver_logic_cpu import StandInMBAR, mirror  # noqa: F401  (fixture)


@pytest.mark.parametrize("name", _fes.FIXTURES)
def test_labels_reproduce_the_reference(name):
    z = _fes.load(name)
    edges = z["bin_edges"][0] if len(z["bin_edges"]) == 1 else z["bin_edges"]
    bin_n, sample_label, nonzero_bins, bin_label, bin_order = hist.histogram_labels(z["x_n"], edges)
    np.testing.assert_array_equal(sample_label, z["sample_label"])
    assert bin_order == z["bin_order"] and list(bin_order) == z["bin_order_labels"].tolist()
    assert len(nonzero_bins) == len(set(nonzero_bins)) and set(bin_label) == set(nonzero_bins)
    assert bin_n.shape == (len(z["x_n"]), len(z["bin_edges"]))
    dense = hist.dense_bins(sample_label, bin_order)
    np.testing.assert_array_equal(dense, [bin_order[s] for s in sample_label])


def test_pseudo_bins_of_the_reference_are_kept():
    """Samples below the grid share label -1, samples above it get the bin count; both are bins of their own, in
    order of first appearance (fes.py:536-570).  With samples on both sides of a 12-bin grid the reference reports
    14 bins with the pseudo-bin -1 first."""
    z = _fes.load("fes_hist_1d")
    _, sample_label, _, bin_label, bin_order = hist.histogram_labels(z["x_n"], z["bin_edges"][0])
    assert len(bin_order) == 14 and list(bin_order)[0] == -1 and 12 in bin_order
    assert bin_label[(-1,)] == -1 and bin_label[(12,)] == 12
    # hand-made: below, inside, above, below again, a 2-D sample below in one dimension only
    x = np.array([-5.0, 0.5, 9.0, -7.0, 1.5])
    _, lab, nz, bl, bo = hist.histogram_labels(x, np.array([0.0, 1.0, 2.0]))
    assert lab.tolist() == [-1, 0, 2, -1, 1] and nz == [(-1,), (0,), (2,), (1,)] and bo == {-1: 0, 0: 1, 2: 2, 1: 3}
    x2 = np.array([[0.5, -1.0], [0.5, 0.5], [3.0, 1.5], [-1.0, 0.5]])
    e = [np.array([0.0, 1.0, 2.0, 3.0]), np.array([0.0, 1.0, 2.0, 3.0])]
    _, lab, nz, bl, bo = hist.histogram_labels(x2, e)
    # label = b0 + b1 * len(edges[1]): the reference's formula, above-grid index 3 in dimension 0
    assert lab.tolist() == [-1, 0, 3 + 1 * 4, -1] and nz == [(0, -1), (0, 0), (3, 1), (-1, 0)]
    assert bl[(-1, 0)] == -1 and bo == {-1: 0, 0: 1, 7: 2}


@pytest.mark.parametrize("name", _fes.FIXTURES)
def test_assembly_gives_the_reference_uncertainties(name):
    """G_aug = [[G, C], [C^T, diag D]] from the reference's W_aug^T W_aug blocks -> Theta -> df_i."""
    z = _fes.load(name)
    K = len(z["N_k"])
    G_aug = hist.augmented_moments(z["G"], z["C"], z["D"])
    np.testing.assert_array_equal(G_aug[:K, :K], z["G"])
    np.testing.assert_array_equal(G_aug[:K, K:], z["C"])
    np.testing.assert_array_equal(G_aug[K:, :K], z["C"].T)
    np.testing.assert_array_equal(G_aug[K:, K:], np.diag(z["D"]))
    # the bin block of the reference is diagonal: every sample lies in one bin
    assert z["bin_block_offdiag_max"] == 0.0
    Theta = est.asymptotic_covariance(G_aug, np.concatenate([z["N_k"], np.zeros(len(z["D"]))]), "svd-ew")
    hd = _histogram_data(z)
    for tag, ref in (("lowest", "from-lowest"), ("specified", "from-specified")):
        r = hist.query(hd, z["queries"], ref, _reference(z),
                       lambda j: hist.bin_uncertainties(Theta, K, j, len(z["f"])))
        np.testing.assert_allclose(r["f_i"], z[f"f_i_{tag}"], rtol=0, atol=1e-12)
        np.testing.assert_allclose(r["df_i"], z[f"df_i_{tag}"], rtol=1e-5, atol=1e-12)


@pytest.mark.parametrize("name", _fes.FIXTURES)
def test_oracle_bin_moments_reproduce_the_reference_blocks(name):
    z = _fes.load(name)
    dense = hist.dense_bins(z["sample_label"], z["bin_order"])
    nb = len(z["bin_order"])
    f_bin, C, D = _fes.bin_moments(z["u_kn"], z["N_k"], z["f_k"], z["u_n"], dense, nb)
    np.testing.assert_allclose(f_bin, z["f"][:nb], rtol=0, atol=1e-12)
    assert not np.any(z["f"][nb:])          # the reference's f has one entry per bin tuple, the extra ones 0
    np.testing.assert_allclose(C, z["C"], rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(D, z["D"], rtol=1e-12, atol=1e-300)


def test_query_errors_follow_the_reference():
    from pymbar_b200.utils import ParameterError

    z = _fes.load("fes_hist_1d")
    hd = _histogram_data(z)
    for ref in ("from-normalization", "all-differences"):
        with pytest.raises(ParameterError):
            hist.query(hd, z["queries"], ref, None)
    with pytest.raises(ParameterError):
        hist.query(hd, z["queries"], "from-specified", None)
    with pytest.raises(ParameterError):
        hist.query(hd, z["queries"], "from-specified", -50.0)         # reference point below the grid
    # above the grid the reference's check (index == number of edges) never fires: the pseudo-bin is the reference
    r = hist.query(hd, z["queries"], "from-specified", 50.0)
    assert r["f_i"][0] == z["f"][hd["bin_order"][0]] - z["f"][hd["bin_order"][12]]
    r = hist.query(hd, z["queries"], "from-lowest", None)
    assert "df_i" not in r and np.isnan(r["f_i"][-2:]).all()           # points off the grid report NaN


@pytest.fixture()
def facade_fes(mirror):  # noqa: F811
    """StandInFES over StandInMBAR over the mirror, facade installed on both; DeviceProblem answers bin_moments
    with numpy."""
    from pymbar_b200 import facade

    mirror.DeviceProblem = _fes.OracleFESProblem
    StandInMBAR.solvers = mirror
    _fes.StandInFES.mbar_class = StandInMBAR
    facade.install_on(StandInMBAR)
    facade.install_fes_on(_fes.StandInFES)
    yield _fes.StandInFES
    facade.uninstall_from(_fes.StandInFES)
    facade.uninstall_from(StandInMBAR)


@pytest.mark.parametrize("name", _fes.FIXTURES)
def test_facade_on_an_fes_shaped_class(facade_fes, name):
    _fes.check_fes_facade(facade_fes, _fes.load(name))


def test_facade_falls_through_and_uninstalls(facade_fes):
    from pymbar_b200 import facade

    z = _fes.load("fes_hist_1d")
    fes = facade_fes(z["u_kn"], z["N_k"])
    # bootstraps, and bootstrap uncertainties, are the original's
    with pytest.raises(AssertionError, match="facade replaces"):
        fes.generate_fes(z["u_n"], z["x_n"], histogram_parameters={"bin_edges": z["bin_edges"][0]}, n_bootstraps=2)
    fes.generate_fes(z["u_n"], z["x_n"], histogram_parameters={"bin_edges": z["bin_edges"][0]})
    with pytest.raises(AssertionError, match="facade replaces"):
        fes.get_fes(z["queries"], uncertainty_method="bootstrap")
    # the unnormalised log weights of MBAR come from the backend's log denominators
    lw = fes.mbar._computeUnnormalizedLogWeights(z["u_n"])
    ref = -z["u_n"] - np.log(np.exp(z["f_k"][:, None] - z["u_kn"]).T @ z["N_k"])
    np.testing.assert_allclose(lw, ref, rtol=0, atol=1e-9)
    facade.uninstall_from(facade_fes)
    assert facade_fes.__dict__["generate_fes"] is facade_fes.__dict__["_replaced"]
    assert "w_kn" not in facade_fes.__dict__
    facade.install_fes_on(facade_fes)                  # (the fixture uninstalls again)


def _reference(z):
    return z["fes_reference"].tolist() if z["fes_reference"].ndim else float(z["fes_reference"])


def _histogram_data(z):
    edges = z["bin_edges"]
    bin_n, sample_label, nonzero_bins, bin_label, bin_order = hist.histogram_labels(z["x_n"], edges)
    return {"dims": len(edges), "bins": edges, "bin_n": bin_n, "nonzero_bins": nonzero_bins,
            "sample_label": sample_label, "bin_order": bin_order, "bin_label": bin_label, "f": z["f"]}

"""FES bootstrap replicates on the CPU: the resampling stream against the unmodified reference's replicates and its
global generator (tests/golden/fes_bootstrap.npz, tools/make_fes_bootstrap_golden.py), the histogram and KDE
bootstrap paths of the facade over the CPU mirror with numpy stand-ins for the device, every fall-back rule, the new
entry points in the header and the ctypes table, and the sm_90a build of the replicate kernels."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from pymbar_b200 import fes as hist
from pymbar_b200 import fes_bootstrap as fb
from tests import _fes, _kde
from tests.test_driver_logic_cpu import StandInMBAR, mirror  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = dict(np.load(os.path.join(_fes.GOLDEN, "fes_bootstrap.npz"), allow_pickle=False))
CASES = [(str(s), int(seed)) for s in G["sources"] for seed in G["seeds"]]
NB = int(G["n_bootstraps"])


def _same_state(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def hist_case(source):
    dims = 1 if source.endswith("1d") else 2
    edges = [G[f"{source}_hist_edges_{d}"] for d in range(dims)]
    r = G[f"{source}_hist_reference"]
    return (edges[0] if dims == 1 else edges), G[f"{source}_hist_queries"], (r.tolist() if r.ndim else float(r))


@pytest.mark.parametrize("source,seed", CASES)
def test_stream_reproduces_the_reference(source, seed):
    """The regenerated indices give every replicate's x_nb (the reference's kdes[b].tree_.data) and the generator
    ends where the reference leaves it, bit for bit."""
    z = _fes.load(source)
    p = f"{source}_s{seed}_"
    np.random.seed(seed)
    states = fb.draw_replicates(z["N_k"], NB)
    after = np.random.random()
    assert after == G[p + "kde_after"] == G[p + "hist_after"]
    x = z["x_n"].reshape(len(z["x_n"]), -1)
    for b, state in enumerate(states):
        np.testing.assert_array_equal(x[fb.replicate_indices(state, z["N_k"])], G[p + "kde_x"][b])
    # regenerating does not touch the global generator
    s0 = np.random.get_state()
    fb.replicate_indices(states[0], z["N_k"])
    assert _same_state(s0, np.random.get_state())


class WeightedOracleProblem(_fes.OracleFESProblem):
    """OracleFESProblem with set_sample_weights: the solve runs on the gathered replicate (each sample repeated by
    its multiplicity), the bin sums take the multiplicities (tests/_fes.bin_moments)."""

    def __init__(self, u_kn, N_k, device=0, N_local=None):
        super().__init__(u_kn, N_k, device, N_local)
        self.u0, self.c = self.u, None

    def set_sample_weights(self, w):
        self.c = None if w is None else np.asarray(w, np.float64)
        self.u = self.u0 if w is None else self.u0[:, np.repeat(np.arange(self.u0.shape[1]), self.c.astype(np.int64))]

    def bin_moments(self, f_k, u_n, bin_n, nbins, want_C=True):
        f_bin, C, D = _fes.bin_moments(self.u0, self.N_k, f_k, u_n, np.asarray(bin_n), int(nbins), mult=self.c)
        return (f_bin, C, D) if want_C else (f_bin, None, None)


class ReplicateNumpyKde(_kde.NumpyKde):
    """NumpyKde with the replicate entry points, answered replicate by replicate by the fp64 restatement."""

    def set_replicates(self, V):
        self.V = np.array(V, np.float64)
        self.B = len(self.V)

    def log_sum_replicates(self, kernel, h, y):
        return np.array([_kde.log_sum_f64(kernel, h, self.x, v, _kde._as2d(y)) for v in self.V])


@pytest.fixture()
def boot_fes(mirror, monkeypatch):  # noqa: F811
    """A KDE-capable FES stand-in over StandInMBAR over the mirror, facade installed; the device is replaced by
    WeightedOracleProblem and ReplicateNumpyKde."""
    pytest.importorskip("sklearn")
    from pymbar_b200 import facade

    monkeypatch.setattr(mirror, "DeviceKde", ReplicateNumpyKde)
    monkeypatch.setattr(mirror, "DeviceProblem", WeightedOracleProblem)
    StandInMBAR.solvers = mirror
    cls = _kde.kde_stand_in()
    cls.mbar_class = StandInMBAR
    facade.install_on(StandInMBAR)
    facade.install_fes_on(cls)
    yield cls
    facade.uninstall_from(cls)
    facade.uninstall_from(StandInMBAR)


def check_histogram_bootstrap(cls, source, seed, atol_f=1e-7):
    """generate_fes / get_fes with bootstrap replicates against the reference, no Log_W_nk download and no call of an
    original method."""
    from pymbar_b200 import facade

    z = _fes.load(source)
    p = f"{source}_s{seed}_"
    edges, queries, ref = hist_case(source)
    s0 = dict(facade.STATS)
    fes = cls(z["u_kn"], z["N_k"])
    fes.generate_fes(z["u_n"], z["x_n"], histogram_parameters={"bin_edges": edges}, n_bootstraps=NB, seed=seed)
    assert np.random.random() == G[p + "hist_after"]
    np.testing.assert_allclose(fes.histogram_data["f"], G[p + "hist_f0"], rtol=0, atol=1e-8)
    assert len(fes.histogram_datas) == NB
    np.testing.assert_allclose([h["f"] for h in fes.histogram_datas], G[p + "hist_f"], rtol=0, atol=atol_f)
    for tag, rp in (("lowest", "from-lowest"), ("specified", "from-specified")):
        r = fes.get_fes(queries, reference_point=rp, fes_reference=ref, uncertainty_method="bootstrap")
        np.testing.assert_array_equal(np.isnan(r["f_i"]), np.isnan(G[p + "hist_f_" + tag]))
        np.testing.assert_allclose(r["f_i"], G[p + "hist_f_" + tag], rtol=0, atol=1e-8)
        np.testing.assert_allclose(r["df_i"], G[p + "hist_df_" + tag], rtol=0, atol=atol_f)
    assert facade.STATS["fes_boot_solves"] == s0["fes_boot_solves"] + NB
    assert facade.STATS["fes_boot_fallbacks"] == s0["fes_boot_fallbacks"]
    assert facade.STATS["redeemed"] == s0["redeemed"] and facade.STATS["fes_w_kn"] == s0["fes_w_kn"]
    return fes


@pytest.mark.parametrize("source,seed", CASES)
def test_histogram_replicates_on_the_mirror(boot_fes, source, seed):
    fes = check_histogram_bootstrap(boot_fes, source, seed)
    p = f"{source}_s{seed}_"
    # the lazy keys, built from the regenerated indices on first read, are the reference's
    x = G[p + "kde_x"]
    for b, h in enumerate(fes.histogram_datas):
        assert set(h) == {"dims", "bins", "bin_n", "nonzero_bins", "sample_label", "f"}
        np.testing.assert_array_equal(h["sample_label"], G[p + "hist_sample_label"][b])
        assert h["nonzero_bins"] == [tuple(int(v) for v in t) for t in G[p + "hist_nonzero_bins"][b]]
        want = np.stack([np.digitize(x[b][:, d], h["bins"][d]) - 1 for d in range(h["dims"])], axis=1)
        np.testing.assert_array_equal(h["bin_n"], want)


def check_kde_bootstrap(cls, source, seed, kernel_ids=None, atol=1e-8):
    from pymbar_b200 import facade

    p = f"{source}_s{seed}_"
    kname = str(G["kde_sources"][list(G["sources"]).index(source)])
    g = dict(np.load(os.path.join(_fes.GOLDEN, kname + ".npz"), allow_pickle=False))
    z = _fes.load(source)
    ref = g["fes_reference"].tolist() if g["fes_reference"].ndim else float(g["fes_reference"])
    queries = g["queries"]
    for i, kernel in enumerate(G["kernels"]):
        if kernel_ids is not None and i not in kernel_ids:
            continue
        s0 = dict(facade.STATS)
        fes = cls(z["u_kn"], z["N_k"])
        f0 = cls.fallbacks
        fes.generate_fes(z["u_n"], z["x_n"], fes_type="kde", n_bootstraps=NB, seed=seed,
                         kde_parameters={"kernel": str(kernel), "bandwidth": float(g["bandwidths"][0])})
        assert np.random.random() == G[p + "kde_after"]
        assert len(fes.kdes) == NB and facade.STATS["fes_kde_fits"] == s0["fes_kde_fits"]
        # where every term of a replicate lies below the fp64 range (log density < -700, the far queries) sklearn's
        # tree resolves the sum only to its node bounds: on these fixtures up to 5 nats off the exact sum at a log
        # density near -1.4e4 (DESIGN.md 3.5b).  There the device is held to the exact sum (log_sum per replicate)
        want_score = G[p + "kde_score"][i]
        near = np.all(~np.isfinite(want_score) | (want_score > -700), axis=0)
        for tag, rp in (("lowest", "from-lowest"), ("specified", "from-specified")):
            want_f, want_df = G[p + "kde_f_" + tag][i], G[p + "kde_df_" + tag][i]
            if np.all(np.isnan(want_f)):                # KernelDensity.sample() raises for this kernel
                with pytest.raises(NotImplementedError):
                    fes.get_fes(queries, reference_point=rp, fes_reference=ref, uncertainty_method="bootstrap")
                continue
            r = fes.get_fes(queries, reference_point=rp, fes_reference=ref, uncertainty_method="bootstrap")
            fin = np.isfinite(want_f) & np.isfinite(r["f_i"])
            np.testing.assert_allclose(r["f_i"][fin], want_f[fin], rtol=1e-12, atol=atol)
            # NaN where a replicate reads -inf; where a compact kernel reaches no sample sklearn's tree may report a
            # finite remnant instead (tests/test_kde_cpu.py _same_support), at least e^20 below the densest query
            assert np.all(np.isnan(r["df_i"][np.isnan(want_df)]))
            extra = np.isnan(r["df_i"]) & ~np.isnan(want_df)
            top = np.max(want_score[np.isfinite(want_score)])
            assert np.all(np.min(want_score[:, extra], axis=0) < top - 20)
            fin = np.isfinite(want_df) & near & ~extra
            np.testing.assert_allclose(r["df_i"][fin], want_df[fin], rtol=1e-10, atol=atol)
        assert cls.fallbacks == f0 and facade.STATS["fes_boot_fallbacks"] == s0["fes_boot_fallbacks"]
        assert facade.STATS["redeemed"] == s0["redeemed"] and facade.STATS["fes_kde_fits"] == s0["fes_kde_fits"]
        # the replicates' device scores, and the lazily fitted KernelDensity objects, against the reference's scores
        dev = fes.__dict__["_b200_kde_dev"]
        settings = dev[1]
        score = dev[0].log_sum_replicates(settings["kernel"], settings["h"], queries)
        score = score + hist.kde_log_norm(settings["kernel"], settings["D"], settings["h"]) - dev[2]
        want = want_score
        assert np.all(np.isinf(score[np.isinf(want)]))
        fin = np.isfinite(want) & np.isfinite(score) & near
        assert fin.sum() >= want.size // 2
        np.testing.assert_allclose(score[fin], want[fin], rtol=1e-12, atol=atol)
        fitted = fes.kdes[NB - 1]
        assert facade.STATS["fes_kde_fits"] == s0["fes_kde_fits"] + 1 and fes.kdes[-1] is fitted
        np.testing.assert_array_equal(np.asarray(fitted.tree_.data), G[p + "kde_x"][NB - 1])
        if kernel != "gaussian":
            continue                    # compact kernels: sklearn's node bounds move with the last bits of w_n
        got = fitted.score_samples(queries.reshape(len(queries), -1))
        fin = np.isfinite(want[NB - 1]) & np.isfinite(got) & near
        assert fin.sum() >= len(fin) // 2
        np.testing.assert_allclose(got[fin], want[NB - 1][fin], rtol=1e-12, atol=atol)
    return fes


@pytest.mark.parametrize("source,seed", CASES)
def test_kde_replicates_on_the_mirror(boot_fes, source, seed):
    check_kde_bootstrap(boot_fes, source, seed)


def _falls_back(cls, call):
    """call() reaches the original with numpy's generator where the caller left it."""
    from pymbar_b200 import facade

    n0 = facade.STATS["fes_boot_fallbacks"]
    np.random.seed(99)
    entry = np.random.get_state()
    with pytest.raises(AssertionError, match="facade replaces"):
        call()
    assert _same_state(entry, np.random.get_state())
    assert facade.STATS["fes_boot_fallbacks"] == n0 + 1


def test_fallbacks(boot_fes):
    cls = boot_fes
    # a replicate empties a bin b = 0 occupies: on the 2-D fixture's 10 x 10 grid every replicate does
    z = _fes.load("fes_hist_2d")
    fes = cls(z["u_kn"], z["N_k"])
    _falls_back(cls, lambda: fes.generate_fes(z["u_n"], z["x_n"], histogram_parameters={"bin_edges": z["bin_edges"]},
                                              n_bootstraps=NB, seed=7))
    # a state without samples (randint(0, 0) raises in the reference)
    ze = _fes.load("fes_hist_empty")
    assert np.any(ze["N_k"] == 0)
    fe = cls(ze["u_kn"], ze["N_k"])
    _falls_back(cls, lambda: fe.generate_fes(ze["u_n"], ze["x_n"], fes_type="kde", kde_parameters={"bandwidth": 0.1},
                                             n_bootstraps=2))
    # spline bootstraps
    z1 = _fes.load("fes_hist_1d")
    f1 = cls(z1["u_kn"], z1["N_k"])
    _falls_back(cls, lambda: f1.generate_fes(z1["u_n"], z1["x_n"], fes_type="spline", spline_parameters={},
                                             n_bootstraps=2))
    # from-normalization on a bootstrap KDE surface (the reference raises UnboundLocalError there)
    f1.generate_fes(z1["u_n"], z1["x_n"], fes_type="kde", kde_parameters={"bandwidth": 0.1}, n_bootstraps=3, seed=1)
    q = np.linspace(-1, 1, 5)
    _falls_back(cls, lambda: f1.get_fes(q, reference_point="from-normalization", uncertainty_method="bootstrap"))
    # bootstrap uncertainties of a surface generated without replicates
    f1.generate_fes(z1["u_n"], z1["x_n"], fes_type="kde", kde_parameters={"bandwidth": 0.1})
    _falls_back(cls, lambda: f1.get_fes(q, reference_point="from-lowest", uncertainty_method="bootstrap"))


def test_entry_points_are_declared():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mbar_b200.h")).read(), flags=re.S)
    from pymbar_b200 import _lib

    for name in ("mbar_b200_kde_set_replicates", "mbar_b200_kde_log_sum_replicates"):
        assert re.search(rf"\b{name}\s*\(", src) and name in _lib.SIGNATURES


def test_replicate_kernels_build_for_sm90a_without_spills():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    csrc = os.path.join(ROOT, "pymbar_b200", "csrc")
    out = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v",
                          "-c", os.path.join(csrc, "kde.cu"), "-o", os.devnull],
                         capture_output=True, text=True, check=True).stderr
    blocks = [b for b in out.split("Compiling entry function")[1:] if "kde_replicates_kernel" in b.split("\n")[0]]
    assert len(blocks) == 24                           # D = 1..4, six kernels
    for b in blocks:
        assert "0 bytes spill stores, 0 bytes spill loads" in b, b

#!/usr/bin/env python
"""Generate tests/golden/fes_bootstrap.npz by running the UNMODIFIED reference pymbar.FES with n_bootstraps > 0.

    python tools/make_fes_bootstrap_golden.py /path/to/pymbar-checkout

The samples are those of the histogram fixtures fes_hist_1d / fes_hist_2d, loaded through tests/_fes.load, so no new
sample data is stored; the KDE queries and bandwidths are those of fes_kde_1d / fes_kde_2d.  The 1-D histogram uses
the fixture's bins.  On the 2-D fixture's 10 x 10 grid some bins hold one sample, and every replicate of every seed
tried leaves one of them empty (the reference's replicate f is then shorter than b = 0's), so the 2-D histogram here
is a 4 x 4 grid over [-1, 1]^2 (hist_edges, hist_queries, hist_reference).  For each source and seed
(n_bootstraps = NB) the file holds, with keys prefixed "<source>_s<seed>_":
  * hist_f [NB, nf]: histogram_datas[b]["f"]; hist_sample_label [NB, N] and hist_nonzero_bins [NB, nt, dims];
    hist_f_<ref> / hist_df_<ref>: get_fes(uncertainty_method="bootstrap") for from-lowest and from-specified;
    hist_after: one np.random.random() drawn right after generate_fes returns;
  * kde_x [NB, N, dims]: kdes[b].tree_.data (the replicate's samples x_nb, an independent record of the stream);
    kde_score [kernel, NB, Q]: kdes[b].score_samples(queries) for every sklearn kernel; kde_f_<ref> / kde_df_<ref>
    [kernel, Q]: get_fes(uncertainty_method="bootstrap"), NaN for the kernels whose KernelDensity.sample() raises
    (all but gaussian and tophat); kde_after: the draw after generate_fes.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden")
KERNELS = ("gaussian", "tophat", "epanechnikov", "exponential", "linear", "cosine")
REFS = ("from-lowest", "from-specified")
NB = 5
SEEDS = (7, 2024)
SOURCES = (("fes_hist_1d", "fes_kde_1d"), ("fes_hist_2d", "fes_kde_2d"))


def _ref(r):
    return r.tolist() if r.ndim else float(r)


def histogram_case(source):
    """(bin edges, queries, from-specified reference) of the histogram replicates of `source`."""
    from tests import _fes

    z = _fes.load(source)
    if z["dims"] == 1:
        return z["bin_edges"], z["queries"], z["fes_reference"]
    e = np.linspace(-1.0, 1.0, 5)
    c = 0.5 * (e[1:] + e[:-1])
    q = np.vstack([[[a, b] for a in c for b in c], [[-2.0, 0.0], [0.0, 2.0]]])
    return [e, e.copy()], q, np.array([0.1, -0.1])


def run(source, kde_name, seed, data):
    import pymbar

    from tests import _fes

    z = _fes.load(source)
    g = dict(np.load(os.path.join(OUT, kde_name + ".npz"), allow_pickle=False))
    p = f"{source}_s{seed}_"
    # histogram
    bin_edges, queries, fes_reference = histogram_case(source)
    fes = pymbar.FES(z["u_kn"], z["N_k"])
    edges = bin_edges[0] if len(bin_edges) == 1 else bin_edges
    fes.generate_fes(z["u_n"], z["x_n"], fes_type="histogram", histogram_parameters={"bin_edges": edges},
                     n_bootstraps=NB, seed=seed)
    data[p + "hist_after"] = np.float64(np.random.random())
    hds = fes.histogram_datas
    data[p + "hist_f"] = np.array([h["f"] for h in hds])
    data[p + "hist_f0"] = np.array(fes.histogram_data["f"])
    data[p + "hist_sample_label"] = np.array([h["sample_label"] for h in hds], np.int64)
    data[p + "hist_nonzero_bins"] = np.array([h["nonzero_bins"] for h in hds], np.int64)
    for ref in REFS:
        r = fes.get_fes(queries, reference_point=ref, fes_reference=_ref(fes_reference),
                        uncertainty_method="bootstrap")
        tag = ref.split("-")[1]
        data[p + "hist_f_" + tag], data[p + "hist_df_" + tag] = np.array(r["f_i"]), np.array(r["df_i"])
    # KDE
    bw = float(g["bandwidths"][0])
    Q = len(g["queries"])
    q2 = g["queries"].reshape(Q, -1)
    score = np.zeros((len(KERNELS), NB, Q))
    kf = {tag: np.full((len(KERNELS), Q), np.nan) for tag in ("f_lowest", "df_lowest", "f_specified", "df_specified")}
    for i, kernel in enumerate(KERNELS):
        fes = pymbar.FES(z["u_kn"], z["N_k"])
        fes.generate_fes(z["u_n"], z["x_n"], fes_type="kde", kde_parameters={"kernel": kernel, "bandwidth": bw},
                         n_bootstraps=NB, seed=seed)
        after = np.float64(np.random.random())
        x_nb = np.array([np.asarray(k.tree_.data) for k in fes.kdes])
        if i == 0:
            data[p + "kde_after"], data[p + "kde_x"] = after, x_nb
        assert after == data[p + "kde_after"] and np.array_equal(x_nb, data[p + "kde_x"])
        score[i] = [k.score_samples(q2) for k in fes.kdes]
        for ref in REFS:
            tag = ref.split("-")[1]
            try:
                r = fes.get_fes(g["queries"], reference_point=ref, fes_reference=_ref(g["fes_reference"]),
                                uncertainty_method="bootstrap")
            except NotImplementedError:
                continue
            kf["f_" + tag][i], kf["df_" + tag][i] = r["f_i"], r["df_i"]
    data[p + "kde_score"] = score
    for tag, v in kf.items():
        data[p + "kde_" + tag] = v
    print(f"{p}: hist df_lowest[:3]={data[p + 'hist_df_lowest'][:3]} kde df_lowest[0, :3]={kf['df_lowest'][0, :3]}")


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    data = {"seeds": np.array(SEEDS), "n_bootstraps": np.int64(NB), "kernels": np.array(KERNELS),
            "sources": np.array([s for s, _ in SOURCES]), "kde_sources": np.array([k for _, k in SOURCES])}
    for source, kde_name in SOURCES:
        bin_edges, queries, fes_reference = histogram_case(source)
        for d, e in enumerate(bin_edges):
            data[f"{source}_hist_edges_{d}"] = np.asarray(e, float)
        data[f"{source}_hist_queries"] = np.asarray(queries, float)
        data[f"{source}_hist_reference"] = np.asarray(fes_reference, float)
        for seed in SEEDS:
            run(source, kde_name, seed, data)
    np.savez_compressed(os.path.join(OUT, "fes_bootstrap.npz"), **data)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

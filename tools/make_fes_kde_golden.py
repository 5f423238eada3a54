#!/usr/bin/env python
"""Generate tests/golden/fes_kde_1d.npz and fes_kde_2d.npz by running the UNMODIFIED reference pymbar.FES with
fes_type="kde".

    python tools/make_fes_kde_golden.py /path/to/pymbar-checkout

The samples are those of the histogram fixtures fes_hist_1d / fes_hist_2d, loaded through tests/_fes.load, so no new
sample data is stored.  For each case (every sklearn kernel at a fixed bandwidth, and the gaussian kernel with the
"scott" and "silverman" bandwidths) the file holds the parameters, the query points (grid points, points far from the
data, points beyond the compact kernels' support) and the reference's outputs:
  * f_<ref> [case, Q]: get_fes(queries, reference_point=<ref>)["f_i"] for from-lowest, from-specified and
    from-normalization.  get_fes calls KernelDensity.sample() for the dimension check (fes.py:1560), which sklearn
    implements for the gaussian and tophat kernels only: for the others the reference raises NotImplementedError,
    recorded in get_fes_raises, and the row is NaN;
  * score [case, Q]: score_samples of the reference's fitted KernelDensity (get_kde()), for every kernel.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden")
REFS = ("from-lowest", "from-specified", "from-normalization")
KERNELS = ("gaussian", "tophat", "epanechnikov", "exponential", "linear", "cosine")


def run(name, out_name, h, queries, fes_reference):
    import pymbar

    from tests import _fes

    z = _fes.load(name)
    cases = [(k, repr(h)) for k in KERNELS] + [("gaussian", "scott"), ("gaussian", "silverman")]
    data = {"kernels": np.array([c[0] for c in cases]), "bandwidths": np.array([c[1] for c in cases]),
            "source": np.array(name), "queries": np.asarray(queries, float),
            "fes_reference": np.asarray(fes_reference, float)}
    Q = len(queries)
    q2 = np.asarray(queries, float).reshape(Q, -1)
    for ref in REFS:
        data["f_" + ref.split("-")[1]] = np.full((len(cases), Q), np.nan)
    data["score"] = np.zeros((len(cases), Q))
    data["get_fes_raises"] = np.zeros(len(cases), bool)
    for i, (kernel, bw) in enumerate(cases):
        fes = pymbar.FES(z["u_kn"], z["N_k"])
        params = {"kernel": kernel, "bandwidth": bw if bw in ("scott", "silverman") else float(bw)}
        fes.generate_fes(z["u_n"], z["x_n"], fes_type="kde", kde_parameters=params)
        data["score"][i] = fes.get_kde().score_samples(q2)
        for ref in REFS:
            try:
                r = fes.get_fes(queries, reference_point=ref, fes_reference=fes_reference)
            except NotImplementedError:
                data["get_fes_raises"][i] = True
                continue
            data["f_" + ref.split("-")[1]][i] = r["f_i"]
        print(f"{out_name}: {kernel:12s} {bw:10s} h={fes.get_kde().bandwidth_:.6g} "
              f"f_lowest[:3]={data['f_lowest'][i][:3]}")
    np.savez_compressed(os.path.join(OUT, out_name + ".npz"), **data)


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    # 1-D: grid points over the data, two far points (gaussian terms near -45000 at h = 0.1), points just beyond
    # the reach of every sample for the compact kernels
    from tests import _fes

    x1 = _fes.load("fes_hist_1d")["x_n"]
    grid = np.linspace(-2.0, 2.0, 41)
    beyond = [x1.max() + 0.1 + 1e-3, x1.min() - 0.1 - 1e-3]
    run("fes_hist_1d", "fes_kde_1d", 0.1, np.concatenate([grid, [-30.0, 30.0], beyond]).reshape(-1, 1), 0.05)
    # 2-D: an 11 x 11 grid, far points and points beyond reach
    x2 = _fes.load("fes_hist_2d")["x_n"]
    g = np.linspace(-0.8, 0.8, 11)
    q = np.array([[a, b] for a in g for b in g])
    far = [[-20.0, 0.0], [5.0, 25.0], [x2[:, 0].max() + 0.2, 0.0], [0.0, x2[:, 1].min() - 0.2]]
    run("fes_hist_2d", "fes_kde_2d", 0.15, np.vstack([q, far]), [0.0, 0.0])


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

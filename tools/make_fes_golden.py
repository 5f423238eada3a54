#!/usr/bin/env python
"""Generate tests/golden/fes_hist_*.npz by running the UNMODIFIED reference pymbar.FES (histogram type).

    python tools/make_fes_golden.py /path/to/pymbar-checkout

Imports pymbar from the given checkout through the numexpr stub in oracle/ref_shim, as oracle/make_golden.py does.
Each case is umbrella sampling of a harmonic potential of mean force (a few thousand samples, drawn here with a
seeded numpy generator), stored with the reference's outputs:
  * the inputs: N_k, x_n, the umbrella centres and spring constants (u_kn and u_n are regenerated from them by
    tests/_fes.umbrella_energies), the bin edges, and the reference MBAR's f_k;
  * histogram_data: sample_label, bin_order (as label / index arrays) and f;
  * get_fes at query points (bin centres and points off the grid): f_i / df_i for "from-lowest" and
    "from-specified" with uncertainty_method="analytical";
  * the blocks G, C, D of W_aug^T W_aug of the augmented weight matrix, assembled from the reference MBAR's Log_W_nk
    and _computeUnnormalizedLogWeights exactly as fes.py:1382-1402 fills it, and the largest off-diagonal entry of
    its bin block.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden")


def umbrellas(centres, N_k, K0, Ku, rng):
    """Samples of the biased states of u0(x) = K0/2 |x|^2 + Ku/2 |x - c_k|^2 (Gaussian, exact) and the energies of
    tests/_fes.umbrella_energies, which the tests use to regenerate u_kn and u_n from the stored x_n."""
    from tests._fes import umbrella_energies

    centres = np.atleast_2d(np.asarray(centres, float))
    if centres.shape[0] == 1 and len(N_k) > 1:
        centres = centres.T
    K, dims = centres.shape
    sd = 1.0 / np.sqrt(K0 + Ku)
    x = np.concatenate([rng.normal(Ku * centres[k] / (K0 + Ku), sd, size=(N_k[k], dims)) for k in range(K)])
    x = x[:, 0] if dims == 1 else x
    u_kn, u0 = umbrella_energies(x, centres, K0, Ku)
    return x, u_kn, u0, dict(centres=centres, K0=np.float64(K0), Ku=np.float64(Ku))


def run_case(name, x_n, u_kn, u_n, spec, N_k, bin_edges, queries, fes_reference):
    import pymbar

    fes = pymbar.FES(u_kn, N_k)
    fes.generate_fes(u_n, x_n, fes_type="histogram", histogram_parameters={"bin_edges": bin_edges})
    hd = fes.histogram_data
    mbar = fes.mbar
    K, nb = mbar.K, len(hd["bin_order"])
    # u_kn and u_n are not stored: tests/_fes.load regenerates them from x_n and the umbrella parameters
    data = dict(spec, N_k=np.asarray(N_k, np.int64), x_n=x_n, f_k=np.array(mbar.f_k),
                sample_label=np.array(hd["sample_label"]), f=np.array(hd["f"]),
                bin_order_labels=np.array(list(hd["bin_order"].keys()), np.int64),
                bin_order_index=np.array(list(hd["bin_order"].values()), np.int64),
                queries=np.asarray(queries, float), fes_reference=np.asarray(fes_reference, float))
    edges = hd["bins"]
    data["dims"] = np.int64(len(edges))
    for d, e in enumerate(edges):
        data[f"edges_{d}"] = np.asarray(e, float)
    for tag, ref in (("lowest", "from-lowest"), ("specified", "from-specified")):
        r = fes.get_fes(queries, reference_point=ref, fes_reference=fes_reference, uncertainty_method="analytical")
        data[f"f_i_{tag}"], data[f"df_i_{tag}"] = np.array(r["f_i"]), np.array(r["df_i"])
    # W_aug as fes.py:1386-1402 fills it
    W = np.zeros((mbar.N, K + nb))
    W[:, :K] = np.exp(mbar.Log_W_nk)
    log_w = mbar._computeUnnormalizedLogWeights(fes.u_n)
    for label in hd["bin_label"].values():
        idx = np.where(hd["sample_label"] == label)
        i = hd["bin_order"][label]
        W[idx, K + i] = np.exp(log_w[idx] + hd["f"][i])
    G_aug = W.T @ W
    # the blocks of G_aug: G = W^T W, C, D (the bin block is diagonal: each sample lies in one bin)
    bin_block = G_aug[K:, K:]
    data["G"], data["C"], data["D"] = G_aug[:K, :K], G_aug[:K, K:], np.diag(bin_block).copy()
    data["bin_block_offdiag_max"] = np.float64(np.abs(bin_block - np.diag(np.diag(bin_block))).max())
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **data)
    print(f"{name}: K={K} N={mbar.N} nbins={nb} f_i[:3]={data['f_i_lowest'][:3]}")


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    rng = np.random.RandomState(8642)

    # 1-D: eight windows from -2 to 2 on a 12-bin grid over [-1.2, 1.2]: samples fall off the grid on both sides
    N_k = [300] * 8
    x, u_kn, u0, spec = umbrellas(np.linspace(-2.0, 2.0, 8), N_k, K0=4.0, Ku=40.0, rng=rng)
    edges = np.linspace(-1.2, 1.2, 13)
    centres = 0.5 * (edges[1:] + edges[:-1])
    run_case("fes_hist_1d", x, u_kn, u0, spec, N_k, edges, np.concatenate([centres, [-3.0, 3.0]]), 0.05)

    # 2-D: 7 x 7 windows, a 10 x 10 grid (the shape of the reference's own 2-D FES test)
    g = 0.2 * np.arange(-3, 4)
    cx, cy = np.meshgrid(g, g, indexing="ij")
    N_k = [60] * 49
    x, u_kn, u0, spec = umbrellas(np.stack([cx.ravel(), cy.ravel()], axis=1), N_k, K0=20.0, Ku=100.0, rng=rng)
    lo, hi = 0.2 * (-3 - 0.5), 0.2 * (3 + 0.5)
    e = np.linspace(lo, hi, 11)
    c = 0.5 * (e[1:] + e[:-1])
    q = np.array([[a, b] for a in c for b in c]) + 1e-4
    run_case("fes_hist_2d", x, u_kn, u0, spec, N_k, [e, e.copy()], np.vstack([q, [[-2.0, 0.0], [0.0, 2.0]]]),
             [0.0, 0.0])

    # 1-D with an unsampled window: its W_nk column enters C
    N_k = [400, 400, 0, 400, 400]
    x, u_kn, u0, spec = umbrellas(np.linspace(-1.0, 1.0, 5), N_k, K0=4.0, Ku=30.0, rng=rng)
    edges = np.linspace(-1.0, 1.0, 11)
    centres = 0.5 * (edges[1:] + edges[:-1])
    run_case("fes_hist_empty", x, u_kn, u0, spec, N_k, edges, centres, 0.05)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

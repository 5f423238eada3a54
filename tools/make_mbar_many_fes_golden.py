#!/usr/bin/env python
"""Generate tests/golden/mbar_many_fes.npz by running the UNMODIFIED reference pymbar.FES (histogram type) on each
umbrella problem of tests/_mbar_many_fes.SPECS.

    python tools/make_mbar_many_fes_golden.py /path/to/pymbar-checkout

Imports pymbar from the given checkout through the numexpr stub in oracle/ref_shim, as oracle/make_golden.py does.
The samples are drawn here with one seeded numpy generator (tools/make_fes_golden.umbrellas); u_kn and u_n are not
stored but regenerated from x_n by tests/_fes.umbrella_energies.  For problem i the file holds p<i>_x_n, p<i>_f_k (the
reference MBAR's), p<i>_f, p<i>_sample_label and p<i>_bin_order_{labels,index} (histogram_data), and
p<i>_f_i_<ref>_<unc> / p<i>_df_i_<ref>_analytical: get_fes at the spec's queries (bin centres and points off the grid)
for ref in "lowest" / "specified" and unc in "none" / "analytical".  "names" lists the problems.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "mbar_many_fes.npz")


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    import pymbar
    from make_fes_golden import umbrellas

    from tests import _mbar_many_fes as F

    rng = np.random.RandomState(4321)
    data = {"names": np.array([s["name"] for s in F.SPECS])}
    for i, s in enumerate(F.SPECS):
        x, u_kn, u_n, _ = umbrellas(s["centres"], s["N_k"], s["K0"], s["Ku"], rng)
        fes = pymbar.FES(u_kn, s["N_k"])
        fes.generate_fes(u_n, x, fes_type="histogram", histogram_parameters={"bin_edges": s["bin_edges"]})
        hd = fes.histogram_data
        p = f"p{i}_"
        data[p + "x_n"] = x
        data[p + "f_k"] = np.array(fes.mbar.f_k)
        data[p + "f"] = np.array(hd["f"])
        data[p + "sample_label"] = np.array(hd["sample_label"])
        data[p + "bin_order_labels"] = np.array(list(hd["bin_order"].keys()), np.int64)
        data[p + "bin_order_index"] = np.array(list(hd["bin_order"].values()), np.int64)
        for tag, rp in (("lowest", "from-lowest"), ("specified", "from-specified")):
            for unc in (None, "analytical"):
                r = fes.get_fes(s["queries"], reference_point=rp, fes_reference=s["fes_reference"],
                                uncertainty_method=unc)
                data[f"{p}f_i_{tag}_{unc or 'none'}"] = np.array(r["f_i"])
                if unc:
                    data[f"{p}df_i_{tag}_{unc}"] = np.array(r["df_i"])
        print(f"{s['name']}: K={len(s['N_k'])} N={len(x)} nbins={len(hd['bin_order'])} f[:3]={data[p + 'f'][:3]}")
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

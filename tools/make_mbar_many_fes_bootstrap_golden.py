#!/usr/bin/env python
"""Generate tests/golden/mbar_many_fes_bootstrap.npz by running the UNMODIFIED reference pymbar.FES (histogram type,
n_bootstraps = B) on each umbrella problem of tests/_mbar_many_fes_bootstrap.SPECS.

    python tools/make_mbar_many_fes_bootstrap_golden.py /path/to/pymbar-checkout

Imports pymbar from the given checkout through the numexpr stub in oracle/ref_shim, as oracle/make_golden.py does.
The samples are drawn with one seeded numpy generator (tools/make_fes_golden.umbrellas); u_kn and u_n are regenerated
from x_n by tests/_fes.umbrella_energies.  Two runs:

* "seeded": problem p's generate_fes(..., n_bootstraps=B, seed=SEED0 + p);
* "stream": every FES is constructed first (each MBAR constructor draws from numpy's global generator), then
  np.random.seed(STREAM_SEED) once and generate_fes(..., n_bootstraps=B, seed=-1) on each problem in turn;
  "stream_next" is the np.random.randint(2**31 - 1) that follows.

For problem i and run r the file holds p<i>_x_n, p<i>_<r>_f (b = 0's histogram f), p<i>_<r>_boot_f [B, len(f)] (the
replicates' f) and p<i>_<r>_{f_i,df_i}_<ref> of get_fes(uncertainty_method="bootstrap") at the spec's queries for ref in
"lowest" / "specified".  Every replicate must draw from every bin tuple of b = 0 (asserted here).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "mbar_many_fes_bootstrap.npz")


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    import pymbar
    from make_fes_golden import umbrellas

    from tests import _mbar_many_fes_bootstrap as FB

    rng = np.random.RandomState(2468)
    data = {"names": np.array([s["name"] for s in FB.SPECS]), "n_bootstraps": np.int64(FB.B)}
    inputs = []
    for i, s in enumerate(FB.SPECS):
        x, u_kn, u_n, _ = umbrellas(s["centres"], s["N_k"], s["K0"], s["Ku"], rng)
        data[f"p{i}_x_n"] = x
        inputs.append((x, u_kn, u_n))

    def record(i, s, fes, run):
        p = f"p{i}_{run}_"
        hd = fes.histogram_data
        tuples = {tuple(int(v) for v in t) for t in hd["bin_n"]}
        for h in fes.histogram_datas:
            assert {tuple(int(v) for v in t) for t in h["bin_n"]} == tuples, (s["name"], run, "uncovered tuple")
        data[p + "f"] = np.array(hd["f"])
        data[p + "boot_f"] = np.array([h["f"] for h in fes.histogram_datas])
        for tag, rp in (("lowest", "from-lowest"), ("specified", "from-specified")):
            r = fes.get_fes(s["queries"], reference_point=rp, fes_reference=s["fes_reference"],
                            uncertainty_method="bootstrap")
            data[f"{p}f_i_{tag}"] = np.array(r["f_i"])
            data[f"{p}df_i_{tag}"] = np.array(r["df_i"])
        print(f"{s['name']} {run}: K={len(s['N_k'])} N={len(inputs[i][0])} nbins={len(hd['bin_order'])} "
              f"boot_f[0,:3]={data[p + 'boot_f'][0, :3]}", flush=True)

    for i, s in enumerate(FB.SPECS):
        x, u_kn, u_n = inputs[i]
        fes = pymbar.FES(u_kn, s["N_k"])
        fes.generate_fes(u_n, x, fes_type="histogram", histogram_parameters={"bin_edges": s["bin_edges"]},
                         n_bootstraps=FB.B, seed=FB.SEED0 + i)
        record(i, s, fes, "seeded")
    fess = [pymbar.FES(inputs[i][1], s["N_k"]) for i, s in enumerate(FB.SPECS)]
    np.random.seed(FB.STREAM_SEED)
    for i, s in enumerate(FB.SPECS):
        x, _, u_n = inputs[i]
        fess[i].generate_fes(u_n, x, fes_type="histogram", histogram_parameters={"bin_edges": s["bin_edges"]},
                             n_bootstraps=FB.B, seed=-1)
    data["stream_next"] = np.int64(np.random.randint(2 ** 31 - 1))
    for i, s in enumerate(FB.SPECS):
        record(i, s, fess[i], "stream")
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

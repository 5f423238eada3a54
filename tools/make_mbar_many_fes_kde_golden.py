#!/usr/bin/env python
"""Generate tests/golden/mbar_many_fes_kde.npz by running the UNMODIFIED reference pymbar.FES (kde type, with
scikit-learn) on each umbrella problem of tests/_mbar_many_fes_kde.SPECS.

    python tools/make_mbar_many_fes_kde_golden.py /path/to/pymbar-checkout

Imports pymbar from the given checkout through the numexpr stub in oracle/ref_shim, as oracle/make_golden.py does.
The samples are drawn with one seeded numpy generator (tools/make_fes_golden.umbrellas); u_kn and u_n are regenerated
from x_n by tests/_fes.umbrella_energies.  For problem i the file holds p<i>_x_n and:

* b = 0 (generate_fes with n_bootstraps=0): p<i>_f_i_<ref> of get_fes at the spec's queries for ref in "lowest",
  "specified" and "normalization"; for the epanechnikov problem, whose get_fes raises (KernelDensity.sample is not
  implemented for it), p<i>_score (kde.score_samples of the queries) and p<i>_get_fes_raises = 1 instead;
* for the problems of BOOT, two runs of B replicates: "seeded" (generate_fes(..., seed=SEED0 + i)) and "stream" (every
  FES constructed first, then np.random.seed(STREAM_SEED) once and seed=-1 for each problem in turn; "stream_next" is
  the np.random.randint(2**31 - 1) that follows), with p<i>_<run>_{f_i,df_i}_<ref> of
  get_fes(uncertainty_method="bootstrap") for ref in "lowest" and "specified".
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "mbar_many_fes_kde.npz")


def main(reference):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    sys.path.insert(0, os.path.abspath(reference))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ["PYMBAR_DISABLE_JAX"] = "1"
    import pymbar
    from make_fes_golden import umbrellas

    from tests import _mbar_many_fes_kde as FK

    rng = np.random.RandomState(97531)
    data = {"names": np.array(FK.NAMES), "n_bootstraps": np.int64(FK.B)}
    inputs = []
    for i, s in enumerate(FK.SPECS):
        x, u_kn, u_n, _ = umbrellas(s["centres"], s["N_k"], s["K0"], s["Ku"], rng)
        data[f"p{i}_x_n"] = x
        inputs.append((x, u_kn, u_n))

    def queries(s):
        q = np.array(s["queries"])
        return q.reshape(-1, 1) if q.ndim == 1 else q

    for i, s in enumerate(FK.SPECS):
        x, u_kn, u_n = inputs[i]
        fes = pymbar.FES(u_kn, s["N_k"])
        fes.generate_fes(u_n, x, fes_type="kde", kde_parameters=dict(s["kde_parameters"]))
        if i in FK.RAISES:
            data[f"p{i}_score"] = np.array(fes.kde.score_samples(queries(s)))
            data[f"p{i}_get_fes_raises"] = np.int64(1)
            try:
                fes.get_fes(s["queries"], reference_point="from-lowest")
            except NotImplementedError:
                pass
            else:
                raise AssertionError(f"{s['name']}: get_fes did not raise")
            continue
        for tag, rp in FK.REFS:
            r = fes.get_fes(s["queries"], reference_point=rp, fes_reference=s["fes_reference"])
            data[f"p{i}_f_i_{tag}"] = np.array(r["f_i"])
        print(f"{s['name']}: K={len(s['N_k'])} N={len(x)} f_i[:3]={data[f'p{i}_f_i_lowest'][:3]}", flush=True)

    def record(i, s, fes, run):
        for tag, rp in FK.BOOT_REFS:
            r = fes.get_fes(s["queries"], reference_point=rp, fes_reference=s["fes_reference"],
                            uncertainty_method="bootstrap")
            data[f"p{i}_{run}_f_i_{tag}"] = np.array(r["f_i"])
            data[f"p{i}_{run}_df_i_{tag}"] = np.array(r["df_i"])

    for i in FK.BOOT:
        s = FK.SPECS[i]
        x, u_kn, u_n = inputs[i]
        fes = pymbar.FES(u_kn, s["N_k"])
        fes.generate_fes(u_n, x, fes_type="kde", kde_parameters=dict(s["kde_parameters"]), n_bootstraps=FK.B,
                         seed=FK.SEED0 + i)
        record(i, s, fes, "seeded")
    fess = {i: pymbar.FES(inputs[i][1], FK.SPECS[i]["N_k"]) for i in FK.BOOT}
    np.random.seed(FK.STREAM_SEED)
    for i in FK.BOOT:
        s = FK.SPECS[i]
        x, _, u_n = inputs[i]
        fess[i].generate_fes(u_n, x, fes_type="kde", kde_parameters=dict(s["kde_parameters"]), n_bootstraps=FK.B,
                             seed=-1)
    data["stream_next"] = np.int64(np.random.randint(2 ** 31 - 1))
    for i in FK.BOOT:
        record(i, FK.SPECS[i], fess[i], "stream")
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

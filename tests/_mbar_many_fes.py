"""Problems of the MbarMany histogram FES tests and numpy stand-ins of the batch's bin_moments.

SPECS are the umbrella problems of tests/golden/mbar_many_fes.npz (tools/make_mbar_many_fes_golden.py): 1-D problems
with K = 1, 8 and 64, a 2-D 3 x 3 umbrella grid, a 1-D problem with an unsampled window and a K = 70 problem, which
takes the single path.  Every grid leaves samples outside, so pseudo-bins occur, and every problem has its own
bin_edges.  load() rebuilds u_kn and u_n from the stored samples with tests/_fes.umbrella_energies.

FesOracleBatch adds `bin_moments` to tests/_mbar_many_expectations.AugOracleBatch and FesOracleProblem adds it to
AugOracleProblem, both answered by the numpy restatement tests/_fes.bin_moments, so that the routing, waves and host
algebra of MbarMany.generate_fes / get_fes run without a GPU.
"""
import os

import numpy as np

from tests import _fes
from tests import _mbar_many_expectations as E

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mbar_many_fes.npz")


def _centres(edges):
    return 0.5 * (edges[1:] + edges[:-1])


def _specs():
    out = []

    def one_d(name, centres, N_k, K0, Ku, edges, ref):
        q = np.concatenate([_centres(edges), [edges[0] - 2.0, edges[-1] + 2.0]])
        out.append(dict(name=name, centres=np.asarray(centres, float), N_k=np.asarray(N_k, np.int64), K0=K0, Ku=Ku,
                        bin_edges=edges, queries=q, fes_reference=ref))

    one_d("1d_K1", [0.0], [600], 4.0, 10.0, np.linspace(-0.6, 0.6, 9), 0.05)
    one_d("1d_K8", np.linspace(-2.0, 2.0, 8), [200] * 8, 4.0, 40.0, np.linspace(-1.2, 1.2, 13), 0.05)
    one_d("1d_K64", np.linspace(-3.0, 3.0, 64), [40] * 64, 2.0, 60.0, np.linspace(-2.5, 2.5, 41), -0.3)
    g = 0.4 * np.arange(-1, 2)
    cx, cy = np.meshgrid(g, g, indexing="ij")
    e = np.linspace(-0.7, 0.7, 8)
    c = _centres(e)
    q = np.array([[a, b] for a in c for b in c]) + 1e-4
    out.append(dict(name="2d_3x3", centres=np.stack([cx.ravel(), cy.ravel()], axis=1), N_k=np.full(9, 150, np.int64),
                    K0=10.0, Ku=60.0, bin_edges=[e, e.copy()], queries=np.vstack([q, [[-2.0, 0.0], [0.0, 2.0]]]),
                    fes_reference=[0.0, 0.0]))
    one_d("1d_unsampled", np.linspace(-1.0, 1.0, 5), [300, 300, 0, 300, 300], 4.0, 30.0, np.linspace(-1.0, 1.0, 11),
          0.05)
    one_d("1d_K70", np.linspace(-3.0, 3.0, 70), [30] * 70, 2.0, 60.0, np.linspace(-2.0, 2.0, 21), 0.1)
    return out


SPECS = _specs()
TAGS = (("lowest", "from-lowest"), ("specified", "from-specified"))


def load(path=GOLDEN):
    """[case] with the spec's inputs, u_kn, u_n, x_n and the reference's outputs (keys as in the file, without the
    p<i>_ prefix)."""
    z = np.load(path)
    assert [str(n) for n in z["names"]] == [s["name"] for s in SPECS]
    cases = []
    for i, s in enumerate(SPECS):
        p = f"p{i}_"
        c = dict(s, **{k[len(p):]: z[k] for k in z.files if k.startswith(p)})
        c["u_kn"], c["u_n"] = _fes.umbrella_energies(c["x_n"], s["centres"], s["K0"], s["Ku"])
        c["bin_order"] = dict(zip(c["bin_order_labels"].tolist(), c["bin_order_index"].tolist()))
        cases.append(c)
    return cases


def check_case(c, hd, out):
    """histogram_data and get_fes outputs out[(tag, unc)] against the reference, at the bounds of the single-problem
    FES golden checks (tests/_fes.check_fes_facade): f atol 1e-8, df rtol 1e-5 / atol 1e-12."""
    n = c["name"]
    np.testing.assert_array_equal(hd["sample_label"], c["sample_label"], err_msg=n)
    assert hd["bin_order"] == c["bin_order"], n
    np.testing.assert_allclose(hd["f"], c["f"], rtol=0, atol=1e-8, err_msg=n)
    for tag, _ in TAGS:
        for unc in ("none", "analytical"):
            r = out[(tag, unc)]
            want = c[f"f_i_{tag}_{unc}"]
            np.testing.assert_array_equal(np.isnan(r["f_i"]), np.isnan(want), err_msg=n)
            np.testing.assert_allclose(r["f_i"], want, rtol=0, atol=1e-8, err_msg=f"{n} {tag} {unc}")
            if unc == "analytical":
                np.testing.assert_allclose(r["df_i"], c[f"df_i_{tag}_analytical"], rtol=1e-5, atol=1e-12,
                                           err_msg=f"{n} {tag} df")
            else:
                assert "df_i" not in r


def run_all(m, cases, skip=()):
    """generate_fes then the four get_fes queries of the fixture on every case (None for the indices in skip):
    {(tag, unc): [out per problem]}."""
    sel = [None if i in skip else c for i, c in enumerate(cases)]
    m.generate_fes([None if c is None else c["u_n"] for c in sel], [None if c is None else c["x_n"] for c in sel],
                   histogram_parameters=[None if c is None else {"bin_edges": c["bin_edges"]} for c in sel])
    out = {}
    for tag, rp in TAGS:
        for unc in ("none", "analytical"):
            out[(tag, unc)] = m.get_fes([None if c is None else c["queries"] for c in sel], reference_point=rp,
                                        fes_reference=[None if c is None else c["fes_reference"] for c in sel],
                                        uncertainty_method=None if unc == "none" else unc)
    return out


class FesOracleBatch(E.AugOracleBatch):
    """AugOracleBatch with bin_moments.  `bin_flagged` names problem indices (in this batch) whose bin_moments
    requests report the flag (`bin_flagged_C`: only those with want_C); calls are recorded in AugOracleBatch.calls as
    ("bin_moments", problems, want_C)."""

    bin_flagged = ()
    bin_flagged_C = ()

    def bin_moments(self, problems, f_list, u_n_list, bin_list, nbins_list, want_C=True):
        E.AugOracleBatch.calls.append(("bin_moments", [int(p) for p in problems], bool(want_C)))
        out, flags = [], []
        for p, f, u, b, nb in zip(problems, f_list, u_n_list, bin_list, nbins_list):
            f_bin, C, D = _fes.bin_moments(self.u[p], self.N_k[p], f, u, np.asarray(b), int(nb))
            out.append((f_bin, C, D) if want_C else (f_bin, None, None))
            flags.append(p in self.bin_flagged or (want_C and p in self.bin_flagged_C))
        return out, np.array(flags, bool)


class FesOracleProblem(E.AugOracleProblem):
    """AugOracleProblem with bin_moments."""

    def bin_moments(self, f_k, u_n, bin_n, nbins, want_C=True):
        f_bin, C, D = _fes.bin_moments(self.u, self.N_k, f_k, u_n, np.asarray(bin_n), int(nbins))
        return (f_bin, C, D) if want_C else (f_bin, None, None)

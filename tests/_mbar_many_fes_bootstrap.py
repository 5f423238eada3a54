"""Problems of the MbarMany bootstrap histogram FES tests and numpy stand-ins of the weighted bin pass.

SPECS are the umbrella problems of tests/golden/mbar_many_fes_bootstrap.npz (tools/make_mbar_many_fes_bootstrap_golden.py):
1-D problems with K = 1, 8 and 32, a 2-D 3 x 3 umbrella grid and a K = 70 problem, which takes the single path.  No
state is empty, every grid leaves many samples outside (pseudo-bins, and in 2-D several out-of-grid tuples sharing
label -1), and every bin tuple holds enough samples that each replicate of the file draws from all of them.  The file
holds two runs of B replicates: "seeded" (seed = SEED0 + p per problem) and "stream" (np.random.seed(STREAM_SEED) once,
then seed=-1 for each problem in turn, and the next np.random.randint(2**31 - 1) after the last).

FesBootOracleBatch adds replicate slots (tests/_mbar_many_boot.WeightedOracleBatch) and replicate_bin_moments to
tests/_mbar_many_fes.FesOracleBatch; FesBootOracleProblem adds set_sample_weights to FesOracleProblem.  Both answer in
float64 numpy (tests/_fes.bin_moments with the multiplicities), so that the draws, waves, routing and host algebra of
MbarMany.generate_fes(..., n_bootstraps=B) run without a GPU.
"""
import os

import numpy as np

from tests import _fes
from tests import _mbar_many_boot as W
from tests import _mbar_many_fes as F

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mbar_many_fes_bootstrap.npz")
B = 8
SEED0 = 1000
STREAM_SEED = 777
RUNS = ("seeded", "stream")
TAGS = F.TAGS


def _centres(edges):
    return 0.5 * (edges[1:] + edges[:-1])


def _specs():
    out = []

    def one_d(name, centres, N_k, K0, Ku, edges, ref):
        q = np.concatenate([_centres(edges), [edges[0] - 2.0, edges[-1] + 2.0]])
        out.append(dict(name=name, centres=np.asarray(centres, float), N_k=np.asarray(N_k, np.int64), K0=K0, Ku=Ku,
                        bin_edges=edges, queries=q, fes_reference=ref))

    one_d("1d_K1", [0.0], [800], 4.0, 10.0, np.linspace(-0.5, 0.5, 6), 0.05)
    one_d("1d_K8", np.linspace(-2.0, 2.0, 8), [300] * 8, 4.0, 40.0, np.linspace(-1.5, 1.5, 11), 0.05)
    one_d("1d_K32", np.linspace(-3.0, 3.0, 32), [100] * 32, 2.0, 60.0, np.linspace(-2.5, 2.5, 21), -0.3)
    g = 0.4 * np.arange(-1, 2)
    cx, cy = np.meshgrid(g, g, indexing="ij")
    e = np.linspace(-0.3, 0.3, 4)
    c = _centres(e)
    q = np.array([[a, b] for a in c for b in c]) + 1e-4
    out.append(dict(name="2d_3x3", centres=np.stack([cx.ravel(), cy.ravel()], axis=1), N_k=np.full(9, 300, np.int64),
                    K0=10.0, Ku=60.0, bin_edges=[e, e.copy()], queries=np.vstack([q, [[-2.0, 0.0], [0.0, 2.0]]]),
                    fes_reference=[0.0, 0.0]))
    one_d("1d_K70", np.linspace(-3.0, 3.0, 70), [30] * 70, 2.0, 60.0, np.linspace(-2.0, 2.0, 11), 0.1)
    return out


SPECS = _specs()


def load(path=GOLDEN):
    """[case] with the spec's inputs, u_kn, u_n, x_n and the reference's outputs of both runs (keys as in the file,
    without the p<i>_ prefix), plus "stream_next"."""
    z = np.load(path)
    assert [str(n) for n in z["names"]] == [s["name"] for s in SPECS]
    assert int(z["n_bootstraps"]) == B
    cases = []
    for i, s in enumerate(SPECS):
        p = f"p{i}_"
        c = dict(s, **{k[len(p):]: z[k] for k in z.files if k.startswith(p)})
        c["u_kn"], c["u_n"] = _fes.umbrella_energies(c["x_n"], s["centres"], s["K0"], s["Ku"])
        cases.append(c)
    return cases, int(z["stream_next"])


def seeds(cases):
    return [SEED0 + i for i in range(len(cases))]


def args(cases):
    return [c["u_kn"] for c in cases], [c["N_k"].astype(np.float64) for c in cases]


def fes_args(cases):
    return ([c["u_n"] for c in cases], [c["x_n"] for c in cases],
            [{"bin_edges": c["bin_edges"]} for c in cases])


def run(m, cases, run_name, skip=()):
    """generate_fes with B replicates in the fixture's seed mode, then the two bootstrap get_fes queries:
    ({tag: [out per problem]}, the next randint after the draws for "stream")."""
    sel = [None if i in skip else c for i, c in enumerate(cases)]
    u, x, hp = fes_args(cases)
    pick = [None if c is None else v for c, v in zip(sel, u)], [None if c is None else v for c, v in zip(sel, x)]
    if run_name == "seeded":
        m.generate_fes(*pick, histogram_parameters=hp, n_bootstraps=B, seed=seeds(cases))
        nxt = None
    else:
        np.random.seed(STREAM_SEED)
        m.generate_fes(*pick, histogram_parameters=hp, n_bootstraps=B)
        nxt = int(np.random.randint(2 ** 31 - 1))
    out = {}
    for tag, rp in TAGS:
        out[tag] = m.get_fes([None if c is None else c["queries"] for c in sel], reference_point=rp,
                             fes_reference=[None if c is None else c["fes_reference"] for c in sel],
                             uncertainty_method="bootstrap")
    return out, nxt


def check_case(c, run_name, m, i, out, atol=1e-8):
    """Problem i's replicates and bootstrap get_fes outputs against the reference's run `run_name`."""
    n = f"{c['name']} {run_name}"
    reps = m.replicate_histogram_datas[i]
    assert len(reps) == B, n
    got = np.array([h["f"] for h in reps])
    np.testing.assert_allclose(got, c[f"{run_name}_boot_f"], rtol=0, atol=atol, err_msg=n)
    np.testing.assert_allclose(m.histogram_datas[i]["f"], c[f"{run_name}_f"], rtol=0, atol=atol, err_msg=n)
    for tag, _ in TAGS:
        r = out[tag][i]
        for key in ("f_i", "df_i"):
            want = c[f"{run_name}_{key}_{tag}"]
            np.testing.assert_array_equal(np.isnan(r[key]), np.isnan(want), err_msg=f"{n} {tag} {key}")
            np.testing.assert_allclose(r[key], want, rtol=0, atol=atol, err_msg=f"{n} {tag} {key}")


def max_errors(c, run_name, m, i, out):
    """{key: largest absolute difference from the reference} of problem i in run `run_name`."""
    got = np.array([h["f"] for h in m.replicate_histogram_datas[i]])
    e = dict(boot_f=float(np.max(np.abs(got - c[f"{run_name}_boot_f"]))))
    for tag, _ in TAGS:
        for key in ("f_i", "df_i"):
            a, b = np.asarray(out[tag][i][key]), c[f"{run_name}_{key}_{tag}"]
            ok = ~np.isnan(b)
            e[f"{key}_{tag}"] = float(np.max(np.abs(a[ok] - b[ok]))) if ok.any() else 0.0
    return e


class FesBootOracleBatch(F.FesOracleBatch, W.WeightedOracleBatch):
    """FesOracleBatch with replicate slots and replicate_bin_moments.  `rep_bin_flagged` names batch problem indices
    whose replicate_bin_moments requests report the flag; calls are recorded in AugOracleBatch.calls as
    ("replicate_bin_moments", target problems, slot problems)."""

    rep_bin_flagged = ()

    def replicate_bin_moments(self, target_problems, u_n_list, bin_list, nbins_list, slots, targets, f_list):
        F.FesOracleBatch.calls.append(("replicate_bin_moments", [int(p) for p in target_problems],
                                       [int(self.slot_problems[s]) for s in slots]))
        out, flags = [], []
        for s, t, f in zip(slots, targets, f_list):
            p = int(self.slot_problems[s])
            assert int(target_problems[t]) == p
            with np.errstate(divide="ignore"):
                f_bin, _, _ = _fes.bin_moments(self.u[p], self.N_k[p], f, u_n_list[t], np.asarray(bin_list[t]),
                                               int(nbins_list[t]), mult=self.slot_counts[s])
            out.append(f_bin)
            flags.append(p in self.rep_bin_flagged)
        return out, np.array(flags, bool)


class FesBootOracleProblem(F.FesOracleProblem):
    """FesOracleProblem with set_sample_weights: bin_moments then counts each sample by its multiplicity, and
    bootstrap.bootstrap_f_k is replaced by tests/_mbar_many_boot.oracle_bootstrap_f_k (the solve on u[:, rints])."""

    def __init__(self, u_kn, N_k, device=0):
        super().__init__(u_kn, N_k, device)
        self.c = None

    def set_sample_weights(self, w):
        self.c = None if w is None else np.asarray(w, np.float64)

    def bin_moments(self, f_k, u_n, bin_n, nbins, want_C=True):
        with np.errstate(divide="ignore"):
            f_bin, C, D = _fes.bin_moments(self.u, self.N_k, f_k, u_n, np.asarray(bin_n), int(nbins), mult=self.c)
        return (f_bin, C, D) if want_C else (f_bin, None, None)

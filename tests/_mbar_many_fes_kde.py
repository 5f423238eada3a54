"""Problems of the MbarMany KDE surface tests and numpy stand-ins of the batch's log_weights and of DeviceKdeMany.

SPECS are the umbrella problems of tests/golden/mbar_many_fes_kde.npz (tools/make_mbar_many_fes_kde_golden.py): 1-D
problems with K = 1, 8 and 64, a 2-D 3 x 3 umbrella grid, a K = 70 problem (the single path), a problem with an
unsampled window (b = 0 only) and one epanechnikov problem, whose get_fes raises in the reference (KernelDensity.sample
is not implemented for it) and whose score_samples is recorded instead.  Bandwidths: fixed, "scott" and "silverman";
kernels gaussian, tophat and epanechnikov.  Queries lie on the grid, far from the data and beyond the compact
supports.  The file holds every problem's b = 0 f_i for the three reference points and, for the problems in BOOT,
two runs of B bootstrap replicates ("seeded": seed = SEED0 + p; "stream": np.random.seed(STREAM_SEED) once, then
seed=-1 for each problem in turn, and the next np.random.randint(2**31 - 1) after the last) with f_i and df_i for
"from-lowest" and "from-specified".

KdeOracleBatch adds log_weights to tests/_mbar_many_fes_bootstrap.FesBootOracleBatch, KdeOracleProblem adds
log_denominator to FesBootOracleProblem, and NumpyKdeMany answers DeviceKdeMany.log_sum with the fp64 restatement
tests/_kde.log_sum, so that MbarMany's KDE surfaces run without a GPU.
"""
import os

import numpy as np

from oracle import mbar_oracle as orc
from tests import _fes
from tests import _kde
from tests import _mbar_many_expectations as E
from tests import _mbar_many_fes_bootstrap as FB

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mbar_many_fes_kde.npz")
B = 5
SEED0 = 2000
STREAM_SEED = 4321
RUNS = ("seeded", "stream")
REFS = (("lowest", "from-lowest"), ("specified", "from-specified"), ("normalization", "from-normalization"))
BOOT_REFS = REFS[:2]


def _specs():
    out = []

    def one_d(name, centres, N_k, K0, Ku, params, ref, lo, hi):
        q = np.concatenate([np.linspace(lo, hi, 25), [lo - 6.0, hi + 6.0]])
        out.append(dict(name=name, centres=np.asarray(centres, float), N_k=np.asarray(N_k, np.int64), K0=K0, Ku=Ku,
                        kde_parameters=params, queries=q, fes_reference=ref))

    one_d("1d_K1", [0.0], [400], 4.0, 10.0, {"bandwidth": 0.1}, 0.05, -0.6, 0.6)
    one_d("1d_K8", np.linspace(-2.0, 2.0, 8), [150] * 8, 4.0, 40.0, {"bandwidth": "scott"}, 0.05, -1.5, 1.5)
    one_d("1d_K64", np.linspace(-3.0, 3.0, 64), [20] * 64, 2.0, 60.0, {"bandwidth": "silverman"}, -0.3, -2.5, 2.5)
    g = 0.4 * np.arange(-1, 2)
    cx, cy = np.meshgrid(g, g, indexing="ij")
    c = np.linspace(-0.6, 0.6, 5)
    q = np.array([[a, b] for a in c for b in c]) + 1e-4
    out.append(dict(name="2d_3x3", centres=np.stack([cx.ravel(), cy.ravel()], axis=1), N_k=np.full(9, 100, np.int64),
                    K0=10.0, Ku=60.0, kde_parameters={"bandwidth": 0.15, "kernel": "gaussian"},
                    queries=np.vstack([q, [[-6.0, 0.0], [0.0, 6.0]]]), fes_reference=[0.0, 0.0]))
    one_d("1d_unsampled", np.linspace(-1.0, 1.0, 5), [200, 200, 0, 200, 200], 4.0, 30.0,
          {"bandwidth": 0.2, "kernel": "tophat"}, 0.05, -1.2, 1.2)
    one_d("1d_K70", np.linspace(-3.0, 3.0, 70), [15] * 70, 2.0, 60.0, {"bandwidth": 0.1}, 0.1, -2.0, 2.0)
    one_d("1d_epanechnikov", np.linspace(-1.0, 1.0, 4), [150] * 4, 4.0, 30.0,
          {"bandwidth": 0.3, "kernel": "epanechnikov"}, 0.0, -1.5, 1.5)
    return out


SPECS = _specs()
NAMES = [s["name"] for s in SPECS]
BOOT = [NAMES.index(n) for n in ("1d_K1", "1d_K8", "1d_K64", "2d_3x3", "1d_K70")]   # bootstrapped in the fixture
RAISES = [NAMES.index("1d_epanechnikov")]                                        # get_fes raises in the reference


def load(path=GOLDEN):
    """([case], stream_next): the spec's inputs, u_kn, u_n, x_n and the reference's outputs (keys as in the file,
    without the p<i>_ prefix)."""
    z = np.load(path)
    assert [str(n) for n in z["names"]] == NAMES
    assert int(z["n_bootstraps"]) == B
    cases = []
    for i, s in enumerate(SPECS):
        p = f"p{i}_"
        c = dict(s, **{k[len(p):]: z[k] for k in z.files if k.startswith(p)})
        c["u_kn"], c["u_n"] = _fes.umbrella_energies(c["x_n"], s["centres"], s["K0"], s["Ku"])
        cases.append(c)
    return cases, int(z["stream_next"])


def args(cases):
    return [c["u_kn"] for c in cases], [c["N_k"] for c in cases]


def select(cases, keep, key):
    return [c[key] if i in keep else None for i, c in enumerate(cases)]


def query(m, cases, keep, rp, unc=None):
    return m.get_fes(select(cases, keep, "queries"), reference_point=rp,
                     fes_reference=select(cases, keep, "fes_reference"), uncertainty_method=unc)


def generate(m, cases, keep, n_bootstraps=0, seed=None):
    m.generate_fes(select(cases, keep, "u_n"), select(cases, keep, "x_n"), fes_type="kde",
                   kde_parameters=select(cases, keep, "kde_parameters"), n_bootstraps=n_bootstraps, seed=seed)


def check_plain(c, out, tag, atol=1e-8):
    """b = 0's f_i against the reference, at the bound of the single-problem KDE golden checks."""
    want = c[f"f_i_{tag}"]
    np.testing.assert_array_equal(np.isinf(out["f_i"]), np.isinf(want), err_msg=c["name"])
    fin = np.isfinite(want)
    np.testing.assert_allclose(out["f_i"][fin], want[fin], rtol=0, atol=atol, err_msg=f"{c['name']} {tag}")
    assert out["df_i"] is None


def check_boot(c, out, run, tag, atol=1e-8, rtol_df=1e-6):
    want = c[f"{run}_f_i_{tag}"]
    fin = np.isfinite(want)
    np.testing.assert_allclose(out["f_i"][fin], want[fin], rtol=0, atol=atol, err_msg=f"{c['name']} {run} {tag}")
    wdf = c[f"{run}_df_i_{tag}"]
    fin = np.isfinite(wdf)
    np.testing.assert_array_equal(np.isfinite(out["df_i"]), fin, err_msg=c["name"])
    np.testing.assert_allclose(out["df_i"][fin], wdf[fin], rtol=rtol_df, atol=1e-10,
                               err_msg=f"{c['name']} {run} {tag} df")


class KdeOracleBatch(FB.FesBootOracleBatch):
    """FesBootOracleBatch with log_weights in numpy fp64.  `lw_flagged` names problem indices (in this batch) whose
    requests report the flag; calls are recorded in AugOracleBatch.calls as ("log_weights", problems)."""

    lw_flagged = ()

    def log_weights(self, problems, f_list, u_n_list):
        E.AugOracleBatch.calls.append(("log_weights", [int(p) for p in problems]))
        out, flags = [], []
        for p, f, u in zip(problems, f_list, u_n_list):
            N_k = np.asarray(self.N_k[p], np.float64)
            s = N_k > 0
            f = np.asarray(f, np.float64)
            out.append(-np.asarray(u, np.float64) - orc.log_denominator_n(self.u[p][s], N_k[s], f[s]))
            flags.append(p in self.lw_flagged)
        return out, np.array(flags, bool)


class KdeOracleProblem(FB.FesBootOracleProblem):
    """FesBootOracleProblem with log_denominator."""

    def log_denominator(self, f):
        N_k = np.asarray(self.N_k, np.float64)
        s = N_k > 0
        return orc.log_denominator_n(np.asarray(self.u)[s], N_k[s], np.asarray(f, np.float64)[s])


class NumpyKdeMany:
    """DeviceKdeMany in numpy fp64 (tests/_kde.log_sum); every log_sum call is recorded in `calls` as the list of its
    requests' sets, and `created` counts constructions and `closed` closes."""

    calls = []
    created = 0
    closed = 0

    def __init__(self, x_list, device=0):
        self.x = [np.asarray(x, np.float64).reshape(len(x), -1) for x in x_list]
        NumpyKdeMany.created += 1
        self._open = True

    def log_sum(self, sets, kernels, hs, w_list, y_list):
        assert self._open
        NumpyKdeMany.calls.append([int(s) for s in sets])
        return [_kde.log_sum_f64(k, h, self.x[s], w, np.asarray(y, np.float64).reshape(-1, self.x[s].shape[1]))
                for s, k, h, w, y in zip(sets, kernels, hs, w_list, y_list)]

    def last_stats(self):
        return dict(ms=0.0, launches=2, pairs=0)

    def close(self):
        if self._open:
            NumpyKdeMany.closed += 1
        self._open = False

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

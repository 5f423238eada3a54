"""Problems of the MbarMany estimator tests and numpy stand-ins of the batch with appended rows.

expectation_problems() are the inputs of tests/golden/mbar_many_expectations.npz
(tools/make_mbar_many_expectations_golden.py): problems of tests/_mbar_many.golden_problems() with K = 1, 2, 9, 33, 64
(3K = 192 rows for entropy and enthalpy) and 65 (the single path), the empty-first, empty-middle and unsampled-far
problems, and two harmonic ladders with K = 21 and 22 (3K = 63 and 66 rows, on both sides of one 64-row boundary).

requests(u_kn) gives the estimator inputs the golden file records for a problem: the last state's energies as the
observable (averages), the state-dependent energies as observables (differences), and the midpoints of neighbouring
rows as perturbed states.

AugOracleBatch adds `set_unsampled` and `augmented_moments` to tests/_mbar_many.OracleBatch, and AugOracleProblem the
augmented problem of the single path to OracleProblem, both in float64 numpy, so that the routing, waves and host
algebra of pymbar_b200.mbar_many.MbarMany run without a GPU.
"""
import numpy as np

from tests import _mbar_many as H

GOLDEN = "mbar_many_expectations.npz"
PICK = ("harmonic_K1", "harmonic_K2", "exponential_K9", "harmonic_K33", "harmonic_K64", "harmonic_K65",
        "empty_first", "empty_middle", "unsampled_far")


def expectation_problems():
    """[(name, (u_kn, N_k))] in the order of the golden file."""
    base = dict(H.golden_problems())
    out = [(n, base[n]) for n in PICK]
    out.insert(3, ("harmonic_K21", H.harmonic(21, 60, 21, spacing=0.6)))
    out.insert(4, ("harmonic_K22", H.harmonic(22, 60, 22, spacing=0.6)))
    return out


def requests(u_kn):
    """(A_n for averages [N], A_n for state-dependent differences [K, N], u_ln of the perturbed states [L, N])."""
    u = np.asarray(u_kn, np.float64)
    u_ln = 0.5 * (u[:-1] + u[1:]) if u.shape[0] > 1 else np.vstack([u[0], 0.5 * u[0]])
    return u[-1].copy(), u.copy(), u_ln


KEYS = {
    "avg": ("mu", "sigma"),
    "diff": ("mu", "sigma"),
    "pert": ("Delta_f", "dDelta_f"),
    "ent": ("Delta_f", "dDelta_f", "Delta_u", "dDelta_u", "Delta_s", "dDelta_s"),
    "ovl": ("scalar", "eigenvalues", "matrix"),
    "neff": ("N_eff",),
}


def load(path):
    """The problems with the reference's results: case["avg"]["mu"] and so on."""
    z = np.load(path)
    probs = expectation_problems()
    assert [str(n) for n in z["names"]] == [n for n, _ in probs]
    cases = []
    for i, (name, (u, N_k)) in enumerate(probs):
        c = dict(name=name, u_kn=u, N_k=N_k)
        for what, keys in KEYS.items():
            c[what] = {k: z[f"p{i}_{what}_{k}"] for k in keys if f"p{i}_{what}_{k}" in z}
        cases.append(c)
    return cases


def _close(a, b, rtol, atol, what):
    np.testing.assert_allclose(np.real(a), np.real(b), rtol=rtol, atol=atol, err_msg=what)


def check_case(c, avg, diff, pert, ent, ovl, neff):
    """The bounds of tests/test_expectations.py: mu rtol 1e-8 / atol 1e-9, sigma and dDelta rtol 1e-5 / atol 1e-8,
    Delta atol 1e-8."""
    n = c["name"]
    _close(avg["mu"], c["avg"]["mu"], 1e-8, 1e-9, n + " avg mu")
    _close(avg["sigma"], c["avg"]["sigma"], 1e-5, 1e-8, n + " avg sigma")
    _close(diff["mu"], c["diff"]["mu"], 1e-8, 1e-9, n + " diff mu")
    _close(diff["sigma"], c["diff"]["sigma"], 1e-5, 1e-8, n + " diff sigma")
    _close(pert["Delta_f"], c["pert"]["Delta_f"], 0, 1e-8, n + " pert Delta_f")
    _close(pert["dDelta_f"], c["pert"]["dDelta_f"], 1e-5, 1e-8, n + " pert dDelta_f")
    for k in ("Delta_f", "Delta_u", "Delta_s"):
        _close(ent[k], c["ent"][k], 0, 1e-8, n + " ent " + k)
        _close(ent["d" + k], c["ent"]["d" + k], 1e-5, 1e-8, n + " ent d" + k)
    if "scalar" in c["ovl"]:
        _close(ovl["matrix"], c["ovl"]["matrix"], 1e-6, 1e-9, n + " overlap")
        _close(ovl["scalar"], c["ovl"]["scalar"], 1e-6, 1e-9, n + " overlap scalar")
    _close(neff["N_eff"], c["neff"]["N_eff"], 1e-6, 1e-9, n + " N_eff")


def run_all(m, cases):
    reqs = [requests(c["u_kn"]) for c in cases]
    return (m.compute_expectations([r[0] for r in reqs]),
            m.compute_expectations([r[1] for r in reqs], output="differences", state_dependent=True),
            m.compute_perturbed_free_energies([r[2] for r in reqs]),
            m.compute_entropy_and_enthalpy(),
            m.compute_overlap(),
            m.compute_effective_sample_number())


class AugOracleBatch(H.OracleBatch):
    """OracleBatch with appended rows.  `aug_flagged` names problem indices (in this batch) whose augmented requests
    report the flag; `calls` records (entry point, problems) of every set_unsampled / augmented_moments call."""

    aug_flagged = ()
    calls = []

    def __init__(self, u_kn_list, N_k_list, device=0):
        super().__init__(u_kn_list, N_k_list, device)
        self.rows = {}

    def set_unsampled(self, problems, rows_list):
        AugOracleBatch.calls.append(("set_unsampled", list(problems)))
        self.rows = {int(p): np.asarray(r, np.float64) for p, r in zip(problems, rows_list)}

    def augmented_moments(self, f_list, want_G=False, problems=None):
        problems = range(len(f_list)) if problems is None else problems
        AugOracleBatch.calls.append(("augmented_moments", list(problems)))
        out = []
        for f, p in zip(f_list, problems):
            extra = self.rows[p]
            u = np.vstack([self.u[p], extra])
            N_k = np.concatenate([self.N_k[p], np.zeros(extra.shape[0])])
            with np.errstate(over="ignore", invalid="ignore"):
                S, logS, sL, G = H.ghat_np(u, N_k, np.asarray(f, np.float64), True)
            d = dict(S=S, log_S=logS, sum_L=sL, flag=p in self.aug_flagged)
            if want_G:
                d["G"] = G
            out.append(d)
        return out

    def last_stats(self):
        return dict(ms=0.0, launches=0, iterations=0, bytes_read=0)


class AugOracleProblem(H.OracleProblem):
    """OracleProblem with the augmented problem and the self-consistent update expectations_inner uses."""

    created = []

    def __init__(self, u_kn, N_k, device=0):
        super().__init__(u_kn, N_k, device)
        AugOracleProblem.created.append(self)

    def augmented(self, extra):
        return AugOracleProblem(np.vstack([self.u, extra]), np.concatenate([self.N_k, np.zeros(len(extra))]))

    def self_consistent_update(self, f):
        with np.errstate(over="ignore", invalid="ignore"):
            _, logS, _, _ = H.ghat_np(self.u, self.N_k, np.asarray(f, np.float64), True)
        return np.asarray(f, np.float64) - logS

    def weight_moments(self, f):
        with np.errstate(over="ignore", invalid="ignore"):
            return super().weight_moments(f)

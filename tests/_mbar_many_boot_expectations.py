"""Problems of the MbarMany bootstrap estimator tests and a numpy stand-in of the weighted batch with appended rows.

boot_problems() are the inputs of tests/golden/mbar_many_boot_expectations.npz
(tools/make_mbar_many_boot_expectations_golden.py): the problems of tests/_mbar_many_expectations.expectation_problems()
with K = 2, 9, 21, 22, 33, 64 and 65 (the single path), and the empty-first and empty-middle problems; problem i is
drawn with rseed = seed0 + i.

BootOracleBatch serves every entry point MbarMany's bootstrap estimators call (replicate slots, appended rows, and
augmented_moments with slots=) in float64 numpy: a slot with counts c evaluates its problem, appended rows included, as
the gathered array u[:, repeat(n, c_n)], which is what the reference evaluates for that replicate.  BootOracleProblem
adds replicate_unsampled to the single path's stand-in on the same gathered arrays.
"""
import numpy as np

from tests import _mbar_many as H
from tests import _mbar_many_boot as W
from tests import _mbar_many_expectations as E

GOLDEN = "mbar_many_boot_expectations.npz"
PICK = ("harmonic_K2", "exponential_K9", "harmonic_K21", "harmonic_K22", "harmonic_K33", "harmonic_K64",
        "harmonic_K65", "empty_first", "empty_middle")


def boot_problems():
    """[(name, (u_kn, N_k))] in the order of the golden file."""
    base = dict(E.expectation_problems())
    return [(n, base[n]) for n in PICK]


def load(path):
    """The problems with their seeds and the reference's bootstrap results: case["avg_sigma"] and so on."""
    z = np.load(path)
    probs = boot_problems()
    assert [str(n) for n in z["names"]] == [n for n, _ in probs]
    B, seed0 = int(z["n_bootstraps"]), int(z["seed0"])
    keys = ("avg_sigma", "diff_sigma", "pert_dDelta_f", "ent_dDelta_f", "ent_dDelta_u", "ent_dDelta_s",
            "inner_bootstrapped_observables", "inner_bootstrapped_f", "f_k_boots")
    return [dict(name=name, u_kn=u, N_k=N_k, seed=seed0 + i, B=B, **{k: z[f"p{i}_{k}"] for k in keys})
            for i, (name, (u, N_k)) in enumerate(probs)]


def run_boot(m, cases):
    """The four bootstrap requests the golden file records, on an MbarMany of `cases`."""
    reqs = [E.requests(c["u_kn"]) for c in cases]
    return (m.compute_expectations([r[0] for r in reqs], uncertainty_method="bootstrap"),
            m.compute_expectations([r[1] for r in reqs], output="differences", state_dependent=True,
                                   uncertainty_method="bootstrap"),
            m.compute_perturbed_free_energies([r[2] for r in reqs], uncertainty_method="bootstrap"),
            m.compute_entropy_and_enthalpy(uncertainty_method="bootstrap"))


def check_boot_case(c, avg, diff, pert, ent, atol=1e-8):
    """Every bootstrap key against the reference's within `atol`."""
    n = c["name"]

    def close(a, b, what):
        np.testing.assert_allclose(a, b, rtol=0, atol=atol, err_msg=n + " " + what)

    close(avg["bootstrapped_observables"], c["inner_bootstrapped_observables"], "bootstrapped_observables")
    close(avg["bootstrapped_f"], c["inner_bootstrapped_f"], "bootstrapped_f")
    close(avg["sigma"], c["avg_sigma"], "avg sigma")
    close(diff["sigma"], c["diff_sigma"], "diff sigma")
    close(pert["dDelta_f"], c["pert_dDelta_f"], "pert dDelta_f")
    for k in ("dDelta_f", "dDelta_u", "dDelta_s"):
        close(ent[k], c["ent_" + k], "ent " + k)


def max_errors(c, avg, diff, pert, ent):
    """{key: largest absolute difference from the reference} of one case."""
    pairs = dict(bootstrapped_observables=(avg["bootstrapped_observables"], c["inner_bootstrapped_observables"]),
                 bootstrapped_f=(avg["bootstrapped_f"], c["inner_bootstrapped_f"]),
                 avg_sigma=(avg["sigma"], c["avg_sigma"]), diff_sigma=(diff["sigma"], c["diff_sigma"]),
                 pert_dDelta_f=(pert["dDelta_f"], c["pert_dDelta_f"]),
                 **{"ent_" + k: (ent[k], c["ent_" + k]) for k in ("dDelta_f", "dDelta_u", "dDelta_s")})
    return {k: float(np.max(np.abs(np.asarray(a) - np.asarray(b)))) for k, (a, b) in pairs.items()}


class BootOracleBatch(E.AugOracleBatch, W.WeightedOracleBatch):
    """AugOracleBatch with replicate slots (WeightedOracleBatch) and weighted augmented requests.  `slot_flagged`
    names batch problem indices whose weighted augmented requests report the flag."""

    slot_flagged = ()

    def augmented_moments(self, f_list, want_G=False, problems=None, slots=None):
        if slots is None:
            return super().augmented_moments(f_list, want_G, problems)
        assert problems is None and not want_G
        BootOracleBatch.calls.append(("replicate_augmented_moments", [int(self.slot_problems[s]) for s in slots]))
        out = []
        for f, s in zip(f_list, slots):
            p = int(self.slot_problems[s])
            extra = self.rows[p]
            u = W.gathered(np.vstack([self.u[p], extra]), self.slot_counts[s])
            N_k = np.concatenate([self.N_k[p], np.zeros(extra.shape[0])])
            with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
                S, logS, sL, _ = H.ghat_np(u, N_k, np.asarray(f, np.float64), True)
            out.append(dict(S=S, log_S=logS, sum_L=sL, flag=p in self.slot_flagged))
        return out


class BootOracleProblem(E.AugOracleProblem):
    """AugOracleProblem with replicate_unsampled, as expectations_inner(..., replicates=) calls it."""

    replicate_calls = []

    def augmented(self, extra):
        return BootOracleProblem(np.vstack([self.u, extra]), np.concatenate([self.N_k, np.zeros(len(extra))]))

    def replicate_unsampled(self, counts, F):
        BootOracleProblem.replicate_calls.append(np.asarray(counts).copy())
        un = ~(self.N_k > 0)
        out = np.empty((len(counts), int(un.sum())))
        for b, c in enumerate(counts):
            f = np.asarray(F[b], np.float64)
            with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
                _, logS, _, _ = H.ghat_np(W.gathered(self.u, c), self.N_k, f, True)
            out[b] = (f - logS)[un]
        return out

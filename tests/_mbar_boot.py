"""Shared pieces of the MBAR bootstrap tests (test infrastructure): an MBAR-shaped stand-in whose constructor restates
the reference's bootstrap loop, the public estimators restated on top of compute_expectations_inner, a numpy
stand-in for a weighted DeviceProblem, and the checks of every quantity tests/golden/mbar_bootstrap.npz records."""
import os

import numpy as np
from scipy.special import logsumexp

from tests import _cases
from tests.test_driver_logic_cpu import OracleProblem, StandInMBAR

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mbar_bootstrap.npz")


def golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


class BootMBAR(StandInMBAR):
    """StandInMBAR with the reference constructor's random stream and bootstrap loop (mbar.py:264-275, :297,
    :417-451): x_kindices, the generator and its duplicate-state draw, then per replicate the draws state by state,
    an optional BAR start on the gathered columns and a solve of the gathered u_kn[:, rints]."""

    def __init__(self, u_kn, N_k, initialize="zeros", solver_protocol=None, x_kindices=None, n_bootstraps=0,
                 bootstrap_solver_protocol=None, rseed=None, verbose=False):
        ms = type(self).solvers
        self.u_kn = np.array(u_kn, dtype=np.float64)
        self.N_k = np.asarray(N_k, dtype=np.int64)
        self.K, self.N = self.u_kn.shape
        self.x_kindices = np.repeat(np.arange(self.K), self.N_k) if x_kindices is None else np.asarray(x_kindices)
        self.rng = np.random.default_rng(rseed)
        self.rng.choice(np.arange(self.N), min(50, self.N))
        self.samestates = []
        self.states_with_samples = np.where(self.N_k != 0)[0]
        f_k = self._initialize_with_bar(self.u_kn) if initialize == "BAR" else np.zeros(self.K)
        protocol = {None: ms.DEFAULT_SOLVER_PROTOCOL, "default": ms.DEFAULT_SOLVER_PROTOCOL,
                    "robust": ms.ROBUST_SOLVER_PROTOCOL}.get(solver_protocol, solver_protocol)
        protocol = tuple({k: (dict(v) if isinstance(v, dict) else v) for k, v in st.items()} for st in protocol)
        self.f_k = ms.solve_mbar_for_all_states(self.u_kn, self.N_k, f_k, self.states_with_samples, protocol)
        if n_bootstraps > 0:
            boot_protocol = tuple({k: (dict(v) if isinstance(v, dict) else v) for k, v in st.items()}
                                  for st in ms.BOOTSTRAP_SOLVER_PROTOCOL)
            self.n_bootstraps = n_bootstraps
            self.f_k_boots = np.zeros([n_bootstraps, self.K])
            self.bootstrap_rints = np.zeros([n_bootstraps, self.N], int)
            for b in range(n_bootstraps):
                f_k_init = np.array(self.f_k.copy())
                rints = np.zeros(self.N, int)
                for k in range(self.K):
                    k_indices = np.where(self.x_kindices == k)[0]
                    rints[k_indices] = k_indices[self.rng.integers(int(self.N_k[k]), size=int(self.N_k[k]))]
                if initialize == "BAR":
                    f_k_init = self._initialize_with_bar(self.u_kn[:, rints], f_k_init=self.f_k)
                self.f_k_boots[b, :] = ms.solve_mbar_for_all_states(self.u_kn[:, rints], self.N_k, f_k_init,
                                                                    self.states_with_samples, boot_protocol)
                self.bootstrap_rints[b, :] = rints
        self.Log_W_nk = ms.mbar_log_W_nk(self.u_kn, self.N_k, self.f_k)


# ---- the public estimators of mbar.py on top of compute_expectations_inner, "bootstrap" only ----------------------
def expectations(m, A_n, u_kn=None, output="averages", state_dependent=False):
    u = m.u_kn if u_kn is None else u_kn
    Ks = 1 if np.ndim(u) == 1 else np.shape(u)[0]
    state_map = np.zeros([2, Ks], int)
    state_map[0] = np.arange(Ks)
    state_map[1] = np.arange(Ks) if state_dependent else 0
    r = m.compute_expectations_inner(A_n, u, state_map, return_theta=True, uncertainty_method="bootstrap")
    A, Ab = r["observables"], r["bootstrapped_observables"]
    if output == "averages":
        return {"mu": A, "sigma": np.std(Ab, axis=0)}
    return {"mu": A - np.vstack(A), "sigma": np.std(np.array([a - np.vstack(a) for a in Ab]), axis=0)}


def multiple_expectations(m, A_in, u_n):
    state_map = np.zeros([2, len(A_in)], int)
    state_map[1] = np.arange(len(A_in))
    r = m.compute_expectations_inner(A_in, u_n, state_map, return_theta=True, uncertainty_method="bootstrap")
    Ab = r["bootstrapped_observables"]
    return {"mu": r["observables"], "sigma": np.std(Ab, axis=0), "covariances": np.cov(Ab.T)}


def perturbed(m, u_ln):
    r = m.compute_expectations_inner(np.array([0]), u_ln, np.arange(len(u_ln)), return_theta=True,
                                     uncertainty_method="bootstrap")
    f = r["f"]
    return {"Delta_f": f - np.vstack(f), "dDelta_f": np.std(r["bootstrapped_f"], axis=0)}


def entropy_and_enthalpy(m):
    K = m.u_kn.shape[0]
    state_map = np.array([np.arange(K), np.arange(K)])
    r = m.compute_expectations_inner(m.u_kn.copy(), m.u_kn, state_map, return_theta=True,
                                     uncertainty_method="bootstrap")
    f, u = r["f"], r["observables"]
    s = u - f
    out = {"Delta_f": f - np.vstack(f), "Delta_u": u - np.vstack(u), "Delta_s": s - np.vstack(s)}

    def spread(rows):
        return np.std(np.array([x - np.vstack(x) for x in rows]), axis=0)

    out["dDelta_f"] = spread(m.f_k_boots)
    out["dDelta_u"] = spread(r["bootstrapped_observables"])
    out["dDelta_s"] = spread(r["bootstrapped_observables"] - m.f_k_boots)
    return out


def check_case(m, g, name, seed, rtol_obs=1e-8, rtol_sigma=1e-6, atol_sigma=1e-9, tol_f=1e-8):
    """Every golden quantity of (name, seed) from the MBAR `m` (built with n_bootstraps=NB, rseed=seed)."""
    z = _cases.load(name)
    p = f"{name}_s{seed}_"
    x, u = z["x_n"], z["u_kn"]
    K = len(z["N_k"])
    np.testing.assert_allclose(m.f_k_boots, g[p + "f_k_boots"], rtol=0, atol=tol_f)

    def close(a, b):
        np.testing.assert_allclose(a, b, rtol=rtol_sigma, atol=atol_sigma)

    close(m.compute_free_energy_differences(uncertainty_method="bootstrap")["dDelta_f"], g[p + "fed_dDelta_f"])
    r = m.compute_free_energy_differences(uncertainty_method="bootstrap", return_theta=True)
    close(r["dDelta_f"], g[p + "fed_theta_dDelta_f"])
    np.testing.assert_allclose(r["Theta"], g[p + "fed_Theta"], rtol=1e-5, atol=1e-9)
    for tag, kw in (("avg", {}), ("diff", {"output": "differences"})):
        r = expectations(m, x.copy(), **kw)
        np.testing.assert_allclose(r["mu"], g[p + tag + "_mu"], rtol=rtol_obs, atol=1e-10)
        close(r["sigma"], g[p + tag + "_sigma"])
    r = expectations(m, u.copy(), state_dependent=True)
    np.testing.assert_allclose(r["mu"], g[p + "sd_mu"], rtol=rtol_obs, atol=1e-10)
    close(r["sigma"], g[p + "sd_sigma"])
    r = multiple_expectations(m, np.array([x, x ** 2]), u[0].copy())
    np.testing.assert_allclose(r["mu"], g[p + "mult_mu"], rtol=rtol_obs, atol=1e-10)
    close(r["sigma"], g[p + "mult_sigma"])
    close(r["covariances"], g[p + "mult_cov"])
    r = perturbed(m, z["pert_u_ln"].copy())
    np.testing.assert_allclose(r["Delta_f"], g[p + "pert_Delta_f"], atol=1e-8)
    close(r["dDelta_f"], g[p + "pert_dDelta_f"])
    r = entropy_and_enthalpy(m)
    for key in ("Delta_f", "Delta_u", "Delta_s"):
        np.testing.assert_allclose(r[key], g[p + "ee_" + key], atol=1e-8)
    for key in ("dDelta_f", "dDelta_u", "dDelta_s"):
        close(r[key], g[p + "ee_" + key])
    state_map = np.array([np.arange(K), np.zeros(K, int)])
    r = m.compute_expectations_inner(x.copy()[None], u.copy(), state_map, uncertainty_method="bootstrap")
    np.testing.assert_allclose(r["bootstrapped_observables"], g[p + "inner_obs"], rtol=rtol_obs, atol=1e-10)
    np.testing.assert_allclose(r["bootstrapped_f"], g[p + "inner_f"], rtol=rtol_obs, atol=1e-10)


# ---- a weighted DeviceProblem in numpy ----------------------------------------------------------------------------
def replicate_unsampled(u_kn, N_k, counts, F):
    """mbar_b200_replicate_unsampled restated: [B, n_u] of -log sum_n c_bn exp(-u_jn - L_bn)."""
    u = np.asarray(u_kn, dtype=np.float64)
    N_k = np.asarray(N_k, dtype=np.float64)
    s = N_k > 0
    out = np.empty((len(counts), int(np.sum(~s))))
    for b, (c, f) in enumerate(zip(np.asarray(counts, dtype=np.float64), np.asarray(F))):
        L = logsumexp(f[s, None] + np.log(N_k[s, None]) - u[s], axis=0)
        with np.errstate(divide="ignore"):
            out[b] = -logsumexp(-u[~s] - L + np.log(c), axis=1)
    return out


class WeightedOracleProblem(OracleProblem):
    """OracleProblem with integer multiplicities (set_sample_weights, the gathered columns of each replicate) and
    replicate_unsampled.  `fail_on` names the weighted uploads (1-based) that raise MbarB200Error instead."""

    fail_on = ()
    uploads = 0
    replicate_calls = 0

    def __init__(self, u_kn, N_k, device=0, N_local=None):
        super().__init__(u_kn, N_k, device, N_local)
        self.base = self.u

    def set_sample_weights(self, w):
        from pymbar_b200._lib import MbarB200Error

        if w is None:
            self.u = self.base
            self.K, self.N = self.u.shape
            return
        cls = WeightedOracleProblem
        cls.uploads += 1
        if cls.uploads in cls.fail_on:
            raise MbarB200Error(-2, "injected device failure")
        self.u = np.repeat(self.base, np.asarray(w).astype(np.int64), axis=1)

    def augmented(self, u_extra):
        u_extra = np.atleast_2d(np.asarray(u_extra, float))
        return WeightedOracleProblem(np.vstack([self.base, u_extra]),
                                     np.concatenate([self.N_k, np.zeros(len(u_extra))]))

    def replicate_unsampled(self, counts, F):
        c = np.asarray(counts)
        if c.size and c.max() > 65535:
            raise ValueError("replicate counts must lie in [0, 65535]")
        WeightedOracleProblem.replicate_calls += 1
        return replicate_unsampled(self.base, self.N_k, c, F)

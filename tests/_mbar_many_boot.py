"""A weighted numpy stand-in of DeviceMbarBatch for the mbar_many bootstrap tests, and the bootstrap fixture.

WeightedOracleBatch adds replicate slots to tests/_mbar_many.OracleBatch: a slot with counts c evaluates its problem
as the gathered array u[:, repeat(n, c_n)], which is what the reference solves for that replicate.  It records every
set_replicates call, and `flagged_counts` names (batch problem, counts bytes) pairs whose solve reports status 2.
oracle_bootstrap_f_k stands in for bootstrap.bootstrap_f_k on the same gathered arrays.
"""
import numpy as np

from oracle import mbar_oracle as orc
from tests import _mbar_many as H

GOLDEN = "mbar_many_bootstrap.npz"


def gathered(u, c):
    return u[:, np.repeat(np.arange(u.shape[1]), np.asarray(c, np.int64))]


class WeightedOracleBatch(H.OracleBatch):
    flagged_counts = set()
    uploads = []          # [(problems, counts)] of every set_replicates call

    def __init__(self, u_kn_list, N_k_list, device=0):
        super().__init__(u_kn_list, N_k_list, device)
        self.slot_problems = np.zeros(0, np.int32)
        self.slot_counts = []

    def set_replicates(self, problems, counts):
        self.slot_problems = np.asarray(problems, np.int32)
        self.slot_counts = [np.asarray(c, np.uint16) for c in counts]
        for p, c in zip(self.slot_problems, self.slot_counts):
            assert int(c.astype(np.int64).sum()) == self.u[p].shape[1]
        WeightedOracleBatch.uploads.append((self.slot_problems.copy(), [c.copy() for c in self.slot_counts]))

    def moments(self, f_list, want_G=False, all_rows=False, problems=None, slots=None):
        if slots is None:
            return super().moments(f_list, want_G, all_rows, problems)
        out = []
        for f, s in zip(f_list, slots):
            p = self.slot_problems[s]
            S, logS, sL, G = H.ghat_np(gathered(self.u[p], self.slot_counts[s]), self.N_k[p],
                                       np.asarray(f, np.float64), all_rows)
            d = dict(S=S, log_S=logS, sum_L=sL, flag=False)
            if want_G:
                d["G"] = G
            out.append(d)
        return out

    def solve_replicates(self, f_list, tol=1e-12, maxiter=10000, min_sc_iter=0, gamma=1.0):
        S = len(self.slot_problems)
        fs, status, iters = [], np.zeros(S, np.int32), np.zeros(S, np.int32)
        for s in range(S):
            p = self.slot_problems[s]
            f0 = np.array(f_list[s], np.float64)
            if (int(p), self.slot_counts[s].tobytes()) in self.flagged_counts:
                status[s] = 2
                fs.append(f0)
                continue
            sw = self.N_k[p] > 0
            if sw.sum() < 2:
                f0[sw] = 0.0
                fs.append(f0)
                continue
            u = gathered(self.u[p], self.slot_counts[s])
            f, _ = orc.solve_mbar_once(u[sw], self.N_k[p][sw], f0[sw] - f0[sw][0], method="adaptive", tol=tol,
                                       options=dict(min_sc_iter=min_sc_iter, gamma=gamma, maxiter=maxiter))
            out = f0.copy()
            out[sw] = f - f[0]
            fs.append(out)
            iters[s] = 1
        return fs, status, iters


class WeightedOracleProblem(H.OracleProblem):
    """DeviceProblem stand-in that the single replicate path opens (its u_kn and N_k only)."""

    opened = []

    def __init__(self, u_kn, N_k, device=0):
        super().__init__(u_kn, N_k, device)
        WeightedOracleProblem.opened.append(self)


def oracle_bootstrap_f_k(problem, f_k, N_k, rints=None, n_bootstraps=0, rseed=None, x_kindices=None,
                         solver_protocol=None):
    """bootstrap.bootstrap_f_k on the numpy oracle: each replicate solved on u[:, rints] from f_k."""
    N_k = np.asarray(N_k, np.int64)
    sw = np.flatnonzero(N_k > 0)
    out = np.zeros((len(rints), len(N_k)))
    for b, r in enumerate(rints):
        out[b] = orc.solve_mbar_for_all_states(problem.u[:, r], N_k.astype(float), np.array(f_k, np.float64), sw,
                                               solver_protocol)
    return out


def load(path):
    """The golden problems with the reference's bootstrap results: f_k_boots [B, K], dDelta_f, seed and B."""
    z = np.load(path)
    probs = H.golden_problems()
    assert [str(n) for n in z["names"]] == [n for n, _ in probs]
    B, seed0 = int(z["n_bootstraps"]), int(z["seed0"])
    return [dict(name=name, u_kn=u, N_k=N_k, f_init=H.golden_f_init(name, len(N_k)), seed=seed0 + i, B=B,
                 f_k_boots=z[f"p{i}_f_k_boots"], dDelta_f=z[f"p{i}_dDelta_f"])
            for i, (name, (u, N_k)) in enumerate(probs)]

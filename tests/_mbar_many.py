"""Problems of the mbar_many tests and a numpy stand-in of DeviceMbarBatch.

golden_problems() are the inputs of tests/golden/mbar_many.npz (tools/make_mbar_many_golden.py): harmonic and
exponential ladders with K = 1, 2, 5, 8, 9, 16, 33, 64 and 65, an empty first state, an empty middle state, an
unsampled state far from every sample and a problem whose free energies span more than 700 kT.  Each has N <= 2000.

OracleBatch serves `moments` and `solve` from the float64 numpy oracle (oracle/mbar_oracle.py), with the contract of
DeviceMbarBatch, so the routing and post-processing of pymbar_b200.mbar_many run without a GPU.
"""
import numpy as np

from oracle import mbar_oracle as orc

GOLDEN = "mbar_many.npz"


def harmonic(K, n_per, seed, spacing=1.0, unsampled=(), offsets=None, centres=None):
    """u_kn [K, N], N_k of harmonic states of unit spring constant with centres `spacing` apart (or at `centres`)."""
    rng = np.random.RandomState(seed)
    centres = spacing * np.arange(K, dtype=np.float64) if centres is None else np.asarray(centres, np.float64)
    N_k = np.full(K, n_per, np.int64)
    N_k[list(unsampled)] = 0
    owner = np.repeat(np.arange(K), N_k)
    x = centres[owner] + rng.normal(size=owner.size)
    u = 0.5 * (x[None, :] - centres[:, None]) ** 2
    if offsets is not None:
        u = u + np.asarray(offsets, np.float64)[:, None]
    return u, N_k.astype(np.float64)


def exponential(K, n_per, seed):
    """u_kn [K, N], N_k of exponential distributions with rates 1 .. 2 (x >= 0, u_k = rate_k x)."""
    rng = np.random.RandomState(seed)
    rates = np.linspace(1.0, 2.0, K)
    N_k = np.full(K, n_per, np.int64)
    owner = np.repeat(np.arange(K), N_k)
    x = rng.exponential(1.0 / rates[owner])
    return rates[:, None] * x[None, :], N_k.astype(np.float64)


def golden_problems():
    """[(name, (u_kn, N_k))] in the order of the golden file."""
    out = [
        ("harmonic_K1", harmonic(1, 300, 1)),
        ("harmonic_K2", harmonic(2, 400, 2)),
        ("exponential_K5", exponential(5, 200, 5)),
        ("harmonic_K8", harmonic(8, 150, 8, spacing=0.8)),
        ("exponential_K9", exponential(9, 120, 9)),
        ("harmonic_K16", harmonic(16, 100, 16, spacing=0.7)),
        ("harmonic_K33", harmonic(33, 50, 33, spacing=0.5)),
        ("harmonic_K64", harmonic(64, 30, 64, spacing=0.4)),
        ("harmonic_K65", harmonic(65, 30, 65, spacing=0.4)),
        ("empty_first", harmonic(6, 200, 61, unsampled=(0,))),
        ("empty_middle", harmonic(7, 200, 71, unsampled=(3,))),
    ]
    # state 5 is centred 45 standard deviations from the nearest sample's state: its weights are about e^-900
    out.append(("unsampled_far", harmonic(6, 200, 81, unsampled=(5,), centres=[0, 1, 2, 3, 4, 49.0])))
    # f spans 750 kT; the solve starts from f_init = the offsets (from zeros the reference's protocol fails here)
    out.append(("span_750kT", harmonic(16, 100, 91, spacing=0.5, offsets=50.0 * np.arange(16))))
    return out


def golden_f_init(name, K):
    """Starting free energies of a golden problem: zeros, except the offsets for span_750kT."""
    return 50.0 * np.arange(K) if name == "span_750kT" else np.zeros(K)


def load(path):
    """The golden problems with their inputs (u_kn, N_k, f_init) and the reference's results."""
    z = np.load(path)
    probs = golden_problems()
    assert [str(n) for n in z["names"]] == [n for n, _ in probs]
    cases = []
    for i, (name, (u, N_k)) in enumerate(probs):
        p = f"p{i}_"
        cases.append(dict(name=name, u_kn=u, N_k=N_k, f_init=golden_f_init(name, len(N_k)),
                          **{k: z[p + k] for k in ("f_k", "Delta_f", "dDelta_f", "Theta")}))
    return cases


def ghat_np(u, N_k, f, all_rows):
    """(S, log S, sum L, Ghat) of one problem in float64 numpy: Ghat's rows scaled by N_k (sampled) and by 1
    (unsampled, all_rows) or 0."""
    s = N_k > 0
    c = f[s] + np.log(N_k[s])
    a = c[:, None] - u[s]
    m = a.max(axis=0)
    L = m + np.log(np.exp(a - m).sum(axis=0))
    logW = f[:, None] - u - L[None, :]
    top = logW.max(axis=1, keepdims=True)
    with np.errstate(invalid="ignore"):
        logS = (top + np.log(np.exp(logW - top).sum(axis=1, keepdims=True)))[:, 0]
    logS[~np.isfinite(top[:, 0])] = -np.inf
    scale = np.where(s, N_k, 1.0 if all_rows else 0.0)
    w = np.exp(logW) * scale[:, None]
    return np.exp(logS), logS, float(L.sum()), w @ w.T


class OracleBatch:
    """Numpy stand-in of pymbar_b200.DeviceMbarBatch.  `flagged` names problem indices (in this batch) whose every
    moments request reports the range flag; solve reports status 2 for them."""

    flagged = ()
    created = []

    def __init__(self, u_kn_list, N_k_list, device=0):
        self.u = [np.asarray(u, np.float64) for u in u_kn_list]
        self.N_k = [np.asarray(n, np.float64) for n in N_k_list]
        self.P = len(self.u)
        self.K = np.array([u.shape[0] for u in self.u])
        OracleBatch.created.append(self)

    def close(self):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        pass

    def moments(self, f_list, want_G=False, all_rows=False, problems=None):
        problems = range(len(f_list)) if problems is None else problems
        out = []
        for f, p in zip(f_list, problems):
            S, logS, sL, G = ghat_np(self.u[p], self.N_k[p], np.asarray(f, np.float64), all_rows)
            d = dict(S=S, log_S=logS, sum_L=sL, flag=p in self.flagged)
            if want_G:
                d["G"] = G
            out.append(d)
        return out

    def solve(self, f_list=None, tol=1e-12, maxiter=10000, min_sc_iter=0, gamma=1.0):
        fs, status, iters = [], np.zeros(self.P, np.int32), np.zeros(self.P, np.int32)
        for p in range(self.P):
            f0 = np.zeros(self.K[p]) if f_list is None else np.array(f_list[p], np.float64)
            s = self.N_k[p] > 0
            if p in self.flagged:
                status[p] = 2
                fs.append(f0)
                continue
            if s.sum() < 2:
                f0[s] = 0.0
                fs.append(f0)
                continue
            f, r = orc.solve_mbar_once(self.u[p][s], self.N_k[p][s], f0[s] - f0[s][0], method="adaptive", tol=tol,
                                       options=dict(min_sc_iter=min_sc_iter, gamma=gamma, maxiter=maxiter))
            out = f0.copy()
            out[s] = f - f[0]
            fs.append(out)
            iters[p] = 1
        return fs, status, iters


def oracle_all_states(u_kn, N_k, f_k, states_with_samples, solver_protocol):
    """Stand-in of mbar_solvers.solve_mbar_for_all_states on the numpy oracle."""
    return orc.solve_mbar_for_all_states(u_kn, N_k, f_k, states_with_samples, solver_protocol)


class OracleProblem:
    """Stand-in of DeviceProblem for the single-problem path: weight_moments only."""

    def __init__(self, u_kn, N_k, device=0):
        self.u, self.N_k = np.asarray(u_kn, np.float64), np.asarray(N_k, np.float64)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        pass

    def weight_moments(self, f):
        S, _, _, Ghat = ghat_np(self.u, self.N_k, np.asarray(f, np.float64), True)
        s = np.where(self.N_k > 0, self.N_k, 1.0)
        return S, Ghat / np.outer(s, s)


def random_problem(rng, K, N, empty=0):
    """A random harmonic problem with K states, about N samples and `empty` unsampled states.  Spring constants differ
    between states, so the free energies are O(1) apart: with every f_k near 0, the adaptive solver's relative-change
    test at tol = 1e-12 falls below the rounding noise of any pass and convergence becomes a matter of luck."""
    centres = np.sort(rng.uniform(0, 0.6 * K, size=K))
    spring = rng.uniform(0.5, 2.0, size=K)
    N_k = np.zeros(K, np.int64)
    sampled = np.sort(rng.choice(K, size=max(K - empty, 1), replace=False))
    counts = rng.multinomial(max(N - len(sampled), 0), np.ones(len(sampled)) / len(sampled)) + 1
    N_k[sampled] = counts
    owner = np.repeat(np.arange(K), N_k)
    x = centres[owner] + rng.normal(size=owner.size) / np.sqrt(spring[owner])
    u = 0.5 * spring[:, None] * (x[None, :] - centres[:, None]) ** 2
    return u, N_k.astype(np.float64)


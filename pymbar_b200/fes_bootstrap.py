"""Bootstrap replicates of pymbar's FES (fes.py:388-430) for fes_type="histogram", "kde" and "spline", from the
resident problem.

The reference resamples every state's block of samples and, inside the loop over states, builds a full MBAR on the
gathered u_kn[:, idx] for each block (fes.py:395-406): K solves, K gathers of 8 K N bytes and K draws of the MBAR
constructor's seed (mbar.py:273-274) per replicate, of which only the last solve is used.  Here:

* the resampling stream is drawn from numpy's global generator exactly as the reference draws it (the blocks by
  position, and one randint(2^31 - 1) after each block for the constructor), so that `seed=` reproduces the same
  replicates and the generator ends where the reference leaves it.  The generator's state before each replicate's
  draws is kept instead of its N indices, and replicate_indices regenerates them on demand;
* a histogram replicate is one weighted solve on the resident problem (bootstrap.bootstrap_f_k with the
  multiplicities c_n = #{i : idx[i] = n}, the solve of the last MBAR of the loop: same data, same start), then the
  bin free energies f_i = -log sum_{n in i} c_n exp(-u_n - L_n) from the device's bin kernel with the same
  multiplicities.  bin_n, sample_label and nonzero_bins are built from the regenerated indices on first read;
* a KDE replicate needs no solve: the reference fits replicate b to x_n[idx_b] with the weights of b = 0 by position
  (fes.py:696), so its weight on sample n is V_bn = sum of w_m over the positions m with idx_b[m] = n, and
  DeviceKde.log_sum_replicates scores every replicate in one device call.  FES.kdes becomes a ReplicateKdes whose
  item b is fitted as the reference fits it when something reads it;
* a spline replicate's fit needs only its sample terms v_b (fes.spline_sample_terms): with samples in block order and
  c_bn = #{m : idx_b[m] = n}, v_b[i] = sum_n V_bn B_i(x_n) with V_bn = c_bn ("biasedstates"), c_bn N / (K N_{s_n})
  ("simplesum") or N c_bn e^{-u_n - L^{(b)}_n} / Z_b ("unbiasedstate", where L^{(b)} comes from one weighted solve
  and Z_b normalises as fes.py:412-414 does).  spline_replicates draws the stream and builds V; one
  DeviceBSpline.replicate_sums call then gives every v_b.
"""
from __future__ import annotations

from collections.abc import Mapping, Sequence

import numpy as np

from . import fes as hist

_SEED_BOUND = np.iinfo(np.int32).max


def _draw(rng, N_k):
    N = int(np.sum(N_k))
    idx = np.empty(N, dtype=np.int64)
    index = 0
    for n in N_k:
        n = int(n)
        idx[index:index + n] = index + rng.randint(0, n, size=n)
        index += n
        rng.randint(_SEED_BOUND)            # MBAR.__init__ draws its seed after every block (mbar.py:273-274)
    return idx


def draw_replicates(N_k, n_bootstraps, each=None):
    """Advance numpy's global generator as the reference's bootstrap loop does for n_bootstraps replicates and
    return the generator state before each replicate's draws; each(b, idx), when given, sees every replicate's
    indices as they are drawn.  Every N_k[k] must be >= 1 (randint(0, 0) raises in the reference)."""
    rng = np.random.mtrand._rand
    states = []
    for b in range(int(n_bootstraps)):
        states.append(rng.get_state())
        idx = _draw(rng, N_k)
        if each is not None:
            each(b, idx)
    return states


def replicate_indices(state, N_k):
    """The reference's bootstrap_indices [N] of the replicate drawn from `state`, on a private generator."""
    rng = np.random.RandomState()
    rng.set_state(state)
    return _draw(rng, N_k)


def tuple_index(bin_n):
    """(index of each sample's bin tuple [N], number of distinct tuples)."""
    tuples, inv = np.unique(bin_n, axis=0, return_inverse=True)
    return np.asarray(inv).ravel(), len(tuples)


def covers_every_tuple(idx, tuples, n_tuples):
    """True when the replicate keeps at least one sample in every bin tuple b = 0 occupies.  Otherwise the
    reference's f of the replicate is shorter than b = 0's (fes.py:579-592): IndexError there, or a shape error in
    get_fes."""
    return bool(np.all(np.bincount(tuples[idx], minlength=n_tuples) > 0))


class ReplicateHistogram(Mapping):
    """histogram_datas[b] with the reference's keys (fes.py:509-595): "dims", "bins" and "f" are held; "bin_n",
    "sample_label" and "nonzero_bins" are built from the regenerated indices and b = 0's labels on first read."""

    KEYS = ("dims", "bins", "bin_n", "nonzero_bins", "sample_label", "f")

    def __init__(self, f, base, state, N_k):
        self._d = {"dims": base["dims"], "bins": base["bins"], "f": f}
        self._source = (base, state, N_k)

    def __getitem__(self, key):
        if key not in self._d and key in self.KEYS:
            base, state, N_k = self._source
            idx = replicate_indices(state, N_k)
            bin_n = base["bin_n"][idx]
            self._d["bin_n"] = bin_n
            self._d["sample_label"] = base["sample_label"][idx]
            self._d["nonzero_bins"] = [tuple(int(v) for v in bin_n[n]) for n in hist._first_rows(bin_n)]
        return self._d[key]

    def __iter__(self):
        return iter(self.KEYS)

    def __len__(self):
        return len(self.KEYS)


def solver_protocol(default_protocol, maximum_iterations=10000):
    """`default_protocol` as MBAR.__init__ normalises it (mbar.py:391-406) for MBAR(u_kn, N_k, initial_f_k=...)."""
    out = []
    for st in default_protocol:
        st = {k: (dict(v) if isinstance(v, dict) else v) for k, v in st.items()}
        st.setdefault("options", {})
        st.setdefault("continuation", None)
        opts = st["options"]
        opts["maxiter"] = max(opts.get("maxiter", maximum_iterations), maximum_iterations)
        opts.setdefault("verbose", False)
        out.append(st)
    return tuple(out)


def histogram_replicates(problem, f_k, N_k, u_n, base, states, protocol, on_solve=None):
    """histogram_datas of fes.py:388-430 for the replicates drawn from `states`, on the resident `problem`
    (a DeviceProblem holding (u_kn, N_k)); base is b = 0's histogram_data.  Every replicate must cover every bin
    tuple of b = 0 (covers_every_tuple)."""
    from .bootstrap import bootstrap_f_k

    N = int(np.sum(N_k))
    dense = hist.dense_bins(base["sample_label"], base["bin_order"])
    nb = len(base["bin_order"])
    u = np.asarray(u_n, dtype=np.float64)
    out = []
    for state in states:
        idx = replicate_indices(state, N_k)
        f_b = bootstrap_f_k(problem, f_k, N_k, rints=idx[None], solver_protocol=protocol)[0]
        try:
            problem.set_sample_weights(np.bincount(idx, minlength=N).astype(np.float64))
            f_bin, _, _ = problem.bin_moments(f_b, u, dense, nb, want_C=False)
        finally:
            problem.set_sample_weights(None)
        f = np.zeros(len(base["f"]))
        f[:nb] = f_bin
        out.append(ReplicateHistogram(f, base, state, N_k))
        if on_solve is not None:
            on_solve()
    return out


def bootstrap_df(histogram_datas, j, n_out):
    """np.std over the replicates of f_b - f_b[j] (fes.py:1417-1422)."""
    fall = np.zeros([n_out, len(histogram_datas)])
    for b, h in enumerate(histogram_datas):
        fall[:, b] = h["f"] - h["f"][j]
    return np.std(fall, axis=1)


class ReplicateKdes(Sequence):
    """FES.kdes of a bootstrap KDE surface: item b is the reference's KernelDensity of replicate b (a new
    KernelDensity with b = 0's parameters fitted to x_n[idx_b] with sample_weight=w_n, fes.py:689-699), fitted the
    first time it is read."""

    def __init__(self, params, x_n, w_n, N_k, states, on_fit=None):
        self._params, self._x, self._w, self._N_k, self._states = dict(params), x_n, w_n, N_k, states
        self._fitted = [None] * len(states)
        self._on_fit = on_fit

    def __len__(self):
        return len(self._states)


    def __getitem__(self, b):
        if isinstance(b, slice):
            return [self[i] for i in range(*b.indices(len(self)))]
        b = range(len(self))[b]
        if self._fitted[b] is None:
            from sklearn.neighbors import KernelDensity

            x = self._x[replicate_indices(self._states[b], self._N_k)]
            if np.ndim(x) == 1:
                x = x.reshape(-1, 1)
            kde = KernelDensity()
            kde.set_params(**self._params)
            kde.fit(x, sample_weight=self._w)
            self._fitted[b] = kde
            if self._on_fit is not None:
                self._on_fit()
        return self._fitted[b]


def in_block_order(x_kindices, N_k):
    """True when the samples are in block order (state k's N_k[k] samples after those of states < k)."""
    N_k = np.asarray(N_k, dtype=np.int64)
    return np.array_equal(np.asarray(x_kindices), np.repeat(np.arange(len(N_k)), N_k))


def replicate_weights(c, log_w):
    """V_n = c_n e^{log_w_n} / sum_m c_m e^{log_w_m}: the reference's normalised replicate weights w_nb (fes.py:410-414)
    summed over the positions that repeat sample n.  Samples the replicate does not draw get 0."""
    V = np.zeros(len(c))
    sel = c > 0
    e = c[sel] * np.exp(log_w[sel] - np.max(log_w[sel]))
    V[sel] = e / np.sum(e)
    return V


def spline_replicates(N_k, n_bootstraps, spline_weights, replicate_log_weights=None):
    """(states, V [B, N]): the generator states of n_bootstraps replicates drawn as the reference draws them
    (draw_replicates) and the weight of every resident sample in each replicate's spline sample terms, with samples in
    block order.  V_b is c_b ("biasedstates"), c_b N / (K N_{s_n}) ("simplesum"), or replicate_weights(c_b,
    replicate_log_weights(idx_b)) ("unbiasedstate"; the callable returns -u_n - L^{(b)}_n of the replicate's solve,
    and the caller multiplies the sums by N).  Every N_k[k] must be >= 1."""
    N_k = np.asarray(N_k, dtype=np.int64)
    K, N = len(N_k), int(np.sum(N_k))
    V = np.empty((int(n_bootstraps), N))
    scale = np.repeat(N / (K * N_k.astype(np.float64)), N_k) if spline_weights == "simplesum" else None

    def each(b, idx):
        c = np.bincount(idx, minlength=N).astype(np.float64)
        if spline_weights == "unbiasedstate":
            V[b] = replicate_weights(c, replicate_log_weights(idx))
        elif spline_weights == "simplesum":
            V[b] = c * scale
        elif spline_weights == "biasedstates":
            V[b] = c
        else:
            raise ValueError(f"spline_weights {spline_weights!r} is not one of {hist.SPLINE_WEIGHTS}")

    return draw_replicates(N_k, n_bootstraps, each), V


def spline_replicate_samples(state, N_k, x_n, V_b, spline_weights):
    """(x_nb, w_nb): the samples and weights the reference passes to _generate_fes_spline for the replicate drawn from
    `state` (fes.py:406-430).  w_nb is rebuilt from V_b for "unbiasedstate"; the other weightings never read it and
    get None, as no solve is run for them."""
    idx = replicate_indices(state, N_k)
    if spline_weights != "unbiasedstate":
        return x_n[idx], None
    c = np.bincount(idx, minlength=len(V_b)).astype(np.float64)
    return x_n[idx], V_b[idx] / c[idx]


def kde_bootstrap_query(kde, settings, x, reference_point, fes_reference, log_sum_w):
    """_get_fes_kde with uncertainty_method="bootstrap" (fes.py:1523-1609) for "from-lowest" and "from-specified":
    f_i from kde_query and df_i = std over the replicates of -score_b(x) - fmin, every replicate scored by one
    DeviceKde.log_sum_replicates call (the replicates share b = 0's weight sum, as sklearn normalises them)."""
    out, fmin = hist.kde_query(kde, settings, x, reference_point, fes_reference, log_sum_w, with_fmin=True)
    kernel, h, D = settings["kernel"], settings["h"], settings["D"]
    y = np.asarray(x, dtype=np.float64).reshape(-1, D)
    return kde_bootstrap_finish(settings, out, fmin, kde.log_sum_replicates(kernel, h, y), log_sum_w)


def kde_bootstrap_finish(settings, out, fmin, log_sums, log_sum_w):
    """kde_bootstrap_query's df_i from the replicates' log sums [B, Q] at the queries (fes.py:1590-1601); out and fmin
    are kde_query's (with_fmin=True).  Returns out with df_i set."""
    score = np.array(log_sums, dtype=np.float64)
    score += hist.kde_log_norm(settings["kernel"], settings["D"], settings["h"])
    score -= log_sum_w
    fall = -score.T - fmin
    out["df_i"] = np.std(fall, axis=1)
    return out

"""The seeded series and cases of tests/golden/timeseries_many.npz (tools/make_timeseries_many_golden.py), and a numpy
stand-in for the segmented `DeviceAcf.inefficiency_series`."""
import hashlib

import numpy as np

from tests import _timeseries as tsr

# (fast, nskip) for detect_equilibration_many, (B, fast, mintime) for statistical_inefficiency_many ("cross": B is
# the list of partner series), (conservative, g) for subsample_correlated_data_many (g None: computed)
EQ_CASES = [(True, 1), (False, 1), (True, 3), (False, 3)]
SI_CASES = [(b, fast, mintime) for b in ("auto", "cross") for fast in (False, True) for mintime in (0, 3, 20)]
SUB_CASES = [(False, None), (True, None), (False, 3.7), (True, 3.7), (False, "per-series")]
LONG = 20000                   # the one long series: the numpy stand-in skips it in detect_equilibration
SHORT = {1: 520, 3: 800}       # detect_equilibration on the CPU stand-in: series up to this length per nskip


def ar1(rng, T, tau):
    a = np.exp(-1.0 / tau)
    x = np.empty(T)
    x[0] = rng.standard_normal()
    e = rng.standard_normal(T) * np.sqrt(1 - a * a)
    for n in range(1, T):
        x[n] = a * x[n - 1] + e[n]
    return x


def series():
    """(names, A list, B list): about 30 seeded series of mixed lengths and kinds."""
    rng = np.random.RandomState(20261018)
    s = []
    for T in (2, 3, 511, 512, 513, 1025):
        s.append((f"ar_{T}", ar1(rng, T, 4.0)))
    s.append(("white_700", rng.standard_normal(700)))
    for T, tau, amp in ((600, 3.0, 5.0), (1500, 5.0, 10.0), (2000, 8.0, 100.0), (900, 2.0, 1.0)):
        s.append((f"trans_{T}", ar1(rng, T, tau) + amp * np.exp(-np.arange(T) / (T / 20.0))))
    s.append(("offset_1500", 1.0e6 + ar1(rng, 1500, 5.0)))
    s.append(("int_1200", np.round(40.0 * ar1(rng, 1200, 5.0)).astype(np.int64)))
    s.append(("int_small_800", np.round(3.0 * ar1(rng, 800, 3.0)).astype(np.int64)))
    x = ar1(rng, 700, 5.0) + 3.0 * np.exp(-np.arange(700) / 40.0)
    s.append(("tail_exact", np.concatenate([x, np.full(80, 3.0)])))
    s.append(("tail_inexact", np.concatenate([x[:600], np.full(90, 0.1)])))
    s.append(("tail_one", np.concatenate([ar1(rng, 300, 3.0), [7.25]])))
    s.append(("constant_400", np.full(400, 2.5)))
    for k, T in enumerate((1000, 1300, 1700, 2500, 3000, 750, 1100, 1900, 2200, 1400)):
        s.append((f"ar_mix_{k}", ar1(rng, T, 2.0 + 3.0 * k)))
    s.append((f"long_{LONG}", ar1(rng, LONG, 5.0)))
    names = [n for n, _ in s]
    A = [x for _, x in s]
    B = [0.6 * np.asarray(x, np.float64) + 0.8 * ar1(rng, np.size(x), 3.0) for x in A]
    return names, A, B


def digest(A, B):
    """sha256 of every series and partner, in order: identifies the fixture's inputs without storing them"""
    h = hashlib.sha256()
    for a, b in zip(A, B):
        h.update(np.ascontiguousarray(a).tobytes())
        h.update(np.ascontiguousarray(b).tobytes())
    return h.hexdigest()


class SeriesNumpyAcf(tsr.NumpyAcf):
    """tests/_timeseries.NumpyAcf with `inefficiency_series`: each request answered by NumpyAcf on its series alone."""

    def inefficiency_series(self, series, starts, fast=False, mintime=3):
        from pymbar_b200 import _lib

        k = np.atleast_1d(np.asarray(series, np.int64))
        s = np.atleast_1d(np.asarray(starts, np.int64))
        if self.lengths is None or k.size < 1 or k.shape != s.shape:
            raise _lib.MbarB200Error(-1, "inefficiency_series: bad requests or an unsegmented object")
        off = np.concatenate([[0], np.cumsum(self.lengths)])
        if np.any(k < 0) or np.any(k >= self.lengths.size) or np.any(s < 0) or np.any(s >= self.lengths[k % max(
                self.lengths.size, 1)]):
            raise _lib.MbarB200Error(-1, "inefficiency_series: series or start out of range")
        self.calls += 1
        n = s.size
        out = {key: np.empty(n) for key in ("mean_a", "mean_b", "sigma2", "g")}
        out["last_lag"] = np.empty(n, np.int64)
        out["status"] = np.empty(n, np.int32)
        for q in np.unique(k):
            idx = np.flatnonzero(k == q)
            one = tsr.NumpyAcf(self.a[off[q]:off[q + 1]], self.b[off[q]:off[q + 1]] if self.cross else None)
            r = one.inefficiency(s[idx], fast=fast, mintime=mintime)
            for key in out:
                out[key][idx] = r[key]
        return out

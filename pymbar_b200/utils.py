"""Exception and validation surface shared with pymbar.utils (utils.py:117-232, :401-422)."""
import warnings

import numpy as np


class ParameterError(Exception):
    """pymbar.utils.ParameterError (utils.py:401)."""


class ConvergenceError(Exception):
    """pymbar.utils.ConvergenceError (utils.py:408)."""


class BoundsError(Exception):
    """pymbar.utils.BoundsError (utils.py:413)."""


class TypeCastPerformanceWarning(RuntimeWarning):
    """pymbar.utils.TypeCastPerformanceWarning (utils.py:36)."""


def ensure_type(val, dtype, ndim, name, shape=None, warn_on_cast=True):
    """Same contract as pymbar.utils.ensure_type (utils.py:117-232) for the cases the solver path
    uses: ndarray only, cast to dtype with a warning, ndim / shape checks, C-contiguous result."""
    if not isinstance(val, np.ndarray):
        raise TypeError(f"{name} must be numpy array.  You supplied type {type(val)}")
    dtype = np.dtype(np.float64 if dtype == "float" else dtype)
    if val.dtype != dtype:
        if warn_on_cast:
            warnings.warn(f"Casting {name} dtype={val.dtype} to {dtype} ", TypeCastPerformanceWarning)
        val = val.astype(dtype)
    if val.ndim != ndim:
        raise ValueError(f"{name} must be ndim {ndim}. You supplied {val.ndim}")
    val = np.ascontiguousarray(val)
    if shape is not None:
        if len(shape) != val.ndim or any(s is not None and s != t for s, t in zip(shape, val.shape)):
            raise ValueError(f"{name} must be shape {tuple(shape)}. You supplied  {val.shape}")
    return val


def kln_to_kn(kln, N_k=None, cleanup=False):
    """Vectorised pymbar.utils.kln_to_kn (utils.py:41-75): [K, L, N_max] -> [L, N] in block order.

    The reference copies one column per Python iteration (N iterations); this copies one state block
    per iteration (K iterations), which matters once the solve itself takes milliseconds
    (SURVEY.md 8f, row N4).  Same semantics, including N_k = None meaning N_max samples per state."""
    kln = np.asarray(kln)
    K, L, N_max = kln.shape
    if N_k is None:
        N_k = N_max * np.ones([L], dtype=np.int64)
    N_k = np.asarray(N_k, dtype=np.int64)
    N = int(np.sum(N_k[:K]))
    kn = np.zeros([L, N], dtype=np.float64)
    i = 0
    for k in range(K):
        n = int(N_k[k])
        kn[:, i:i + n] = kln[k, :, :n]
        i += n
    return kn


def kn_to_n(kn, N_k=None, cleanup=False):
    """Vectorised pymbar.utils.kn_to_n (utils.py:78-114): [K, N_max] -> [N] in block order."""
    kn = np.asarray(kn)
    K, N_max = kn.shape
    if N_k is None:
        N_k = N_max * np.ones([K], dtype=np.int64)
    N_k = np.asarray(N_k, dtype=np.int64)
    return np.concatenate([kn[k, :int(N_k[k])] for k in range(K)]).astype(np.float64) if K else np.zeros(0)

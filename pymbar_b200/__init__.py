"""pymbar_b200 — the MBAR solve hot path of pymbar on NVIDIA H100 (sm_90a).

Public surface:
  * :mod:`pymbar_b200.mbar_solvers` — same names/signatures as ``pymbar.mbar_solvers``;
  * :class:`pymbar_b200.DeviceProblem` — explicit residency handle (one GPU, one shard of samples);
  * :class:`pymbar_b200.DeviceKde` — weighted samples resident for kernel-density sums (FES with fes_type="kde");
  * :class:`pymbar_b200.DeviceKdeMany` — many sample sets resident for the kernel-density sums of many problems and
    their bootstrap replicates in one call;
  * :class:`pymbar_b200.DeviceBSpline` — samples resident for B-spline basis sums (FES with fes_type="spline");
  * :class:`pymbar_b200.DeviceAcf` — a series resident for the lag sums of ``pymbar.timeseries``
    (:mod:`pymbar_b200.timeseries`);
  * :class:`pymbar_b200.DeviceWork` — work vectors resident for the sums of ``pymbar.other_estimators`` (BAR, EXP,
    Gaussian EXP; :mod:`pymbar_b200.other_estimators`, including ``bar_many`` for many pairs in lockstep);
  * :class:`pymbar_b200.DeviceMbarBatch` — many small MBAR problems (up to 64 states each) resident together;
    :func:`pymbar_b200.mbar_many.mbar_many` solves all of them in lockstep, one device call per iteration, and
    returns each problem's free energies and uncertainties, and :class:`pymbar_b200.MbarMany` keeps them resident
    for batched expectations, perturbed free energies, entropies and enthalpies, overlaps, effective sample
    numbers and histogram and kernel-density free-energy surfaces (``generate_fes`` / ``get_fes``);
  * :func:`pymbar_b200.install` — rebind ``pymbar.mbar_solvers`` so unmodified ``pymbar.MBAR`` uses it.

Everything numerical runs in libmbar_b200.so (C ABI in include/mbar_b200.h).  No CPU fallback.
"""
from . import _lib
from .problem import DeviceAcf, DeviceBSpline, DeviceKde, DeviceKdeMany, DeviceMbarBatch, DeviceProblem, DeviceWork, PinnedArray
from .utils import ParameterError

__all__ = ["DeviceProblem", "DeviceKde", "DeviceKdeMany", "DeviceBSpline", "DeviceAcf", "DeviceWork", "DeviceMbarBatch", "PinnedArray", "ParameterError", "install", "uninstall", "trim", "mbar_solvers", "MbarMany"]

_SAVED = {}
_PATCHED = (
    "self_consistent_update", "mbar_gradient", "mbar_objective", "mbar_objective_and_gradient",
    "mbar_hessian", "mbar_log_W_nk", "mbar_W_nk", "precondition_u_kn", "adaptive",
    "solve_mbar_once", "solve_mbar", "solve_mbar_for_all_states",
    "jax_self_consistent_update", "jax_mbar_gradient", "jax_mbar_objective",
    "jax_mbar_objective_and_gradient", "jax_mbar_hessian", "jax_mbar_log_W_nk", "jax_mbar_W_nk",
    "jax_precondition_u_kn",
)


def install(target=None, patch_layout_helpers=True, patch_mbar=True):
    """Route ``pymbar.mbar_solvers`` (or `target`, a module object) through the GPU backend.

    pymbar looks its solver entry points up as module attributes at call time (mbar.py:413, :437,
    :455, :910), so rebinding them is the whole integration; nothing in pymbar is edited."""
    from . import mbar_solvers as backend

    _lib.load()
    if target is None:
        import pymbar.mbar_solvers as target  # noqa: F811
    for name in _PATCHED:
        if hasattr(target, name) and (target, name) not in _SAVED:
            _SAVED[(target, name)] = getattr(target, name)
        setattr(target, name, getattr(backend, name))
    if target.__name__ == "pymbar.mbar_solvers":
        # raise pymbar's own exception type so that `except pymbar.utils.ParameterError` keeps working
        try:
            from pymbar.utils import ParameterError as _PE

            from . import utils as _u

            if ("ParameterError",) not in _SAVED:
                _SAVED[("ParameterError",)] = (backend.ParameterError, _u.ParameterError)
            backend.ParameterError = _PE
            _u.ParameterError = _PE
        except ImportError:
            pass
    if patch_layout_helpers and target.__name__ == "pymbar.mbar_solvers":
        # MBAR.__init__ converts 3-D input with a per-column Python loop (mbar.py:238, utils.py:68-71);
        # it looks the helper up in its own module namespace
        import pymbar.mbar as mbar_mod

        from . import utils as u

        for name in ("kln_to_kn", "kn_to_n"):
            if hasattr(mbar_mod, name):
                if (mbar_mod, name) not in _SAVED:
                    _SAVED[(mbar_mod, name)] = getattr(mbar_mod, name)
                setattr(mbar_mod, name, getattr(u, name))
    if patch_mbar and target.__name__ == "pymbar.mbar_solvers":
        # lazy Log_W_nk + estimators / expectations from device moments (see facade.py)
        import pymbar.mbar as mbar_mod

        from . import facade

        facade.install_on(mbar_mod.MBAR)
        # histogram free-energy surfaces from the same resident problem (pymbar.FES, when importable)
        try:
            import pymbar.fes as fes_mod
        except ImportError:
            fes_mod = None
        if fes_mod is not None and hasattr(fes_mod, "FES"):
            facade.install_fes_on(fes_mod.FES)
        # pymbar.timeseries (statistical inefficiencies, equilibration detection), when importable
        try:
            import pymbar.timeseries as ts_mod
        except ImportError:
            ts_mod = None
        if ts_mod is not None:
            facade.install_timeseries_on(ts_mod)
        # pymbar.other_estimators (BAR, EXP, Gaussian EXP), when importable; pymbar re-exports those names at import
        try:
            import pymbar.other_estimators as oe_mod
        except ImportError:
            oe_mod = None
        if oe_mod is not None:
            import pymbar as pkg

            originals = {name: oe_mod.__dict__.get(name) for name in facade.OE_NAMES}
            facade.install_other_estimators_on(oe_mod)
            for name in facade.OE_NAMES:
                if originals[name] is not None and pkg.__dict__.get(name) is originals[name]:
                    if (pkg, name) not in _SAVED:
                        _SAVED[(pkg, name)] = originals[name]
                    setattr(pkg, name, getattr(oe_mod, name))
    return target


def uninstall():
    from . import facade

    for cls in list(facade._SAVED):
        facade.uninstall_from(cls)
    for key, fn in list(_SAVED.items()):
        if key == ("ParameterError",):
            from . import mbar_solvers as backend
            from . import utils as _u

            backend.ParameterError, _u.ParameterError = fn
        else:
            setattr(key[0], key[1], fn)
        del _SAVED[key]


def trim():
    """Give back the device / pinned buffers parked by closed DeviceProblems (mbar_b200_trim)."""
    _lib.check(_lib.load().mbar_b200_trim())


def _autoinstall():
    """PYMBAR_B200=1 in the environment: `import pymbar_b200` alone routes pymbar through the GPU backend (the
    switch SURVEY.md section 5 asks for, in the style of PYMBAR_DISABLE_JAX)."""
    import os

    if os.environ.get("PYMBAR_B200", "").lower() in ("1", "true", "yes"):
        try:
            install()
        except ImportError:          # pymbar itself not importable here: nothing to route
            pass


def __getattr__(name):
    if name == "mbar_solvers":
        import importlib

        return importlib.import_module(".mbar_solvers", __name__)
    if name == "MbarMany":
        from .mbar_many import MbarMany

        return MbarMany
    raise AttributeError(name)


_autoinstall()

"""CPU-only checks of the drop-in boundary: the shared library loads, exports every function that
include/mbar_b200.h declares, the ctypes table matches the header, and the product package refuses
to run without a GPU (no CPU fallback).  No compute calls are made here."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "mbar_b200.h")


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mbar_b200_[a-z_0-9A-Z]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    from pymbar_b200 import build

    build.build()
    from pymbar_b200 import _lib

    return _lib


def test_header_functions_are_exported(lib):
    names = declared_functions()
    assert len(names) >= 29
    dll = ctypes.CDLL(lib.LIB_PATH)
    for n in names:
        assert hasattr(dll, n), f"{n} declared in include/mbar_b200.h but not exported"


def test_ctypes_table_matches_header(lib):
    assert sorted(lib.SIGNATURES) == declared_functions()
    lib.load()
    assert lib.load().mbar_b200_abi_version() == 1


def test_max_states_matches_header():
    """The facade decides up front whether an augmented problem fits a context: its limit must be the library's."""
    from pymbar_b200 import _lib

    m = re.search(r"#define\s+MBAR_B200_MAX_STATES\s+(\d+)", open(HEADER).read())
    assert m and int(m.group(1)) == _lib.MAX_STATES


def test_no_internal_symbols_leak(lib):
    import subprocess

    out = subprocess.run(["nm", "-D", "--defined-only", lib.LIB_PATH], capture_output=True, text=True).stdout
    exported = [l.split()[-1] for l in out.splitlines() if " T " in l]
    assert exported and all(s.startswith("mbar_b200_") for s in exported), exported


def test_fails_loudly_without_gpu(lib):
    import pymbar_b200

    if lib.device_count() > 0:
        pytest.skip("a GPU is visible here")
    with pytest.raises(lib.MbarB200Error) as e:
        pymbar_b200.DeviceProblem(np.zeros((2, 8)), np.array([4.0, 4.0]))
    assert e.value.status == -3 and "no CPU fallback" in str(e.value)
    from pymbar_b200 import mbar_solvers as ms

    with pytest.raises(lib.MbarB200Error):
        ms.mbar_gradient(np.zeros((2, 8)), np.array([4, 4]), np.zeros(2))


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under pymbar_b200/ may import or reference it."""
    pkg = os.path.join(ROOT, "pymbar_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, fn)).read()
                assert "oracle" not in txt.replace("test oracle", ""), f"{fn} mentions the oracle"


def test_mirror_has_reference_surface():
    """Same public names as pymbar.mbar_solvers for the path (SURVEY.md 8b)."""
    from pymbar_b200 import mbar_solvers as ms

    for name in ("self_consistent_update", "mbar_gradient", "mbar_objective", "mbar_objective_and_gradient",
                 "mbar_hessian", "mbar_log_W_nk", "mbar_W_nk", "precondition_u_kn", "adaptive",
                 "solve_mbar_once", "solve_mbar", "solve_mbar_for_all_states", "validate_inputs",
                 "DEFAULT_SOLVER_PROTOCOL", "ROBUST_SOLVER_PROTOCOL", "BOOTSTRAP_SOLVER_PROTOCOL",
                 "JAX_SOLVER_PROTOCOL", "scipy_minimize_options", "scipy_root_options"):
        assert hasattr(ms, name), name
    assert ms.DEFAULT_SOLVER_PROTOCOL[0]["method"] == "hybr"
    with pytest.raises(TypeError):
        ms.validate_inputs(np.zeros((2, 3)), [1, 2], np.zeros(2))
    with pytest.raises(ValueError):
        ms.validate_inputs(np.zeros((2, 3)), np.zeros(3), np.zeros(2))

"""MBAR bootstrap replicates through the facade, without a GPU: the replicate stream against the reference's, every
bootstrap estimator over the CPU mirror (a weighted numpy stand-in for DeviceProblem) against
tests/golden/mbar_bootstrap.npz (tools/make_mbar_bootstrap_golden.py, the unmodified reference), every fall-back rule,
the ABI entries and the spill-free build of replicates.cu."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from tests import _cases
from tests import _mbar_boot as mb
from tests.test_driver_logic_cpu import mirror  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = mb.golden()
CASES = [str(c) for c in G["cases"]]
SEEDS = [int(s) for s in G["seeds"]]
NB = int(G["n_bootstraps"])


@pytest.fixture()
def boot_mbar(mirror, monkeypatch):  # noqa: F811
    """BootMBAR over the mirror with multiplicities, facade installed."""
    from pymbar_b200 import facade
    from pymbar_b200 import mbar_solvers as ms

    monkeypatch.setattr(ms, "DeviceProblem", mb.WeightedOracleProblem)
    monkeypatch.setattr(mb.WeightedOracleProblem, "fail_on", ())
    monkeypatch.setattr(mb.WeightedOracleProblem, "uploads", 0)
    mb.BootMBAR.solvers = mirror
    facade.install_on(mb.BootMBAR)
    yield mb.BootMBAR
    facade.uninstall_from(mb.BootMBAR)


# ---- the stream --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_stream_block_and_interleaved(name):
    """draw_mbar_replicates + replicate_rints reproduce the reference's bootstrap_rints and leave the generator where
    the reference leaves it, for samples in block order and interleaved."""
    from pymbar_b200 import bootstrap as bs

    z = _cases.load(name)
    N_k = z["N_k"]
    runs = [(f"{name}_s{s}_", s, np.repeat(np.arange(len(N_k)), N_k)) for s in SEEDS]
    perm = G[f"{name}_perm"]
    runs.append((f"{name}_il_", SEEDS[0], np.repeat(np.arange(len(N_k)), N_k)[perm]))
    for p, seed, x in runs:
        rng = np.random.default_rng(seed)
        rng.choice(np.arange(int(N_k.sum())), min(50, int(N_k.sum())))
        members = bs.state_members(N_k, x)
        seen = []
        states, counts = bs.draw_mbar_replicates(rng, N_k, members, NB, lambda b, r: seen.append(r.copy()))
        np.testing.assert_array_equal(np.array(seen), G[p + "bootstrap_rints"])
        after = rng.bit_generator.state
        regen = np.array([bs.replicate_rints(rng, st, N_k, members) for st in states])
        np.testing.assert_array_equal(regen, G[p + "bootstrap_rints"])
        assert rng.bit_generator.state == after                  # regenerating does not advance the generator
        assert rng.random() == G[p + "after"]
        want = np.array([np.bincount(r, minlength=int(N_k.sum())) for r in G[p + "bootstrap_rints"]])
        assert counts.dtype == np.uint16 and np.array_equal(counts, want)


def test_state_members_rejects_undefined_labellings():
    from pymbar_b200 import bootstrap as bs

    N_k = np.array([2, 1])
    assert bs.state_members(N_k, np.array([0, 1, 0]))[0].tolist() == [0, 2]
    assert bs.state_members(N_k, np.array([0, 1, 1])) is None              # counts differ from N_k
    assert bs.state_members(N_k, np.array([0, 2, 0])) is None              # a state outside [0, K)
    assert bs.state_members(N_k, np.array([0.0, 1.0, 0.0])) is None        # not integers


# ---- the facade over the mirror ----------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("name", CASES)
def test_facade_against_golden(boot_mbar, name, seed):
    from pymbar_b200 import facade

    z = _cases.load(name)
    s0 = dict(facade.STATS)
    m = boot_mbar(z["u_kn"], z["N_k"], n_bootstraps=NB, rseed=seed)
    assert facade.STATS["mbar_boot_solves"] == s0["mbar_boot_solves"] + NB
    assert facade.STATS["mbar_boot_fallbacks"] == s0["mbar_boot_fallbacks"]
    assert m.n_bootstraps == NB and "bootstrap_rints" not in m.__dict__
    assert isinstance(m.__dict__["_b200_rints"], facade.RintsTicket)
    state = m.rng.bit_generator.state
    mb.check_case(m, G, name, seed)
    assert facade.STATS["redeemed"] == s0["redeemed"]                    # no Log_W_nk, no original method
    assert facade.STATS["expectations_boot"] == s0["expectations_boot"] + 7
    assert facade.STATS["expectations_fallbacks"] == s0["expectations_fallbacks"]
    assert facade.STATS["boot_rints_built"] == s0["boot_rints_built"]
    np.testing.assert_array_equal(m.bootstrap_rints, G[f"{name}_s{seed}_bootstrap_rints"])
    assert facade.STATS["boot_rints_built"] == s0["boot_rints_built"] + 1
    assert m.rng.bit_generator.state == state                           # reading the property drew nothing
    assert m.rng.random() == G[f"{name}_s{seed}_after"]


@pytest.mark.parametrize("name", CASES)
def test_bar_start_and_interleaved_samples(boot_mbar, name):
    z = _cases.load(name)
    seed = SEEDS[0]
    m = boot_mbar(z["u_kn"], z["N_k"], n_bootstraps=NB, rseed=seed, initialize="BAR")
    np.testing.assert_allclose(m.f_k_boots, G[f"{name}_bar_f_k_boots"], rtol=0, atol=1e-8)
    # the installed BAR returns a fresh array: f_k stays the solution of the full data
    np.testing.assert_allclose(m.f_k, z["fk_default"], atol=1e-8)
    perm = G[f"{name}_perm"]
    labels = np.repeat(np.arange(len(z["N_k"])), z["N_k"])[perm]
    m = boot_mbar(z["u_kn"][:, perm], z["N_k"], n_bootstraps=NB, rseed=seed, x_kindices=labels)
    np.testing.assert_allclose(m.f_k_boots, G[f"{name}_il_f_k_boots"], rtol=0, atol=1e-8)
    np.testing.assert_array_equal(m.bootstrap_rints, G[f"{name}_il_bootstrap_rints"])
    assert m.rng.random() == G[f"{name}_il_after"]


# ---- fall-backs --------------------------------------------------------------------------------------------------
class _RecordingInner(mb.BootMBAR):
    calls = []
    __init__ = mb.BootMBAR.__init__          # the facade patches a class's own constructor

    def compute_expectations_inner(self, *args, **kwargs):
        type(self).calls.append(kwargs.get("uncertainty_method"))
        return {"original": True}


@pytest.fixture()
def recording_mbar(mirror, monkeypatch):  # noqa: F811
    from pymbar_b200 import facade
    from pymbar_b200 import mbar_solvers as ms

    monkeypatch.setattr(ms, "DeviceProblem", mb.WeightedOracleProblem)
    monkeypatch.setattr(mb.WeightedOracleProblem, "fail_on", ())
    _RecordingInner.solvers = mirror
    _RecordingInner.calls = []
    facade.install_on(_RecordingInner)
    yield _RecordingInner
    facade.uninstall_from(_RecordingInner)


@pytest.mark.parametrize("n", [None, -4, 0, 100.3, True, np.float64(3.0)])
def test_non_positive_int_runs_the_original(recording_mbar, n):
    from pymbar_b200 import facade

    z = _cases.load("small_osc_8x40")
    s0 = dict(facade.STATS)
    try:
        m = recording_mbar(z["u_kn"], z["N_k"], n_bootstraps=n, rseed=1)
    except TypeError:
        assert n is None or isinstance(n, (float, bool))                # the original's own error
        assert facade.STATS["mbar_boot_solves"] == s0["mbar_boot_solves"]
        return
    assert facade.STATS["mbar_boot_solves"] == s0["mbar_boot_solves"]
    if isinstance(n, np.floating):                                       # the original's loop ran (numpy accepts it)
        assert m.f_k_boots.shape == (3, 8) and isinstance(m.__dict__["_b200_rints"], np.ndarray)
        return
    assert not hasattr(m, "f_k_boots")
    m.compute_expectations_inner(z["x_n"].copy(), m.u_kn, np.array([[0], [0]]), uncertainty_method="bootstrap")
    assert recording_mbar.calls == ["bootstrap"]


def test_device_error_in_one_replicate(boot_mbar):
    """Replicate 2 of 5 fails on the device: only it is solved on the gathered columns; results and stream are the
    reference's."""
    from pymbar_b200 import facade

    name, seed = "small_osc_8x40", SEEDS[0]
    z = _cases.load(name)
    mb.WeightedOracleProblem.fail_on = (3,)
    s0 = dict(facade.STATS)
    m = boot_mbar(z["u_kn"], z["N_k"], n_bootstraps=5, rseed=seed)
    assert facade.STATS["mbar_boot_fallbacks"] == s0["mbar_boot_fallbacks"] + 1
    assert facade.STATS["mbar_boot_solves"] == s0["mbar_boot_solves"] + 4
    np.testing.assert_allclose(m.f_k_boots, G[f"{name}_s{seed}_f_k_boots"][:5], rtol=0, atol=1e-8)
    np.testing.assert_array_equal(m.bootstrap_rints, G[f"{name}_s{seed}_bootstrap_rints"][:5])


def test_expectation_fallbacks(recording_mbar, monkeypatch):
    from pymbar_b200 import _lib

    z = _cases.load("small_osc_8x40")
    m = recording_mbar(z["u_kn"], z["N_k"], n_bootstraps=3, rseed=5)
    K = m.K
    sm = np.array([np.arange(K), np.zeros(K, int)])
    # past MAX_STATES
    monkeypatch.setattr(_lib, "MAX_STATES", K + 2 * K - 1)
    assert m.compute_expectations_inner(z["x_n"].copy(), m.u_kn, sm, uncertainty_method="bootstrap")["original"]
    monkeypatch.setattr(_lib, "MAX_STATES", 8192)
    # a count above 65535 (the constructor keeps no counts then)
    m.__dict__["_b200_boot_counts"] = None
    assert m.compute_expectations_inner(z["x_n"].copy(), m.u_kn, sm, uncertainty_method="bootstrap")["original"]
    del m.__dict__["_b200_boot_counts"]
    # a device error
    monkeypatch.setattr(mb.WeightedOracleProblem, "replicate_unsampled",
                        lambda self, c, F: (_ for _ in ()).throw(_lib.MbarB200Error(-6, "injected")))
    assert m.compute_expectations_inner(z["x_n"].copy(), m.u_kn, sm, uncertainty_method="bootstrap")["original"]
    assert recording_mbar.calls == ["bootstrap"] * 3


def test_counts_from_assigned_rints(boot_mbar):
    """bootstrap_rints assigned after construction: the counts come from its rows."""
    name, seed = "small_osc_8x40", SEEDS[0]
    z = _cases.load(name)
    m = boot_mbar(z["u_kn"], z["N_k"], n_bootstraps=NB, rseed=seed)
    m.bootstrap_rints = G[f"{name}_s{seed}_bootstrap_rints"].copy()
    assert "_b200_boot_counts" not in m.__dict__
    mb.check_case(m, G, name, seed)
    m.bootstrap_rints = np.zeros((NB, m.N), int) + np.arange(m.N) % 2      # sample 0 / 1 drawn N / 2 times
    from pymbar_b200 import facade

    counts = facade._replicate_counts(m)
    assert counts is not None and counts[0, 0] == m.N // 2


def test_binding_rejects_large_counts():
    from pymbar_b200.problem import DeviceProblem

    p = DeviceProblem.__new__(DeviceProblem)
    p.K, p.N, p.N_k = 2, 3, np.array([3.0, 0.0])
    with pytest.raises(ValueError):
        p.replicate_unsampled(np.array([[1, 65536, 0]]), np.zeros((1, 2)))
    with pytest.raises(ValueError):
        p.replicate_unsampled(np.array([[1, -1, 0]]), np.zeros((1, 2)))


# ---- ABI and build -----------------------------------------------------------------------------------------------
def test_header_and_ctypes_entries():
    from pymbar_b200 import _lib

    header = open(os.path.join(ROOT, "include", "mbar_b200.h")).read()
    for name in ("mbar_b200_replicate_unsampled", "mbar_b200_last_replicate_stats"):
        assert re.search(r"\bint " + name + r"\(", header), name
        assert name in _lib.SIGNATURES
    res, args = _lib.SIGNATURES["mbar_b200_replicate_unsampled"]
    assert len(args) == 5 and args[2]._type_ is __import__("ctypes").c_uint16
    assert len(_lib.SIGNATURES["mbar_b200_last_replicate_stats"][1]) == 4


def test_replicates_cu_builds_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "pymbar_b200", "csrc", "replicates.cu")
    out = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v",
                          "-c", src, "-o", str(tmp_path / "replicates.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    log = out.stdout + out.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)'", log)
    assert any("rep_partial_kernel" in k for k in kernels) and any("rep_combine_kernel" in k for k in kernels)
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert spills and all(a == "0" and b == "0" for a, b in spills), log
    assert "bytes stack frame" in log and all(s == "0" for s in re.findall(r"(\d+) bytes stack frame", log))

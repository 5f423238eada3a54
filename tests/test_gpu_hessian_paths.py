"""Every Hessian kernel path, entry by entry, against the extended-precision reference of tests/_moments.py.

Ghat = (N W)^T (N W) is a sum of non-negative products, so every entry -- down to couplings of 1e-300 between states
that barely overlap, which decide the Newton step of a poorly overlapping problem -- must match the reference to
the relative tolerance of _moments.entry_tol.  Which kernel answers depends on K, on whether the fused pass stored
the weights, on all-rows moments and on whether the 8 K N weight buffer fits; each test asserts the kernel name so
that a parametrisation cannot silently collapse onto one path:

  P1  streaming_pass(want_G) / hessian after the fused pass stored the weights (WST)
  P2  the same after set_kernel("generic"): in-register small kernel (K <= 64) or weights_kernel
  P3  weight_moments: all rows, in-register small kernel or weights_kernel
  P4  streaming_pass(want_G) with per-sample multiplicities (zeros included)

The in-place kernel is checked twice: forced for every K in a subprocess (the switch is read once per process),
and chosen by the library itself at the C5 shape, where u_kn and the weights do not both fit on an 80 GB H100.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import mbar_oracle as orc
from tests import _moments as M

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = list(M.cases())
HEADROOM = {}          # (path label) -> largest |dGhat| / tol seen
SUBNORMAL = {}         # (path label) -> [entries with 0 < Ghat < 2^-1022, of which the device kept nonzero]

_CASES, _REFS = {}, {}


def case(name):
    if name not in _CASES:
        _CASES[name] = M.build(name)
    return _CASES[name]


def ref(name, path):
    key = (name, "P1" if path == "P2" else path)
    if key not in _REFS:
        _REFS[key] = M.reference(case(name), key[1])
    return _REFS[key]


@pytest.fixture(scope="module")
def lib():
    import pymbar_b200
    from pymbar_b200 import _lib

    _lib.load()
    if _lib.device_count() == 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    yield pymbar_b200
    for label in sorted(HEADROOM):
        sub = SUBNORMAL.get(label, [0, 0])
        print(f"\n[hessian paths] {label}: max |dGhat|/tol = {HEADROOM[label]:.3g}; subnormal reference entries "
              f"{sub[0]}, nonzero on the device {sub[1]}")


def check_moments(name, path, d, expect, label):
    """The checks every path must pass; d holds two calls (S0, G0, S1, G1, name0, name1) and, for P1 / P2, H0 / H1."""
    c = case(name)
    S_ref, Ghat, A, rows = ref(name, path)
    s = c["N"] > 0
    for i in range(2):
        assert expect in d[f"name{i}"], (expect, d[f"name{i}"])
    # two calls are bit-identical
    assert np.array_equal(d["G0"], d["G1"]) and np.array_equal(d["S0"], d["S1"])
    S, G = d["S0"], d["G0"]
    assert np.array_equal(G, G.T)
    if path != "P3":
        assert np.all(G[~s] == 0) and np.all(G[:, ~s] == 0)
    sc = M.row_scale(c["N"], path)
    Gd = G * sc[:, None] * sc[None, :]
    N = c["u"].shape[1]
    wmax = float(np.sqrt(np.max(np.diag(Ghat).astype(np.float64))))
    tol = M.entry_tol(Ghat, A, N, wmax)
    mask = rows[:, None] & rows[None, :]
    r = M.excess(Gd, Ghat, tol, mask)
    HEADROOM[label] = max(HEADROOM.get(label, 0.0), r)
    sub = mask & (Ghat > 0) & (Ghat < M.LD(2.0 ** -1022))
    acc = SUBNORMAL.setdefault(label, [0, 0])
    acc[0] += int(sub.sum())
    acc[1] += int((sub & (Gd != 0)).sum())
    worst = np.unravel_index(np.argmax(np.where(mask, np.abs(Gd.astype(M.LD) - Ghat) / tol, 0)), G.shape)
    assert r <= 1.0, (r, worst, Gd[worst], Ghat[worst], tol[worst])
    # row sums: sum_{j sampled} Ghat_ij = s_i S_i, against S of the same call (the pass kernel's own exp)
    lhs = Gd[:, s].astype(M.LD).sum(axis=1)
    rhs = (sc * S).astype(M.LD)
    bound = 2 * tol[:, s].sum(axis=1)
    rr = np.abs(lhs - rhs)[rows] / bound[rows]
    assert rr.max() <= 1.0, (rr.max(), np.argmax(rr))
    if "H0" in d:
        assert np.array_equal(d["H0"], d["H1"])
        assert expect in d["hname"], d["hname"]
        off = np.outer(s, s) & ~np.eye(len(s), dtype=bool)
        np.testing.assert_allclose(-d["H0"][off], Gd[off], rtol=4 * M.EPS, atol=1e-300)
        assert np.all(d["H0"][~s] == 0) and np.all(d["H0"][:, ~s] == 0)


@pytest.mark.parametrize("path", M.PATHS)
@pytest.mark.parametrize("name", NAMES)
def test_paths_in_process(lib, name, path):
    c = case(name)
    with lib.DeviceProblem(c["u"], c["N"]) as p:
        d = M.device_moments(p, c, path)
    expect = M.expected_kernel(c, path)
    check_moments(name, path, d, expect, f"{path} {expect.split(' (')[0]}")


# ---- the in-place kernel, forced ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def inplace(lib, tmp_path_factory):
    out = str(tmp_path_factory.mktemp("inplace") / "inplace.npz")
    env = dict(os.environ, MBAR_B200_HESSIAN_INPLACE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hessian_inplace_worker.py"), out],
                       capture_output=True, text=True, timeout=1800, cwd=ROOT, env=env)
    assert r.returncode == 0 and "INPLACE_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    z = np.load(out)
    data = {k: z[k] for k in z.files if k != "names"}
    data.update(json.loads(str(z["names"])))
    return data


@pytest.mark.parametrize("path", M.PATHS)
@pytest.mark.parametrize("name", NAMES)
def test_inplace_kernel_forced(inplace, name, path):
    keys = ("S0", "G0", "S1", "G1", "name0", "name1", "H0", "H1", "hname")
    d = {k: inplace[f"{name}|{path}|{k}"] for k in keys if f"{name}|{path}|{k}" in inplace}
    check_moments(name, path, d, M.expected_kernel(case(name), path, inplace=True),
                  f"{path} hessian_inplace_kernel (forced)")


@pytest.mark.parametrize("K", [17, 65])
def test_inplace_kernel_forced_solves(inplace, K):
    """Device-resident adaptive solves (batch 2 and 16, kernel by kernel and from a captured graph) and the stepped
    solve, every Hessian from the in-place kernel, against the oracle's adaptive() and each other."""
    c = M.solve_ladder(K, seed=K)
    ref = orc.adaptive(c["u"], c["N"], np.zeros(K), tol=1e-12, options=dict(min_sc_iter=0))
    assert ref["success"]
    assert "hessian_inplace_kernel" in inplace[f"solve{K}|hname"], inplace[f"solve{K}|hname"]
    assert inplace[f"solve{K}|graph_launches"] > 0
    fs = inplace[f"solve{K}|stepped"]
    assert inplace[f"solve{K}|stepped|ok"]
    assert np.max(np.abs(fs - ref["x"])) < 1e-8
    for batch in (2, 16):
        for rep in range(2):
            f = inplace[f"solve{K}|b{batch}|{rep}"]
            assert inplace[f"solve{K}|b{batch}|{rep}|ok"]
            assert np.max(np.abs(f - ref["x"])) < 1e-8, (batch, rep)
            assert np.max(np.abs(f - fs)) < 1e-9, (batch, rep)


# ---- the in-place kernel, chosen by the library at the C5 shape ---------------------------------------------------
def test_c5_inplace_chosen_by_library(lib):
    """K = 512, N = 1.25e7 (BASELINE C5 per GPU): u_kn is 51.2 GB, the weights would be another 51.2 GB.  Unless
    the device has room for both, the library answers with hessian_inplace_kernel; ten shards of 1.25e6 samples
    whose weights do fit give the same S and Ghat through the materialised path.  A device-resident adaptive
    solve on the full problem then converges, and the Hessian of its last enqueued iteration, which runs past
    convergence, exits at once."""
    import torch

    K, N, n_shards = 512, 12_500_000, 10
    Ns = N // n_shards
    N_k = np.full(K, N // K, float)
    N_k[-1] += N - N_k.sum()
    O, kk = M.harmonic_c5(K)
    fa = M.analytic_f(kk)
    lib.trim()          # parked buffers must neither cause the fallback nor hide it
    free, _ = torch.cuda.mem_get_info()
    fits = free >= 2 * 8 * K * N
    p = lib.DeviceProblem(None, N_k, N_local=N)
    try:
        p.synthesize(O, kk, seed=1)
        S, _, G = p.streaming_pass(fa, want_G=True)
        name = p.last_kernels()["hessian_kernel"]
        ms = p.last_hessian_ms()["hessian_ms"]
    finally:
        p.close()
    lib.trim()
    assert ("hessian_inplace_kernel" in name) != fits, (name, free)
    if fits:
        assert "weights stored by the fused pass (WST)" in name, name
    print(f"\n[C5] free before the context {free / 1e9:.1f} GB; {name}; Hessian {ms:.1f} ms")
    S_sum = np.zeros(K, M.LD)
    G_sum = np.zeros((K, K), M.LD)
    for r in range(n_shards):
        with lib.DeviceProblem(None, N_k, N_local=Ns) as q:
            q.synthesize(O, kk, seed=1, n_offset=r * Ns, N_global=N)
            Sr, _, Gr = q.streaming_pass(fa, want_G=True)
            assert "weights stored by the fused pass (WST)" in q.last_kernels()["hessian_kernel"]
            S_sum += Sr
            G_sum += Gr
    lib.trim()
    NN = np.outer(N_k, N_k)
    Ghat_shards = G_sum * NN
    Ghat_full = G * NN
    # A bound that holds for every state: only weights in the normal range carry the argument term
    tol = M.entry_tol(Ghat_shards, -M.LOG_NORMAL, N, 1.0)
    assert M.excess(Ghat_full, Ghat_shards, 2 * tol) <= 1.0
    np.testing.assert_allclose(S, S_sum.astype(np.float64), rtol=1e-12)
    lhs = Ghat_full.astype(M.LD).sum(axis=1)
    assert np.all(np.abs(lhs - N_k * S) <= 2 * tol.sum(axis=1))
    assert np.array_equal(G, G.T)

    p = lib.DeviceProblem(None, N_k, N_local=N)
    try:
        p.synthesize(O, kk, seed=1)
        p.set_loop_mode("device", 16)
        f, r = p.solve_adaptive(np.zeros(K), tol=1e-12, min_sc_iter=0)
        assert r["success"], r
        assert ("hessian_inplace_kernel" in p.last_kernels()["hessian_kernel"]) != fits
        hms = p.last_hessian_ms()["hessian_ms"]
        print(f"[C5] adaptive: {r['iterations']} iterations; Hessian of the last enqueued iteration {hms:.3f} ms")
        assert hms < 1.0, hms
        S, _, _ = p.streaming_pass(f)
        np.testing.assert_allclose(S, 1.0, atol=1e-9)
        assert np.max(np.abs(p.gradient(f))) < 1e-8 * N_k.max()
        np.testing.assert_allclose(p.self_consistent_update(f), f, atol=1e-9)
        assert np.max(np.abs(f - fa)) < 0.02
    finally:
        p.close()
        lib.trim()

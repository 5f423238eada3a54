#!/usr/bin/env python
"""MBAR bootstrap replicates at user-sized shapes, one run:

  1. harmonic oscillators (oracle/testsystems.oscillators) at --K states, --N samples, --B replicates: the wall time of
     MBAR(u_kn, N_k, n_bootstraps=B) through the facade (on the MBAR-shaped stand-in of the tests, with the device
     backend), against the old gather path's per-replicate time (solve_mbar_for_all_states on u_kn[:, rints], a fresh
     upload each) timed on --gather-B replicates in the same process;
  2. compute_expectations(bootstrap) of one observable at every state on the same object: the replicate_unsampled
     kernel time (CUDA events) and its call time (counts upload included), against a loop of B per-replicate
     set_sample_weights + self_consistent_update on the same augmented context; both alternately, --reps times,
     after a warm-up; and the exps per second from the call's counter;
  3. the same comparison at --big-K, --big-N, --big-B on a synthesised problem (no host u_kn) augmented with one
     state of interest and one observable (two appended rows);
  4. the card name, its power limit and its max SM clock, read in the same run.
Not run by bench.py.

    python tools/quick_mbar_bootstrap.py [--K 64] [--N 1000000] [--B 200] [--gather-B 5]
        [--big-K 256] [--big-N 10000000] [--big-B 50] [--reps 3] [--out quick_mbar_bootstrap.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import testsystems as ots  # noqa: E402
from pymbar_b200 import DeviceProblem, facade  # noqa: E402
from pymbar_b200 import expectations as ex  # noqa: E402
from pymbar_b200 import mbar_solvers as ms  # noqa: E402
from tests import _mbar_boot as mb  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def compare(q, counts, F, reps):
    """(replicate_unsampled timings, per-replicate loop timings) on the augmented context q, alternately."""
    s = q.N_k > 0
    q.replicate_unsampled(counts[:1], F[:1])                  # warm-up of both paths
    q.set_sample_weights(counts[0].astype(np.float64))
    q.self_consistent_update(F[0])
    q.set_sample_weights(None)
    calls, loops = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        R = q.replicate_unsampled(counts, F)
        t1 = time.perf_counter()
        st = q.last_replicate_stats()
        calls.append({"call_s": t1 - t0, "kernel_ms": st["ms"], "batches": st["batches"], "exps": st["exps"],
                      "exps_per_s_kernel": st["exps"] / (st["ms"] * 1e-3)})
        t0 = time.perf_counter()
        ref = []
        for c, f in zip(counts, F):
            q.set_sample_weights(c.astype(np.float64))
            ref.append(q.self_consistent_update(f)[~s])
        q.set_sample_weights(None)
        loops.append({"loop_s": time.perf_counter() - t0})
        ref = np.array(ref)
        fin = np.isfinite(ref)
        rel = float(np.max(np.abs(R[fin] - ref[fin]) / np.maximum(1.0, np.abs(ref[fin]))))
        calls[-1]["max_rel_diff_vs_loop"] = rel
    return calls, loops


def flagship(a, out):
    u_kn, N_k = ots.oscillators(a.K, a.N // a.K, seed=1)
    K, N = u_kn.shape
    mb.BootMBAR.solvers = ms
    facade.install_on(mb.BootMBAR)
    try:
        t0 = time.perf_counter()
        m = mb.BootMBAR(u_kn, N_k, n_bootstraps=a.B, rseed=5)
        ctor = time.perf_counter() - t0
        # the old path: gather u_kn[:, rints] and solve it as a new problem (upload included), per replicate
        protocol = tuple({k: (dict(v) if isinstance(v, dict) else v) for k, v in st.items()}
                         for st in ms.BOOTSTRAP_SOLVER_PROTOCOL)
        rints = m.bootstrap_rints[:a.gather_B]
        t0 = time.perf_counter()
        for r in rints:
            ms.solve_mbar_for_all_states(np.ascontiguousarray(u_kn[:, r]), N_k, m.f_k.copy(), np.flatnonzero(N_k > 0),
                                         protocol)
        gather = (time.perf_counter() - t0) / len(rints)
        out["flagship"] = {"K": K, "N": N, "B": a.B, "constructor_s": ctor, "gather_per_replicate_s": gather,
                           "gather_replicates_timed": len(rints), "gather_estimate_for_B_s": gather * a.B}
        x = np.linspace(-1.0, 1.0, N)
        t0 = time.perf_counter()
        m.compute_expectations_inner(x[None], m.u_kn, np.array([np.arange(K), np.zeros(K, int)]),
                                     uncertainty_method="bootstrap")
        out["flagship"]["expectations_inner_bootstrap_s"] = time.perf_counter() - t0
        # the kernel against the per-replicate loop on the same augmented context
        sm = np.array([np.arange(K), np.zeros(K, int)])
        of_state, of_obs, wanted = ex._appended(sm)
        floor = x.min() - abs(4 * np.finfo(float).eps * x.min())
        extra = np.vstack([u_kn[wanted], u_kn[of_state] - np.log(x - floor)])
        counts = m.__dict__["_b200_boot_counts"]
        F = np.concatenate([m.f_k_boots, np.zeros((a.B, len(extra)))], axis=1)
        with ms._borrow(m.u_kn, N_k.astype(np.float64)) as p, p.augmented(extra) as q:
            calls, loops = compare(q, counts, F, a.reps)
        out["flagship"]["replicate_unsampled"] = calls
        out["flagship"]["per_replicate_loop"] = loops
    finally:
        facade.uninstall_from(mb.BootMBAR)
        ms.clear_cache()


def big(a, out):
    K, N, B = a.big_K, a.big_N, a.big_B
    N_k = np.full(K, N // K, dtype=np.float64)
    N_k[-1] += N - N_k.sum()
    with DeviceProblem(None, N_k, device=0, N_local=N) as p:
        p.synthesize(np.linspace(1, 5, K), np.linspace(1, 3, K), seed=11)
        f, _ = p.solve_adaptive(np.zeros(K), tol=1e-10, min_sc_iter=0)
        rng = np.random.default_rng(2)
        counts = rng.poisson(1.0, (B, N)).astype(np.uint16)
        F = np.tile(np.concatenate([f, [0.0, 0.0]]), (B, 1)) + np.concatenate(
            [rng.normal(0, 1e-3, (B, K)), np.zeros((B, 2))], axis=1)
        # a state of interest with energies of the oscillators' scale, and one observable x in [0.5, 1.5] at it
        x = np.linspace(0.5, 1.5, N)
        u_l = rng.uniform(0.0, 5.0, N)
        extra = np.vstack([u_l, u_l - np.log(x)])
        with p.augmented(extra) as q:
            calls, loops = compare(q, counts, F, a.reps)
    out["big"] = {"K": K, "N": N, "B": B, "appended_rows": 2, "replicate_unsampled": calls,
                  "per_replicate_loop": loops}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, default=64)
    ap.add_argument("--N", type=int, default=1_000_000)
    ap.add_argument("--B", type=int, default=200)
    ap.add_argument("--gather-B", type=int, default=5)
    ap.add_argument("--big-K", type=int, default=256)
    ap.add_argument("--big-N", type=int, default=10_000_000)
    ap.add_argument("--big-B", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = {"card": card()}
    flagship(a, out)
    if a.big_N > 0:
        big(a, out)
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()

"""The data path in and out of HBM (ctx.cu, logw.cu) against the restatements of tests/_datapath.py.

Uploads, downloads and appends are compared bit for bit with the restated image: each stored value is one IEEE
operation on host and device alike.  Shapes are chosen so that every copy loop runs several chunks, including a
ragged last one (the chunk counts are asserted from the restated geometry).  Reused contexts, and contexts built on
parked buffers, must give bit-identical results to a fresh context holding the same data."""
import numpy as np
import pytest

from oracle import mbar_oracle as orc
from tests import _datapath as D
from tests import _edges as E

pytestmark = pytest.mark.gpu

K_BIG, N_BIG = 384, 3 * 21824 + 45          # upload: 4 chunks (last ragged); log W: 4 chunks
K_THIN, N_THIN = 5, 1677696 + 1000          # upload: 2 chunks, the last packed serially
ERR_INVALID, ERR_NAN, ERR_RANGE = -1, -5, -6


@pytest.fixture(scope="module")
def lib():
    import pymbar_b200
    from pymbar_b200 import _lib

    _lib.load()
    if _lib.device_count() == 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return pymbar_b200


def err(lib):
    from pymbar_b200._lib import MbarB200Error

    return MbarB200Error


def assert_bits(a, b, what=""):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    bad = a.view(np.int64) != b.view(np.int64)
    if bad.any():
        idx = np.argwhere(bad)
        i = tuple(idx[0])
        raise AssertionError(f"{what}: {bad.sum()} of {bad.size} entries differ, first at {i}: {a[i]!r} vs {b[i]!r}")


def energies(K, N, seed, unsampled=(), inf_at=()):
    """Random energies with row offsets; N_k sums to N; `unsampled` rows get N_k = 0."""
    rng = np.random.default_rng(seed)
    u = rng.standard_normal((K, N)) * 3.0 + np.linspace(0.0, 4.0, K)[:, None]
    N_k = np.zeros(K)
    s = np.setdiff1d(np.arange(K), unsampled)
    N_k[s] = N // len(s)
    N_k[s[-1]] += N - N_k.sum()
    for k, n in inf_at:
        u[k, n] = np.inf
    return u, N_k


@pytest.fixture(scope="module")
def big(lib):
    inf_at = [(1, 0), (7, 21823), (7, 21824), (300, N_BIG - 1), (383, 2 * 21824 + 5)]
    u, N_k = energies(K_BIG, N_BIG, 1, unsampled=(3, 200), inf_at=inf_at)
    p = lib.DeviceProblem(u, N_k)
    yield dict(u=u, N_k=N_k, p=p, image=D.download_image(u, N_k), inf_at=inf_at)
    p.close()


# ------------------------------------------------------------------------------------- 1. upload routes
def _routes(lib, u):
    import torch

    K, N = u.shape
    view = np.empty((K, N + 37))
    view[:, :N] = u
    yield "contiguous", lambda p: p.upload(u)
    yield "view ld > N", lambda p: p.upload(view[:, :N])
    yield "fortran", lambda p: p.upload(np.asfortranarray(u))
    pin = lib.PinnedArray((K, N))
    pin.array[:] = u
    yield "pinned", lambda p: p.upload(pin.array)
    pin.free()
    t = torch.empty((K, N + 29), dtype=torch.float64, device="cuda")
    t[:, :N].copy_(torch.from_numpy(u))
    torch.cuda.synchronize()
    yield "device ld > N", lambda p: p.upload_device_ptr(t.data_ptr(), N + 29)
    del t


@pytest.mark.parametrize("shape", ["big", "thin"])
def test_upload_routes(lib, shape):
    if shape == "big":
        K, N, chunks = K_BIG, N_BIG, 4
        u, N_k = energies(K, N, 2, unsampled=(5,), inf_at=[(0, 21824), (9, N - 1)])
    else:
        K, N, chunks = K_THIN, N_THIN, 2
        u, N_k = energies(K, N, 3, unsampled=(2,), inf_at=[(4, 1677696), (1, N - 1)])
        assert D.upload_serial_pack(K, N, 1)
    assert D.upload_chunks(K, N) == chunks
    image = D.download_image(u, N_k)
    f = np.linspace(0.0, 1.0, K)
    first = None
    for name, up in _routes(lib, u):
        with lib.DeviceProblem(None, N_k, N_local=N) as p:
            up(p)
            assert_bits(p.download(), image, name)
            S, sumL, _ = p.streaming_pass(f)
            L = p.log_denominator(f)
        got = (S, np.array([sumL]), L)
        if first is None:
            first = got
        for a, b in zip(got, first):
            assert_bits(a, b, f"{name}: pass outputs")


# ------------------------------------------------------------------------------------- 2. download slices
@pytest.mark.parametrize("n0,n", [(5, 100), (37, 10944), (37, 10945), (1001, 2 * 10944 + 77),
                                  (N_BIG - 45, 45), (N_BIG - 10944 - 13, 10944 + 13), (0, N_BIG)])
def test_download_slices(big, n0, n):
    assert D.download_chunks(K_BIG, n) == -(-n // D.download_cols(K_BIG, n))
    got = big["p"].download(n0, n)
    assert_bits(got, big["image"][:, n0:n0 + n], "download")
    wide = np.full((K_BIG, n + 7), -1234.5)
    big["p"].download(n0, n, out=wide[:, :n])
    assert_bits(wide[:, :n], big["image"][:, n0:n0 + n], "download ld > n")
    assert np.all(wide[:, n:] == -1234.5)


# ------------------------------------------------------------------------------------- 3. log W
@pytest.fixture(scope="module")
def logw_ref(big):
    u, N_k = big["u"], big["N_k"]
    f = np.linspace(0.0, 0.5, K_BIG)
    return f, orc.mbar_log_W_nk(u, N_k, f)


def test_log_w_against_oracle(lib, big, logw_ref):
    f, ref = logw_ref
    p = big["p"]
    assert D.logw_chunks(K_BIG, N_BIG) == 4
    lw = p.log_W_nk(f)
    fin = np.isfinite(ref)
    np.testing.assert_allclose(lw[fin], ref[fin], rtol=0, atol=1e-10)
    for k, n in big["inf_at"]:
        assert ref[n, k] == -np.inf and lw[n, k] == -np.inf
    assert np.array_equal(np.isfinite(lw), fin)
    W = p.log_W_nk(f, exponentiate=True)
    np.testing.assert_allclose(W[fin], np.exp(ref[fin]), rtol=1e-10, atol=0)
    for k, n in big["inf_at"]:
        assert W[n, k] == 0.0


def test_log_w_pages_and_destinations(lib, big, logw_ref):
    f, _ = logw_ref
    p = big["p"]
    full = p.log_W_nk(f)
    for row0, rows in ((21824 - 160, 3000), (3 * 21824 - 64, 64 + 45), (0, 2 * 21824 + 1), (32, N_BIG - 32),
                       (N_BIG - 45, 45)):
        assert_bits(p.log_W_nk(f, rows=rows, row0=row0), full[row0:row0 + rows], f"rows {row0}+{rows}")
    assert_bits(p.log_W_nk(f, row0=64), full[64:], "row0 only")
    pin = lib.PinnedArray((N_BIG, K_BIG))
    p.log_W_nk(f, out=pin.array)
    assert_bits(pin.array, full, "pinned destination")
    pin.free()
    for pinned in (False, True):
        holder = lib.PinnedArray((N_BIG, K_BIG + 5)) if pinned else None
        wide = holder.array if pinned else np.empty((N_BIG, K_BIG + 5))
        wide[:] = -7.25
        p.log_W_nk(f, out=wide[:, :K_BIG])
        assert_bits(wide[:, :K_BIG], full, f"ld > K (pinned={pinned})")
        assert np.all(wide[:, K_BIG:] == -7.25)
        if pinned:
            holder.free()
    page = np.full((3000, K_BIG + 3), -7.25)
    p.log_W_nk(f, out=page[:, :K_BIG], rows=3000, row0=21824 - 160)
    assert_bits(page[:, :K_BIG], full[21824 - 160:21824 + 2840], "paged, ld > K")
    assert np.all(page[:, K_BIG:] == -7.25)
    for row0, rows in ((16, 32), (N_BIG, 1), (-32, 64), (0, N_BIG + 1)):
        with pytest.raises(err(lib)) as e:
            p.log_W_nk(f, rows=rows, row0=row0)
        assert e.value.status == ERR_INVALID


# ------------------------------------------------------------------------------------- 4. append
@pytest.mark.parametrize("source", ["pageable", "pinned", "view"])
def test_append_chunks(lib, source):
    K, E_, N = 4, 200, 3 * 20960 + 17
    assert D.append_chunks(E_, N) == 4
    u, N_k = energies(K, N, 4)
    rng = np.random.default_rng(5)
    extra = rng.standard_normal((E_, N)) * 2.0 + np.linspace(-3.0, 6.0, E_)[:, None]
    extra[7, 20960] = np.inf
    extra[150, N - 1] = np.inf
    w = rng.integers(0, 3, N).astype(float)
    if source == "pinned":
        holder = lib.PinnedArray((E_, N))
        holder.array[:] = extra
        src = holder.array
    elif source == "view":
        wide = np.empty((E_, N + 11))
        wide[:, :N] = extra
        src = wide[:, :N]
    else:
        src = extra
    stacked = np.vstack([u, extra])
    N_aug = np.concatenate([N_k, np.zeros(E_)])
    f = np.concatenate([np.linspace(0.0, 0.3, K), np.zeros(E_)])
    with lib.DeviceProblem(u, N_k) as base:
        base.set_sample_weights(w)
        with base.augmented(src) as q:
            assert_bits(q.download(), D.appended_image(u, N_k, extra), "augmented download")
            assert_bits(q.download(), D.download_image(stacked, N_aug), "stacked image")
            got = (q.self_consistent_update(f), *q.weight_moments(f), q.last_kernels()["pass_kernel"])
    with lib.DeviceProblem(stacked, N_aug) as fresh:
        fresh.set_sample_weights(w)
        want = (fresh.self_consistent_update(f), *fresh.weight_moments(f), fresh.last_kernels()["pass_kernel"])
    for a, b in zip(got[:3], want[:3]):
        assert_bits(a, b, "augmented vs fresh")
    assert got[3] == want[3]
    if source == "pinned":
        holder.free()


# ------------------------------------------------------------------------------------- 5. synthesis
SYNTH_CASES = [
    ("empty first/middle/last", [0, 300, 250, 0, 190, 0]),
    ("K = 1", [1001]),
    ("K = 513", [0] + [3] * 255 + [0] + [2] * 255 + [7]),
]


def _synth_check(lib, O, k, N_k, seed, n_offset, N_local):
    N_g = int(np.sum(N_k))
    with lib.DeviceProblem(None, N_k, N_local=N_local) as p:
        p.synthesize(O, k, seed=seed, n_offset=n_offset, N_global=N_g)
        got = p.download()
    want, aux = D.synth(O, k, N_k, seed, n_offset, N_local, N_g)
    tol = D.synth_tolerance(aux)
    bad = np.abs(got - want) > tol
    assert not bad.any(), (f"{bad.sum()} entries beyond the bound, worst excess "
                           f"{np.max((np.abs(got - want) - tol)[bad])}")
    return got


@pytest.mark.parametrize("name,N_k", SYNTH_CASES, ids=[c[0] for c in SYNTH_CASES])
def test_synthesize_against_restatement(lib, name, N_k):
    N_k = np.array(N_k, float)
    K, N = len(N_k), int(N_k.sum())
    assert N % 32
    O, k = np.linspace(1.0, 5.0, K), np.linspace(1.0, 3.0, K)
    whole = _synth_check(lib, O, k, N_k, 17, 0, N)
    n1 = N // 3 + 5
    a = _synth_check(lib, O, k, N_k, 17, 0, n1)
    b = _synth_check(lib, O, k, N_k, 17, n1, N - n1)
    assert_bits(np.hstack([a, b]), whole, "two shards vs the whole")


def test_synthesize_bench_family(lib):
    import bench

    K, N = 256, 100_003
    O, k = bench.workload_params(K)
    N_k = bench.global_N_k(K, N)
    _synth_check(lib, O, k, N_k, 0, 0, N)


# ------------------------------------------------------------------------------------- 6. reused contexts
def _results(p, f):
    S, sumL, _ = p.streaming_pass(f)
    fa, r = p.solve_adaptive(f)
    return [np.array([p.objective(f)]), S, np.array([sumL]), fa, p.self_consistent_update(f)]


@pytest.mark.parametrize("weighted", [False, True])
def test_reupload_matches_fresh(lib, weighted):
    u1, N_k = energies(6, 5000, 7, unsampled=(4,))
    u2, _ = energies(6, 5000, 8, unsampled=(4,))
    u2 += np.random.default_rng(9).uniform(0, 50, 5000)        # different shifts
    w = np.random.default_rng(10).integers(0, 4, 5000).astype(float) if weighted else None
    f = np.linspace(0.0, 1.0, 6)
    with lib.DeviceProblem(u1, N_k) as p:
        if weighted:
            p.set_sample_weights(w)
        _results(p, f)
        p.upload(u2)
        got = _results(p, f)
    with lib.DeviceProblem(u2, N_k) as q:
        if weighted:
            q.set_sample_weights(w)
        want = _results(q, f)
    for a, b in zip(got, want):
        assert_bits(a, b, "re-upload vs fresh")


def test_synthesize_into_weighted_context(lib):
    K, N = 8, 4000
    N_k = np.full(K, N / K)
    O, k = np.linspace(1.0, 5.0, K), np.linspace(1.0, 3.0, K)
    u, _ = energies(K, N, 11)
    w = np.random.default_rng(12).integers(0, 4, N).astype(float)
    f = np.linspace(0.0, 0.5, K)
    with lib.DeviceProblem(u, N_k) as p:
        p.set_sample_weights(w)
        p.synthesize(O, k, seed=3)
        got = _results(p, f)
    with lib.DeviceProblem(None, N_k, N_local=N) as q:
        q.synthesize(O, k, seed=3)
        q.set_sample_weights(w)
        want = _results(q, f)
    for a, b in zip(got, want):
        assert_bits(a, b, "synthesize into a weighted context vs fresh")


def test_rejected_upload_leaves_no_trace(lib):
    case = E.with_unsampled(2500.0, sign=-1.0)
    u_bad, N_k = case["u"].copy(), case["N"]
    u_bad[1, 17] = np.nan
    good = E.with_unsampled(5.0, sign=-1.0)["u"]
    f = np.array([0.0, 5.0, -5.0])
    with lib.DeviceProblem(None, N_k, N_local=u_bad.shape[1]) as p:
        with pytest.raises(err(lib)) as e:
            p.upload(u_bad)
        assert e.value.status == ERR_NAN
        p.upload(good)
        got = (p.self_consistent_update(f), p.last_kernels()["pass_kernel"])
    with lib.DeviceProblem(good, N_k) as q:
        want = (q.self_consistent_update(f), q.last_kernels()["pass_kernel"])
    assert got[1] == want[1]
    assert_bits(got[0], want[0], "after a rejected upload vs fresh")


def test_parked_buffers_behave_like_fresh(lib):
    K, N = 32, 5000
    u, N_k = energies(K, N, 13, unsampled=(3,))
    f = np.linspace(0.0, 1.0, K)

    def run():
        with lib.DeviceProblem(None, N_k, N_local=N) as p:
            p.upload(u)
            assert_bits(p.download(), D.download_image(u, N_k), "download")
            return _results(p, f)

    lib.trim()
    want = run()
    for Kp, Np in ((40, 5000), (16, 10000)):         # larger, and differently shaped, predecessors
        lib.trim()
        junk, Nj = energies(Kp, Np, 14, unsampled=(0,))
        with lib.DeviceProblem(junk * 7.0 - 100.0, Nj) as pred:
            pred.streaming_pass(np.zeros(Kp))
        for a, b in zip(run(), want):
            assert_bits(a, b, f"context on parked buffers of [{Kp}, {Np}]")
    lib.trim()
    for a, b in zip(run(), want):
        assert_bits(a, b, "after trim()")


# ------------------------------------------------------------------------------------- 7. fresh-context sequences
def _small():
    case = E.with_unsampled(5.0, sign=-1.0, n=48)
    return case["u"], case["N"]


FIRST_CALLS = {
    "sci_iterate(f, 0)": lambda p, f: p.sci_iterate(f, 0),
    "sci_iterate(f, 1)": lambda p, f: p.sci_iterate(f, 1),
    "solve_sci": lambda p, f: p.solve_sci(f),
    "solve_adaptive": lambda p, f: p.solve_adaptive(f),
    "pass_multi": lambda p, f: p.pass_multi(np.stack([f, f + 0.1])),
    "log_W_nk": lambda p, f: p.log_W_nk(f),
    "weight_moments": lambda p, f: p.weight_moments(f),
    "bin_moments": lambda p, f: p.bin_moments(f, np.zeros(p.N), np.arange(p.N) % 3, 3),
    "last_pass_ms": lambda p, f: p.last_pass_ms(),
    "last_loop_ms": lambda p, f: p.last_loop_ms(),
    "last_hessian_ms": lambda p, f: p.last_hessian_ms(),
}


@pytest.mark.parametrize("first", list(FIRST_CALLS))
def test_fresh_context_then_gradient(lib, first):
    u, N_k = _small()
    f = np.array([0.0, 4.0, -3.0])
    s = N_k > 0
    with lib.DeviceProblem(u, N_k) as p:
        FIRST_CALLS[first](p, f)
        g = p.gradient(f)
    np.testing.assert_allclose(g[s], orc.mbar_gradient(u[s], N_k[s], f[s]), rtol=0, atol=1e-10)


def test_sci_iterate_zero_then_one(lib):
    u, N_k = _small()
    s = N_k > 0
    f0 = np.array([0.0, 4.0, -3.0])
    with lib.DeviceProblem(u, N_k) as p:
        assert_bits(p.sci_iterate(f0, 0), f0, "zero iterations")
        f1 = p.sci_iterate(f0, 1)
    nxt = orc.self_consistent_update(u[s], N_k[s], f0[s])
    np.testing.assert_allclose(f1[s], nxt - nxt[0], rtol=0, atol=1e-10)
    assert f1[2] == f0[2]


# ------------------------------------------------------------------------------------- 8. the clamp
def _match_or_range(lib, fn, check):
    """Either the result matches the reference, or the call is refused with ERR_RANGE; never another answer."""
    try:
        out = fn()
    except err(lib) as e:
        assert e.status == ERR_RANGE, e
        return False
    check(out)
    return True


@pytest.mark.parametrize("c", [9.99e5, 1.0e6, 2.0e6, np.inf])
@pytest.mark.parametrize("how", ["unsampled", "appended"])
def test_energies_at_and_past_the_clamp(lib, c, how):
    u0 = E.base_samples(128, 21)
    u = np.stack([u0, u0 + 5.0, u0 + c])
    N_k = np.array([64.0, 64.0, 0.0])
    s = N_k > 0
    f_s = np.array([0.0, 5.0])
    f = np.array([0.0, 5.0, c if np.isfinite(c) else 0.0])
    scale = 1e-13 * max(1.0, abs(f[2]))
    ref_f = orc.self_consistent_update(u, N_k, f)
    ref_lw = orc.mbar_log_W_nk(u, N_k, f)
    ref_W = np.exp(ref_lw)
    if how == "unsampled":
        p = lib.DeviceProblem(u, N_k)
        extra = None
    else:
        extra = lib.DeviceProblem(u[:2], N_k[:2])
        p = extra.augmented(u[2:])
    try:
        def check_f(out):
            np.testing.assert_allclose(out[s], ref_f[s], rtol=0, atol=1e-10)
            if np.isfinite(ref_f[2]):
                np.testing.assert_allclose(out[2], ref_f[2], rtol=0, atol=1e-10 + 8 * scale * 1e3)
            else:
                assert out[2] == ref_f[2]

        def check_moments(out):
            S, G = out
            want_S = ref_W.sum(axis=0)
            np.testing.assert_allclose(S, want_S, rtol=1e-9, atol=0)
            np.testing.assert_allclose(G, ref_W.T @ ref_W, rtol=1e-9, atol=1e-300)

        def check_lw(out):
            fin = np.isfinite(ref_lw)
            assert np.array_equal(np.isfinite(out), fin)
            np.testing.assert_allclose(out[fin], ref_lw[fin], rtol=0, atol=1e-9)
            assert np.all(out[~fin] == ref_lw[~fin])

        answered = [
            _match_or_range(lib, lambda: p.self_consistent_update(f), check_f),
            _match_or_range(lib, lambda: p.weight_moments(f), check_moments),
            _match_or_range(lib, lambda: p.log_W_nk(f), check_lw),
        ]
        if c == 9.99e5 or c == np.inf:
            assert all(answered), answered          # inside the stored range: must answer
        if c == 2.0e6:
            assert not any(answered), answered      # 1e6 past every shift: must refuse
        # sampled-state entry points never read the unsampled row
        np.testing.assert_allclose(p.gradient(f)[s], orc.mbar_gradient(u[s], N_k[s], f_s), rtol=0, atol=1e-10)
        if how == "appended":
            from pymbar_b200 import expectations as ex

            def run():
                return ex.expectations_inner(u[:2], N_k[:2], f_s, np.ones((1, u.shape[1])), u[2:], [0],
                                             problem=extra)

            def check_exp(out):
                # (the appended state's f does not depend on its own entry of f)
                if np.isfinite(ref_f[2]):
                    np.testing.assert_allclose(out["f"][0], ref_f[2], rtol=1e-13, atol=1e-10)
                else:
                    assert out["f"][0] == ref_f[2]

            _match_or_range(lib, run, check_exp)
    finally:
        p.close()
        if extra is not None:
            extra.close()


@pytest.mark.parametrize("how", ["unsampled", "appended", "sampled"])
def test_minus_inf_energy_is_rejected(lib, how):
    u0 = E.base_samples(128, 23)
    u = np.stack([u0, u0 + 5.0, u0 - 1.0])
    N_k = np.array([64.0, 64.0, 0.0])
    u[2 if how != "sampled" else 1, 40] = -np.inf   # (lane 8 of its tile: every lane must report)
    with pytest.raises(err(lib)) as e:
        if how == "appended":
            with lib.DeviceProblem(u[:2], N_k[:2]) as b:
                b.augmented(u[2:]).close()
        else:
            lib.DeviceProblem(u, N_k).close()
    assert e.value.status == ERR_NAN
    assert ("no finite energy" in str(e.value)) == (how == "sampled")
    assert ("-inf" in str(e.value)) == (how != "sampled")


# ------------------------------------------------------------------------------------- 9. device-pointer ordering
def test_device_upload_is_ordered_after_torch_copy(lib, big):
    import torch

    u, N_k = big["u"], big["N_k"]
    host = torch.from_numpy(u).pin_memory()
    t = torch.empty((K_BIG, N_BIG), dtype=torch.float64, device="cuda")
    t.fill_(np.nan)
    torch.cuda.synchronize()
    with lib.DeviceProblem(None, N_k, N_local=N_BIG) as p:
        t.copy_(host, non_blocking=True)            # on torch's current stream, no synchronisation after it
        p.upload_device_ptr(t.data_ptr(), N_BIG)
        assert_bits(p.download(), big["image"], "device upload after a non-blocking copy")

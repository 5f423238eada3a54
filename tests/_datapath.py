"""numpy restatements of what the device stores when u_kn moves in and out of HBM (ctx.cu, logw.cu).

* `upload_image` / `download_image`: the per-sample shift x_n = min over sampled k of u_kn, the stored
  u'_kn = min(u_kn - x_n, 1e6) (`retile_kernel`, `append_rows_kernel`), the per-row lowest shifted energy rounded
  down (`row_min_push`), the per-row flag of finite energies at or past 1e6 - 800 and the rows of +inf only
  (`row_clamp_push`).  `download()` returns
  u' + x.  Both the image and its inverse are single IEEE operations on host and device alike, so a download is
  compared bit for bit.
* The chunk geometry of every copy loop (`ensure_staging`, `mbar_b200_download_u_kn`, `launch_logw`,
  `mbar_b200_create_augmented`), so a test can assert that its shape reaches the number of chunks it was chosen for.
* `synth`: `synth_kernel` — Philox-4x32-10 (counter = global sample index, key = seed), 53-bit uniforms,
  Box-Muller with cospi, the state of origin from the cumulative N_k, the per-sample shift over sampled states and
  the clamp.  The device's log, cospi and rsqrt are not correctly rounded: `synth_tolerance` states the bound.

tests/test_datapath_cpu.py checks these restatements; tests/test_gpu_datapath.py checks the device against them.
"""
import numpy as np

TILE_N = 32
U_CLAMP = 1.0e6
U_NEAR_CLAMP = U_CLAMP - 800.0      # a finite shifted energy from here up flags its row (internal.cuh)
EPS = np.finfo(np.float64).eps


# ---------------------------------------------------------------------------------------------- upload image
def upload_image(u, N_k):
    """dict(x [N], up [K, N], rowmin [K], clamped [K]) of u [K, N] as an upload stores it.

    rowmin[k] = min over n of floor(u'_kn) where negative (floored at -2^30), else 0: only an unsampled row can
    lie below its sample's shift.  clamped[k]: some finite u_kn - x_n >= 1e6 - 800; far[k]: every entry is (an unsampled row
    with both cannot be answered: ERR_RANGE); allinf[k]: the row is +inf only."""
    u = np.asarray(u, np.float64)
    s = np.asarray(N_k, np.float64) > 0
    x = u[s].min(axis=0)
    d = u - x
    up = np.minimum(d, U_CLAMP)
    with np.errstate(invalid="ignore"):
        neg = np.where(up < 0.0, np.maximum(np.floor(up), -1073741824.0), 0.0)
    rowmin = neg.min(axis=1)
    clamped = np.any(np.isfinite(d) & (d >= U_NEAR_CLAMP), axis=1)
    far = np.all(d >= U_NEAR_CLAMP, axis=1)
    return dict(x=x, up=up, rowmin=rowmin, clamped=clamped, far=far, allinf=np.all(np.isposinf(d), axis=1))


def download_image(u, N_k):
    """What `download()` returns after uploading u: u' + x, bit for bit."""
    im = upload_image(u, N_k)
    return im["up"] + im["x"]


def appended_image(u_base, N_k, u_extra):
    """`download()` of base.augmented(u_extra): the appended rows are shifted by the base's x_n and clamped."""
    x = upload_image(u_base, N_k)["x"]
    return np.vstack([download_image(u_base, N_k), np.minimum(np.asarray(u_extra, np.float64) - x, U_CLAMP) + x])


# ---------------------------------------------------------------------------------------------- chunk geometry
def ceil_div(a, b):
    return -(-a // b)


def upload_stage_cols(K, N):
    """`ensure_staging`: columns per upload chunk, ~64 MiB per staging buffer in whole tiles, at most the padded N."""
    cols = (64 << 20) // (8 * K)
    cols = cols // TILE_N * TILE_N
    cols = max(cols, TILE_N)
    return min(cols, ceil_div(N, TILE_N) * TILE_N)


def upload_chunks(K, N):
    return ceil_div(N, upload_stage_cols(K, N))


def upload_serial_pack(K, N, chunk):
    """Whether pageable chunk `chunk` is packed by the calling thread alone (fewer than 2^16 elements)."""
    cols = upload_stage_cols(K, N)
    w = min(cols, N - chunk * cols)
    return w * K < (1 << 16)


def download_cols(K, n):
    """`mbar_b200_download_u_kn`: columns per download chunk for a slice of n columns."""
    max_cols = (32 << 20) // (8 * K) // TILE_N * TILE_N + TILE_N
    return min(n, max_cols)


def download_chunks(K, n):
    return ceil_div(n, download_cols(K, n))


def logw_rows_per_chunk(K, n):
    """`launch_logw`: rows of log W per chunk (whole tiles, ~64 MiB) for a request of n rows."""
    tiles = ceil_div(n, TILE_N)
    tpc = max(1, (64 << 20) // (K * TILE_N * 8))
    return min(tpc, tiles) * TILE_N


def logw_chunks(K, n):
    tiles = ceil_div(n, TILE_N)
    return ceil_div(tiles, logw_rows_per_chunk(K, n) // TILE_N)


def append_cols(E, N):
    """`mbar_b200_create_augmented`: columns per chunk of the E appended rows (~32 MiB, whole tiles)."""
    cols = (32 << 20) // (8 * E)
    cols = max(cols // TILE_N * TILE_N, TILE_N)
    return min(cols, ceil_div(N, TILE_N) * TILE_N)


def append_chunks(E, N):
    return ceil_div(N, append_cols(E, N))


# ---------------------------------------------------------------------------------------------- synthesis
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox-4x32-10 on uint32 arrays (Salmon et al., SC'11), the rounds of `philox4x32_10` in ctx.cu."""
    c = [np.asarray(v, np.uint32).copy() for v in (c0, c1, c2, c3)]
    k0, k1 = np.uint32(k0), np.uint32(k1)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = c[0].astype(np.uint64) * _M0
            p1 = c[2].astype(np.uint64) * _M1
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & _LO).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & _LO).astype(np.uint32)
            c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
            k0 = np.uint32(k0 + _W0)
            k1 = np.uint32(k1 + _W1)
    return c


def cospi(t):
    """cos(pi t), reduced exactly to [0, 1/4] first (a few ulp; np.cos(np.pi * t) loses more near the zeros)."""
    t = np.abs(np.asarray(t, np.float64)) % 2.0
    t = np.where(t > 1.0, 2.0 - t, t)                 # cos(pi t) = cos(pi (2 - t))
    sign = np.where(t > 0.5, -1.0, 1.0)
    t = np.where(t > 0.5, 1.0 - t, t)                 # cos(pi t) = -cos(pi (1 - t))
    out = np.where(t <= 0.25, np.cos(np.pi * t), np.sin(np.pi * (0.5 - t)))
    return sign * out


def origin(N_k, g):
    """State of origin of global sample g: the largest s < K with cumN[s] <= g (empty states are skipped)."""
    cum = np.concatenate([[0.0], np.cumsum(np.asarray(N_k, np.float64))])
    K = len(N_k)
    return np.minimum(np.searchsorted(cum[:K], np.asarray(g, np.float64), side="right") - 1, K - 1)


def synth(O_k, k_k, N_k, seed, n_offset, N_local, N_global):
    """u [K, N_local] (original frame, as `download()` returns it) of the samples [n_offset, n_offset + N_local) of
    the synthetic family, and dict(x, z, s, state, shift) for the tolerance.  The state of origin follows the
    cumulative N_k, so N_global (what the caller passes to `synthesize`) must be their sum."""
    O_k, k_k, N_k = (np.asarray(a, np.float64) for a in (O_k, k_k, N_k))
    assert N_global == N_k.sum(), "N_global must be the sum of N_k"
    g = np.arange(n_offset, n_offset + N_local, dtype=np.uint64)
    seed = int(seed)
    r = philox4x32_10((g & _LO).astype(np.uint32), (g >> np.uint64(32)).astype(np.uint32), 0, 0,
                      seed & 0xFFFFFFFF, seed >> 32)
    r64 = [v.astype(np.uint64) for v in r]
    u1 = (((r64[0] << np.uint64(32)) | r64[1]) >> np.uint64(11)).astype(np.float64)
    u2 = (((r64[2] << np.uint64(32)) | r64[3]) >> np.uint64(11)).astype(np.float64)
    u1 = (u1 + 0.5) * 2.0 ** -53
    u2 = (u2 + 0.5) * 2.0 ** -53
    z = np.sqrt(-2.0 * np.log(u1)) * cospi(2.0 * u2)
    st = origin(N_k, g)
    sc = 1.0 / np.sqrt(k_k[st])
    x = O_k[st] + z * sc
    d = x[None, :] - O_k[:, None]
    e = 0.5 * k_k[:, None] * d * d
    sh = e[N_k > 0].min(axis=0)
    u = np.minimum(e - sh, U_CLAMP) + sh
    return u, dict(x=x, z=z, s=sc, state=st, shift=sh, d=d, k=k_k)


def synth_tolerance(aux):
    """Bound on |download() - synth()| per entry.  z carries the device's log (1 ulp), cospi (2 ulp) and two
    roundings, the scale its rsqrt (2 ulp): |dx| <= 8 eps |z s| + eps |x|; then u = k d^2 / 2 moves by k |d| |dx| and
    the shift, its subtraction and the re-addition round at most 4 times: 4 eps (u + shift).  Twice that is allowed."""
    x, zs = np.abs(aux["x"]), np.abs(aux["z"] * aux["s"])
    dx = EPS * (8.0 * zs + x)
    u = 0.5 * aux["k"][:, None] * aux["d"] ** 2
    return 2.0 * (aux["k"][:, None] * np.abs(aux["d"]) * dx[None, :] + 4.0 * EPS * (u + aux["shift"][None, :]))

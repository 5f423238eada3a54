"""Up to 2048 states: the fused pass's launch plan, its variant matrix, and the state-constant reads of its CTAs.

`fused_plan` restates `fused_prepare` and `fused_enqueue` (pass_fused.cu): the cluster size CL, the states per CTA Kh,
the warps per sample group Wk and sample groups per CTA Wn, the register rows per warp Rw and the instantiated R, the
FULL / MASKED and MODE choice, tiles per warp per stage TPW, the ring (stage bytes with the padding for masked reads, NS
stages) and the grid, and the exact `last_kernels()["pass_kernel"]` string the launch prints.  `instantiations` lists
the 90 kernels the three PICK tables of `fused_enqueue` can launch, `variant_matrix` the cases that reach each of them
in each sample-count regime, and `constant_reads` what each CTA of a cluster initialises of its state constants and
what its warps read.  The extended-precision reference and the tolerances are those of tests/_large_k.py: a plan
carries the `depth` entries its reduction and tolerance functions read.
"""
import numpy as np

from tests import _large_k as LK

K_MAX = LK.FUSED_K_MAX
SPREAD_MAX = 1200.0          # FUSED_SPREAD: max c - min c the fused pass accepts
SPREAD_MULT = 600.0          # above this the state constant enters the exponent (MODE = 1)
LOG_EPS_UNSAMPLED = -80.0    # log of the count an unsampled state carries in an all-state pass
SMEM = 225 * 1024            # dynamic shared memory the plan may take, less 16 KB for the exp table
TILE = 32

# fused_enqueue's PICK tables: (R, CL, first id) per table
PICK = ((8, 1, 0), (16, 1, 4), (32, 1, 8), (32, 2, 12), (32, 4, 16), (32, 8, 20),
        (24, 1, 60), (24, 2, 64), (24, 4, 68), (24, 8, 72))
PICKW = ((32, 1, 24), (32, 2, 28), (32, 4, 32), (32, 8, 36), (16, 1, 52), (8, 1, 56),
         (24, 1, 76), (24, 2, 80), (24, 4, 84), (24, 8, 88))
PICKM = ((8, 1, 40), (16, 1, 42), (16, 2, 44), (16, 4, 46), (16, 8, 48))


def slots(CL):
    return CL * 8 if CL > 1 else 16


def smem_header(K, CL, M=1):
    """fused_smem_header: tab | c_s[M][K + 32] | xD | sred | sumL | bad | mbarriers, 128-byte aligned."""
    b = 256 + M * ((K + 32) * 8 + 2 * slots(CL) * 32 * 8 + 256 * 8 + 128 + 128) + 64 + 64
    return (b + 127) & ~127


def mode_of(spread):
    """fused_mode without the development switch: 3 (multiplicative constant) up to a spread of 600, else 1."""
    return 1 if spread > SPREAD_MULT else 3


def r_of(Rw, M):
    return 8 if Rw <= 8 else 16 if Rw <= 16 else 24 if (Rw <= 24 and M == 1) else 32


def geometry(K, M=1):
    """CL, Kh, Wk, Wn, Rw and R of a K-state launch with M candidates (independent of N)."""
    rmax = 16 if M == 2 else 32
    per = 8 * rmax
    CL = 8 if K > 4 * per else 4 if K > 2 * per else 2 if K > per else 1
    Kh = -(-K // CL)
    if CL > 1:
        Kh = (Kh + 1) & ~1
    Wk = 1
    while Wk * rmax < Kh:
        Wk *= 2
    Rw = -(-Kh // Wk)
    Rw = (Rw + 1) & ~1
    return dict(CL=CL, Kh=Kh, Wk=Wk, Wn=8 // Wk, Rw=Rw, R=r_of(Rw, M))


def full_shape(K, M=1):
    """True when every warp of every CTA owns exactly R states (the FULL family, given all rows take part)."""
    g = geometry(K, M)
    return g["Rw"] == g["R"] and K == g["CL"] * g["Wk"] * g["Rw"]


def ring(K, M=1):
    """TPW, stageBytes and NS (fused_prepare), or None when fewer than two stages fit."""
    g = geometry(K, M)
    cta = g["Kh"] * TILE * 8
    tpw = 65536 // (g["Wn"] * cta)
    TPW = min(8, max(1, tpw))
    stage = g["Wn"] * TPW * cta
    over = (g["Wk"] - 1) * g["Rw"] + g["R"] - g["Kh"]      # masked reads past the CTA's last state
    if over > 0:
        stage += over * TILE * 8
    stage = (stage + 127) & ~127
    header = smem_header(K, g["CL"], M)
    ns = (SMEM - header - 16384) // stage
    while ns < 2 and TPW > 1:
        pad = stage - g["Wn"] * TPW * cta
        TPW //= 2
        stage = ((g["Wn"] * TPW * cta + pad) + 127) & ~127
        ns = (SMEM - header - 16384) // stage
    NS = min(8, ns)
    if NS < 2:
        return None
    return dict(TPW=TPW, stageBytes=stage, NS=NS, header=header)


def fused_plan(K, N, *, M=1, all_states=False, want_w=False, weighted=False, n_active=None, spread=0.0,
               sm_count=132, m2_clusters=False):
    """The launch of one fused pass, or None where fused_prepare declines.  `spread` is max c - min c over the rows
    that take part (every row in an all-state pass); `n_active` the sampled states (default K); `want_w` a pass
    that feeds the Hessian (streaming_pass(want_G) / hessian); `m2_clusters` the MBAR_B200_M2_CLUSTERS switch."""
    n_active = K if n_active is None else n_active
    if K > K_MAX or not spread < SPREAD_MAX:
        return None
    mode = mode_of(spread)
    if M == 2 and (mode != 3 or K > 1024 or K < 2 or all_states or want_w):
        return None
    if M == 2 and K > 128 and not m2_clusters:
        return None
    g = geometry(K, M)
    r = ring(K, M)
    if r is None:
        return None
    n_tiles = -(-int(N) // TILE)
    tps = g["Wn"] * r["TPW"]
    n_stages = -(-n_tiles // tps)
    groups = min(n_stages, sm_count // g["CL"])
    grid = groups * g["CL"]
    R, CL = g["R"], g["CL"]
    full = full_shape(K, M) and (n_active == K or all_states) and not weighted
    wst = want_w and not all_states and M == 1
    table = PICKM if M == 2 else (PICKW if wst else PICK)
    base = next(i for (r_, c_, i) in table if r_ == R and c_ == CL)
    if M == 2:
        which = base + (1 if full else 0)
    else:
        which = base + (2 if full else 0) + (1 if mode == 3 else 0)
    desc = "LDS table + multiplicative state constant" if mode == 3 else "LDS table"
    extra = ", M=2 (two candidates per launch)" if M == 2 else ", WST (weights stored for the Hessian)" if wst else ""
    name = (f"pass_fused_kernel<R={R}, {'FULL' if full else 'MASKED'}, CW=8, BATCH=8, MODE={mode} ({desc}), "
            f"CL={CL}{extra}> grid={grid} NS={r['NS']} TPW={r['TPW']}")
    stages_per_group = -(-n_stages // groups)
    tiles_per_lane = stages_per_group * r["TPW"]
    # S_k: a lane's tiles, the warp butterfly, the Wn sample groups of a CTA, the CTA groups in order
    depth = tiles_per_lane + 5 + g["Wn"] + groups
    # sum L: the same chain over the 8 warps of a CTA (one per sample group carries it), and the final + sumW mid
    sumL_depth = tiles_per_lane + 5 + 8 + groups + 2
    return dict(g, K=K, N=int(N), M=M, mode=mode, full=full, wst=wst, TPW=r["TPW"], stageBytes=r["stageBytes"],
                NS=r["NS"], header=r["header"], n_tiles=n_tiles, tiles_per_stage=tps, n_stages=n_stages,
                groups=groups, grid=grid, which=which, name=name, stages_per_group=stages_per_group,
                depth=depth, sumL_depth=sumL_depth, logprod=not weighted,
                inst=(R, CL, full, mode, wst, M))


# ---- the 90 instantiations --------------------------------------------------------------------------------------------
def instantiations():
    """{(R, CL, FULL, MODE, WST, M): sorted K values whose geometry reaches it}.  MODE and the MASKED family reach
    every K (a spread above 600, an unsampled row or multiplicities); FULL needs a FULL shape."""
    out = {}
    for M, tables in ((1, (PICK, PICKW)), (2, (PICKM,))):
        for table in tables:
            for (R, CL, _) in table:
                wst = table is PICKW
                for full in (False, True):
                    for mode in ((3,) if M == 2 else (1, 3)):
                        out[(R, CL, full, mode, wst, M)] = []
    for M in (1, 2):
        for K in range(2 if M == 2 else 1, (1024 if M == 2 else K_MAX) + 1):
            g = geometry(K, M)
            for key in out:
                R, CL, full, mode, wst, m = key
                if m == M and R == g["R"] and CL == g["CL"] and (not full or full_shape(K, M)):
                    out[key].append(K)
    return out


def bands(M=1):
    """[(R, CL, K_first, K_last)]: the runs of K with one (R, CL)."""
    out = []
    for K in range(2 if M == 2 else 1, (1024 if M == 2 else K_MAX) + 1):
        g = geometry(K, M)
        if out and out[-1][:2] == [g["R"], g["CL"]]:
            out[-1][3] = K
        else:
            out.append([g["R"], g["CL"], K, K])
    return [tuple(b) for b in out]


# ---- state constants: what a CTA initialises and what its warps read --------------------------------------------------
def constant_reads(K, M=1, pad=None):
    """Per CTA of the cluster: (highest c_s index a warp reads, highest index the CTA initialises).  `pad` restates
    the kernel's zeroing: None for the current one (up to max(Kl + 32, (Wk - 1) Rw + R)), an int for a fixed count
    past Kl (32 before the fix)."""
    g = geometry(K, M)
    out = []
    for half in range(g["CL"]):
        Kl = max(0, min(g["Kh"], K - half * g["Kh"])) if g["CL"] > 1 else K
        read = (g["Wk"] - 1) * g["Rw"] + g["R"] - 1
        end = max(Kl + 32, read + 1) if pad is None else Kl + pad
        out.append((read, end - 1))
    return out


def kernel_zeroing(path=None):
    """The zeroing of c_s past Kl that pass_fused.cu compiles, in the form `constant_reads` takes: None for 32 entries
    and, in the masked variants (the FULL ones read their own rows only), on up to (Wk - 1) Rw + R; an int n for a
    fixed n entries.  Anything else is an error: the restatement has to be brought up to date with the kernel."""
    import os
    import re

    path = path or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pymbar_b200", "csrc",
                                "pass_fused.cu")
    src = open(path).read()
    m = re.search(r"for \(int i = threadIdx\.x; i < (\d+); i \+= blockDim\.x\) c_s\[Kl \+ i\] = 0\.0;", src)
    if m and re.search(r"if constexpr \(!FULL\)\s+for \(int i = Kl \+ " + m.group(1) + r" \+ threadIdx\.x; "
                       r"i < \(p\.Wk - 1\) \* p\.Rw \+ R; i \+= blockDim\.x\) c_s\[i\] = 0\.0;", src):
        assert m.group(1) == "32", m.group(0)
        return None
    if m:
        return int(m.group(1))
    raise AssertionError("pass_fused.cu: zeroing of the state constants past Kl not recognised")


def overrun_ks(M=1, pad=32):
    """K <= 2048 (<= 1024 for M = 2) at which some CTA reads a constant it did not initialise under `pad`."""
    top = 1024 if M == 2 else K_MAX
    return [K for K in range(2 if M == 2 else 1, top + 1)
            if any(r > i for r, i in constant_reads(K, M, pad=pad))]


# ---- sample counts --------------------------------------------------------------------------------------------------
REGIMES = LK.REGIMES


def regime_n(K, regime, M=1, sm_count=132):
    """A sample count N (never a multiple of 32) that gives fewer stages than CTA groups ('few'), one stage per group
    ('one', the last tile partial), or at least 2 NS + 1 stages per group with a partial last stage ('several': every
    ring slot wraps at least twice)."""
    g = geometry(K, M)
    r = ring(K, M)
    G = sm_count // g["CL"]
    tps = g["Wn"] * r["TPW"]
    if regime == "few":
        return TILE * tps * max(1, G // 3) - 7
    if regime == "one":
        return TILE * tps * G - 11
    return TILE * (tps * (2 * r["NS"] + 1) * G + max(1, tps // 2)) - 11


def stages_per_group(K, N, M=1, sm_count=132):
    g = geometry(K, M)
    r = ring(K, M)
    n_stages = -(-(-(-N // TILE)) // (g["Wn"] * r["TPW"]))
    groups = min(n_stages, sm_count // g["CL"])
    return n_stages, groups


# ---- the case matrix ------------------------------------------------------------------------------------------------
CONTENTS = ("plain", "unsampled", "mult")


def c_spread(f, N_k, all_states):
    """max c - min c with c = f + log N_k over the sampled rows (every row, unsampled at log N = -80, when
    all_states)."""
    N_k = np.asarray(N_k, np.float64)
    s = N_k > 0
    c = np.where(s, f + np.log(np.where(s, N_k, 1.0)), f + LOG_EPS_UNSAMPLED)
    c = c if all_states else c[s]
    return float(np.max(c) - np.min(c))


def case_sampling(K, N, content):
    """(unsampled state indices, ladder gaps, N_k) of a case: 'unsampled' leaves state K // 2 without samples; fewer
    samples than states leave about N / 1.5 evenly spread states sampled on a ladder compressed to 200 units
    (the permutation strings unsampled states together: every one of them stays within reach of a sample).
    The fused all-state pass hands an unsampled row whose S leaves (1e-250, 1e12) to the generic kernel."""
    import tests._moments as M_

    if N < K:
        uns = LK.few_sampled(K, N, 0)
        gaps = (min(39.0, 200.0 / K),)
    elif content == "unsampled" and K > 1:
        # an all-state pass needs the unsampled state's S inside (1e-250, 1e12), and with MODE 1 its raw sum
        # e^-80 N S above the floor test's 2^53 N 2^-1020 e^(mid - c_min) ~ N e^-260: gaps of at most 12 keep the
        # state within about e^-80 of its neighbours' samples
        uns = (K // 2,)
        gaps = tuple(min(g, 12.0) for g in M_.GAPS)
    else:
        uns = ()
        gaps = M_.GAPS
    sampled = np.ones(K, bool)
    sampled[list(uns)] = False
    N_k = np.zeros(K)
    N_k[sampled] = LK._counts(int(sampled.sum()), N / sampled.sum())
    return tuple(uns), gaps, N_k


def case_plans(K, N, M, mode, content, sm_count=132):
    """[(entry point, plan)] of one case, with a nominal spread for its MODE (the case's own data decide the actual
    one; the test asserts that it gives the same MODE).  'pass': streaming_pass, gradient, objective,
    log_denominator, sci_iterate; 'update': self_consistent_update (all states when some are unsampled); 'weights':
    streaming_pass(want_G); 'pass_multi' (M = 2 cases)."""
    spread = 800.0 if mode == 1 else 10.0
    n_act = int(np.sum(case_sampling(K, N, content)[2] > 0))
    w = content == "mult"
    kw = dict(n_active=n_act, weighted=w, spread=spread, sm_count=sm_count)
    out = [("pass", fused_plan(K, N, **kw)),
           ("update", fused_plan(K, N, all_states=(n_act < K), **kw)),
           ("weights", fused_plan(K, N, want_w=True, **kw))]
    if M == 2:
        out.append(("pass_multi", fused_plan(K, N, M=2, m2_clusters=True, **kw)))
    return out


def variant_matrix(sm_count=132):
    """(K, regime, M, mode, content) cases.  Per (R, CL) band: both K edges, and for a band with FULL shapes one of
    them; MODE 3 in every regime, MODE 1 in one regime rotating over the K values.  A FULL K runs 'plain' (FULL,
    FULL WST) and one of 'unsampled' (MASKED, FULL all-state update) / 'mult' (weighted MASKED) in every regime;
    any other K runs one content per regime, rotating.  M = 2 cases run the M = 1 entry points too."""
    rows = []
    i = 0
    for M in (1, 2):
        for (R, CL, k0, k1) in bands(M):
            fulls = [K for K in range(k0, k1 + 1) if full_shape(K, M)]
            ks = sorted({k0, k1} | ({fulls[len(fulls) // 2]} if fulls else set()))
            for K in ks:
                i += 1
                for j, regime in enumerate(REGIMES):
                    if full_shape(K, M):
                        contents = ("plain", ("unsampled", "mult")[(i + j) % 2])
                    else:
                        contents = (CONTENTS[(i + j) % 3],)
                    if K == 1:
                        contents = tuple(c for c in contents if c != "unsampled") or ("mult",)
                    rows += [(K, regime, M, 3, c) for c in contents]
                if M == 1 and K > 2:             # MODE 1 needs two sampled states whose constants differ
                    # (a FULL K needs a sample per state for its FULL pass: a regime with at least K samples)
                    regs = [r for r in REGIMES if not full_shape(K, M) or regime_n(K, r, M, sm_count) >= K]
                    regime = regs[i % len(regs)]
                    other = ("unsampled", "mult")[i % 2]
                    contents = ("plain", other) if full_shape(K, M) else (("plain",) + CONTENTS[1:])[i % 3:][:1]
                    rows += [(K, regime, M, 1, c) for c in contents]
    return rows


def matrix_coverage(rows, sm_count=132):
    """{instantiation: set of regimes} over every entry point of every case."""
    cov = {}
    for (K, regime, M, mode, content) in rows:
        N = regime_n(K, regime, M, sm_count)
        for _, plan in case_plans(K, N, M, mode, content, sm_count):
            if plan is not None:
                cov.setdefault(plan["inst"], set()).add(regime)
    return cov

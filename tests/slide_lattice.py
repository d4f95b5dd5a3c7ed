"""The tensor-core SlidingScorer's index arithmetic restated in Python, and the case tables of
tests/test_gpu_slide_lattice.py.  No GPU and no library: tests/test_slide_lattice_host.py uses the mirror to show that
the tables reach every window phase, the exact / tensor-core split, every split point of the projection's ring wrap and
a front-end ring store across slot L.

Each function names the C++ it restates (csrc/b2cnn_slide.cu, csrc/b2cnn_tc.cu, csrc/b2cnn_tc_fused.cuh).  Sample
indices are stream indices: push n (from 1) carries samples [(n - 1) S, n S), window n is [n S - W, n S)."""
from collections import namedtuple

R_OF = {"mycnn5": 24, "mycnn3": 16}          # receptive field of a feature in samples (slide_create: s->R)
FOFF_OF = {"mycnn5": 3, "mycnn3": 2}         # step j of the stream emits features 2j - foff, 2j - foff + 1
SPLIT = 32                                   # tc_ring_block (slide_push / slide_admit): Q >= 32 features run on tensor cores
W_OF_PHI = {0: 1532, 3: 1533, 2: 1530, 1: 1531}


def fdiv4(a):
    """fdiv(a, 4): floor division"""
    return a // 4


def cdiv4(a):
    """-fdiv(-a, 4): ceiling division (slide_admit's g_lo)"""
    return -((-a) // 4)


def phi_of(W):
    """slide_create: s->phi = (F - W % F) % F with F = 4, stream feature g starts at sample 4 g + phi"""
    return (4 - W % 4) % 4


def L_of(kind, W):
    return (W - R_OF[kind]) // 4 + 1


def n0_of(W, S):
    """the first push with a complete window: n S >= W"""
    return -(-W // S)


def window_head(kind, W, S, n):
    """window_head: G_n = fdiv(n S - W - phi, 4), window n's first stream feature"""
    return fdiv4(n * S - W - phi_of(W))


def push_lattice(kind, W, S, n1, g_done):
    """slide_push for push n1 (from 1) after a push whose last computed feature was g_done (-1: none):
    {g_hi, g_m0, g_lo, Q, tc, slot0, g_done} (g_done after the push)"""
    R, phi, L = R_OF[kind], phi_of(W), L_of(kind, W)
    n = n1 - 1
    g_hi = fdiv4(n1 * S - R - phi)                   # last feature whose samples have all arrived
    g_m0 = n * S // 4                                # first feature that starts inside the segment
    g_lo = max(g_done + 1, window_head(kind, W, S, n1))
    Q = g_hi - g_m0 + 1
    return dict(g_hi=g_hi, g_m0=g_m0, g_lo=g_lo, Q=Q, tc=Q >= SPLIT, slot0=g_m0 % L,
                g_done=g_hi if g_hi >= g_lo else g_done)


def push_Q(kind, W, S):
    """Q of every push: floor((S - R - phi) / 4) + 1, whatever n"""
    return (S - R_OF[kind] - phi_of(W)) // 4 + 1


def pushes(kind, W, S, n_push):
    """push_lattice of pushes 1 .. n_push in order"""
    out, g_done = [], -1
    for n1 in range(1, n_push + 1):
        p = push_lattice(kind, W, S, n1, g_done)
        g_done = p["g_done"]
        out.append(p)
    return out


def seam_features(kind, W, S, n1, g_lo, g_m0, g_hi):
    """slide_push's seam features [g_lo, min(g_hi, g_m0 - 1)] as sample ranges [first, last]"""
    phi, R = phi_of(W), R_OF[kind]
    return [(4 * g + phi, 4 * g + phi + R - 1) for g in range(g_lo, min(g_hi, g_m0 - 1) + 1)]


def admit_lattice(kind, W, S, n, H):
    """slide_admit of H history samples after n pushes: {g_lo, g_hi, Q, off, tc, slot0}; off is the history sample of
    feature g_lo, the shift of its staging copy"""
    R, phi = R_OF[kind], phi_of(W)
    nS = n * S
    g_lo = max(cdiv4(nS - H - phi), window_head(kind, W, S, n))
    g_hi = fdiv4(nS - R - phi)
    Q = g_hi - g_lo + 1
    off = 4 * g_lo + phi - (nS - H)
    return dict(g_lo=g_lo, g_hi=g_hi, Q=Q, off=off, tc=H > 0 and Q >= SPLIT, slot0=g_lo % Q if Q > 0 else None)


def tiles_per_cta_for(L, tiles_env=None):
    """tiles_per_cta_for (b2cnn_tc.cu): B2CNN_TC_TILES when set, else about 33 ranges, at least 4 tiles"""
    if tiles_env is not None and 1 <= tiles_env <= 16384:
        return tiles_env
    return max(((L + 32) // 33 + 4 + 2 * 3 - 1) // (2 * 3), 4)


def ranges_of(L, tiles_env=None):
    """tc_prepare: (feats_per_cta = 6 tiles - 4, chunks_per_cta, n_ranges)"""
    t = tiles_per_cta_for(L, tiles_env)
    fpc = 6 * t - 4
    return fpc, (3 * t + 7) // 8, -(-L // fpc)


def proj_wraps(kind, W, S, n1, tiles_env=None):
    """slide_ring_proj_kernel at push n1: per (range, chunk) whose 16 slots wrap past L (first_slot(m) + 16 > L),
    (range, m, split) with split = L - first_slot(m) in 1..15, the first chunk position read from the second box, kept
    when that position lies inside the range [lo, hi) (else the second box feeds only masked positions)"""
    L, foff = L_of(kind, W), FOFF_OF[kind]
    fpc, nch, nr = ranges_of(L, tiles_env)
    head = window_head(kind, W, S, n1) % L
    out = []
    for r in range(nr):
        lo, hi = r * fpc, min(L, r * fpc + fpc)
        for m in range(nch):
            s0 = (head + lo + 16 * m - foff) % L
            q0 = lo + 16 * m - foff
            if s0 + 16 > L and lo <= q0 + (L - s0) < hi:
                out.append((r, m, L - s0))
    return out


def ring_store_straddles(kind, W, S, n1, tiles_env=None):
    """tc_stream_kernel's kOutRing store at push n1 (a tensor-core push): which wraps of the slot past ring_cap = L
    occur -- "cta": a CTA's positions run across slot L (the `slot -= ring_cap` branch); "pair": one step's two features
    land in slots L - 1 and 0 (the `++slot == ring_cap` branch)"""
    L, foff = L_of(kind, W), FOFF_OF[kind]
    p = push_lattice(kind, W, S, n1, -1)
    Q, slot0 = p["Q"], p["slot0"]
    if Q < SPLIT:
        return set()
    fpc = 6 * tiles_per_cta_for(Q, tiles_env) - 4                 # the segment's own ranges (tc_ring_features)
    got = set()
    for p0 in range(0, Q, fpc):
        nfeat = min(fpc, Q - p0)
        if slot0 + p0 < L <= slot0 + p0 + nfeat - 1:
            got.add("cta")
        for pr0 in range(-foff, nfeat, 2):
            if pr0 >= 0 and pr0 + 1 < nfeat and slot0 + p0 + pr0 == L - 1:
                got.add("pair")
    return got


# ------------------------------------------------------------------ case tables
# dtype "bf16" / "f32"; C in-channels; P patients
Case = namedtuple("Case", "kind W S C dtype P")


def _phase_cases():
    """every phase in both geometries and dtypes; strides with Q >= 32 that do not divide W"""
    out, strides = {}, [388, 276, 452, 340]
    i = 0
    for kind in ("mycnn5", "mycnn3"):
        for dtype in ("bf16", "f32"):
            for phi in (0, 3, 2, 1):
                W = W_OF_PHI[phi]
                out[f"{kind}-{dtype}-w{W}"] = Case(kind, W, strides[i % 4], 1 + i % 3, dtype, 130)
                i += 1
    out["mycnn5-bf16-w7501"] = Case("mycnn5", 7501, 1876, 3, "bf16", 130)
    return out


PHASE_CASES = _phase_cases()

# the strides whose pushes have Q = 31, 32 and 33 features: phase 0, then phases 1, 2, 3
Q_STRIDES = {"mycnn5": {0: (144, 148, 152), 1: (148, 152, 156)},
             "mycnn3": {0: (136, 140, 144), 1: (140, 144, 148)}}


def _q_cases():
    out, i = {}, 0
    for kind in ("mycnn5", "mycnn3"):
        for phi in (0, 1, 2, 3):
            W = W_OF_PHI[phi]
            for q, S in zip((31, 32, 33), Q_STRIDES[kind][min(phi, 1)]):
                out[f"{kind}-w{W}-q{q}"] = Case(kind, W, S, 1 + i % 3, ("bf16", "f32")[i % 2], 130)
                i += 1
    return out


Q_CASES = _q_cases()

# long runs: W = 1533 (L = 378, phase 3), S = 164 (S / 4 = 41 odd: the head visits every residue mod 16, Q = 35)
LONG_W, LONG_S = 1533, 164
LONG_EXTRA = 37                               # pushes past the first window: 7 tiles reach split 8 only at the last
LONG_CASES = {f"p{P}-tiles{t or 'default'}": (Case("mycnn5", LONG_W, LONG_S, C, dtype, P), t)
              for (P, C, dtype) in ((128, 2, "f32"), (257, 3, "bf16")) for t in (None, 7)}


def long_pushes():
    return n0_of(LONG_W, LONG_S) + LONG_EXTRA


# smallest windows: L = 32 in both geometries, S = 4 and the largest multiple of 4 that is <= W
SMALL_CASES = {f"{kind}-w{W}-s{S}": Case(kind, W, S, 1 + (W + S) % 3, ("bf16", "f32")[S == 4], 130)
               for kind, Ws in (("mycnn5", (148, 151)), ("mycnn3", (140, 143))) for W in Ws for S in (4, W // 4 * 4)}


def inject_sites(c):
    """(patient, channel, stream sample, value, what) of one patient per phase case: +inf at a seam sample (the second
    to last sample of push n0 - 1, read from the tail by push n0's seam features), -inf among the first phi samples
    of push n0 + 1 (its first sample at phase 0), NaN at the last sample of window n0 + 1, which no feature of that
    window covers unless (W - R) % 4 == 0"""
    n0, phi = n0_of(c.W, c.S), phi_of(c.W)
    p = c.P - 2
    return [(p, c.C - 1, (n0 - 1) * c.S - 2, float("inf"), "seam"),
            (p, 0, n0 * c.S + max(phi - 1, 0), float("-inf"), "first-phi"),
            (p, c.C // 2, (n0 + 1) * c.S - 1, float("nan"), "uncovered")]


def feature_samples(kind, W, S, n):
    """the stream samples window n's features cover: [4 G_n + phi, 4 (G_n + L - 1) + phi + R - 1]"""
    G, phi, R, L = window_head(kind, W, S, n), phi_of(W), R_OF[kind], L_of(kind, W)
    return 4 * G + phi, 4 * (G + L - 1) + phi + R - 1


# admissions at odd phase: W = 1533 (phase 3) MyCNN5 and W = 1531 (phase 1) MyCNN3, S = 164
ADMIT_CASES = {"mycnn5-bf16-w1533": Case("mycnn5", 1533, 164, 3, "bf16", 96),
               "mycnn3-f32-w1531": Case("mycnn3", 1531, 164, 3, "f32", 96)}
ADMIT_AT = (0, 3)                             # admissions before push 1 and before push 4
ADMIT_PUSHES = 16


def admit_q_history(kind, W, S, q):
    """the smallest history length whose admission has Q = q features and a staging shift off != 0"""
    for H in range(1, W + 1):
        a = admit_lattice(kind, W, S, 0, H)
        if a["Q"] == q and a["off"] != 0:
            return H
    raise ValueError((kind, W, q))


def admit_histories(c):
    """(name, H, unaligned view) of each admitted group"""
    R, W = R_OF[c.kind], c.W
    hs = [("W", W), ("W-1", W - 1), ("W-2", W - 2), ("W-3", W - 3), ("R-1", R - 1), ("R", R), ("0", 0),
          ("q31", admit_q_history(c.kind, W, c.S, 31)), ("q32", admit_q_history(c.kind, W, c.S, 32))]
    return [(name, H, False) for name, H in hs] + [("W-2-unaligned", W - 2, True)]


# heads and state: the long run's lattice at P = 130, exported after EXPORT_AT pushes into a scorer of RESTORE_P
HEADS_CASE = Case("mycnn5", LONG_W, LONG_S, 3, "bf16", 130)
EXPORT_AT = n0_of(LONG_W, LONG_S) + 3
RESTORE_P = 70
HEADS_PUSHES = EXPORT_AT + 3

# push staging: phase 0 (W = 1532), so only the view's pitch or pointer stages the segment
STAGING_CASES = {"f32-offset": Case("mycnn5", 1532, 392, 3, "f32", 130),
                 "bf16-pitch": Case("mycnn3", 1532, 392, 2, "bf16", 130)}

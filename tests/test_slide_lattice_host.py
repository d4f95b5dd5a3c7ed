"""CPU: the case tables of tests/test_gpu_slide_lattice.py reach the edges of the tensor-core SlidingScorer's index
arithmetic, shown with the Python mirror of tests/slide_lattice.py: every window phase in both geometries, pushes of
Q = 31, 32 and 33 features at every phase, admissions of Q = 31 and 32 with a staging shift, every split point of the
projection's ring wrap inside a position range, and a front-end ring store across slot L."""
import pytest

import slide_lattice as M

KINDS = ("mycnn5", "mycnn3")


def test_mirror_matches_the_documented_lattice():
    """window n is stream features G_n .. G_n + L - 1, the last L computed; Q is the same for every push"""
    for kind in KINDS:
        for W in (148, 151, 1530, 1531, 1532, 1533, 7501):
            L, phi, R = M.L_of(kind, W), M.phi_of(W), M.R_OF[kind]
            for S in (4, 40, 144, 148, 164):
                if S > W:
                    continue
                for p in M.pushes(kind, W, S, M.n0_of(W, S) + 5):
                    assert p["Q"] == M.push_Q(kind, W, S)
                for n in range(M.n0_of(W, S), M.n0_of(W, S) + 5):
                    first, last = M.feature_samples(kind, W, S, n)
                    assert n * S - W <= first < n * S - W + 4          # the window's first phi samples uncovered
                    assert n * S - 4 < last + 1 <= n * S and (n * S - 1 - last) == (W - R) % 4
                    assert M.push_lattice(kind, W, S, n, -1)["g_hi"] == M.window_head(kind, W, S, n) + L - 1
                assert (first - phi) % 4 == 0


def test_tiles_and_ranges():
    """tc_prepare's ranges at L = 378 (W = 1533): 4 tiles by default (19 ranges of 20), 10 of 38 with 7 tiles; L = 32"""
    assert M.tiles_per_cta_for(378) == 4 and M.ranges_of(378) == (20, 2, 19)
    assert M.ranges_of(378, 7) == (38, 3, 10)
    assert M.ranges_of(18745) == (572, 36, 33)
    assert M.ranges_of(32) == (20, 2, 2)


def test_every_phase_in_both_geometries_and_dtypes():
    seen = {(c.kind, c.dtype, M.phi_of(c.W)) for c in M.PHASE_CASES.values()}
    assert seen == {(k, d, phi) for k in KINDS for d in ("bf16", "f32") for phi in range(4)}
    assert {c.C for c in M.PHASE_CASES.values()} == {1, 2, 3}
    for name, c in M.PHASE_CASES.items():
        assert c.W % c.S and c.S % 4 == 0, name
        assert M.push_Q(c.kind, c.W, c.S) >= M.SPLIT, name              # the tensor-core front end runs
        assert c.W <= 2100 or name == "mycnn5-bf16-w7501"
    assert M.PHASE_CASES["mycnn5-bf16-w7501"] == M.Case("mycnn5", 7501, 1876, 3, "bf16", 130)


@pytest.mark.parametrize("name", sorted(M.PHASE_CASES))
def test_injected_samples_land_where_named(name):
    """the seam sample is read by a seam feature of push n0, the first-phi sample sits in front of push n0 + 1's
    lattice, the uncovered one lies past window n0 + 1's last feature and inside window n0 + 2's"""
    c = M.PHASE_CASES[name]
    n0, phi = M.n0_of(c.W, c.S), M.phi_of(c.W)
    sites = {what: t for _, _, t, _, what in M.inject_sites(c)}
    ps = M.pushes(c.kind, c.W, c.S, n0 + 2)
    p = ps[n0 - 1]
    seams = M.seam_features(c.kind, c.W, c.S, n0, p["g_lo"], p["g_m0"], p["g_hi"])
    assert any(a <= sites["seam"] <= b for a, b in seams)
    t = sites["first-phi"]
    assert t - n0 * c.S == max(phi - 1, 0)
    assert phi == 0 or t < 4 * ps[n0]["g_m0"] + phi                      # before the segment's first main feature
    t = sites["uncovered"]
    first, last = M.feature_samples(c.kind, c.W, c.S, n0 + 1)
    assert (t > last) == (phi != 0) and t >= first
    first, last = M.feature_samples(c.kind, c.W, c.S, n0 + 2)
    assert first <= t <= last
    for n in (n0, n0 + 1):                                               # every site lies in a judged window
        assert all(n * c.S - c.W <= s < (n + 2) * c.S for s in sites.values())


def test_q_split_at_every_phase():
    got = {}
    for name, c in M.Q_CASES.items():
        got.setdefault((c.kind, M.phi_of(c.W)), set()).add(M.push_Q(c.kind, c.W, c.S))
        assert c.S % 4 == 0 and M.n0_of(c.W, c.S) >= 2, name
    assert got == {(k, phi): {31, 32, 33} for k in KINDS for phi in range(4)}
    # the strides the lattice gives, written out
    assert [M.push_Q("mycnn5", 1532, S) for S in (144, 148, 152)] == [31, 32, 33]
    for W in (1531, 1530, 1533):
        assert [M.push_Q("mycnn5", W, S) for S in (148, 152, 156)] == [31, 32, 33]
        assert M.push_Q("mycnn3", W, 144) == 32
    assert M.push_Q("mycnn3", 1532, 140) == 32


@pytest.mark.parametrize("name", sorted(M.LONG_CASES))
def test_long_runs_reach_every_projection_split_and_a_ring_store_wrap(name):
    """over the emitted pushes of the long run, the projection reads a wrapping chunk at each split offset 1..15 with
    the first position past the wrap inside [lo, hi); the front end stores across slot L, within a CTA and within one
    step's pair of features"""
    c, tiles = M.LONG_CASES[name]
    n0 = M.n0_of(c.W, c.S)
    assert M.L_of(c.kind, c.W) == 378 and M.push_Q(c.kind, c.W, c.S) == 35 and (c.S // 4) % 2 == 1
    assert M.long_pushes() >= n0 + 20
    splits, stores = set(), set()
    for n1 in range(1, M.long_pushes() + 1):
        stores |= M.ring_store_straddles(c.kind, c.W, c.S, n1, tiles)
        if n1 >= n0:
            splits |= {s for _, _, s in M.proj_wraps(c.kind, c.W, c.S, n1, tiles)}
    assert splits == set(range(1, 16))
    assert stores == {"cta", "pair"}


def test_long_run_range_starts_differ_between_tilings():
    """7 tiles put the range starts on other residues mod 16 than the default 4"""
    fd, _, nd = M.ranges_of(378)
    f7, _, n7 = M.ranges_of(378, 7)
    assert (nd, n7) == (19, 10)
    assert {r * f7 % 16 for r in range(n7)} - {r * fd % 16 for r in range(nd)}


def test_smallest_windows():
    got = set()
    for name, c in M.SMALL_CASES.items():
        assert M.L_of(c.kind, c.W) == 32, name
        got.add((c.kind, c.W, c.S))
    assert got == {("mycnn5", 148, 4), ("mycnn5", 148, 148), ("mycnn5", 151, 4), ("mycnn5", 151, 148),
                   ("mycnn3", 140, 4), ("mycnn3", 140, 140), ("mycnn3", 143, 4), ("mycnn3", 143, 140)}
    # one step below is not a tensor-core geometry (L = 31)
    assert M.L_of("mycnn5", 147) == 31 and M.L_of("mycnn3", 139) == 31
    # the S = W pushes straddle the split: Q = 32 at phase 0, 31 at phase 1
    assert M.push_Q("mycnn5", 148, 148) == 32 and M.push_Q("mycnn5", 151, 148) == 31


@pytest.mark.parametrize("name", sorted(M.ADMIT_CASES))
def test_admissions_reach_both_sides_of_the_split_with_a_shift(name):
    c = M.ADMIT_CASES[name]
    assert M.phi_of(c.W) % 2 == 1
    hs = M.admit_histories(c)
    R = M.R_OF[c.kind]
    assert {H for _, H, _ in hs} >= {c.W, c.W - 1, c.W - 2, c.W - 3, R - 1, R, 0}
    assert any(u for _, _, u in hs)
    for n in M.ADMIT_AT:
        a = {nm: M.admit_lattice(c.kind, c.W, c.S, n, H) for nm, H, _ in hs}
        assert a["q31"]["Q"] == 31 and a["q31"]["off"] != 0 and not a["q31"]["tc"]
        assert a["q32"]["Q"] == 32 and a["q32"]["off"] != 0 and a["q32"]["tc"]
        assert a["W"]["Q"] == M.L_of(c.kind, c.W) and a["W"]["off"] == 0
        assert {a[k]["off"] for k in ("W-1", "W-2", "W-3")} == {1, 2, 3}
        assert a["R-1"]["Q"] <= 0 and a["0"]["Q"] <= 0
        # the scratch ring of a q32 admission starts past slot 0, so its front-end store wraps
        assert a["q32"]["slot0"] != 0
    # patients: two rounds of admissions plus untouched ones
    assert c.P >= 2 * len(hs) * 4 + 4


def test_heads_export_at_a_wrapping_push():
    c = M.HEADS_CASE
    assert M.phi_of(c.W) == 3 and M.EXPORT_AT >= M.n0_of(c.W, c.S)
    assert M.proj_wraps(c.kind, c.W, c.S, M.EXPORT_AT)
    assert M.RESTORE_P != c.P and M.HEADS_PUSHES > M.EXPORT_AT


def test_staging_cases_are_phase_zero_with_tensor_core_pushes():
    for c in M.STAGING_CASES.values():
        assert M.phi_of(c.W) == 0 and M.push_Q(c.kind, c.W, c.S) >= M.SPLIT
        assert c.S % 8 == 0                    # contiguous rows of 16-byte multiples in both dtypes: only a view stages
    bf = M.STAGING_CASES["bf16-pitch"]
    assert bf.dtype == "bf16" and (bf.S + 2) % 8 != 0

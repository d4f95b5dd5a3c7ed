"""GPU: the bf16 streaming kernel's pool1 in the conv1 accumulator layout, element by element against the float64
reference of oracle/infer_ref.py at the grants of tests/test_gpu_infer_elem.py.

Each lane of the accumulator fragment pools every shift of one conv1 out channel for four windows, takes tap 9 of the
previous block's position 7 from the tile, carries positions 6 and 7 to the next block, and hands the pooled
activations to thread == window through a buffer that alternates with the block's parity.  These tests aim at the
parts a lane-to-channel or parity mix-up would break:

- impulses in every input channel at its own amplitude and sample offset, spaced 37 samples apart, so every sample
  phase mod 24 (a tile's advance) meets both a tile seam and a position-range seam, 8 j + 7 and the tap-9 feed 8 j + 8
  included;
- NaN and +-inf samples at every phase within 24 samples of a range seam (those windows are flagged and recomputed, and
  their neighbours in the same CTA must not be);
- B2CNN_TC_TILES = 4 and 5: ranges of 12 and 15 blocks, so both buffer parities end a range;
- B = 1, 127, 129, 300: one window, partial row halves and a partial last CTA;
- features() at C = 1..4 (MyCNN5 geometry), logits at C = 1..3 in both geometries with 2 and 3 weight pieces, and a
  SlidingScorer whose pushes end at window phases that are not multiples of 8 (the ring kernel)."""
import pytest
import torch

import tskd_b200
from oracle import mycnn_torch as O
from oracle.infer_ref import TC_FEATURES_BETA, infer_reference
from oracle.train_ref import BETA
from test_gpu_infer_elem import BETA_TC_LOGITS, _check, _model
from test_gpu_tc_pairs import _two_piece

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
W = 1528
BF = torch.bfloat16


def _impulses(B, C, Wn, seed):
    """small noise plus, in channel c of window b, an impulse of amplitude (-1)^c 8 (c + 1) at every sample t with
    (t + 7 b + 5 c) % 37 == 0"""
    x = tskd_b200.synth.make_windows(B, C, Wn, "normal", seed=seed) * 0.1
    t = torch.arange(Wn)
    for c in range(C):
        hit = ((t[None, :] + 7 * torch.arange(B)[:, None] + 5 * c) % 37) == 0
        x[:, c][hit] += (-1) ** c * 8.0 * (c + 1)
    return x.to(BF)


def _range_samples(tiles):
    return 4 * (6 * tiles - 4)        # samples per position range: 4 x the range's feature count (b2cnn_tc.cu)


@pytest.mark.parametrize("tiles", [4, 5])
@pytest.mark.parametrize("C,B", [(1, 1), (2, 127), (3, 129), (4, 300)])
def test_features_impulses(monkeypatch, tiles, C, B):
    monkeypatch.setenv("B2CNN_TC_TILES", str(tiles))       # read by tc_prepare when the weights are set
    seed = 300 + 10 * C + tiles
    ref = O.make_ref(O.stretched(O.ARCHS["mycnn5"], C, W), seed=seed)
    x = _impulses(B, C, W, seed)
    age = tskd_b200.synth.make_ages(B, seed=seed)
    truth, ref32 = infer_reference(ref, x, age), infer_reference(ref, x, age, dtype=torch.float32)
    m = _model(ref, "tensorcore")
    got = m.features(x.to(DEV))
    assert m.last_path == "tensorcore"
    _check([("features", got, truth["features"], ref32["features"], TC_FEATURES_BETA)])


@pytest.mark.parametrize("tiles", [4, 5])
@pytest.mark.parametrize("C", [1, 4])
def test_features_nonfinite_at_range_seams(monkeypatch, tiles, C):
    """window b: one NaN, +inf or -inf at sample seam + (b % 48) - 24 of a range seam, in channel b % C; every fourth
    window stays finite"""
    monkeypatch.setenv("B2CNN_TC_TILES", str(tiles))
    B, seed = 200, 400 + 10 * C + tiles
    ref = O.make_ref(O.stretched(O.ARCHS["mycnn5"], C, W), seed=seed)
    x = _impulses(B, C, W, seed).float()
    R = _range_samples(tiles)
    for b in range(B):
        if b % 4 == 3:
            continue
        seam = R * (2 + (b // 48) % 8)
        x[b, b % C, seam + (b % 48) - 24] = (float("nan"), float("inf"), float("-inf"))[b % 4]
    x = x.to(BF)
    age = tskd_b200.synth.make_ages(B, seed=seed)
    truth, ref32 = infer_reference(ref, x, age), infer_reference(ref, x, age, dtype=torch.float32)
    m = _model(ref, "tensorcore")
    got = m.features(x.to(DEV))
    assert m.last_path == "tensorcore"
    _check([("features", got, truth["features"], ref32["features"], TC_FEATURES_BETA)])


@pytest.mark.parametrize("splits", [2, 3])
@pytest.mark.parametrize("kind", ["mycnn5", "mycnn3"])
@pytest.mark.parametrize("C,B,tiles", [(1, 127, 4), (2, 300, 5), (3, 129, 4), (3, 1, 5)])
def test_logits_impulses(monkeypatch, C, B, tiles, kind, splits):
    monkeypatch.setenv("B2CNN_TC_TILES", str(tiles))
    seed = 500 + 10 * C + tiles + (kind == "mycnn3")
    ref = O.make_ref(O.stretched(O.ARCHS[kind], C, W), seed=seed)
    x = _impulses(B, C, W, seed)
    age = tskd_b200.synth.make_ages(B, seed=seed)
    want = _two_piece(ref) if splits == 2 else ref
    truth, ref32 = infer_reference(want, x, age), infer_reference(want, x, age, dtype=torch.float32)
    m = _model(ref, "tensorcore", tc_splits=splits)
    got = m.predict(x.to(DEV), age.to(DEV))
    assert m.last_path == "tensorcore"
    _check([("z", got, truth["z"], ref32["z"], BETA_TC_LOGITS)])


@pytest.mark.parametrize("kind", ["mycnn5", "mycnn3"])
def test_sliding_scorer_impulses(kind):
    """pushes of 372 samples (4 mod 8): each push's new segment starts at a window phase that is not a multiple of 8"""
    P, S, C, seed = 129, 372, 3, 600 + (kind == "mycnn3")
    ref = O.make_ref(O.stretched(O.ARCHS[kind], C, W), seed=seed)
    n0 = -(-W // S)
    n_push = n0 + 2
    stream = _impulses(P, C, n_push * S, seed)
    age = tskd_b200.synth.make_ages(P, seed=seed)
    m = _model(ref)
    sc = tskd_b200.SlidingScorer(m, P, S, BF)
    assert sc.path == "tensorcore"
    sd = stream.to(DEV)
    pairs = []
    for n in range(1, n_push + 1):
        got = sc.push(sd[:, :, (n - 1) * S:n * S], age.to(DEV))
        if n * S < W:
            assert got is None
            continue
        win = stream[:, :, n * S - W:n * S]
        truth, ref32 = infer_reference(ref, win, age), infer_reference(ref, win, age, dtype=torch.float32)
        pairs.append((f"z[{n}]", got.clone(), truth["z"], ref32["z"], BETA))
        pairs.append((f"features[{n}]", sc.features(), truth["features"], ref32["features"], TC_FEATURES_BETA))
    assert len(pairs) == 2 * (n_push - n0 + 1)
    sc.close()
    _check(pairs)

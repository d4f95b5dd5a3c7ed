"""GPU: the bf16 streaming kernels at window-tile seams and with the two-piece weight option, element by element
against oracle/infer_ref.py at the grants of tests/test_gpu_infer_elem.py:

- logits of predict() (the fused kernel, conv1 weights in three and in two bf16 pieces; the two-piece logits are judged
  against the truth of the two-piece weights, which the kernel multiplies exactly) at B = 63, 64, 65, 127 and 129 in
  both geometries, with clean windows and with NaN / +-inf samples next to every 64-window boundary (windows 63 / 64
  and 127 / 128: the last and first windows of a CTA tile for tiles of 64 or of 128 windows);
- features() (the features-out kernel, MyCNN5 geometry) on the same windows;
- every push of a SlidingScorer at P = 130 (the ring-store kernel), logits and stored features."""
import copy

import pytest
import torch

import tskd_b200
from oracle import mycnn_torch as O
from oracle.infer_ref import TC_FEATURES_BETA, infer_reference
from oracle.train_ref import BETA
from test_gpu_infer_elem import BETA_TC_LOGITS, _check, _model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
W = 1528
SEAM_BS = [63, 64, 65, 127, 129]


def _two_piece(ref):
    """conv1 weights as the sum of two bf16 pieces: what tc_splits=2 multiplies exactly, so the truth of its logits"""
    r = copy.deepcopy(ref)
    with torch.no_grad():
        w = r.conv1.weight
        hi = w.bfloat16().float()
        w.copy_(hi + (w - hi).bfloat16().float())
    return r


def _inject_seams(x):
    """NaN / +-inf samples in the last window before every multiple of 64 and in the first window after it, in the
    first and the last input channel, early, mid-window and at the last sample"""
    B, C, n = x.shape
    for start in range(0, B, 64):
        last = min(start + 63, B - 1)
        x[last, 0, 5] = float("nan")
        x[last, C - 1, n // 2] = float("inf")
        if start + 64 < B:
            x[start + 64, C - 1, n // 3] = float("-inf")
            x[start + 64, 0, n - 1] = float("nan")


@pytest.mark.parametrize("bad", [False, True], ids=["clean", "nan-inf"])
@pytest.mark.parametrize("splits", [3, 2])
@pytest.mark.parametrize("kind", ["mycnn5", "mycnn3"])
@pytest.mark.parametrize("B", SEAM_BS)
def test_predict_and_features_at_tile_seams(B, kind, splits, bad):
    seed = 100 + B + (kind == "mycnn3") * 7 + splits + 11 * bad
    ref = O.make_ref(O.stretched(O.ARCHS[kind], 3, W), seed=seed)
    x = tskd_b200.synth.make_windows(B, 3, W, "normal", seed=seed, dtype=torch.bfloat16)
    if bad:
        _inject_seams(x)
    age = tskd_b200.synth.make_ages(B, seed=seed)
    want = _two_piece(ref) if splits == 2 else ref
    truth, ref32 = infer_reference(want, x, age), infer_reference(want, x, age, dtype=torch.float32)
    if bad:
        assert truth["z"].isnan().any() and not truth["z"].isnan().all()
    m = _model(ref, "tensorcore", tc_splits=splits)
    got = m.predict(x.to(DEV), age.to(DEV))
    assert m.last_path == "tensorcore"
    pairs = [("z", got, truth["z"], ref32["z"], BETA_TC_LOGITS)]
    if kind == "mycnn5" and splits == 3:
        f = m.features(x.to(DEV))
        assert m.last_path == "tensorcore"
        pairs.append(("features", f, truth["features"], ref32["features"], TC_FEATURES_BETA))
    _check(pairs)


@pytest.mark.parametrize("bad", [False, True], ids=["clean", "nan-inf"])
@pytest.mark.parametrize("kind", ["mycnn5", "mycnn3"])
def test_sliding_scorer_push_at_130_patients(kind, bad):
    """P = 130: a partial last window tile; every push's logits and stored features against the explicit window"""
    P, S = 130, 384
    ref = O.make_ref(O.stretched(O.ARCHS[kind], 3, W), seed=120 + bad)
    n0 = -(-W // S)
    n_push = n0 + 2
    stream = tskd_b200.synth.make_windows(P, 3, n_push * S, "normal", seed=120 + bad, dtype=torch.bfloat16)
    if bad:                                                 # in the segment of the first scored push
        _inject_seams(stream[:, :, (n0 - 1) * S:n0 * S])
    age = tskd_b200.synth.make_ages(P, seed=120 + bad)
    m = _model(ref)
    sc = tskd_b200.SlidingScorer(m, P, S, torch.bfloat16)
    sd = stream.to(DEV)
    pairs, emitted = [], 0
    for n in range(1, n_push + 1):
        got = sc.push(sd[:, :, (n - 1) * S:n * S], age.to(DEV))
        if n * S < W:
            assert got is None
            continue
        win = stream[:, :, n * S - W:n * S]
        truth, ref32 = infer_reference(ref, win, age), infer_reference(ref, win, age, dtype=torch.float32)
        if bad:
            assert truth["z"].isnan().any() and not truth["z"].isnan().all()
        pairs.append((f"z[{n}]", got.clone(), truth["z"], ref32["z"], BETA))
        pairs.append((f"features[{n}]", sc.features(), truth["features"], ref32["features"], TC_FEATURES_BETA))
        emitted += 1
    assert emitted == n_push - n0 + 1
    sc.close()
    _check(pairs)

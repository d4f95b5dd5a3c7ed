"""GPU: the bf16 streaming kernels at one and two input channels, element by element against oracle/infer_ref.py at
the grants of tests/test_gpu_infer_elem.py, for the instantiations the other suites reach only at three channels:

- logits of predict() with conv1 weights in two bf16 pieces (the gates kernel, SPLITS = 2), judged against the truth
  of the two-piece weights, in both geometries;
- every push of a bf16 SlidingScorer (the ring-store kernel), logits and stored features, in both geometries."""
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


@pytest.mark.parametrize("kind", ["mycnn5", "mycnn3"])
@pytest.mark.parametrize("C", [1, 2])
def test_two_piece_predict_at_one_and_two_channels(C, kind):
    B, seed = 131, 200 + 10 * C + (kind == "mycnn3")
    ref = O.make_ref(O.stretched(O.ARCHS[kind], C, W), seed=seed)
    x = tskd_b200.synth.make_windows(B, C, W, "normal", seed=seed, dtype=torch.bfloat16)
    age = tskd_b200.synth.make_ages(B, seed=seed)
    want = _two_piece(ref)
    truth, ref32 = infer_reference(want, x, age), infer_reference(want, x, age, dtype=torch.float32)
    m = _model(ref, "tensorcore", tc_splits=2)
    got = m.predict(x.to(DEV), age.to(DEV))
    assert m.last_path == "tensorcore"
    _check([("z", got, truth["z"], ref32["z"], BETA_TC_LOGITS)])


@pytest.mark.parametrize("kind", ["mycnn5", "mycnn3"])
@pytest.mark.parametrize("C", [1, 2])
def test_sliding_scorer_at_one_and_two_channels(C, kind):
    P, S, seed = 130, 384, 220 + 10 * C + (kind == "mycnn3")
    ref = O.make_ref(O.stretched(O.ARCHS[kind], C, W), seed=seed)
    n0 = -(-W // S)
    n_push = n0 + 2
    stream = tskd_b200.synth.make_windows(P, C, n_push * S, "normal", seed=seed, dtype=torch.bfloat16)
    age = tskd_b200.synth.make_ages(P, seed=seed)
    m = _model(ref)
    sc = tskd_b200.SlidingScorer(m, P, S, torch.bfloat16)
    assert sc.path == "tensorcore"
    sd = stream.to(DEV)
    pairs, emitted = [], 0
    for n in range(1, n_push + 1):
        got = sc.push(sd[:, :, (n - 1) * S:n * S], age.to(DEV))
        if n * S < W:
            assert got is None
            continue
        win = stream[:, :, n * S - W:n * S]
        truth, ref32 = infer_reference(ref, win, age), infer_reference(ref, win, age, dtype=torch.float32)
        pairs.append((f"z[{n}]", got.clone(), truth["z"], ref32["z"], BETA))
        pairs.append((f"features[{n}]", sc.features(), truth["features"], ref32["features"], TC_FEATURES_BETA))
        emitted += 1
    assert emitted == n_push - n0 + 1
    sc.close()
    _check(pairs)

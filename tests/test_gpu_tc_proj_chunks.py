"""GPU: the streaming gate kernels' LSTM input projection at the edges of a position range, element by element against
the float64 reference (oracle/infer_ref.py).  A range's chunks of 16 positions are projected one block after the
chunk ends, from double-buffered A tiles, and its last chunk after the range's loop.  B2CNN_TC_TILES = 1, 2 and 3 give
every range of a 1528-sample window 3, 6 or 9 steps:

  * 1, 2: the range is a single partial chunk, projected only after the loop;
  * 3: a full chunk, then a chunk of one step, so the range ends with both chunks' MMAs in flight.

Both geometries, bf16 windows (the tensor-core kernel) and fp32 windows (the CUDA-core conv1 kernel)."""
import pytest
import torch

import tskd_b200
from oracle import mycnn_torch as O
from oracle.infer_ref import infer_reference
from test_gpu_infer_elem import BETA_STREAM_LOGITS, BETA_TC_LOGITS, _check, _model, _oarch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F32 = torch.bfloat16, torch.float32


@pytest.mark.parametrize("tiles", [1, 2, 3])
@pytest.mark.parametrize("kind,dtype", [("mycnn5", BF), ("mycnn3", BF), ("mycnn5", F32), ("mycnn3", F32)])
def test_projection_chunk_edges(monkeypatch, tiles, kind, dtype):
    monkeypatch.setenv("B2CNN_TC_TILES", str(tiles))       # read by tc_prepare when the weights are set
    W, B, seed = 1528, 130, 90 + tiles
    ref = O.make_ref(_oarch(kind, 3, W), seed=seed)
    x = tskd_b200.synth.make_windows(B, 3, W, "normal", seed=seed, dtype=dtype)
    age = tskd_b200.synth.make_ages(B, seed=seed)
    truth = infer_reference(ref, x, age)
    ref32 = infer_reference(ref, x, age, dtype=torch.float32)
    m = _model(ref, "tensorcore")
    got = m.predict(x.to(DEV), age.to(DEV))
    assert m.last_path == ("tensorcore" if dtype == BF else "stream")
    _check([("z", got, truth["z"], ref32["z"], BETA_TC_LOGITS if dtype == BF else BETA_STREAM_LOGITS)])

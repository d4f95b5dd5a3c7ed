"""GPU: the wgmma / TMA front end (b2cnn_tc.cu) against the PyTorch-CPU oracle and against
the exact generic kernel.  path="tensorcore" makes the library refuse instead of falling back,
so a pass here is a pass of the tensor-core kernel itself."""
from dataclasses import replace

import numpy as np
import pytest
import torch

import tskd_b200
from conftest import rel_err
from oracle import mycnn_torch as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4


def _pair(C, W, path="tensorcore", tc_splits=3, seed=0, kind="mycnn5"):
    oarch = O.stretched(O.ARCHS[kind], C, W)
    ref = O.make_ref(oarch, seed=seed)
    arch = replace(tskd_b200.ARCH_PRESETS[kind].with_shape(C, W), age_coef=oarch.age_coef)
    m = tskd_b200.B200MyCNN(arch, has_out12=oarch.has_out12, path=path, tc_splits=tc_splits).to(DEV)
    m.load_state_dict(ref.state_dict())
    return ref, m


@pytest.mark.parametrize("C,W,B,dist", [
    (3, 1528, 5, "normal"), (3, 7504, 128, "normal"), (3, 7504, 200, "physio"),
    (1, 2048, 130, "normal"), (2, 4000, 64, "normal"), (4, 3000, 257, "physio"),
    (3, 75000, 9, "normal"),
])
def test_tc_features_and_logits(C, W, B, dist):
    ref, m = _pair(C, W)
    x = tskd_b200.synth.make_windows(B, C, W, dist, seed=21, dtype=torch.bfloat16)
    ages = tskd_b200.synth.make_ages(B, seed=21)
    fw = O.ref_features(ref, x.float()).numpy()
    fg = m.features(x.to(DEV)).cpu().numpy()
    assert m.last_path == "tensorcore"
    err = np.abs(fg - fw)
    assert err.max() < 2e-5, (err.max(), np.unravel_index(err.argmax(), err.shape))
    want = O.ref_independent(ref, x.float(), ages).numpy()
    got = m.predict(x.to(DEV), ages.to(DEV)).cpu().numpy()
    assert m.last_path == "tensorcore" and rel_err(got, want) <= TOL, rel_err(got, want)


def test_tc_sequence_mode():
    ref, m = _pair(3, 1528)
    x = tskd_b200.synth.make_windows(40, 3, 1528, "normal", seed=6, dtype=torch.bfloat16)
    ages = tskd_b200.synth.make_ages(40, seed=6)
    want = O.ref_sequence(ref, x.float(), ages).numpy()
    got = m(x.to(DEV), ages.to(DEV)).cpu().numpy()
    assert m.last_path == "tensorcore" and rel_err(got, want) <= TOL


def test_tc_matches_generic_kernel():
    _, mt = _pair(3, 7504, path="tensorcore")
    _, mg = _pair(3, 7504, path="generic")
    x = tskd_b200.synth.make_windows(300, 3, 7504, "normal", seed=8, dtype=torch.bfloat16).to(DEV)
    ft, fg = mt.features(x), mg.features(x)
    assert mt.last_path == "tensorcore" and mg.last_path == "generic"
    assert (ft - fg).abs().max().item() < 5e-6
    ages = tskd_b200.synth.make_ages(300, seed=8).to(DEV)
    assert rel_err(mt.predict(x, ages).cpu().numpy(), mg.predict(x, ages).cpu().numpy()) < 2e-5


def test_tc_two_piece_weights_still_inside_tolerance():
    """tc_splits=2 keeps 16 mantissa bits of every conv1 weight (6 instead of 9 MMAs per block): an option, not the
    default; logits stay well inside the north-star tolerance but are no longer fp32-equivalent."""
    ref, m2 = _pair(3, 7504, tc_splits=2)
    _, m3 = _pair(3, 7504, tc_splits=3)
    x = tskd_b200.synth.make_windows(300, 3, 7504, "physio", seed=12, dtype=torch.bfloat16)
    ages = tskd_b200.synth.make_ages(300, seed=12)
    want = O.ref_independent(ref, x.float(), ages).numpy()
    got2 = m2.predict(x.to(DEV), ages.to(DEV)).cpu().numpy()
    got3 = m3.predict(x.to(DEV), ages.to(DEV)).cpu().numpy()
    assert m2.last_path == "tensorcore" and rel_err(got2, want) <= TOL
    assert rel_err(got3, want) <= rel_err(got2, want) + 1e-7


def test_tc_nan_inf_windows_are_recomputed_exactly():
    """Band zeros turn inf/NaN samples into NaN blocks; flagged windows are recomputed by the
    exact kernel so the result has the reference's NaN pattern (+inf saturates, NaN propagates)."""
    ref, m = _pair(3, 7504)
    x = tskd_b200.synth.make_windows(140, 3, 7504, "edge", seed=4, dtype=torch.bfloat16)
    x[77, 1, 7503] = float("inf")
    x[139, 2, 0] = float("nan")
    ages = torch.full((140,), 65.0)
    want = O.ref_independent(ref, x.float(), ages).numpy()
    got = m.predict(x.to(DEV), ages.to(DEV)).cpu().numpy()
    assert m.last_path == "tensorcore"
    assert np.array_equal(np.isnan(want), np.isnan(got))
    assert np.isnan(want[0]) and np.isfinite(want[1]) and np.isfinite(want[77]) and np.isnan(want[139])
    ok = ~np.isnan(want)
    assert rel_err(got[ok], want[ok]) <= TOL
    fw = O.ref_features(ref, x.float()).numpy()
    fg = m.features(x.to(DEV)).cpu().numpy()
    assert np.array_equal(np.isnan(fw), np.isnan(fg))
    assert np.nanmax(np.abs(fg - fw)) < 2e-5


def test_tc_flag_state_is_clean_between_calls():
    """The NaN-exception flag state lives in the handle and is put back to zero by the head kernel instead of a
    per-call memset: calls with different flagged windows, clean calls, another stream (workspace copy + memset),
    a sequence-mode call (no cleaning head) and a different batch size in between must all match the oracle."""
    ref, m = _pair(3, 7504)
    base = tskd_b200.synth.make_windows(300, 3, 7504, "normal", seed=9, dtype=torch.bfloat16)
    ages = tskd_b200.synth.make_ages(300, seed=9)
    clean_want = O.ref_independent(ref, base.float(), ages).numpy()

    def run(bad, n=300, stream=None):
        x = base[:n].clone()
        for b, c, i, v in bad:
            x[b, c, i] = v
        want = O.ref_independent(ref, x.float(), ages[:n]).numpy() if bad else clean_want[:n]
        if stream is None:
            got = m.predict(x.to(DEV), ages[:n].to(DEV)).cpu().numpy()
        else:
            xd, ad = x.to(DEV), ages[:n].to(DEV)
            torch.cuda.synchronize()
            with torch.cuda.stream(stream):
                got = m.predict(xd, ad)
            stream.synchronize()
            got = got.cpu().numpy()
        assert m.last_path == "tensorcore"
        assert np.array_equal(np.isnan(want), np.isnan(got)), bad
        ok = ~np.isnan(want)
        assert rel_err(got[ok], want[ok]) <= TOL
        return got

    inf, nan = float("inf"), float("nan")
    g0 = run([])
    run([(5, 0, 100, inf), (257, 2, 7000, inf), (299, 1, 7503, nan)])
    g1 = run([])                                    # the flags of 5 / 257 / 299 must be gone
    assert np.array_equal(g0, g1)
    run([(5, 1, 3000, inf), (6, 0, 0, inf)])        # a window flagged before, and a new one
    run([(100, 0, 50, inf)], n=140)                 # other batch size
    side = torch.cuda.Stream()
    run([(7, 2, 4000, inf)], stream=side)           # not the owning stream: workspace copy
    seq = m(base[:24].to(DEV), ages[:24].to(DEV)).cpu().numpy()      # sequence mode: no cleaning head, memset next time
    assert rel_err(seq, O.ref_sequence(ref, base[:24].float(), ages[:24]).numpy()) <= TOL
    run([(8, 0, 1234, inf), (299, 2, 5, inf)])
    g2 = run([])
    assert np.array_equal(g0, g2)


@pytest.mark.parametrize("kind,C,W,B,dist", [
    ("mycnn5", 3, 7500, 150, "normal"),     # W % 8 == 4: rows staged into a 16-byte-pitch scratch for TMA
    ("mycnn5", 3, 37500, 20, "physio"),
    ("mycnn5", 2, 1533, 40, "normal"),      # odd W
    ("mycnn3", 3, 7504, 200, "normal"),     # MyCNN2/3/4 geometry (k1=5, pool(2,2)) on the fused kernel
    ("mycnn3", 3, 7500, 130, "physio"),
    ("mycnn3", 1, 2048, 64, "normal"),
    ("mycnn3", 3, 75000, 6, "normal"),
])
def test_tc_other_geometries_and_unaligned_windows(kind, C, W, B, dist):
    ref, m = _pair(C, W, kind=kind)
    x = tskd_b200.synth.make_windows(B, C, W, dist, seed=41, dtype=torch.bfloat16)
    ages = tskd_b200.synth.make_ages(B, seed=41)
    want = O.ref_independent(ref, x.float(), ages).numpy()
    got = m.predict(x.to(DEV), ages.to(DEV)).cpu().numpy()
    assert m.last_path == "tensorcore" and rel_err(got, want) <= TOL, rel_err(got, want)
    if kind == "mycnn5":
        fw = O.ref_features(ref, x.float()).numpy()
        fg = m.features(x.to(DEV)).cpu().numpy()
        assert m.last_path == "tensorcore" and np.abs(fg - fw).max() < 2e-5
    seq = m(x[:24].to(DEV), ages[:24].to(DEV)).cpu().numpy()
    assert rel_err(seq, O.ref_sequence(ref, x[:24].float(), ages[:24]).numpy()) <= TOL


def test_tc_refuses_unsupported_shapes_instead_of_falling_back():
    ref = O.make_ref(O.stretched(O.ARCH_MYCNN5, 5, 2048), seed=0)       # 5 channels: no tensor-core instantiation
    m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(5, 2048), path="tensorcore").to(DEV)
    m.load_state_dict(ref.state_dict())
    with pytest.raises(RuntimeError, match="tensor"):
        m.predict(torch.zeros(4, 5, 2048, dtype=torch.bfloat16, device=DEV))
    _, m = _pair(3, 7504)
    m.predict(torch.zeros(4, 3, 7504, dtype=torch.float32, device=DEV))       # fp32 input: the streaming kernel
    assert m.last_path == "stream"
    _, m = _pair(3, 7502)
    with pytest.raises(RuntimeError, match="tensor"):
        m.predict(torch.zeros(4, 3, 7502, dtype=torch.float32, device=DEV))   # fp32 rows that TMA cannot describe


@pytest.mark.parametrize("C,W,B,dist", [(3, 7504, 300, "normal"), (3, 7504, 513, "physio"), (1, 2048, 130, "normal"),
                                        (2, 4000, 64, "normal"), (3, 75000, 9, "normal"), (3, 1528, 5, "normal")])
def test_tc_unfused_kernels_agree_with_fused(C, W, B, dist):
    """tc_fused=0: tensor-core front end -> features in HBM -> CUDA-core projection (the first
    version of the path).  Both variants must meet the oracle and each other."""
    ref, m = _pair(C, W)
    x = tskd_b200.synth.make_windows(B, C, W, dist, seed=31, dtype=torch.bfloat16).to(DEV)
    ages = tskd_b200.synth.make_ages(B, seed=31).to(DEV)
    fused = m.predict(x, ages).cpu().numpy()
    m.set_option("tc_fused", 0)
    unfused = m.predict(x, ages).cpu().numpy()
    assert m.last_path == "tensorcore"
    want = O.ref_independent(ref, x.float().cpu(), ages.cpu()).numpy()
    assert rel_err(fused, want) <= TOL and rel_err(unfused, want) <= TOL
    assert rel_err(fused, unfused) <= 2e-5


def test_tc_fused_prefix_and_permutation_consistency():
    _, m = _pair(3, 7504)
    x = tskd_b200.synth.make_windows(700, 3, 7504, "normal", seed=33, dtype=torch.bfloat16).to(DEV)
    ages = tskd_b200.synth.make_ages(700, seed=33).to(DEV)
    y = m.predict(x, ages)
    assert torch.equal(m.predict(x[:300], ages[:300]), y[:300])
    perm = torch.randperm(700, device=DEV)
    assert torch.equal(m.predict(x[perm], ages[perm]), y[perm])


@pytest.mark.parametrize("kind,C,W,B", [("mycnn5", 3, 7504, 2100), ("mycnn2", 2, 4000, 4100), ("mycnn5", 3, 1528, 9000)])
def test_tc_fused_persistent_grid_many_items_per_cta(kind, C, W, B):
    """More (window-tile pair, position range) items than SMs: every persistent CTA walks several items with different
    ranges (a shorter last range included), carrying its barrier phases across them.  Checked against the exact generic
    kernel on the whole batch and against the oracle on both ends of it."""
    ref, m = _pair(C, W, kind=kind)
    _, mg = _pair(C, W, path="generic", kind=kind)
    x = tskd_b200.synth.make_windows(B, C, W, "physio", seed=77, dtype=torch.bfloat16).to(DEV)
    ages = tskd_b200.synth.make_ages(B, seed=77).to(DEV)
    got = m.predict(x, ages)
    assert m.last_path == "tensorcore"
    exact = mg.predict(x, ages)
    assert rel_err(got.cpu().numpy(), exact.cpu().numpy()) <= 2e-5
    sel = torch.cat([torch.arange(0, 48), torch.arange(B - 48, B)])
    want = O.ref_independent(ref, x[sel.to(DEV)].float().cpu(), ages[sel.to(DEV)].cpu()).numpy()
    assert rel_err(got[sel.to(DEV)].cpu().numpy(), want) <= TOL
    # the same windows in a small batch (one item per CTA at most): bit-identical
    assert torch.equal(m.predict(x[:300], ages[:300]), got[:300])


# ---- fp32 windows: streaming kernel (CUDA-core conv1 + wgmma projection), csrc/b2cnn_tc_fused.cuh ----

@pytest.mark.parametrize("kind,C,W,B,dist", [
    ("mycnn5", 3, 7504, 200, "normal"), ("mycnn5", 3, 7504, 300, "physio"), ("mycnn5", 1, 2048, 300, "normal"),
    ("mycnn5", 2, 4000, 300, "normal"), ("mycnn3", 3, 7504, 257, "physio"), ("mycnn3", 2, 3000, 290, "normal"),
    ("mycnn5", 3, 75000, 9, "normal"), ("mycnn5", 3, 7500, 33, "normal"), ("mycnn5", 3, 1528, 261, "normal"),
])
def test_f32_stream_kernel_matches_oracle_and_generic(kind, C, W, B, dist):
    ref, m = _pair(C, W, path="auto", kind=kind)
    _, mg = _pair(C, W, path="generic", kind=kind)
    x = tskd_b200.synth.make_windows(B, C, W, dist, seed=61, dtype=torch.float32)
    ages = tskd_b200.synth.make_ages(B, seed=61)
    y = m.predict(x.to(DEV), ages.to(DEV))
    assert m.last_path == "stream"
    yg = mg.predict(x.to(DEV), ages.to(DEV))
    assert mg.last_path == "generic"
    want = O.ref_independent(ref, x, ages).numpy()
    assert rel_err(y.cpu().numpy(), want) <= TOL
    assert rel_err(y.cpu().numpy(), yg.cpu().numpy()) <= 2e-5
    # batch-as-sequence semantics (reference model(x_batch)) share the front end
    ys = m(x[:7].to(DEV), ages[:7].to(DEV))
    assert rel_err(ys.cpu().numpy(), O.ref_sequence(ref, x[:7], ages[:7]).numpy()) <= TOL
    # a window's logit does not depend on its batch (bit-for-bit while the same kernel serves the smaller batch;
    # short windows in small batches take the single-launch kernel instead)
    yh = m.predict(x[: B // 2].to(DEV), ages[: B // 2].to(DEV))
    if m.last_path == "stream":
        assert torch.equal(yh, y[: B // 2])
    else:
        assert rel_err(yh.cpu().numpy(), y[: B // 2].cpu().numpy()) <= 1e-6


def test_f32_stream_kernel_nan_inf_pattern():
    ref, m = _pair(3, 7504, path="auto")
    x = tskd_b200.synth.make_windows(150, 3, 7504, "edge", seed=62, dtype=torch.float32)
    x[3, 1, 100] = float("nan"); x[77, 0, 7503] = float("inf"); x[149, 2, 0] = float("-inf")
    ages = torch.full((150,), 65.0)
    want = O.ref_independent(ref, x, ages).numpy()
    got = m.predict(x.to(DEV), ages.to(DEV)).cpu().numpy()
    assert m.last_path == "stream"
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    assert rel_err(got[ok], want[ok]) <= TOL


def test_f32_falls_back_to_generic_when_rows_are_not_16_byte_multiples():
    ref, m = _pair(3, 7502, path="auto")           # W % 4 != 0: no TMA row pitch -> exact generic kernel
    x = tskd_b200.synth.make_windows(20, 3, 7502, "normal", seed=63, dtype=torch.float32)
    ages = tskd_b200.synth.make_ages(20, seed=63)
    y = m.predict(x.to(DEV), ages.to(DEV))
    assert m.last_path == "generic"
    assert rel_err(y.cpu().numpy(), O.ref_independent(ref, x, ages).numpy()) <= TOL


@pytest.mark.parametrize("kind,C,W,B,dtype,path", [
    ("mycnn5", 3, 7500, 150, torch.bfloat16, "tensorcore"),     # W % 8 == 4: TMA straight from the padded rows, no re-pitching copy
    ("mycnn5", 3, 37500, 12, torch.bfloat16, "tensorcore"),
    ("mycnn3", 3, 7500, 130, torch.bfloat16, "tensorcore"),
    ("mycnn5", 2, 1533, 300, torch.bfloat16, "tensorcore"),     # odd W
    ("mycnn5", 3, 7501, 70, torch.float32, "stream"),           # fp32: W % 4 != 0 is generic when contiguous, streamed when padded
    ("mycnn5", 3, 7501, 33, torch.float32, "generic"),          # the generic kernels honour the pitch too
    ("mycnn3", 3, 1502, 40, torch.bfloat16, "generic"),         # ... and the single-launch small-window kernel
])
def test_row_padded_windows_need_no_staging_copy(kind, C, W, B, dtype, path):
    """b2cnn_forward_pitched: a producer that pads its rows to 16 bytes (B200MyCNN.empty_windows) gets the same logits as
    the contiguous tensor -- bit for bit on the tensor-core paths, where the only difference is the skipped staging copy."""
    ref, m = _pair(C, W, path="auto", kind=kind)
    x = tskd_b200.synth.make_windows(B, C, W, "normal", seed=11, dtype=dtype, device=DEV)
    ages = tskd_b200.synth.make_ages(B, seed=11, device=DEV)
    if path == "generic":
        m.set_path("generic")
    y_c = m.predict(x, ages)
    launches_c, path_c = m.gpu_launches, m.last_path
    xp = m.empty_windows(B, dtype=dtype)
    assert not xp.is_contiguous() and xp.stride(1) % (16 // xp.element_size()) == 0 and xp.shape == x.shape
    xp.copy_(x)
    y_p = m.predict(xp, ages)
    assert m.last_path == path, (m.last_path, path_c)
    want = O.ref_independent(ref, x.float().cpu(), ages.cpu()).numpy()
    assert rel_err(y_p.cpu().numpy(), want) <= TOL
    if path == "tensorcore":
        assert torch.equal(y_p, y_c)
        assert m.gpu_launches == launches_c - 1 and m.gpu_launches <= 3         # fused + exact-recompute (empty) + head
    y_s = m.predict(xp[3:9], ages[3:9])                                          # a slice keeps the pitch
    assert rel_err(y_s.cpu().numpy(), want[3:9]) <= TOL

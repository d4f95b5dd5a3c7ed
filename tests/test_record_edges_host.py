"""CPU: tests/record_plan.py, the plan of a whole-recording call restated, against values worked out by hand from
csrc/b2cnn_record.cu's record_plan and score_record's staging grid.  tests/test_gpu_record_edges.py relies on it to
show that each of its cases reaches the branch it is named for, and checks its workspace sizes against the library."""
import pytest

from record_plan import N_for_L_N, record_plan, row_channel, row_samples, stage_block, windows_of_sample


def test_production_shape_strides_the_staging_grid():
    # [4096, 3, 142500] bf16, W = 75000, S = 45000: L_N = (142500 - 24) / 4 + 1, nr = ceil(35620 / 4096),
    # K = ceil(35620 / 9) = 3958 rounded up to 8
    p = record_plan("mycnn5", 75000, 142500, 45000, 4096, 3)
    assert (p.L, p.n_w, p.L_N, p.step, p.nr, p.K, p.pad) == (18745, 2, 35620, 11250, 9, 3960, 20)
    assert (p.rows, p.M, p.row_len, p.Kp) == (36864, 8192, 15860, 15864)
    assert (p.row_channels, p.grid_y, p.stage_strides) == (110592, 65535, True)
    # blocks below 110592 - 65535 = 45057 stage two row-channels; recording 2427's row 2, channel 0 is the first of the
    # second pass
    assert row_channel(p, 3, 2427, 2, 0) == 65535
    assert stage_block(65535) == (0, 1) and stage_block(110591) == (45056, 1) and stage_block(45057) == (45057, 0)
    assert row_samples(p, 2) == (31680, 47539) and row_samples(p, 8) == (126720, 142579)    # past N: the zero fill
    assert windows_of_sample(p, 45000, 40000) == [0] and windows_of_sample(p, 45000, 115000) == [1]
    assert windows_of_sample(p, 45000, 140000) == []


def test_generic_benchmark_shape():
    # the MyCNN5 golden at W = 120 (L = 25) over [1024, 10, 7200]: K = L, nr = ceil(1795 / 25)
    p = record_plan("mycnn5", 120, 7200, 12, 1024, 10, "f32", path="generic")
    assert (p.L, p.L_N, p.K, p.nr, p.rows, p.n_w, p.M) == (25, 1795, 25, 72, 73728, 591, 1024 * 591)
    assert p.row_channels == 737280 and p.stage_strides and p.ws is None


@pytest.mark.parametrize("kind,R", [("mycnn5", 24), ("mycnn3", 16)])
def test_fold_transitions(kind, R):
    assert N_for_L_N(kind, 4096) == 4 * 4095 + R
    p = record_plan(kind, 7504, N_for_L_N(kind, 4096), 752, 3, 3)
    assert (p.L_N, p.nr, p.K, p.pad) == (4096, 1, 4096, 0)
    p = record_plan(kind, 7504, N_for_L_N(kind, 4096) + 3, 752, 3, 3)          # three samples more: still 4096 features
    assert (p.L_N, p.nr) == (4096, 1)
    p = record_plan(kind, 7504, N_for_L_N(kind, 4097), 752, 3, 3)
    assert (p.L_N, p.nr, p.K, p.pad) == (4097, 2, 2056, 15)                   # ceil(4097 / 2) = 2049 -> 2056
    p = record_plan(kind, 7504, N_for_L_N(kind, 8 * 4096 + 1), 752, 3, 3)
    assert (p.L_N, p.nr, p.K, p.pad) == (32769, 9, 3648, 63)                  # ceil(32769 / 9) = 3641 -> 3648


def test_window_counts_at_the_edges():
    W, S = 7504, 752
    assert record_plan("mycnn5", W, W - 1, S, 3, 3).n_w == 0
    assert record_plan("mycnn5", W, W - 1, S, 3, 3).ws == 0
    for N, L_N in ((W, 1871), (W + S - 1, 2058)):                             # (N - 24) / 4 + 1
        p = record_plan("mycnn5", W, N, S, 3, 3)
        assert (p.n_w, p.nr, p.L_N) == (1, 1, L_N)
    assert record_plan("mycnn5", W, W + S, S, 3, 3).n_w == 2


def test_workspace_bytes():
    # MyCNN5, W = 7504 (L = 1871: tiles_per_cta 11, 62 features per range, 31 ranges), one bf16 recording of W samples
    # in 3 channels: K = 1872, row_len = 7508, Kp = 7512; each region rounded up to 256 bytes
    p = record_plan("mycnn5", 7504, 7504, 752, 1, 3)
    stage, feats, flags, partial, age = 45312, 7680, 256, 31 * 256, 256     # 45072, 7488, 12, 7936, 4 bytes
    assert (p.K, p.row_len, p.Kp) == (1872, 7508, 7512)
    assert p.ws == stage + feats + flags + partial + age
    assert record_plan("mycnn5", 7504, 7504, 752, 1, 3, mode="sequence").ws == p.ws + 256     # the [M][64] gates
    assert record_plan("mycnn5", 7504, 7504, 752, 1, 3, "f32").ws == p.ws - stage + 90368   # 90144 bytes of fp32 staging

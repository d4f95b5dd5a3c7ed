"""The plan of a whole-recording call (B200MyCNN.predict_record, b2cnn_score_record) restated in Python: record_plan of
csrc/b2cnn_record.cu and the staging grid score_record launches.  No GPU and no library: tests/test_record_edges_host.py
checks it against hand-computed values, and every case of tests/test_gpu_record_edges.py asserts through it that it
reaches the branch it is named for (more than 65535 staged row-channels, the fold going from 1 to 2 rows, a last row
with features past the recording's end) and that the library's workspace size is the one the plan adds up.

Sample and feature indices are those of one recording: feature g reads samples F g .. F g + R - 1."""
from collections import namedtuple

from slide_lattice import R_OF, ranges_of

F = 4                                        # feature stride of both tensor-core geometries (and the MyCNN5 golden)
REC_ROW_FEATS = 4096                         # kRecRowFeats: the tensor-core path folds into rows of at most ~4096 features
GATES = 64
STAGE_GRID_Y = 65535                         # record_stage_kernel's grid.y: min(row-channels, 65535), strided beyond

Plan = namedtuple("Plan", "F R L n_w L_N step K nr rows Lp row_len Kp M pad row_channels grid_y stage_strides ws")


def L_of(kind, W):
    return (W - R_OF[kind]) // F + 1


def _al256(b):
    return (b + 255) // 256 * 256


def record_plan(kind, W, N, S, B, C, dtype="bf16", mode="independent", path="tensorcore"):
    """record_plan (+ the staging grid and, on the tensor-core path, the workspace bytes) of B recordings of N samples
    in C channels, windows of W samples every S.  pad: features of the last folded row past the recording's last
    feature L_N - 1 (computed from the zero fill); stage_strides: some blockIdx.y stages more than one row-channel."""
    R, L = R_OF[kind], L_of(kind, W)
    assert S >= 1 and S % F == 0
    n_w = (N - W) // S + 1 if N >= W else 0
    if n_w == 0:
        return Plan(F, R, L, 0, *([None] * 13), 0)
    L_N = (N - R) // F + 1
    if path == "tensorcore":
        nr = -(-L_N // REC_ROW_FEATS)
        K = (-(-L_N // nr) + 7) // 8 * 8
    else:
        K = L
        nr = -(-L_N // K)
    rows, M, Lp = B * nr, B * n_w, nr * K
    row_len = F * (K - 1) + R
    Kp = (row_len + 7) // 8 * 8
    rc = rows * C
    grid_y = min(rc, STAGE_GRID_Y)
    ws = None
    if path == "tensorcore":
        esz = 2 if dtype == "bf16" else 4
        ranges = ranges_of(L)[2]
        ws = (_al256(rows * C * Kp * esz) + _al256(4 * B * Lp) + _al256(4 * (2 * rows + 1)) + _al256(4 * ranges * M * GATES)
              + (_al256(4 * M * GATES) if mode == "sequence" else 0) + _al256(4 * M))
    return Plan(F, R, L, n_w, L_N, S // F, K, nr, rows, Lp, row_len, Kp, M, Lp - L_N, rc, grid_y, rc > grid_y, ws)


def stage_block(rc):
    """the blockIdx.y that stages row-channel rc, and its pass through the y loop (0: the first)"""
    return rc % STAGE_GRID_Y, rc // STAGE_GRID_Y


def row_channel(p, C, b, r, c):
    """the staged row-channel index of recording b's folded row r, channel c"""
    return (b * p.nr + r) * C + c


def row_samples(p, r):
    """[first, last] samples of recording row r's staging copy (its halo included; past N is the zero fill)"""
    return r * p.K * F, r * p.K * F + p.row_len - 1


def windows_of_sample(p, S, pos):
    """the windows one of whose features reads sample pos: window w's features cover samples w S .. w S + F (L - 1) +
    R - 1 (the last (W - R) % F samples of a window are in none)"""
    return [w for w in range(p.n_w) if w * S <= pos <= w * S + F * (p.L - 1) + p.R - 1]


def N_for_L_N(kind, L_N):
    """the smallest recording length with L_N features"""
    return F * (L_N - 1) + R_OF[kind]

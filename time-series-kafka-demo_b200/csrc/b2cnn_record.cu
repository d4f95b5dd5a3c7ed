// b2cnn_record.cu -- whole recordings (b2cnn_score_record): every sliding window of B long recordings scored in one
// call, each window feature computed once.  Stateless: a call on a handle, no scorer involved.
#include <algorithm>
#include <cstring>
#include <type_traits>

#include "b2cnn_proj_tc.cuh"

namespace b2cnn {

// A recording of N samples has L_N = (N - R) / F + 1 features on one lattice: feature g reads samples F g .. F g + R - 1.
// Every window starts at a multiple of S (S % F == 0), so window w (samples w S .. w S + W - 1) is features w S / F ..
// w S / F + L - 1 of that lattice (phase 0), and each feature is computed once however many windows hold it.
//   * fold: each recording is cut into nr rows of K features; row r carries samples r K F .. r K F + F (K - 1) + R - 1
//     (the R - F sample halo), copied into 16-byte aligned staging rows [B nr][C][Kp] (zeros past the recording's end).
//     The front end runs once over all B nr rows and stores row (b, r) at feats[b Lp + r K + j], Lp = nr K: one
//     record-major buffer [B][Lp].  Tensor-core path: tc_row_features, K = ceil(L_N / nr) rounded up to 8 with nr =
//     ceil(L_N / kRecRowFeats), so that one 24 h recording still gives ~660 rows; a NaN / inf sample flags (and sends
//     through the exact kernel) its row only.  Generic path: launch_frontend_generic with K = L, predict()'s tile.
//   * projection: the B n_w (recording, window) pairs are the M rows of one launch.  Tensor-core path:
//     slide_record_proj_kernel, the arithmetic of slide_ring_proj_kernel per window with 128 windows per CTA sharing
//     each W_ih chunk; generic path: launch_record_head (proj_body with a per-row base), predict()'s tiles and order.
//   * head: launch_reduce_lstm_head (tensor cores) or reduce_gates + head_independent (generic) over the M rows, with
//     each recording's age repeated over its windows.  Sequence mode (the LSTM carried over each recording's windows,
//     utils.run_model's batch-as-sequence call per recording): reduce_gates over the same partials (tc.n_ranges slices
//     on the tensor-core path, as forward's tensor-core sequence mode sums them), then head_sequence with one warp per
//     recording scanning its n_w gate rows.
// Launches per call: stage, tensor-core front end, flag compaction, exact re-computation, age, projection, head
// (tensor-core path, plus the flag memset; reduction + scan in sequence mode) or stage, front end, age, projection,
// reduction, head (generic path) -- whatever B, N and S.
//   * heads (b2cnn_score_record_heads): rows 0 (the model) .. K (candidate heads of the same front end) share stage,
//     front end, flags and age.  Tensor-core path: the rows run in pairs, one HP = 2 projection per pair into the two
//     partial buffers (each row's partials those of its model's own call), then each row's head on its buffer with its
//     own HeadWeights and age_coef, before the next pair reuses the buffers; an odd last row runs the HP = 1 kernel
//     alone.  Generic path: launch_record_head per row on the one partial / gates buffer.
constexpr int64_t kRecRowFeats = 4096;

struct RecordPlan {
    bool tc, seq;
    int F, R, ranges;
    int64_t n_w, L_N, K, nr, rows, Lp, row_len, Kp, step, M;
    size_t stage, feats, flags, partial, gates, age, partial2, total;   // partial2: the second row of a pair (heads)
};

// the plan of a call; false with *err and *code when an argument is out of range
static bool record_plan(const Dims &d, const TcState &tc, bool use_tc, int64_t B, int64_t N, int64_t stride, int dtype, int mode,
                        int n_heads, RecordPlan *o, int *code, const char **err) {
    RecordPlan &p = *o;
    memset(&p, 0, sizeof p);
    p.tc = use_tc;
    p.seq = mode == B2CNN_MODE_SEQUENCE;
    p.F = d.feature_stride();
    p.R = d.receptive_field();
    *code = B2CNN_EINVAL;
    if (mode != B2CNN_MODE_INDEPENDENT && mode != B2CNN_MODE_SEQUENCE) {
        *err = "mode must be B2CNN_MODE_INDEPENDENT or B2CNN_MODE_SEQUENCE"; return false;
    }
    if (B < 1 || B > 0x7fffffff) { *err = "the recording count must be in [1, 2^31)"; return false; }
    if (N < 0) { *err = "the recording length must be >= 0"; return false; }
    if (stride < 1 || stride % p.F != 0) {
        *err = use_tc ? "stride must be a positive multiple of the feature stride (4 samples)"
                      : "stride must be a positive multiple of the feature stride (pool_s^2 samples)";
        return false;
    }
    p.n_w = N >= d.W ? (N - d.W) / stride + 1 : 0;
    if (p.n_w == 0) return true;
    p.L_N = (N - p.R) / p.F + 1;
    p.step = stride / p.F;
    if (use_tc) {
        p.nr = (p.L_N + kRecRowFeats - 1) / kRecRowFeats;
        p.K = ((p.L_N + p.nr - 1) / p.nr + 7) & ~(int64_t)7;
    } else {
        p.K = d.L;
        p.nr = (p.L_N + p.K - 1) / p.K;
    }
    p.rows = B * p.nr;
    p.M = B * p.n_w;
    // the kernels index rows, windows and their gate rows with 32-bit integers
    if (p.rows > 0x7fffffff / kGates || p.M > 0x7fffffff / kGates) {
        *err = "too many rows: recordings x windows (or x folded rows) must stay below 2^25"; return false;
    }
    p.Lp = p.nr * p.K;
    p.row_len = p.F * (p.K - 1) + p.R;
    p.Kp = (p.row_len + 7) & ~(int64_t)7;
    p.ranges = use_tc ? tc.n_ranges : proj_slices(d.L);
    const int64_t esz = dtype == B2CNN_DTYPE_BF16 ? 2 : 4;
    p.stage = al256((size_t)(p.rows * d.C * p.Kp * esz));
    p.feats = al256(sizeof(float) * (size_t)(B * p.Lp));
    p.flags = use_tc ? al256(sizeof(int) * (size_t)(2 * p.rows + 1)) : 0;
    p.partial = al256(sizeof(float) * (size_t)p.ranges * (size_t)p.M * kGates);
    p.gates = use_tc && !p.seq ? 0 : al256(sizeof(float) * (size_t)p.M * kGates);   // the fused tensor-core head sums in registers
    p.age = al256(sizeof(float) * (size_t)p.M);
    p.partial2 = use_tc && n_heads > 0 ? p.partial : 0;
    p.total = p.stage + p.feats + p.flags + p.partial + p.gates + p.age + p.partial2;
    *code = B2CNN_OK;
    return true;
}

// staging rows: row (b, r) channel c = samples r step_s .. r step_s + row_len - 1 of recording b's channel c, zeros past
// N and past row_len up to Kp; blockIdx.y strides the B nr C row-channels.  A thread writes 16 bytes (Kp % 8 == 0: every
// staging row is 16-byte aligned) from element loads, which take any alignment of the recording.
template <typename T>
__global__ void record_stage_kernel(const T *__restrict__ x, int64_t pitch, int C, int64_t N, int64_t nr, int64_t step_s, int64_t row_len,
                                    int64_t Kp, T *__restrict__ dst, int64_t row_channels) {
    constexpr int V = 16 / sizeof(T);
    for (int64_t rc = blockIdx.y; rc < row_channels; rc += gridDim.y) {
        const int64_t row = rc / C, c = rc - row * C, b = row / nr, r = row - b * nr;
        const T *src = x + (b * C + c) * pitch + r * step_s;
        const int64_t n = min(row_len, N - r * step_s);
        T *out = dst + rc * Kp;
        for (int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * V; i0 < Kp; i0 += (int64_t)gridDim.x * blockDim.x * V) {
            union { uint4 u; T e[V]; } v;
#pragma unroll
            for (int j = 0; j < V; ++j) v.e[j] = i0 + j < n ? __ldg(src + i0 + j) : T(0);
            *reinterpret_cast<uint4 *>(out + i0) = v.u;
        }
    }
}

// age of row m = recording m / n_w's
__global__ void record_age_kernel(const float *__restrict__ age, int64_t n_age, int64_t n_w, int64_t M, float *__restrict__ dst) {
    const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m < M) dst[m] = age[n_age == 1 ? 0 : m / n_w];
}

// The tensor-core projection of whole recordings.  CTA = (128 (recording, window) rows, range); per window the
// arithmetic of slide_ring_proj_kernel (HP = 1): the same ranges, 16-position chunks in the same order, A pieces and 12
// MMAs per chunk with the handle's packed W_ih chunks -- which the CTA's 128 windows share.  A window's features start
// at any float offset (w S / F), so instead of TMA boxes each consumer thread loads its window's 16 consecutive floats
// of the chunk (whole sectors), one chunk ahead: the loads of chunk m + 1 are in flight during chunk m's MMAs.
//   warp 4: the W_ih chunks (bulk copies, two stages); warps 0-3: thread == window.
struct RecordProjParams {
    const float *feats;              // [B][rec_pitch]
    const uint8_t *wpack;            // [n_ranges][chunks_per_cta][kRpWChunk]
    float *partial;                  // [n_ranges][M][64]
    int64_t rec_pitch, step;         // recording pitch and window step in features
    int M, n_w, L, feats_per_cta, chunks_per_cta, foff;
};
// Two rows of a call with heads (score_record with n_heads > 0) per CTA: p's wpack / partial are the first row's, these
// the second's.  HP: rows per CTA, each with its own W_ih chunk slot per stage and its own accumulators.
struct RecordProjPair {
    RecordProjParams p;
    const uint8_t *wpack1;
    float *partial1;
};
template <int HP>
using RecordProjArgs = std::conditional_t<HP == 1, RecordProjParams, RecordProjPair>;
__device__ __forceinline__ const RecordProjParams &rec_base(const RecordProjParams &a) { return a; }
__device__ __forceinline__ const RecordProjParams &rec_base(const RecordProjPair &a) { return a.p; }
template <int HP>
constexpr size_t kRecProjSmemHP = 1024 + 2 * HP * kRpWChunk + 3 * kRpPiece + 64;

// Per row the instructions are those of HP = 1: the A pieces split once from the window's features serve both rows,
// and each row gets the same 12 MMAs per chunk in the same chunk order -- so each row's partials are bit-identical to
// those of its model's own call.
template <int HP>
__global__ void __launch_bounds__(kRpThreads) slide_record_proj_kernel(const __grid_constant__ RecordProjArgs<HP> args) {
    const RecordProjParams &p = rec_base(args);
    auto wpack_of = [&](int j) {
        if constexpr (HP == 1) return p.wpack;
        else return j == 0 ? p.wpack : args.wpack1;
    };
    auto partial_of = [&](int j) {
        if constexpr (HP == 1) return p.partial;
        else return j == 0 ? p.partial : args.partial1;
    };
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t *sW = smem;                                            // [2 stages][HP][6 KB]
    uint8_t *sPc = sW + 2 * HP * kRpWChunk;                        // [3 pieces][4 KB]
    uint64_t *bars = reinterpret_cast<uint64_t *>(sPc + 3 * kRpPiece);
    const uint32_t bar_full = smem_u32(bars + 0), bar_empty = smem_u32(bars + 2);
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
    const int lane = threadIdx.x & 31;
    const int b0 = blockIdx.x * kRpM;
    const int lo = blockIdx.y * p.feats_per_cta, hi = min(p.L, lo + p.feats_per_cta);
    const int nch = p.chunks_per_cta;
    if (threadIdx.x == 0) {
        for (int i = 0; i < 2; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (warp == 4) {
        if (lane == 0) {
            for (int m = 0; m < nch; ++m) {
                const int u = m & 1;
                mbar_wait(bar_empty + 8 * u, ((m >> 1) & 1) ^ 1);
                mbar_expect_tx(bar_full + 8 * u, HP * kRpWChunk);
#pragma unroll
                for (int j = 0; j < HP; ++j)
                    bulk_load_1d(smem_u32(sW + (u * HP + j) * kRpWChunk), wpack_of(j) + ((size_t)blockIdx.y * nch + m) * kRpWChunk,
                                 kRpWChunk, bar_full + 8 * u);
            }
        }
        return;
    }
    const int row = threadIdx.x, b = b0 + row;
    const bool row_ok = b < p.M;
    const float *fr = p.feats;
    if (row_ok) {
        const int r = b / p.n_w;
        fr += (int64_t)r * p.rec_pitch + (int64_t)(b - r * p.n_w) * p.step;
    }
    float gacc[HP][2][32];
#pragma unroll
    for (int j = 0; j < HP; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 32; ++i) gacc[j][h][i] = 0.f;
    uint8_t *arow = sPc + (row >> 3) * 256 + (row & 7) * 16;
    float v[16];
    auto load = [&](int m) {
        const int q0 = lo + 16 * m - p.foff;
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const int q = q0 + k;
            v[k] = row_ok && q >= lo && q < hi ? __ldg(fr + q) : 0.f;
        }
    };
    load(0);
#pragma unroll 1
    for (int m = 0; m < nch; ++m) {
        const int u = m & 1;
        rp_split_row(arow, [&](int k) { return v[k]; });
        fence_proxy_async();
        wg_bar();
        mbar_wait(bar_full + 8 * u, (m >> 1) & 1);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < HP; ++j) rp_mma_chunk(gacc[j], smem_u32(sPc), smem_u32(sW + (u * HP + j) * kRpWChunk));
        wgmma_commit();
        if (m + 1 < nch) load(m + 1);                              // in flight during the MMAs
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * u);
        wg_bar();                                                  // A tile free for the next chunk
    }
#pragma unroll
    for (int j = 0; j < HP; ++j) rp_store_partial(partial_of(j), blockIdx.y, p.M, b0, warp, lane, gacc[j]);
}

int64_t record_workspace_bytes(const Dims &d, const TcState &tc, bool use_tc, int64_t B, int64_t N, int64_t stride, int dtype, int mode,
                               const char **err, int n_heads) {
    RecordPlan p;
    int code;
    if (!record_plan(d, tc, use_tc, B, N, stride, dtype, mode, n_heads, &p, &code, err)) return -1;
    return (int64_t)p.total;
}

int score_record(const Dims &d, const ConvWeights &cw, const HeadWeights &hw, const TcState &tc, bool use_tc, int num_sms, const void *x,
                 int dtype, int64_t B, int64_t N, int64_t pitch, int64_t stride, int mode, const float *age, int64_t n_age, int apply_sigmoid,
                 float *out, void *ws, int64_t ws_bytes, cudaStream_t st, const char **err, const float *state_in, float *state_out,
                 const RecordHead *heads, int n_heads) {
    RecordPlan p;
    int code;
    if (!record_plan(d, tc, use_tc, B, N, stride, dtype, mode, n_heads, &p, &code, err)) return code;
    const int rows = 1 + n_heads;                                  // output rows: the model's, then each head's
    if (pitch < N || pitch < 1) { *err = "pitch must be >= the recording length"; return B2CNN_EINVAL; }
    if (n_age != 1 && n_age != B) { *err = "age must have 1 or B elements"; return B2CNN_EINVAL; }
    if ((state_in || state_out) && !p.seq) { *err = "an LSTM state needs sequence mode"; return B2CNN_EINVAL; }
    if (overlap(state_in, state_out, sizeof(float) * kGates * (size_t)B * rows)) { *err = "state_in and state_out overlap"; return B2CNN_EINVAL; }
    if (p.n_w == 0) {
        // no window: the state passes through unchanged
        const size_t bytes = sizeof(float) * (size_t)B * kGates * rows;
        if (state_out && (state_in ? cudaMemcpyAsync(state_out, state_in, bytes, cudaMemcpyDeviceToDevice, st)
                                   : cudaMemsetAsync(state_out, 0, bytes, st)) != cudaSuccess) {
            *err = "copy of the LSTM state"; return B2CNN_ECUDA;
        }
        return B2CNN_OK;
    }
    if (!ws || ws_bytes < (int64_t)p.total || (reinterpret_cast<uintptr_t>(ws) & 255) != 0) {
        *err = "workspace missing, not 256-byte aligned or smaller than b2cnn_record_workspace_bytes()"; return B2CNN_ESTATE;
    }
    Dims dr = d;                                                   // one folded row
    dr.L = (int)p.K; dr.W = (int)p.row_len; dr.XP = (int)p.Kp;
    if (!use_tc && !frontend_generic_fits(dr)) {
        *err = "the generic front end's tile does not fit shared memory (in_channels * pool_s^2 too large for this window length)";
        return B2CNN_EARCH;
    }
    char *base = static_cast<char *>(ws);
    void *stage = base;
    float *feats = reinterpret_cast<float *>(base + p.stage);
    int *flags = reinterpret_cast<int *>(base + p.stage + p.feats);
    float *partial = reinterpret_cast<float *>(base + p.stage + p.feats + p.flags);
    float *gates = reinterpret_cast<float *>(base + p.stage + p.feats + p.flags + p.partial);
    float *ages = reinterpret_cast<float *>(base + p.stage + p.feats + p.flags + p.partial + p.gates);
    float *partial2 = reinterpret_cast<float *>(base + p.stage + p.feats + p.flags + p.partial + p.gates + p.age);
    // row r: its head weights, packed W_ih chunks, geometry with its age_coef, and its slices of out and the states
    struct Row { const HeadWeights *hw; const TcState *tc; Dims d; float *out; const float *state_in; float *state_out; };
    auto row_of = [&](int r) {
        Row w{r == 0 ? &hw : heads[r - 1].hw, r == 0 ? &tc : heads[r - 1].tc, d, out + (size_t)r * p.M,
              state_in ? state_in + (size_t)r * B * kGates : nullptr, state_out ? state_out + (size_t)r * B * kGates : nullptr};
        if (r > 0) w.d.age_coef = heads[r - 1].age_coef;
        return w;
    };
    // ---- fold: staging rows
    {
        const int64_t rc = p.rows * d.C;
        const int64_t per_block = 256 * (dtype == B2CNN_DTYPE_BF16 ? 8 : 4);
        const dim3 grid((unsigned)std::min<int64_t>((p.Kp + per_block - 1) / per_block, 16), (unsigned)std::min<int64_t>(rc, 65535));
        const int64_t step_s = p.K * p.F;
        if (dtype == B2CNN_DTYPE_BF16)
            record_stage_kernel<uint16_t><<<grid, 256, 0, st>>>(static_cast<const uint16_t *>(x), pitch, d.C, N, p.nr, step_s, p.row_len, p.Kp,
                                                                 static_cast<uint16_t *>(stage), rc);
        else
            record_stage_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float *>(x), pitch, d.C, N, p.nr, step_s, p.row_len, p.Kp,
                                                              static_cast<float *>(stage), rc);
        if (cudaGetLastError() != cudaSuccess) { *err = "staging launch"; return B2CNN_ECUDA; }
    }
    // ---- front end: every row's K features into feats[b Lp + r K + j]
    if (use_tc) {
        if (cudaMemsetAsync(flags, 0, sizeof(int) * (size_t)(2 * p.rows + 1), st) != cudaSuccess) { *err = "memset flags"; return B2CNN_ECUDA; }
        if (tc_row_features(tc, dr, cw, stage, p.Kp, dtype, p.rows, feats, p.K, flags, num_sms, st, err) < 0) return B2CNN_ECUDA;
    } else {
        // the rows hold at most L features, often one tile: four times predict()'s CTAs per SM keep the SMs busy (the
        // grid does not change what a CTA computes)
        const int rc = launch_frontend_generic(dr, cw, stage, dtype, p.rows, feats, p.K, 1, st, 4 * num_sms, err);
        if (rc < 0) return rc == kLaunchArch ? B2CNN_EARCH : B2CNN_ECUDA;
    }
    // ---- each recording's age over its windows
    record_age_kernel<<<(unsigned)((p.M + 255) / 256), 256, 0, st>>>(age, n_age, p.n_w, p.M, ages);
    if (cudaGetLastError() != cudaSuccess) { *err = "age launch"; return B2CNN_ECUDA; }
    // ---- projection + head over the B n_w windows
    if (!use_tc) {
        for (int r = 0; r < rows; ++r) {
            const Row w = row_of(r);
            if (launch_record_head(w.d, *w.hw, feats, p.Lp, (int)p.n_w, p.step, p.M, ages, p.M, mode, apply_sigmoid, w.out, gates, partial, st,
                                   err, w.state_in, w.state_out) < 0)
                return B2CNN_ECUDA;
        }
        return B2CNN_OK;
    }
    RecordProjParams rp;
    rp.feats = feats; rp.wpack = reinterpret_cast<const uint8_t *>(tc.d_wpack); rp.partial = partial;
    rp.rec_pitch = p.Lp; rp.step = p.step;
    rp.M = (int)p.M; rp.n_w = (int)p.n_w; rp.L = d.L;
    rp.feats_per_cta = tc.feats_per_cta; rp.chunks_per_cta = tc.chunks_per_cta; rp.foff = d.K1 == 10 ? 3 : 2;
    const dim3 grid((unsigned)((p.M + kRpM - 1) / kRpM), (unsigned)tc.n_ranges);
    // one row's head over its range partials
    auto head = [&](const Row &w, const float *part) {
        if (p.seq)
            return launch_reduce_gates(part, tc.n_ranges, p.M, *w.hw, gates, st, err) < 0 ||
                           launch_sequence_segments(w.d, *w.hw, gates, B, p.n_w, ages, p.M, apply_sigmoid, w.out, st, err, nullptr,
                                                    w.state_in, w.state_out) < 0
                       ? B2CNN_ECUDA : B2CNN_OK;
        return launch_reduce_lstm_head(w.d, *w.hw, part, tc.n_ranges, p.M, ages, p.M, apply_sigmoid, w.out, st, err) < 0 ? B2CNN_ECUDA
                                                                                                                         : B2CNN_OK;
    };
    for (int r = 0; r < rows; r += 2) {
        const Row w0 = row_of(r);
        rp.wpack = reinterpret_cast<const uint8_t *>(w0.tc->d_wpack);
        if (r + 1 < rows) {
            const Row w1 = row_of(r + 1);
            const RecordProjPair pair{rp, reinterpret_cast<const uint8_t *>(w1.tc->d_wpack), partial2};
            if (cudaFuncSetAttribute(slide_record_proj_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRecProjSmemHP<2>) !=
                cudaSuccess) {
                *err = "projection smem attribute"; return B2CNN_ECUDA;
            }
            slide_record_proj_kernel<2><<<grid, kRpThreads, kRecProjSmemHP<2>, st>>>(pair);
            if (cudaGetLastError() != cudaSuccess) { *err = "projection launch"; return B2CNN_ECUDA; }
            if (int rc = head(w0, partial)) return rc;
            if (int rc = head(w1, partial2)) return rc;
            continue;
        }
        if (cudaFuncSetAttribute(slide_record_proj_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRecProjSmemHP<1>) !=
            cudaSuccess) {
            *err = "projection smem attribute"; return B2CNN_ECUDA;
        }
        slide_record_proj_kernel<1><<<grid, kRpThreads, kRecProjSmemHP<1>, st>>>(rp);
        if (cudaGetLastError() != cudaSuccess) { *err = "projection launch"; return B2CNN_ECUDA; }
        if (int rc = head(w0, partial)) return rc;
    }
    return B2CNN_OK;
}

}  // namespace b2cnn

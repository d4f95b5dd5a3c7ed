// b2cnn_proj_tc.cuh -- the layer-0 projection on wgmma shared by the scorer's ring (slide_ring_proj_kernel,
// b2cnn_slide.cu) and whole recordings (slide_record_proj_kernel, b2cnn_record.cu), and the interface of the latter.
//
// CTA = (128 rows, position range) of kRpThreads: warps 0-3 are the consumer warpgroup, thread == row (a patient or a
// window); warp 4 loads.  Per 16-position chunk the row's 16 features (0 outside the range) are split into three bf16
// pieces written as the K-major A tile (rp_split_row), then 2 row halves x 6 m64n64k16 piece pairs (hh hm mh hl lh mm,
// fp32-equivalent products, as the fused kernel) with the chunk's packed W_ih (rp_mma_chunk) accumulate the row's 64
// gates in registers, stored at the end as partial[range][row][64] (rp_store_partial).  Both kernels issue exactly
// these instructions per chunk, so a window's partials do not depend on which of them computed it.
#pragma once
#include "b2cnn_tc.cuh"
#include "b2cnn_tc_ptx.cuh"

namespace b2cnn {

constexpr int kRpThreads = 160;
constexpr int kRpM = 128;                            // rows per CTA
constexpr int kRpWChunk = 3 * 64 * 16 * 2;           // a packed W_ih chunk (tc_pack_wih_kernel, kFuWChunkBytes)
constexpr int kRpPiece = kRpM * 16 * 2;              // one bf16 piece of the A tile

inline size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

// feat(k), k < 16: the row's features of the chunk, split into hi / mid / lo bf16 pieces at arow, arow + kRpPiece and
// arow + 2 kRpPiece (arow: the row's 16 bytes of its 8-row core matrix)
template <typename Feat>
__device__ __forceinline__ void rp_split_row(uint8_t *arow, Feat feat) {
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
        const float f0 = feat(2 * kk), f1 = feat(2 * kk + 1);
        const uint32_t h = pack_bf16x2(f0, f1);
        const float r1x = f0 - __uint_as_float(h << 16), r1y = f1 - __uint_as_float(h & 0xffff0000u);
        const uint32_t md = pack_bf16x2(r1x, r1y);
        const uint32_t lw = pack_bf16x2(r1x - __uint_as_float(md << 16), r1y - __uint_as_float(md & 0xffff0000u));
        const int off = (kk >> 2) * 128 + (kk & 3) * 4;
        *reinterpret_cast<uint32_t *>(arow + off) = h;
        *reinterpret_cast<uint32_t *>(arow + kRpPiece + off) = md;
        *reinterpret_cast<uint32_t *>(arow + 2 * kRpPiece + off) = lw;
    }
}

// the chunk's 12 MMAs: A pieces at shared address pa, W_ih pieces at pw, into acc[row half][32]
__device__ __forceinline__ void rp_mma_chunk(float (&acc)[2][32], uint32_t pa, uint32_t pw) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        constexpr int kAp[6] = {0, 0, 1, 0, 2, 1}, kWp[6] = {0, 1, 0, 2, 0, 1};
#pragma unroll
        for (int q = 0; q < 6; ++q)
            wgmma_m64n64(acc[hh], gdesc_none_kmajor(pa + kAp[q] * kRpPiece + hh * 2048, 128, 256),
                         gdesc_none_kmajor(pw + kWp[q] * 2048, 128, 256));
    }
}

// acc into part[range][row][64] for the CTA's rows b0 .. b0 + 127 below n_rows (the wgmma D fragment layout)
__device__ __forceinline__ void rp_store_partial(float *part, int range, int n_rows, int b0, int warp, int lane,
                                                 const float (&acc)[2][32]) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) {
            const int bb = b0 + 64 * hh + 16 * warp + (lane >> 2) + 8 * e2;
            if (bb < n_rows) {
                float *dst = part + ((int64_t)range * n_rows + bb) * kGates + 2 * (lane & 3);
#pragma unroll
                for (int e = 2 * e2; e < 32; e += 4)
                    *reinterpret_cast<float2 *>(dst + 8 * (e >> 2)) = make_float2(acc[hh][e], acc[hh][e + 1]);
            }
        }
}

// whole recordings (b2cnn_score_record, b2cnn_record.cu): x [B][C][pitch], out [B][n_w], n_w = (N - W) / stride + 1
// (0 for N < W).  use_tc: the tensor-core path (the caller has checked that the handle's TcState holds the model).  The
// workspace size is -1 (with *err) for bad arguments.  mode: B2CNN_MODE_INDEPENDENT (every window from the zero LSTM
// state) or B2CNN_MODE_SEQUENCE (the LSTM carried over each recording's windows in order, from the zero state per
// recording, or from state_in[b] when state_in is not null; state_out[b] receives recording b's state after its last
// window, state_in[b] (or zeros) when it has none).  state_in / state_out: device [B][64] = h0 | c0 | h1 | c1, null
// or sequence mode only (else B2CNN_EINVAL).
// Candidate heads (b2cnn_score_record_heads): rows 1 .. n_heads of out [1 + n_heads][B][n_w] and of the states [1 +
// n_heads][B][64] are those of heads[i - 1] -- its LSTM / Linear weights, packed W_ih chunks (tensor-core path; the
// model's n_ranges and chunks_per_cta) and age_coef over the model's features (the caller has checked that every head
// has the model's architecture and front-end weights).  Row 0 is the call without heads.  n_heads > 0 adds one range
// partial buffer to the tensor-core workspace.
struct RecordHead {
    const HeadWeights *hw;
    const TcState *tc;
    float age_coef;
};
int64_t record_workspace_bytes(const Dims &d, const TcState &tc, bool use_tc, int64_t B, int64_t N, int64_t stride, int dtype, int mode,
                               const char **err, int n_heads = 0);
int score_record(const Dims &d, const ConvWeights &cw, const HeadWeights &hw, const TcState &tc, bool use_tc, int num_sms, const void *x,
                 int dtype, int64_t B, int64_t N, int64_t pitch, int64_t stride, int mode, const float *age, int64_t n_age, int apply_sigmoid,
                 float *out, void *ws, int64_t ws_bytes, cudaStream_t st, const char **err, const float *state_in = nullptr,
                 float *state_out = nullptr, const RecordHead *heads = nullptr, int n_heads = 0);

}  // namespace b2cnn

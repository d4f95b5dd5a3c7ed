// b2cnn_tc.cuh -- interface of the wgmma (Hopper tensor core) fast path, b2cnn_tc.cu.
#pragma once
#include <cuda.h>

#include "b2cnn_internal.cuh"

namespace b2cnn {

struct TcState {
    // What tc_prepare found for the handle's geometry (both false: every call takes the generic kernels)
    bool features = false;       // the features-out kernel (tc_frontend): MyCNN5 geometry, C <= 4
    bool fused = false;          // the fused / fp32 stream / ring kernels and the packed W_ih: either geometry, C <= 3
    int splits = 3;              // bf16 pieces per fp32 conv1 weight in the fused kernels (3 = fp32-equivalent)
    void *d_bmats = nullptr;     // Toeplitz-expanded conv1 weights, three bf16 pieces (see b2cnn_tc.cu)
    void *d_bmats2 = nullptr;    // the first two pieces only (tc_splits=2)
    void *d_wpack = nullptr;     // W_ih_l0 packed per (position range, 16-position chunk), 3 bf16 pieces
    int tiles_per_cta = 96, feats_per_cta = 572, chunks_per_cta = 36, n_ranges = 1;
    // Flag state of the streaming kernels' NaN exception path (count | flags [cap] | list [cap]) owned by the handle:
    // it is all-zero between calls -- the head kernel that consumes a call's list clears exactly what the call set --
    // so the per-call memset of the workspace copy (one more stream operation and dependent-launch gap per step)
    // disappears.  Only calls on the stream that first used it take it (one stream = serialised); calls on any other
    // stream, batches beyond the capacity and sequence-mode calls keep the workspace copy + memset.
    int *d_flagstate = nullptr;
    int64_t flag_cap = 0;
    bool flags_clean = false;    // host-side: the last call on the owning stream ended with the cleaning head kernel
    bool owner_set = false;
    cudaStream_t owner_stream = nullptr;
    // what the current call uses (read by the caller of tc_gates to hand the cleaning job to the head kernel)
    int *cur_count = nullptr, *cur_flags = nullptr, *cur_list = nullptr;
    bool cur_own = false;
};



const char *tc_error();
int tc_prepare(TcState &s, const Dims &d, const ConvWeights &cw, const float *d_wih0, int splits, cudaStream_t st);
void tc_release(TcState &s);
// Workspace of the tensor-core kernels, after the head's buffers: NaN flags (count, flags [B], list [B]), then the
// pitch-aligned bf16 copy of x that tc_frontend / tc_gates make when the row pitch is not a multiple of 8 samples.
int64_t tc_flags_bytes(int64_t B);
int64_t tc_stage_bytes(const Dims &d, int64_t B);
// returns number of kernel launches, or <0 with *err set
int tc_frontend(TcState &s, const Dims &d, const ConvWeights &cw, const void *x, int64_t B, float *feats,
                int64_t sB, int64_t sP, void *ws, int num_sms, cudaStream_t st, const char **err);
// streaming front end + layer-0 projection of bf16 windows (tensor-core conv1) or fp32 windows (CUDA-core conv1),
// b2cnn_tc_fused.cuh: leaves the range partials partial[n_ranges][B][64] and, with reduce_here, gates[B][64]
// (biases included); without it the caller's head kernel sums the partials itself.
int tc_gates(TcState &s, const Dims &d, const ConvWeights &cw, const HeadWeights &hw, const void *x, int dtype, int64_t B,
             float *partial, float *gates, void *ws, int num_sms, cudaStream_t st, const char **err, bool reduce_here);
int tc_features(TcState &s, const Dims &d, const ConvWeights &cw, const void *x, int64_t B, float *feats,
                int num_sms, cudaStream_t st, const char **err);
// sliding-window scorer (b2cnn_slide.cu): a segment's features into the position-major feature ring
int tc_ring_features(const TcState &s, const Dims &dseg, const ConvWeights &cw, const void *x, int64_t pitch, int dtype,
                     int64_t P, float *ring, int64_t ring_pitch, int cap, int slot0, int *flags, cudaStream_t st, const char **err);
int tc_ring_tmap(const float *ring, int64_t P, int64_t pitch, int L, CUtensorMap *tm, const char **err);
// whole recordings (b2cnn_record.cu, b2cnn_score_record): the features of `rows` staged rows into feats[row sB + j],
// flagged rows recomputed exactly
int tc_row_features(const TcState &s, const Dims &dseg, const ConvWeights &cw, const void *x, int64_t pitch, int dtype,
                    int64_t rows, float *feats, int64_t sB, int *flags, int num_sms, cudaStream_t st, const char **err);

}  // namespace b2cnn

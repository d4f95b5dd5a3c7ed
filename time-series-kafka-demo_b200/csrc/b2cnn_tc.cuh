// b2cnn_tc.cuh -- interface of the wgmma (Hopper tensor core) fast path, b2cnn_tc.cu.
#pragma once
#include <cuda.h>

#include "b2cnn_internal.cuh"

namespace b2cnn {

struct TcState {
    bool ready = false;
    int splits = 3;              // bf16 pieces per fp32 conv1 weight in the fused kernels (3 = fp32-equivalent)
    void *d_bmats = nullptr;     // Toeplitz-expanded conv1 weights, three bf16 pieces (see b2cnn_tc.cu)
    void *d_bmats2 = nullptr;    // the first two pieces only (tc_splits=2)
    void *d_wpack = nullptr;     // W_ih_l0 packed per (position range, 16-position chunk), 3 bf16 pieces
    int tiles_per_cta = 96, feats_per_cta = 572, chunks_per_cta = 36, n_ranges = 1;
    bool has_v1 = false;         // the features-out kernel exists for this geometry (MyCNN5 only)
    bool fused_ready = false;    // fused conv + projection kernels (bf16 and fp32 windows) usable (C <= 3)
    int64_t opt_fused = 1;
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
    // what the current call uses (read by the caller of tc_*_gates to hand the cleaning job to the head kernel)
    int *cur_count = nullptr, *cur_flags = nullptr, *cur_list = nullptr;
    bool cur_own = false;
};



const char *tc_error();
int tc_prepare(TcState &s, const Dims &d, const ConvWeights &cw, const float *d_wih0, const HeadWeights &hw,
               int splits, int num_sms, cudaStream_t st);
void tc_release(TcState &s);
bool tc_supported(const TcState &s, const Dims &d, int dtype, int64_t B, int mode);
bool tc_can_emit_features(const TcState &s);
int64_t tc_workspace_bytes(const TcState &s, const Dims &d, int64_t B);
// returns number of kernel launches, or <0 with *err set
int tc_frontend(TcState &s, const Dims &d, const ConvWeights &cw, const void *x, int64_t B, float *feats,
                int64_t sB, int64_t sP, void *ws, int num_sms, cudaStream_t st, const char **err);
// fused kernel: front end + layer-0 projection; leaves gates[B][64] (biases included).
bool tc_fused_supported(const TcState &s, const Dims &d, int dtype);
int tc_partial_slices(const TcState &s);
int tc_fused_gates(TcState &s, const Dims &d, const ConvWeights &cw, const HeadWeights &hw, const void *x, int64_t B,
                   float *feats, float *partial, float *gates, void *ws, int num_sms, cudaStream_t st, const char **err,
                   bool reduce_here = true, int *slices_out = nullptr);
// fp32 windows: streaming kernel with CUDA-core conv1 + wgmma projection (b2cnn_tc_fused.cuh)
bool tc_stream_supported(const TcState &s, const Dims &d, int dtype);
int tc_stream_gates(TcState &s, const Dims &d, const ConvWeights &cw, const HeadWeights &hw, const void *x, int64_t B,
                    float *feats, float *partial, float *gates, void *ws, int num_sms, cudaStream_t st, const char **err,
                    bool reduce_here = true, int *slices_out = nullptr);
int tc_features(TcState &s, const Dims &d, const ConvWeights &cw, const void *x, int64_t B, float *feats,
                int num_sms, cudaStream_t st, const char **err);
// sliding-window scorer (b2cnn_slide.cu): a segment's features into the position-major feature ring
bool tc_ring_supported(const TcState &s, const Dims &d);
int tc_ring_features(const TcState &s, const Dims &dseg, const ConvWeights &cw, const void *x, int64_t pitch, int dtype,
                     int64_t P, float *ring, int64_t ring_pitch, int cap, int slot0, int *flags, cudaStream_t st, const char **err);
int tc_ring_tmap(const float *ring, int64_t P, int64_t pitch, int L, CUtensorMap *tm, const char **err);

}  // namespace b2cnn

// b2cnn_internal.cuh -- shared declarations of libb2cnn (sm_90a only).
//
// The hot path being replaced is MyCNN.forward (bin/models.py:22-36 of the reference):
//   conv1+tanh (:23) -> pool (:24) -> [dropout = identity in eval (:25)] -> conv2+tanh (:26)
//   -> pool (:27) -> view(-1, MAGICNUM) (:29) -> 2-layer LSTM (:30) -> Linear (:31)
//   -> * relu(age*1e-8+1) (:32-33) -> squeeze (:34)
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "../../include/b2cnn.h"

namespace b2cnn {

constexpr int kCMid = 4;      // conv1 out_channels (models.py:10)
constexpr int kHidden = 16;   // LSTM hidden (models.py:16)
constexpr int kGates = 64;    // 4 * hidden, PyTorch gate order i,f,g,o
constexpr int kMaxW1 = 800;   // 4 * C * K1 floats kept in the kernel-parameter constant bank
constexpr int kMaxK2 = 8;

// Everything derived from b2cnn_config (see RefArch in oracle/mycnn_torch.py for the mirror).
struct Dims {
    int C, K1, K2, PK, PS, W;
    int L1, P1, L2, L;       // conv1 out, pool1 out, conv2 out, pool2 out (= LSTM input size)
    int act, has_affine;
    float age_coef;
    int XP;                  // row pitch of x in elements (>= W): channel rows start XP apart, windows C*XP apart.
                             // == W for a contiguous [B][C][W] tensor; set per call (b2cnn_forward_pitched)

    // consecutive features start F = pool_s^2 samples apart and each reads R samples, so L = (W - R) / F + 1
    int feature_stride() const { return PS * PS; }
    int receptive_field() const { return PS * (PK + K2 - 2) + PK + K1 - 1; }
};

// false when a size is below 1 or the window is too short for the conv/pool stack
inline bool derive_dims(const b2cnn_config &c, Dims &d) {
    d.C = c.in_channels; d.K1 = c.k1; d.K2 = c.k2; d.PK = c.pool_k; d.PS = c.pool_s; d.W = c.window;
    d.act = c.act; d.has_affine = (c.flags & B2CNN_FLAG_AFFINE) ? 1 : 0; d.age_coef = c.age_coef; d.XP = c.window;
    if (d.C < 1 || d.K1 < 1 || d.K2 < 1 || d.PK < 1 || d.PS < 1 || d.W < 1) return false;
    d.L1 = d.W - d.K1 + 1;
    if (d.L1 < d.PK) return false;
    d.P1 = (d.L1 - d.PK) / d.PS + 1;
    d.L2 = d.P1 - d.K2 + 1;
    if (d.L2 < d.PK) return false;
    d.L = (d.L2 - d.PK) / d.PS + 1;
    return d.L >= 1;
}

// Offsets (floats) of the tensors in the packed weight blob (include/b2cnn.h: b2cnn_weight_count is total): the conv
// parameters [w1, wih0), the LSTM and the output layer, then with has_affine the conv-epilogue affine block
// [affine, total) = s1[4], t1[4], s2, t2.
struct BlobOff {
    int64_t w1, b1, w2, b2, wih0, whh0, bih0, bhh0, wih1, whh1, bih1, bhh1, wo, bo, affine, total;
};
__host__ __device__ inline BlobOff blob_offsets(const Dims &d) {
    BlobOff o;
    int64_t p = 0;
    o.w1 = p; p += (int64_t)kCMid * d.C * d.K1;
    o.b1 = p; p += kCMid;
    o.w2 = p; p += kCMid * d.K2;
    o.b2 = p; p += 1;
    o.wih0 = p; p += (int64_t)kGates * d.L;
    o.whh0 = p; p += kGates * kHidden;
    o.bih0 = p; p += kGates;
    o.bhh0 = p; p += kGates;
    o.wih1 = p; p += kGates * kHidden;
    o.whh1 = p; p += kGates * kHidden;
    o.bih1 = p; p += kGates;
    o.bhh1 = p; p += kGates;
    o.wo = p; p += kHidden;
    o.bo = p; p += 1;
    o.affine = p; if (d.has_affine) p += 2 * kCMid + 2;
    o.total = p;
    return o;
}

// The sequence lengths of a _seq call (include/b2cnn.h): a host array of n lengths; on == false for the calls that take
// a mode instead
struct SeqLengths {
    bool on;
    const int64_t *len;
    int64_t n;
};
// off = the n + 1 offsets 0, n_0, n_0 + n_1, ..., B of lengths that are each >= 1 and sum to B; false (with the reason in
// err) for a NULL array, n < 1, a length below 1 or a sum that is not B.  No CUDA call.
inline bool seq_offsets(const SeqLengths &sl, int64_t B, std::vector<int64_t> &off, const char **err) {
    if (!sl.len || sl.n < 1 || sl.n > B) { *err = "seq_lengths: NULL, or n_seq not in [1, B]"; return false; }
    off.resize((size_t)sl.n + 1);
    off[0] = 0;
    for (int64_t s = 0; s < sl.n; ++s) {
        const int64_t v = sl.len[s];
        if (v < 1 || v > B - off[s]) { *err = v < 1 ? "seq_lengths: every length must be >= 1" : "seq_lengths: the lengths add up to more than B"; return false; }
        off[s + 1] = off[s] + v;
    }
    if (off[sl.n] != B) { *err = "seq_lengths: the lengths add up to less than B"; return false; }
    return true;
}

// whether the device arrays of `bytes` bytes at a and at b share a byte (false when either is null)
inline bool overlap(const void *a, const void *b, size_t bytes) {
    if (!a || !b) return false;
    const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
    return x < y + bytes && y < x + bytes;
}

// The windows of a _record training call (include/b2cnn.h): B recordings of N samples, windows of the configuration's W
// samples every S samples, counts[b] of them (a host array) from recording b; on == false for every other call.  The
// _record_state calls (sequence mode) add the LSTM state of each recording, device [B][64] = h0 | c0 | h1 | c1, each
// pointer may be null: state_in (the scan starts from it instead of zero), state_out (the state after the recording's
// last counted window), and for the backward d_state_out (the gradient arriving at state_out) and d_state_in (the
// gradient of state_in).  A recording without windows passes both through.
struct RecordArgs {
    bool on;
    int64_t N, S;
    const int64_t *counts;
    const float *state_in = nullptr;
    float *state_out = nullptr;
    const float *d_state_out = nullptr;
    float *d_state_in = nullptr;
    bool has_state() const { return state_in || state_out || d_state_out || d_state_in; }
    // whether two of the state arrays of B recordings overlap: an output written while an input is still to be read
    bool states_overlap(int64_t B) const {
        const void *p[4] = {state_in, state_out, d_state_out, d_state_in};
        const size_t bytes = sizeof(float) * 64 * (size_t)B;
        for (int i = 0; i < 4; ++i)
            for (int j = i + 1; j < 4; ++j)
                if (overlap(p[i], p[j], bytes)) return true;
        return false;
    }
};

// Makes `device` current for the guard's lifetime and restores the caller's device on every exit path (a call on cuda:1
// must not leave the calling thread on cuda:1: later `device="cuda"` allocations of the host framework would land on the
// wrong GPU).  A negative device leaves the current device as it is.
struct DeviceGuard {
    int prev = -1;
    cudaError_t err = cudaSuccess;
    explicit DeviceGuard(int dev) {
        if (dev < 0) return;
        err = cudaGetDevice(&prev);
        if (err != cudaSuccess) { prev = -1; return; }
        if (prev != dev) err = cudaSetDevice(dev); else prev = -1;     // nothing to restore
    }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
    DeviceGuard(const DeviceGuard &) = delete;
    DeviceGuard &operator=(const DeviceGuard &) = delete;
};

// Conv weights travel as a by-value kernel parameter: they land in the constant bank, so the
// fully unrolled FFMAs of the templated kernels read them as c[0x0][imm] operands.
struct ConvWeights {
    float w1[kMaxW1];          // [c][k][o]  -> (c*K1 + k)*4 + o
    float b1[kCMid];
    float w2[kCMid * kMaxK2];  // [c][k]     -> c*K2 + k
    float b2;
    float s1[kCMid], t1[kCMid], s2, t2;   // optional conv-epilogue affine (folded eval-BN)
};

// Small LSTM / head tensors: device pointers into the handle's copy of the packed blob.
struct HeadWeights {
    const float *wih0T;   // [L][64]  transposed copy of lstm.weight_ih_l0
    const float *whh0;    // [64][16]
    const float *bih0, *bhh0;
    const float *wih1, *whh1;   // [64][16]
    const float *bih1, *bhh1;
    const float *wo, *bo;       // out.weight[16], out.bias[1]
};

struct FrontParams {
    const void *x;        // [B][C][W] f32 or bf16
    float *feats;         // features, element (b, p) at feats[b*sB + p*sP]
    int64_t sB, sP;
    int B;
    int tile_p;           // final positions per tile
    int n_tiles;
    Dims d;
    int xs_stride, a1_stride;   // padded smem row strides (floats)
    const int *win_list;        // optional: indices of the windows to process (device memory)
    const int *win_count;       //           and how many (device memory)
    // gate mode (the exact re-computation behind the streaming tensor-core kernels): instead of writing feature
    // rows, every CTA multiplies the features of its tiles by W_ih_l0^T and writes gate_part[slice][b][64];
    // slice = blockIdx.x covers tiles [slice * tiles_per_slice, ...), slices >= gate_slices_used are zero-filled
    float *gate_part;           // [gate_slices][B][64] or nullptr
    const float *wih0T;         // [L][64]
    int gate_slices, tiles_per_slice;
    ConvWeights cw;
};

// NaN-propagating max, as ATen's max_pool1d ((v > m) || isnan(v)); fmaxf would drop NaNs.
__device__ __forceinline__ float max_nan(float a, float b) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

__device__ __forceinline__ float apply_act(float v, int act) {
    if (act == B2CNN_ACT_TANH) return tanhf(v);
    if (act == B2CNN_ACT_RELU) return (v > 0.f || v != v) ? v : 0.f;
    return v;
}

__device__ __forceinline__ float sigmoid_acc(float v) { return 1.0f / (1.0f + expf(-v)); }

// conflict-free smem index for "thread r reads a window starting at stride*r": one pad word
// every 32 keeps lanes of a warp on distinct banks for strides 4 and 8.
__host__ __device__ __forceinline__ int padi(int g) { return g + (g >> 5); }

// ---- launchers (b2cnn_generic.cu / b2cnn_head.cu) ----------------------------------------
// Each returns the number of kernels it launched, or <0 with the message in `err`: kLaunchArch when the
// configuration exceeds what the kernel can hold (nothing was launched; the API reports B2CNN_EARCH), any other
// negative value for a CUDA error.
constexpr int kLaunchArch = -2;
int launch_frontend_generic(const Dims &d, const ConvWeights &cw, const void *x, int dtype,
                            int64_t B, float *feats, int64_t sB, int64_t sP, cudaStream_t st,
                            int num_sms, const char **err);

int launch_frontend_generic_listed(const Dims &d, const ConvWeights &cw, const void *x, int dtype,
                                   int64_t B, float *feats, int64_t sB, int64_t sP, const int *win_list,
                                   const int *win_count, cudaStream_t st, int num_sms, const char **err);

// whether the generic front end's tile of min(d.L, 508) final positions fits shared memory (else kLaunchArch)
bool frontend_generic_fits(const Dims &d);

// exact gate partials of the listed windows straight into the range-partial buffer the head sums (no feature rows)
int launch_frontend_generic_gates_listed(const Dims &d, const ConvWeights &cw, const void *x, int dtype, int64_t B,
                                         const float *wih0T, float *gate_part, int gate_slices, const int *win_list,
                                         const int *win_count, cudaStream_t st, int num_sms, const char **err);

// seq_off / n_seq (sequence mode only): the scan runs over n_seq sequences, rows [seq_off[s], seq_off[s + 1]) of the
// batch (device memory), instead of over all B rows
int launch_head(const Dims &d, const HeadWeights &hw, const float *feats, int64_t sB, int64_t sP,
                int64_t B, const float *age, int64_t n_age, int mode, int apply_sigmoid,
                float *out, float *gates_ws, float *partial_ws, int ksplit, cudaStream_t st,
                const char **err, const int64_t *seq_off = nullptr, int64_t n_seq = 0);

int launch_reduce_gates(const float *partial, int slices, int64_t B, const HeadWeights &hw, float *gates,
                        cudaStream_t st, const char **err);
int launch_lstm_head(const Dims &d, const HeadWeights &hw, const float *gates, int64_t B, const float *age,
                     int64_t n_age, int mode, int apply_sigmoid, float *out, cudaStream_t st, const char **err,
                     const int64_t *seq_off = nullptr, int64_t n_seq = 0);
// sequence mode over n_seg segments of seg_len consecutive rows of gates [n_seg seg_len][64], age (n_age = 1 or n_seg
// seg_len) and out, each scanned from the zero state; launch_lstm_head's sequence mode is one segment of B rows.
// seg_off != nullptr (device memory, n_seg + 1 offsets): segment s is rows [seg_off[s], seg_off[s + 1]) instead.
// state_in / state_out (device memory, [n_seg][64] = h0 | c0 | h1 | c1, each may be null): segment s starts from
// state_in[s] instead of zero, and its state after its last row is stored to state_out[s]
int launch_sequence_segments(const Dims &d, const HeadWeights &hw, const float *gates, int64_t n_seg, int64_t seg_len, const float *age,
                             int64_t n_age, int apply_sigmoid, float *out, cudaStream_t st, const char **err,
                             const int64_t *seg_off = nullptr, const float *state_in = nullptr, float *state_out = nullptr);
// a sequence-mode sliding scorer's head: for every live patient p (all with seen == nullptr, else seen[p] >= 0 &&
// seen[p] + S >= d.W, the counts before the push advances them), one LSTM step from state[p] [64] = h0 | c0 | h1 | c1,
// its layer-0 gates summed from partial [slices][P][64] as launch_reduce_gates does; out[p] and state[p] written
int launch_seq_step(const Dims &d, const HeadWeights &hw, const float *partial, int slices, int64_t P, const float *age, int64_t n_age,
                    int apply_sigmoid, float *out, float *state, const int64_t *seen, int64_t S, cudaStream_t st, const char **err);

int launch_reduce_lstm_head(const Dims &d, const HeadWeights &hw, const float *partial, int slices, int64_t B,
                            const float *age, int64_t n_age, int apply_sigmoid, float *out, cudaStream_t st, const char **err,
                            int *clean_count = nullptr, int *clean_flags = nullptr, const int *clean_list = nullptr);

int choose_ksplit(int L);
int proj_slices(int L);       // split-K slices launch_head's projection writes for L positions: [slices][B][64] partials

// launch_head of independent windows whose features sit in a sliding scorer's position-major ring (b2cnn_slide.cu):
// position k < d.L of window b in ring[((head + k) mod cap) * pitch + b] (cap >= d.L: the window may be a suffix of the
// ring's); the same tiles and summation order as launch_head
int launch_ring_head(const Dims &d, const HeadWeights &hw, const float *ring, int64_t pitch, int cap, int head, int64_t B,
                     const float *age, int64_t n_age, int apply_sigmoid, float *out, float *gates_ws, float *partial_ws,
                     cudaStream_t st, const char **err);
// launch_ring_head's projection alone: partial_ws [slices][B][64]; returns slices (-1 on error)
int launch_ring_proj(const Dims &d, const HeadWeights &hw, const float *ring, int64_t pitch, int cap, int head, int64_t B, float *partial_ws,
                     cudaStream_t st, const char **err);

// launch_head of the n_w windows of each whole recording (b2cnn_record.cu, b2cnn_score_record, generic path): row b =
// window b mod n_w of recording b / n_w, position k at feats[(b / n_w) rec_pitch + (b mod n_w) step + k]; rows =
// recordings x n_w; the same tiles and summation order as launch_head.  mode B2CNN_MODE_SEQUENCE: one LSTM scan per
// recording over its n_w windows (launch_sequence_segments, from state_in and into state_out) instead of independent windows
int launch_record_head(const Dims &d, const HeadWeights &hw, const float *feats, int64_t rec_pitch, int n_w, int64_t step, int64_t rows,
                       const float *age, int64_t n_age, int mode, int apply_sigmoid, float *out, float *gates_ws, float *partial_ws,
                       cudaStream_t st, const char **err, const float *state_in = nullptr, float *state_out = nullptr);

// b2cnn_small.cu: whole forward pass of short windows in one launch (independent windows only)
bool small_supported(const Dims &d);
int launch_small_forward(const Dims &d, const ConvWeights &cw, const HeadWeights &hw, const void *x, int dtype, int64_t B,
                         const float *age, int64_t n_age, int apply_sigmoid, float *out, cudaStream_t st, const char **err);

// b2cnn_batch.cu: many short windows per launch, one warp per window (the production shape [P, 10, 120])
bool batch_supported(const Dims &d);
int launch_short_batch(const Dims &d, const ConvWeights &cw, const HeadWeights &hw, const void *x, int dtype, int64_t B,
                       const float *age, int64_t n_age, int apply_sigmoid, float *out, int num_sms, cudaStream_t st, const char **err);

// b2cnn_prep.cu: preprocessing + window assembly in front of the model call (f2 + f1)
int64_t prep_window_count(int64_t n_samples, double fs, const b2cnn_prep_config *cfg);
int64_t prep_workspace_bytes(int64_t n_samples, double fs, int n_sel, const b2cnn_prep_config *cfg);
int prep_windows(const int16_t *raw, int64_t n_samples, int n_sig, const int *sel, int n_sel, const double *gains,
                 const double *baselines, double fs, const b2cnn_prep_config *cfg, void *x_out, int dtype, double *t0_out,
                 void *workspace, int64_t ws_bytes, cudaStream_t st, const char **err);

// streaming form of the same preprocessing: per-patient device ring buffers (b2cnn_prep.cu)
struct Ring;
int ring_create(const b2cnn_prep_config *cfg, int n_patients, int n_sig, double fs, int device, Ring **out, const char **err);
void ring_destroy(Ring *r);
int ring_device(const Ring *r);
int ring_reset(Ring *r, cudaStream_t st, const char **err);
int ring_set_signals(Ring *r, int patient, const int *sel, int n_sel, const double *gains, const double *baselines,
                     cudaStream_t st, const char **err);
int ring_push(Ring *r, const void *new_samples, int sample_kind, int64_t n_new, void *x_out, int dtype, int *emitted,
              int64_t *window_out, double *t0_out, cudaStream_t st, const char **err);

// b2cnn_wire.cu: the reference's JSON wire formats decoded on the device (row f3)
int wire_decode_pairs(const uint8_t *bytes, const int64_t *offsets, int64_t n_msgs, int *idx_out, double *val_out,
                      const int64_t *row_of_msg, double *frame, int64_t frame_rows, int n_sig, int *n_bad, cudaStream_t st,
                      const char **err);
int wire_decode_arrays(const uint8_t *bytes, const int64_t *offsets, int64_t n_msgs, int max_vals, double *vals_out, int *counts_out,
                       int *n_bad, cudaStream_t st, const char **err);
double wire_parse_decimal_host(const char *s, int64_t len, int *status);

// b2cnn_train.cu: one training step (row f4).  mode is B2CNN_MODE_*; every entry point checks all its arguments before
// any CUDA call, then makes cfg->device current for the call (a negative device: the current one)
// sl: the sequence lengths of a _seq call (mode is then B2CNN_MODE_SEQUENCE), or {false} for the calls that take a mode
// heads: 0 for the calls that train one model, K in [1, B2CNN_SLIDE_MAX_HEADS] for b2cnn_train_heads_*
int64_t train_workspace_bytes(const b2cnn_config *cfg, int64_t B, const SeqLengths &sl, const RecordArgs &ra, int mode, int heads = 0);
// weighted != 0: BCEWithLogitsLoss(pos_weight=pos_weight), else plain BCEWithLogitsLoss
int train_step(const b2cnn_config *cfg, float *params, float *adam_m, float *adam_v, float *grads, int64_t step, float lr, float beta1,
               float beta2, float eps, int apply_update, const float *x, int64_t B, const float *age, const float *target,
               int weighted, float pos_weight, int mode, const SeqLengths &sl, const RecordArgs &ra, const float *mask1, const float *mask2,
               float *loss_out, void *workspace, int64_t ws_bytes, cudaStream_t st, const char **err);
// the autograd seam
int train_forward(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age, int mode, const SeqLengths &sl,
                  const RecordArgs &ra, const float *mask1, const float *mask2, float *z_out, void *workspace, int64_t ws_bytes, cudaStream_t st, const char **err);
int train_backward(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age, int mode, const SeqLengths &sl,
                   const RecordArgs &ra, const float *mask1, const float *mask2, const float *dz, float *grads, float *dx, float *dage, int flags,
                   void *workspace, int64_t ws_bytes, cudaStream_t st, const char **err);
// b2cnn_train_heads_step / _record: n_heads blobs on the conv weights of `frontend`; params, adam_m, adam_v, grads and lr
// are host arrays of n_heads entries, loss_out a device array of n_heads floats
int train_heads_step(const b2cnn_config *cfg, const float *frontend, int n_heads, float *const *params, float *const *adam_m,
                     float *const *adam_v, float *const *grads, const float *lr, int64_t step, float beta1, float beta2, float eps,
                     int apply_update, const float *x, int64_t B, const float *age, const float *target, int weighted, float pos_weight,
                     int mode, const SeqLengths &sl, const RecordArgs &ra, const float *mask1, const float *mask2, float *loss_out,
                     void *workspace, int64_t ws_bytes, cudaStream_t st, const char **err);

void launch_transpose_wih(const float *wih0, float *wih0T, int L, cudaStream_t st);

// 64-bit FNV-1a over what the features depend on: the front-end geometry and the used conv weights (affine when on);
// b2cnn_slide_state_header's frontend_digest (b2cnn_slide.cu)
uint64_t frontend_digest(const Dims &d, const ConvWeights &cw);

}  // namespace b2cnn

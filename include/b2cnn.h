/*
 * b2cnn.h -- C ABI of the B200-native MyCNN forward pass (libb2cnn.so).
 *
 * The reference (travistangvh/time-series-kafka-demo) has no plugin/FFI seam: the only
 * boundary of its hot path is the Python call `output = model(x_arr, a_arr)`
 * (bin/predictStream.py:157; also bin/utils.py:204,249,682) into `MyCNN.forward`
 * (bin/models.py:22-36).  These entry points are what a ctypes/cffi binding for that call
 * binds; INTEGRATION.md shows the stub.  Plain pointers and sizes only -- no torch types.
 *
 * Ownership: the caller owns x / age / out / workspace; the library owns only its packed
 * weight buffers, 512 KB of NaN-exception state allocated with them (flags of the windows the
 * tensor-core kernels hand to the exact path; zero between calls, used by calls on the first
 * stream a handle sees -- other streams use a copy in the workspace) and, for b2cnn_forward_host,
 * its pinned/device staging buffers.  A handle serves one call at a time.
 * b2cnn_forward makes no allocation and is asynchronous on `stream`.
 * Errors: every call returns 0 on success or a B2CNN_E* code; b2cnn_last_error() returns a
 * thread-local message.  There is no CPU fallback anywhere in this library.
 */
#ifndef B2CNN_H_
#define B2CNN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2CNN_OK 0
#define B2CNN_EINVAL 1      /* bad argument / shape / dtype                                */
#define B2CNN_EARCH 2       /* architecture outside what the kernels support               */
#define B2CNN_EVIEW 3       /* L_out(window) != lstm_input: x.view(-1, MAGICNUM) would      */
                            /* straddle windows (bin/models.py:29) -- rejected, not guessed */
#define B2CNN_ECUDA 4       /* CUDA runtime / driver error                                  */
#define B2CNN_ESTATE 5      /* weights not set, workspace too small, ...                    */

enum { B2CNN_DTYPE_F32 = 0, B2CNN_DTYPE_BF16 = 1 };
/* INDEPENDENT: every window starts from the zero LSTM state == looping the reference one
 *   window at a time (bin/predictStream.py:70,157).
 * SEQUENCE: bit-for-bit the structure of model(x_batch): the LSTM scans the batch axis
 *   (bin/models.py:29-30 with B>1; bin/utils.py:249). */
enum { B2CNN_MODE_INDEPENDENT = 0, B2CNN_MODE_SEQUENCE = 1 };
enum { B2CNN_ACT_TANH = 0, B2CNN_ACT_RELU = 1, B2CNN_ACT_IDENTITY = 2 };
enum { B2CNN_PATH_AUTO = 0, B2CNN_PATH_GENERIC = 1, B2CNN_PATH_TENSORCORE = 2,
       B2CNN_PATH_STREAM = 3 /* reported by b2cnn_last_path only: fp32 windows, streamed CUDA-core conv1 + tcgen05 projection */ };

#define B2CNN_FLAG_AFFINE 1 /* per-channel scale/shift after each conv (folded eval-BatchNorm) */

/* Mirrors the constructor of MyCNN (bin/models.py:6-20). */
typedef struct b2cnn_config {
    int32_t in_channels; /* conv1 in_channels            models.py:10 (10; 7 in MyCNN2/3)    */
    int32_t k1;          /* conv1 kernel_size            models.py:10 (10; 5 in MyCNN2/3/4)  */
    int32_t c_mid;       /* conv1 out_channels           models.py:10 (must be 4)            */
    int32_t k2;          /* conv2 kernel_size            models.py:11 (5)                    */
    int32_t pool_k;      /* MaxPool1d kernel_size        models.py:12 (3; 2 in MyCNN2/3/4)   */
    int32_t pool_s;      /* MaxPool1d stride             models.py:12 (2)                    */
    int32_t hidden;      /* LSTM hidden_size             models.py:16 (must be 16)           */
    int32_t layers;      /* LSTM num_layers              models.py:16 (must be 2)            */
    int32_t window;      /* samples per window W         config.cfg:23 (120)                 */
    int32_t lstm_input;  /* MAGICNUM                     models.py:8  (must equal L_out(W))  */
    int32_t act;         /* B2CNN_ACT_*; the reference uses tanh (models.py:23,26)           */
    int32_t flags;       /* B2CNN_FLAG_*                                                     */
    float age_coef;      /* models.py:32 (1e-8)                                              */
    int32_t device;      /* CUDA device ordinal, or -1 for the current device                */
} b2cnn_config;

typedef struct b2cnn_handle b2cnn_handle;

/* L_out(W): conv1 -> pool -> conv2 -> pool output length (floor pooling); <=0 if invalid. */
int64_t b2cnn_l_out(const b2cnn_config *cfg);

/* Number of floats in the packed weight blob, in this order (== state_dict order of the
 * used tensors, bin/models.py:10-17):
 *   conv1.weight[4][C][K1], conv1.bias[4], conv2.weight[1][4][K2], conv2.bias[1],
 *   lstm.weight_ih_l0[64][L], lstm.weight_hh_l0[64][16], lstm.bias_ih_l0[64], lstm.bias_hh_l0[64],
 *   lstm.weight_ih_l1[64][16], lstm.weight_hh_l1[64][16], lstm.bias_ih_l1[64], lstm.bias_hh_l1[64],
 *   out.weight[16], out.bias[1]
 *   (+ if B2CNN_FLAG_AFFINE: scale1[4], shift1[4], scale2[1], shift2[1]) */
int64_t b2cnn_weight_count(const b2cnn_config *cfg);

/* Replaces `model = torch.load(path); model.eval()` (bin/predictStream.py:36-37). */
int b2cnn_create(const b2cnn_config *cfg, b2cnn_handle **out);
void b2cnn_destroy(b2cnn_handle *h);

/* Replaces load_state_dict: copies the packed blob (host or device memory) into the
 * library's device buffers, enqueued on `stream` (a cudaStream_t, may be NULL). */
int b2cnn_set_weights(b2cnn_handle *h, const float *blob, int64_t n_floats, int blob_on_device,
                      void *stream);

/* Bytes of caller-provided device scratch b2cnn_forward needs for a batch of B windows.
 * b2cnn_workspace_bytes is dtype-blind: enough for any path and any row pitch, the generic path's [B][L_out] feature
 * rows and, where the tensor-core kernels exist for the handle, the B*C*round_up(W,8) bf16 staging rows included
 * (also when W % 8 == 0: a bf16 b2cnn_forward_pitched call whose x_pitch is not a multiple of 8 needs them);
 * b2cnn_workspace_bytes_for is exact for contiguous windows of `dtype`: where the streaming tensor-core kernels apply,
 * the features never leave the SM and the scratch is the range partials only (39 MB instead of 346 MB at
 * [4096,3,75000]).  A pitched call with rows that are not a multiple of 16 bytes may need more than the _for size;
 * it is refused with B2CNN_ESTATE instead. */
int64_t b2cnn_workspace_bytes(b2cnn_handle *h, int64_t B, int mode);
int64_t b2cnn_workspace_bytes_for(b2cnn_handle *h, int64_t B, int mode, int dtype);

/* Replaces `output = model(x, age)` (bin/predictStream.py:157).  All pointers are DEVICE
 * pointers.  x: [B][C][W] contiguous, dtype f32 or bf16.  age: n_age == B or 1 (broadcast).
 * out: [B] floats: the logit (bin/models.py:34), or sigmoid(logit) if apply_sigmoid
 * (bin/predictStream.py:160). */
int b2cnn_forward(b2cnn_handle *h, const void *x, int dtype, int64_t B, const float *age,
                  int64_t n_age, int mode, int apply_sigmoid, float *out, void *workspace,
                  int64_t workspace_bytes, void *stream);

/* b2cnn_forward for windows whose channel rows are `x_pitch` ELEMENTS apart (x_pitch >= W; window b starts at
 * x + b * C * x_pitch): a producer that pads its rows to a multiple of 16 bytes (8 bf16 / 4 fp32 samples) lets TMA
 * stream windows of ANY length straight from `x`; a contiguous tensor with W % 8 != 0 (7500, 37500 ...) has to be
 * re-pitched into scratch first (one extra read + write of the input).  The pad is never read. */
int b2cnn_forward_pitched(b2cnn_handle *h, const void *x, int dtype, int64_t B, int64_t x_pitch, const float *age,
                          int64_t n_age, int mode, int apply_sigmoid, float *out, void *workspace,
                          int64_t workspace_bytes, void *stream);

/* Many sequences in one sequence-mode call: the B windows are n_seq consecutive sequences of seq_lengths[0], ...,
 * seq_lengths[n_seq - 1] windows (a HOST array; every length >= 1, the lengths add up to B), and the LSTM scans each
 * sequence from the zero state, no state crossing from one to the next -- what one b2cnn_forward(mode =
 * B2CNN_MODE_SEQUENCE) call per sequence returns, row for row, with the front end run once for the whole batch.
 * {B} is B2CNN_MODE_SEQUENCE over the batch, {1, ..., 1} is B2CNN_MODE_INDEPENDENT.  x, x_pitch, age, n_age,
 * apply_sigmoid and out as in b2cnn_forward_pitched.  Bad lengths (NULL, n_seq < 1, a length below 1, a sum other
 * than B) are B2CNN_EINVAL before any CUDA call.  workspace: b2cnn_workspace_bytes_seq() bytes, which is
 * b2cnn_workspace_bytes(h, B) plus a region the call copies the sequence offsets into (from the host array, on
 * `stream`); a smaller one is B2CNN_ESTATE before any launch.  The call allocates nothing. */
int64_t b2cnn_workspace_bytes_seq(b2cnn_handle *h, int64_t B, const int64_t *seq_lengths, int64_t n_seq);
int b2cnn_forward_seq(b2cnn_handle *h, const void *x, int dtype, int64_t B, int64_t x_pitch, const float *age, int64_t n_age,
                      const int64_t *seq_lengths, int64_t n_seq, int apply_sigmoid, float *out, void *workspace,
                      int64_t workspace_bytes, void *stream);

/* Same call with HOST pointers (ideally pinned): chunked H2D copy of x overlapped with
 * compute, D2H of the B results; synchronous on return.  Uses library-owned staging. */
int b2cnn_forward_host(b2cnn_handle *h, const void *x_host, int dtype, int64_t B,
                       const float *age_host, int64_t n_age, int mode, int apply_sigmoid,
                       float *out_host);

/* Intermediate of bin/models.py:29 (after the second pool, before the LSTM):
 * feats[B][L_out] floats on the device.  For parity tests. */
int b2cnn_features(b2cnn_handle *h, const void *x, int dtype, int64_t B, float *feats,
                   void *stream);

/* Options: "path" = B2CNN_PATH_*; "tc_splits" = 2|3: bf16 pieces per fp32 conv1 weight on the
 * tensor cores (3, default: exact fp32 weights; 2: weights rounded to 16 mantissa bits);
 * "tc_fused" = 0|1 (default 1): bf16 windows take the fused conv+projection kernel; "small_kernel" = 0|1;
 * "profile" = 0|1: record CUDA events around the stages of each b2cnn_forward on its stream. */
int b2cnn_set_option(b2cnn_handle *h, const char *key, int64_t value);
int64_t b2cnn_get_option(b2cnn_handle *h, const char *key);

/* Kernel launches issued by the most recent forward on this handle (bench: gpu_launches),
 * and which path it took (B2CNN_PATH_GENERIC / B2CNN_PATH_TENSORCORE / B2CNN_PATH_STREAM). */
int64_t b2cnn_last_launch_count(b2cnn_handle *h);
int b2cnn_last_path(b2cnn_handle *h);

/* With option "profile"=1: device time in ms of a stage of the most recent b2cnn_forward
 * (0 = front end conv/pool kernel(s), the dominant kernel; 1 = projection + LSTM head).
 * Synchronises on the stage's end event.  <0 if unavailable. */
double b2cnn_last_stage_ms(b2cnn_handle *h, int stage);

/* ---- The two steps in front of the model call, on the device (SURVEY.md section 8, rows f2 + f1) ----
 * b2cnn_prep_windows replaces, for replay, what reaches bin/predictStream.py:105-139 through Kafka and
 * Spark: the 180 s / 5 s sliding mean with nulls skipped (bin/processStream.py:196-208), forward-fill,
 * back-fill and 0-fill of that grid (bin/processStream.py:62-123), and the 600 s / 60 s window assembly
 * x_arr[0, signal_index, :] with zeros for absent signals (bin/predictStream.py:105-139,245-259).
 *   raw        device pointer, int16 [n_samples][n_sig]: a WFDB format-16 numerics record as on disk
 *              (-32768 = missing; physical = (adc - baseline) / gain, what wfdb.rdrecord returns,
 *              bin/sendStream.py:46)
 *   sel        host array [n_sel]: record columns of the model's signals; position i becomes model
 *              channel i (the message index of bin/sendStream.py:59-64)
 *   gains / baselines  host arrays [n_sig]
 *   x_out      device pointer, [n_windows][n_channels][window_points] in `dtype` (f32 or bf16)
 *   t0_out     device pointer or NULL, [n_windows] window start times in seconds
 * The caller owns every buffer; the call allocates nothing and is asynchronous on `stream`. */
typedef struct b2cnn_prep_config {
    int32_t n_channels;    /* model input channels                 config.cfg CHANNEL_NAMES (10)      */
    int32_t window_points; /* points per window                    config.cfg WINDOWSIZE (120)        */
    int32_t grid_s;        /* slide of the smoothing window        processStream.py:199 (5 s)         */
    int32_t smooth_s;      /* length of the smoothing window       processStream.py:199 (180 s)       */
    int32_t stride_s;      /* slide of the model window            predictStream.py:252 (60 s)        */
} b2cnn_prep_config;
int64_t b2cnn_prep_window_count(int64_t n_samples, double fs, const b2cnn_prep_config *cfg);
int64_t b2cnn_prep_workspace_bytes(int64_t n_samples, double fs, int32_t n_sel, const b2cnn_prep_config *cfg);
int b2cnn_prep_windows(const int16_t *raw, int64_t n_samples, int32_t n_sig, const int32_t *sel, int32_t n_sel,
                       const double *gains, const double *baselines, double fs, const b2cnn_prep_config *cfg,
                       void *x_out, int dtype, double *t0_out, void *workspace, int64_t workspace_bytes, void *stream);

/* ---- The same two steps as a STREAM: per-patient device ring buffers (SURVEY.md section 8, row f1) ----
 * Replaces the per-trigger Python loop of bin/predictStream.py:70-156 (one row per patient, B = 1 each, numpy
 * assembly on the host) by device-resident state for P patients: every trigger appends the new samples of all
 * patients (b2cnn_ring_push), the grid points whose 180 s window is now complete are finalised and forward-filled
 * (bin/processStream.py:62-123,196-208), and the [P][n_channels][window_points] batch of the 600 s window that just
 * completed is written for ONE b2cnn_forward call.  Pushing a record trigger by trigger reproduces
 * b2cnn_prep_windows on the whole record bit-for-bit (tests/test_stream.py).
 *   n_sig        signals per sample frame (columns of the pushed arrays)
 *   fs           sampling rate shared by the ring's patients (1/60 Hz for MIMIC numerics), at least 1 / stride_s
 *   new_samples  DEVICE pointer [n_patients][n_new][n_sig]: B2CNN_SAMPLES_ADC16 = int16 ADC units as in a WFDB
 *                format-16 file (-32768 = missing; gain / baseline from b2cnn_ring_set_signals), or
 *                B2CNN_SAMPLES_F64 = physical values as fp64 (NaN = missing) -- what bin/sendStream.py:59-64 publishes
 *   emitted      host int: 1 when x_out was written (from the 10th trigger on), 0 while the first window fills
 * One push may carry at most stride_s seconds of samples (stride_s / grid_s grid points) and emits at most one window:
 * a push after which the window following the one it emits would also be complete is refused with B2CNN_EINVAL and
 * leaves the ring unchanged.  Pushes cut at cumulative stride boundaries (push n carries the samples with time
 * < n * stride_s) never are.  The ring owns its device buffers; b2cnn_ring_push allocates nothing and is asynchronous
 * on `stream`. */
enum { B2CNN_SAMPLES_ADC16 = 0, B2CNN_SAMPLES_F64 = 1,
       B2CNN_SAMPLES_GRID = 2 /* fp64 5-second grid points [n_patients][n_new][n_sig] as bin/processStream.py:126-131 publishes
                                 them on `call-stream` (already smoothed and filled, 12 per trigger): appended as they are */ };
typedef struct b2cnn_ring b2cnn_ring;
int b2cnn_ring_create(const b2cnn_prep_config *cfg, int32_t n_patients, int32_t n_sig, double fs, int32_t device,
                      b2cnn_ring **out);
void b2cnn_ring_destroy(b2cnn_ring *ring);
int b2cnn_ring_reset(b2cnn_ring *ring, void *stream);
/* sel[n_sel]: frame columns of the model's signals for this patient (position i -> model channel i);
 * gains / baselines: host arrays [n_sig] or NULL (physical input). */
int b2cnn_ring_set_signals(b2cnn_ring *ring, int32_t patient, const int32_t *sel, int32_t n_sel, const double *gains,
                           const double *baselines, void *stream);
int b2cnn_ring_push(b2cnn_ring *ring, const void *new_samples, int sample_kind, int64_t n_new, void *x_out, int dtype,
                    int32_t *emitted, int64_t *window_index, double *t0_seconds, void *stream);

/* ---- Long waveform windows scored incrementally: a per-patient feature ring (csrc/b2cnn_slide.cu) ----
 * The reference scores a patient with a W-sample window that slides by S samples (bin/predictStream.py:248-252: 600 s
 * every 60 s); consecutive windows share W - S samples.  The front end is translation-equivariant with a feature
 * stride of 4 samples, so for S % 4 == 0 feature i of a window is feature i + S/4 of the previous one: a scorer keeps
 * every patient's L = lstm_input features on the device and computes only the S/4 features each push completes, then
 * runs the input projection over the whole feature row and the head.
 *   b2cnn_slide_create   `h` with weights set; n_patients P >= 1; stride S with 1 <= S <= window and S % 4 == 0
 *                        (else B2CNN_EINVAL); dtype of the pushed samples, f32 or bf16.  The geometries and channel
 *                        counts of the streaming tensor-core kernels with both window dtypes and the packed W_ih
 *                        projection (MyCNN5 or MyCNN2/3/4 conv/pool, 1 to 3 channels, tanh, no affine); anything
 *                        else is B2CNN_EARCH.  C = 4 is left out on purpose: the fp32-window kernel and the packed
 *                        W_ih chunks exist for C <= 3 only.  Allocates all device state
 *                        (the fp32 ring, 4 P L bytes, and staging rows for one segment); the handle must outlive
 *                        the scorer.
 *   b2cnn_slide_push     new_samples: DEVICE pointer [P][C][S] in the scorer's dtype, channel rows `pitch` elements
 *                        apart (pitch >= S; window p starts at new_samples + p * C * pitch).  After push n (from 1 on)
 *                        every patient's window is the last W samples of its stream, [n S - W, n S).  Once n S >= W
 *                        the push writes out[P] (logits, or sigmoid(logit) if apply_sigmoid), sets *emitted = 1 and
 *                        *window_index = n - ceil(W / S); before that *emitted = 0 (the features are still stored).
 *                        out[p] == b2cnn_forward(window of p, mode INDEPENDENT) within fp32 rounding; age: n_age == 1
 *                        or P.  Rows 16-byte aligned with W % 4 == 0 stream straight from new_samples; otherwise the
 *                        segment is first copied into the scorer's aligned staging rows -- also when W % 4 != 0 and
 *                        the rows are aligned: the feature lattice then starts phi = (-W) mod 4 samples into the
 *                        segment, and the tensor-core kernel's TMA boxes must start on 16-byte boundaries.  B2CNN_ESTATE after
 *                        b2cnn_set_weights on the handle since the scorer's last reset (its features are stale).
 *                        Allocates nothing; asynchronous on `stream`.
 *   b2cnn_slide_reset    forget every stream (pushes count from 1 again) and accept the handle's current weights.
 *   b2cnn_slide_features feats[P][L] floats on the device: the features of the current windows in window order
 *                        (parity tests); B2CNN_ESTATE before the first window is complete or when the weights
 *                        changed since the last reset.
 * The scorer's patients are independent windows; a push uses no atomics in its value path, so its results do not
 * depend on P, on the ring's rotation or on the run.
 *
 * Per-patient lifecycle (a bed reassigned, a monitor reconnected).  Every patient p has seen[p]: its stream samples
 * since its admission, or -1 once discharged.  b2cnn_slide_reset admits every patient with seen = 0; a push adds S to
 * every admitted patient's count.  `patients` are HOST arrays of n distinct indices in [0, P).
 *   b2cnn_slide_admit    restarts the listed patients' streams.  history: DEVICE pointer [n][C][history_len] in the
 *                        scorer's dtype (`dtype` must name it), channel rows `pitch` elements apart (pitch >=
 *                        history_len; any alignment), or NULL with history_len == 0; 0 <= history_len <= window.  Its
 *                        last sample immediately precedes the next push's first one.  Then seen[p] = history_len, and
 *                        p's window after a later push is the last W samples of (history | pushes since admission),
 *                        defined once seen[p] >= W: with history_len == W at the very next push, and b2cnn_slide_features
 *                        returns that window right away.  Computes the history's features that lie in the current
 *                        window or a later one (the push kernels, into a scratch ring in
 *                        `workspace`, then scattered into the patients' ring columns) and their last 24 samples.
 *                        workspace: DEVICE, >= b2cnn_slide_admit_workspace_bytes(slide, n, history_len) bytes (else
 *                        B2CNN_ESTATE); allocates nothing; asynchronous on `stream` except for two small host-to-device
 *                        copies (the indices and the counts) from pageable memory.  B2CNN_ESTATE after
 *                        b2cnn_set_weights without a reset, as for a push.
 *   b2cnn_slide_discharge  seen[p] = -1 for the listed patients; their samples in later pushes are ignored.
 *   b2cnn_slide_samples_seen  seen[P] into a DEVICE int64 array (asynchronous on `stream`).
 * Once admit or discharge has been called (until the next reset), a push writes out[p] for patients with
 * seen[p] >= W and NaN for every other patient, sets *emitted = 1 when at least one patient has a complete window
 * (*window_index keeps its meaning, n - ceil(W / S), and may be negative), and b2cnn_slide_features writes NaN rows
 * for patients without a complete window and fails with B2CNN_ESTATE when no patient has one.  A scorer that never
 * calls either runs exactly the launches above.  Bad indices (out of range, listed twice), history_len outside
 * [0, window], a NULL history with history_len > 0, pitch < history_len or another dtype: B2CNN_EINVAL.
 *
 * Two implementations (DESIGN.md §6).  b2cnn_slide_create is the tensor-core path described above.
 *   b2cnn_slide_create_path  the same with a path: B2CNN_PATH_TENSORCORE is exactly b2cnn_slide_create;
 *                        B2CNN_PATH_GENERIC is exact fp32 on CUDA cores for every model b2cnn_create accepts (any channel
 *                        count, activation, affine and conv/pool geometry): the feature stride is F = pool_s^2 samples,
 *                        so stride % F == 0 (else B2CNN_EINVAL), and each patient keeps its last R - 1 samples, R =
 *                        pool_s (pool_k + k2 - 2) + pool_k + k1 - 1 the receptive field of one feature.  Its logits are
 *                        b2cnn_forward's with path = generic and small_kernel = 0 on the same windows.  B2CNN_EARCH, before
 *                        allocating anything, where b2cnn_forward on the whole windows would refuse the generic front end
 *                        (its tile does not fit shared memory).  B2CNN_PATH_AUTO: the tensor-core path where
 *                        b2cnn_slide_create succeeds, the generic path where it returns B2CNN_EARCH.  Any other path:
 *                        B2CNN_EINVAL.  Every b2cnn_slide_* call works on either path with the semantics above.
 *   b2cnn_slide_path     B2CNN_PATH_TENSORCORE or B2CNN_PATH_GENERIC: the path a scorer runs (-1 for NULL). */
typedef struct b2cnn_slide b2cnn_slide;
int b2cnn_slide_create(b2cnn_handle *h, int32_t n_patients, int32_t stride, int dtype, b2cnn_slide **out);
int b2cnn_slide_create_path(b2cnn_handle *h, int32_t n_patients, int32_t stride, int dtype, int path, b2cnn_slide **out);
int b2cnn_slide_path(const b2cnn_slide *slide);
void b2cnn_slide_destroy(b2cnn_slide *slide);
int b2cnn_slide_reset(b2cnn_slide *slide, void *stream);
int b2cnn_slide_push(b2cnn_slide *slide, const void *new_samples, int64_t pitch, const float *age, int64_t n_age,
                     int apply_sigmoid, float *out, int32_t *emitted, int64_t *window_index, void *stream);
int b2cnn_slide_features(b2cnn_slide *slide, float *feats, void *stream);
int64_t b2cnn_slide_admit_workspace_bytes(b2cnn_slide *slide, int32_t n, int64_t history_len);
int b2cnn_slide_admit(b2cnn_slide *slide, const int32_t *patients, int32_t n, const void *history, int64_t history_len,
                      int64_t pitch, int dtype, void *workspace, int64_t workspace_bytes, void *stream);
int b2cnn_slide_discharge(b2cnn_slide *slide, const int32_t *patients, int32_t n, void *stream);
int b2cnn_slide_samples_seen(b2cnn_slide *slide, int64_t *seen, void *stream);

/* Sequence mode: every patient scored as the reference's run_model scores a recording (bin/utils.py:671-692, the LSTM
 * running along the batch axis, bin/models.py:29-30), live.  Each patient p keeps its LSTM state (h and c of both
 * layers, 256 bytes) on the device, carried from its previous scored window to the next.
 *   b2cnn_slide_create_ex  b2cnn_slide_create_path with a batch mode.  mode = B2CNN_MODE_INDEPENDENT: exactly
 *                        b2cnn_slide_create_path.  mode = B2CNN_MODE_SEQUENCE: after a push, out[p] is what
 *                        model(windows_p, age) returns for the last row, windows_p all of p's windows scored since its
 *                        admission (or since the last reset), in order: one LSTM step per push from p's stored state.
 *                        On the generic path out[p] is bit-identical to b2cnn_score_record_ex (generic, sequence) over
 *                        those windows.  Any other mode: B2CNN_EINVAL.
 *   b2cnn_slide_mode     B2CNN_MODE_INDEPENDENT or B2CNN_MODE_SEQUENCE (-1 for NULL).
 * The state starts at zero at create, b2cnn_slide_reset, b2cnn_slide_admit (with or without history: the history's own
 * window is not scored, the first step is at the first push with seen[p] >= W) and b2cnn_slide_discharge, and is not
 * advanced for a patient whose output is NaN because its window is incomplete or it is discharged.  The age enters the
 * output scale only, never the state.  A NaN sample makes its patient's output NaN from the first window holding it on
 * (the state is poisoned, as in run_model) without touching the other patients; b2cnn_slide_admit starts it again.  A
 * sequence-mode scorer takes no extra heads: b2cnn_slide_set_heads{,_ex} with n > 0 is B2CNN_EINVAL and changes
 * nothing (n == 0 and b2cnn_slide_push_heads with no heads work).  A push runs the launches of an independent-mode
 * push with one step kernel in place of the head's launches, allocates nothing, and its results do not depend on P
 * or on the run. */
int b2cnn_slide_create_ex(b2cnn_handle *h, int32_t n_patients, int32_t stride, int dtype, int path, int mode, b2cnn_slide **out);
int b2cnn_slide_mode(const b2cnn_slide *slide);

/* Warm-started admission (DESIGN.md §6, state across calls).  The LSTM state of one patient or recording is 64 floats,
 * [layer][h | c][unit] = h0 | c0 | h1 | c1 of 16 units each (b2cnn_slide_export_ex's rows, b2cnn_score_record_state's).
 *   b2cnn_slide_admit_ex  b2cnn_slide_admit plus lstm: DEVICE float [n][64], row j the state patients[j]'s next LSTM step
 *                        starts from, or NULL to zero the rows as b2cnn_slide_admit does.  A non-NULL lstm on an
 *                        independent-mode scorer is B2CNN_EINVAL.  Every check of b2cnn_slide_admit runs first; the rows
 *                        are written before the counts are committed, so a call that fails changes neither.  The
 *                        handoff from a backtest to a live scorer: admit a stay of T >= W samples with history = its last
 *                        W samples and lstm = b2cnn_score_record_state's state_out over samples (T - W) mod S .. T - 1;
 *                        every later push then scores what b2cnn_score_record_state scores over the whole stream. */
int b2cnn_slide_admit_ex(b2cnn_slide *slide, const int32_t *patients, int32_t n, const void *history, int64_t history_len,
                         int64_t pitch, int dtype, const float *lstm, void *workspace, int64_t workspace_bytes, void *stream);

/* Every sliding window of whole recordings in one call (DESIGN.md §7), each window feature computed once.
 *   b2cnn_score_record  x: DEVICE [B][C][pitch] samples of `dtype` (channel rows pitch >= N samples apart, recordings
 *                        C pitch apart; any alignment), N samples per recording.  out: DEVICE float [B][n_w], n_w =
 *                        (N - W) / stride + 1 (0 when N < W: nothing runs).  out[b][w] is the logit (sigmoid with
 *                        apply_sigmoid) of the window x[b][:][w stride .. w stride + W - 1], as b2cnn_forward scores it in
 *                        independent mode.  age: DEVICE float, n_age = 1 or B (one per recording, for all its windows).
 *                        path: B2CNN_PATH_TENSORCORE (the models b2cnn_slide_create holds; else B2CNN_EARCH),
 *                        B2CNN_PATH_GENERIC (every model, exact fp32: logits bit-identical to b2cnn_forward with path =
 *                        generic and small_kernel = 0 on the windows) or B2CNN_PATH_AUTO (tensor cores where they hold).
 *                        stride: a positive multiple of the feature stride pool_s^2 (4 on the tensor-core path); it may
 *                        exceed W.  A fixed number of launches whatever B, N and stride; nothing allocated, nothing
 *                        synchronised.  Every check runs before the first launch: B2CNN_EINVAL for a bad stride, shape,
 *                        dtype, path, pitch < N, n_age or more than 2^25 rows (B n_w, or B times the folded rows per
 *                        recording); B2CNN_ESTATE for a workspace that is missing, not 256-byte aligned or smaller than
 *                        b2cnn_record_workspace_bytes; B2CNN_EARCH as above.
 *   b2cnn_record_workspace_bytes  DEVICE workspace of that call (-1 for bad arguments, with b2cnn_last_error).
 *   b2cnn_score_record_ex  the same call with a batch mode.  mode = B2CNN_MODE_INDEPENDENT: exactly b2cnn_score_record.
 *                        mode = B2CNN_MODE_SEQUENCE: out[b] is what model(windows_b, age_b) returns, windows_b the n_w
 *                        windows of recording b in order -- the LSTM carried across a recording's windows (batch as
 *                        sequence, as bin/utils.py run_model scores one recording), from the zero state at each
 *                        recording's first window and never from one recording to the next.  The scan is causal:
 *                        out[b][0 .. k-1] do not depend on windows k and later, and a NaN window makes its own and
 *                        every later output of its recording NaN.  On the generic path each row is bit-identical to
 *                        b2cnn_forward (path = generic, small_kernel = 0, mode = sequence) on the recording's windows.
 *                        A fixed number of launches whatever B, N and stride; nothing allocated, nothing synchronised.
 *                        Every check of b2cnn_score_record runs before the first launch, and a mode that is neither
 *                        value is B2CNN_EINVAL.  Tensor-core sequence mode needs B n_w x 256 bytes more workspace than
 *                        independent mode: size it with b2cnn_record_workspace_bytes_ex and the same mode. */
int64_t b2cnn_record_workspace_bytes(b2cnn_handle *h, int64_t B, int64_t N, int64_t pitch, int64_t stride, int dtype, int path);
int b2cnn_score_record(b2cnn_handle *h, const void *x, int dtype, int64_t B, int64_t N, int64_t pitch, int64_t stride, int path,
                       const float *age, int64_t n_age, int apply_sigmoid, float *out, void *workspace, int64_t workspace_bytes,
                       void *stream);
int64_t b2cnn_record_workspace_bytes_ex(b2cnn_handle *h, int64_t B, int64_t N, int64_t pitch, int64_t stride, int dtype, int path,
                                        int mode);
int b2cnn_score_record_ex(b2cnn_handle *h, const void *x, int dtype, int64_t B, int64_t N, int64_t pitch, int64_t stride, int path,
                          int mode, const float *age, int64_t n_age, int apply_sigmoid, float *out, void *workspace,
                          int64_t workspace_bytes, void *stream);

/* A recording scored in chunks (DESIGN.md §7, state across calls).
 *   b2cnn_score_record_state  b2cnn_score_record_ex in sequence mode with the LSTM state as an input and an output.
 *                        state_in: DEVICE float [B][64] (layout above), recording b's scan starts from state_in[b]
 *                        instead of zero; NULL: the zero state.  state_out: DEVICE float [B][64], recording b's state
 *                        after its last window, or NULL.  With n_w = 0 no head kernel runs and state_out = state_in (zeros
 *                        for a NULL state_in).  A NaN in state_in[b] makes recording b's outputs and state_out[b] NaN
 *                        and no other recording's.  Cutting a recording x at window k into A = x[.., 0 .. (k - 1) S + W)
 *                        and B = x[.., k S ..] and passing A's state_out as B's state_in gives A's and B's outputs and a
 *                        final state that are bit-identical to one call over x, on both paths.  mode must be
 *                        B2CNN_MODE_SEQUENCE (else B2CNN_EINVAL).  state_in and state_out must not overlap (else
 *                        B2CNN_EINVAL): carry the state between calls in two buffers.  The same workspace as
 *                        b2cnn_score_record_ex in sequence mode (b2cnn_record_workspace_bytes_ex); every check runs
 *                        before the first launch. */
int b2cnn_score_record_state(b2cnn_handle *h, const void *x, int dtype, int64_t B, int64_t N, int64_t pitch, int64_t stride, int path,
                             int mode, const float *age, int64_t n_age, int apply_sigmoid, float *out, const float *state_in,
                             float *state_out, void *workspace, int64_t workspace_bytes, void *stream);

/* Candidate heads over whole recordings (DESIGN.md §7, backtesting heads): the model and up to B2CNN_SLIDE_MAX_HEADS
 * handles that share its front end scored over the same recordings, the features computed once.
 *   b2cnn_score_record_heads  out: DEVICE float [1 + n_heads][B][n_w].  out[0] is exactly what b2cnn_score_record_state
 *                        (b2cnn_score_record_ex when both states are NULL) writes with the same arguments; out[i] exactly
 *                        what that call on heads[i - 1] writes -- its own LSTM, Linear and age_coef, the same records,
 *                        ages, path and mode.  state_in / state_out: NULL or DEVICE float [1 + n_heads][B][64] (the
 *                        layout above), row i model i's start and final states; sequence mode only, and they must not
 *                        overlap.  n_heads = 0 is exactly b2cnn_score_record_state (or _ex): the same launches and bits.
 *                        Every head needs the model's architecture (b2cnn_config apart from age_coef and device), weights
 *                        set, the model's device and the model's front-end digest (b2cnn_slide_state_header); on the
 *                        tensor-core path also its packed W_ih chunks in the model's layout (any handle of the model's
 *                        b2cnn_config has them).  A head may be the model's own handle.  Stage, front end and ages run
 *                        once; on the tensor-core path the rows' projections run two per launch (the features split once
 *                        for both), then each row's head.  Nothing allocated, nothing synchronised.
 *   b2cnn_record_workspace_bytes_heads  DEVICE workspace of that call: b2cnn_record_workspace_bytes_ex's, plus on the
 *                        tensor-core path one range-partial buffer (4 * n_ranges * B n_w * 64 bytes, rounded up to 256)
 *                        when n_heads > 0; -1 for bad arguments or n_heads outside [0, B2CNN_SLIDE_MAX_HEADS].
 * Every check runs before the first launch.  B2CNN_EINVAL: a NULL handle or argument, n_heads outside [0,
 * B2CNN_SLIDE_MAX_HEADS], a head without weights or on another device, a state outside sequence mode, overlapping states
 * and every refusal of b2cnn_score_record_ex.  B2CNN_EARCH: a head of another architecture, or without packed W_ih chunks
 * of the model's layout on the tensor-core path.  B2CNN_ESTATE: a head with other front-end (conv / affine) weights than
 * the model's (the message names the head), and the workspace refusals of b2cnn_score_record. */
int64_t b2cnn_record_workspace_bytes_heads(b2cnn_handle *h, int32_t n_heads, int64_t B, int64_t N, int64_t pitch, int64_t stride,
                                           int dtype, int path, int mode);
int b2cnn_score_record_heads(b2cnn_handle *h, b2cnn_handle *const *heads, int32_t n_heads, const void *x, int dtype, int64_t B,
                             int64_t N, int64_t pitch, int64_t stride, int path, int mode, const float *age, int64_t n_age,
                             int apply_sigmoid, float *out, const float *state_in, float *state_out, void *workspace,
                             int64_t workspace_bytes, void *stream);

/* Export and import of patients (a restart, beds moved to another scorer or GPU, new LSTM / head weights).  A
 * patient's state is its current window's L features in window order, raw and unmasked (for a complete window
 * bit-identical to its b2cnn_slide_features row), its T-sample tail (the stream's last T samples per channel, fp32;
 * T = 24 on the tensor-core path, R - 1 on the generic path) and its sample count seen (as b2cnn_slide_samples_seen).
 * It does not depend on the ring's rotation, the push count, P, the patient's slot or the stride, so it can be imported
 * into any scorer of the same path, dtype, C, W, L, F and T whose handle has the same front-end weights.
 * The header's frontend_digest is 64-bit FNV-1a over the bit patterns of the conv1 / conv2 weights and biases, the
 * affine scales and shifts when B2CNN_FLAG_AFFINE is set, and the front-end geometry (C, k1, k2, pool_k, pool_s, act,
 * affine flag) -- not the LSTM, Linear or head weights, which the features do not depend on.
 *   b2cnn_slide_describe_state  the header of this scorer's state (the digest of the handle's current weights).
 *   b2cnn_slide_state_workspace_bytes  DEVICE workspace both calls need for n patients (-1 for n outside [0, P]).
 *   b2cnn_slide_export   features [n][L] and tails [n][C][T] into DEVICE fp32 arrays, seen [n] into a HOST int64 array,
 *                        *header filled.  Reads the scorer and changes nothing in it.
 *   b2cnn_slide_import   writes the listed patients' windows and tails, then seen[p] = seen_host[j], as an admission with
 *                        a full history does (the per-patient masking is on afterwards): a patient with seen >= W is
 *                        in b2cnn_slide_features at once and scored at the next push, one with seen == -1 stays
 *                        discharged.  Patient p's window after a later push is the last W samples of (the exported
 *                        stream | pushes since the import).
 * `patients`: HOST arrays of n distinct indices in [0, P); row j belongs to patients[j].  Both calls allocate nothing
 * and are asynchronous on `stream` apart from the pageable host-to-device copy of the indices (and, for an import, of
 * the counts).  Every check runs before the first launch.  B2CNN_EINVAL: bad indices, NULL arrays with n > 0, a bad
 * magic or version, a path, dtype, C, W, L, F or T that is not the scorer's, a seen value below -1.  B2CNN_ESTATE: a
 * digest that is not the handle's (the features come from other conv weights), a scorer whose handle's weights changed
 * since its last reset, or a workspace smaller than b2cnn_slide_state_workspace_bytes. */
#define B2CNN_SLIDE_STATE_MAGIC 0x53533242u /* "B2SS" */
#define B2CNN_SLIDE_STATE_VERSION 1
typedef struct b2cnn_slide_state_header {
    uint32_t magic;              /* B2CNN_SLIDE_STATE_MAGIC */
    uint16_t version;            /* B2CNN_SLIDE_STATE_VERSION */
    uint16_t path;               /* B2CNN_PATH_TENSORCORE or B2CNN_PATH_GENERIC */
    int32_t dtype, in_channels, window;
    int32_t lstm_input;          /* L: features per patient */
    int32_t feature_stride;      /* F: 4 on the tensor-core path, pool_s^2 on the generic path */
    int32_t tail_len;            /* T: tail samples per patient and channel */
    uint64_t frontend_digest;
} b2cnn_slide_state_header;
int b2cnn_slide_describe_state(b2cnn_slide *slide, b2cnn_slide_state_header *out);
int64_t b2cnn_slide_state_workspace_bytes(b2cnn_slide *slide, int32_t n);
int b2cnn_slide_export(b2cnn_slide *slide, const int32_t *patients, int32_t n, float *features, float *tails, int64_t *seen_host,
                       b2cnn_slide_state_header *header, void *workspace, int64_t workspace_bytes, void *stream);
int b2cnn_slide_import(b2cnn_slide *slide, const int32_t *patients, int32_t n, const b2cnn_slide_state_header *header,
                       const float *features, const float *tails, const int64_t *seen_host, void *workspace,
                       int64_t workspace_bytes, void *stream);
/* The same calls with a sequence-mode scorer's LSTM state (b2cnn_slide_create_ex): lstm is NULL or a DEVICE fp32
 * array [n][2 layers][h, c][16 units].
 *   b2cnn_slide_export_ex  b2cnn_slide_export, plus the listed patients' state rows into lstm when it is not NULL.
 *   b2cnn_slide_import_ex  b2cnn_slide_import, plus the listed patients' state rows from lstm; with lstm == NULL (and
 *                        with b2cnn_slide_import) a sequence-mode scorer zeroes them, as an admission does.
 * A non-NULL lstm for an independent-mode scorer is B2CNN_EINVAL.  Every check runs before the first write, and the
 * header, the workspace and the other arrays are those of b2cnn_slide_export / _import. */
int b2cnn_slide_export_ex(b2cnn_slide *slide, const int32_t *patients, int32_t n, float *features, float *tails, int64_t *seen_host,
                          float *lstm, b2cnn_slide_state_header *header, void *workspace, int64_t workspace_bytes, void *stream);
int b2cnn_slide_import_ex(b2cnn_slide *slide, const int32_t *patients, int32_t n, const b2cnn_slide_state_header *header,
                          const float *features, const float *tails, const int64_t *seen_host, const float *lstm, void *workspace,
                          int64_t workspace_bytes, void *stream);

/* Extra heads over one scorer's features (shadow scoring a retrained head, ensembles of heads over one front end).
 * The stored ring holds everything a head needs, so K extra heads cost one projection over the ring each (on the
 * tensor-core path two per CTA, sharing the ring reads and the bf16 split of the features) plus their LSTM heads.
 *   b2cnn_slide_set_heads  replaces the scorer's heads with SNAPSHOTS of heads[0 .. n) (0 <= n <= B2CNN_SLIDE_MAX_HEADS;
 *                        a head may be the scorer's own handle): each one's LSTM / Linear weights, W_ih^T, age_coef and,
 *                        on the tensor-core path, its packed W_ih chunks are copied, so a later b2cnn_set_weights on a
 *                        head's handle has no effect until the next b2cnn_slide_set_heads.  Every head needs the scorer's
 *                        architecture (b2cnn_config apart from age_coef and device), weights set, the scorer's device and
 *                        the same front-end digest (b2cnn_slide_state_header) as the scorer's weights.  Every check runs
 *                        before anything changes: a failed call leaves the previous heads.  Allocates here (a push still
 *                        allocates nothing), per head: 4 * 3345 bytes of LSTM / Linear weights + 4 * L * 64 of W_ih^T,
 *                        each rounded up to 256, plus on the tensor-core path the packed chunks (n_ranges *
 *                        chunks_per_cta * 6144 bytes, as the handle's) and the range partials 4 * n_ranges * P * 64.
 *                        Synchronises `stream`.
 *   b2cnn_slide_n_heads  the number of heads attached (-1 for NULL).
 *   b2cnn_slide_push_heads  b2cnn_slide_push, with out [1 + n_heads][P] on the DEVICE: row 0 exactly what
 *                        b2cnn_slide_push writes, row i head i - 1's logits (or probabilities) of the same windows with
 *                        its own LSTM, Linear and age_coef and the same ages, NaN for the patients whose row 0 is NaN.
 *                        A head attached at push n scores from push n on, as a scorer of its model running since the
 *                        start would.
 * B2CNN_EINVAL: a NULL argument, n outside [0, B2CNN_SLIDE_MAX_HEADS], a head without weights or on another device.
 * B2CNN_EARCH: a head of another architecture.  B2CNN_ESTATE: a head whose front-end digest is not the scorer's (at
 * set_heads, or at push_heads after a reset that took other conv weights; the message names the head), or a scorer whose
 * handle's weights changed since its last reset.
 *
 * Heads with shorter windows (risk over the last 60 s, 300 s and 600 s from one scorer).  The front end is
 * translation-equivariant with feature stride F (4 on the tensor-core path, pool_s^2 on the generic path), so a window
 * W_k <= W that ends where the scorer's ends, with (W - W_k) % F == 0, is the same stream features on the same lattice:
 * its L_k = lstm_input features are the last L_k of the scorer's window, positions d .. L - 1 with d = (W - W_k) / F.
 *   b2cnn_slide_set_heads_ex  b2cnn_slide_set_heads with flags; flags == 0 is exactly b2cnn_slide_set_heads.  With
 *                        B2CNN_SLIDE_HEADS_SHORTER_WINDOWS a head may also differ from the scorer's b2cnn_config in window
 *                        and lstm_input: window <= W, (W - window) % F == 0, lstm_input == L_out(window) and, on the
 *                        tensor-core path, the packed W_ih chunks of the streaming kernels for its own L_k (any
 *                        handle b2cnn_create accepted on the tensor-core geometries has them); anything else is
 *                        B2CNN_EARCH.  Any other flag bit: B2CNN_EINVAL.  The digest check is unchanged (the window
 *                        is not part of the digest), and every check runs before anything changes.  Memory per head
 *                        as above with its own L_k and range count: 4 * L_k * 64 of W_ih^T and on the tensor-core path
 *                        n_ranges_k * chunks_per_cta_k * 6144 of packed chunks and 4 * n_ranges_k * P * 64 of partials.
 *   b2cnn_slide_push_heads  then writes row i NaN for every patient whose window W_i for that row is incomplete
 *                        (seen < W_i, or n S < W_i before any lifecycle call; row 0 keeps W), sets *emitted = 1 once any
 *                        row has a complete window for at least one patient (a push before the scorer's own first
 *                        window may emit, row 0 all NaN; *window_index keeps n - ceil(W / S) and may be negative), and
 *                        runs no projection for a row whose window is incomplete for every patient.  Row i equals what a
 *                        scorer of head i - 1's model at window W_i and the same stride computes from the same pushes.
 *                        b2cnn_slide_push, features, admit, discharge, export, import and reset do not change, and a
 *                        scorer whose heads all have window W runs the launches it runs with b2cnn_slide_set_heads. */
#define B2CNN_SLIDE_MAX_HEADS 8
#define B2CNN_SLIDE_HEADS_SHORTER_WINDOWS 1
int b2cnn_slide_set_heads(b2cnn_slide *slide, b2cnn_handle *const *heads, int32_t n, void *stream);
int b2cnn_slide_set_heads_ex(b2cnn_slide *slide, b2cnn_handle *const *heads, int32_t n, int32_t flags, void *stream);
int b2cnn_slide_n_heads(const b2cnn_slide *slide);
int b2cnn_slide_push_heads(b2cnn_slide *slide, const void *new_samples, int64_t pitch, const float *age, int64_t n_age,
                           int apply_sigmoid, float *out, int32_t *emitted, int64_t *window_index, void *stream);

/* ---- The reference's wire formats, decoded on the device (SURVEY.md section 8, row f3) ----
 * A trigger's Kafka messages as one DEVICE byte buffer + offsets [n_msgs + 1] (message t = bytes[offsets[t] .. offsets[t+1])).
 * b2cnn_decode_sample_messages: value = json.dumps([i, val]) (bin/sendStream.py:62): idx_out[t] = i, val_out[t] = val
 *   (either may be NULL); with `frame` [frame_rows][n_sig] fp64 (first filled with NaN = missing) and row_of_msg[t]
 *   (the frame row = patient * n_new + sample the message belongs to, from its key / arrival order; < 0 = skip) the
 *   value is scattered to frame[row][i] -- the array b2cnn_ring_push(B2CNN_SAMPLES_F64) takes.
 * b2cnn_decode_array_messages: value = "[v0,v1,...]" (bin/processStream.py:128, read back at bin/predictStream.py:241):
 *   vals_out[t][0 .. max_vals) (NaN-padded), counts_out[t] = number of values (-1: malformed).
 * Numbers are converted with correct rounding (== json.loads / float() / Double.parseDouble) for up to 19 significant
 * digits and |decimal exponent| <= 27; NaN / Infinity / null (quoted or not) are accepted; JSON whitespace may separate
 * the tokens, nothing may follow the closing bracket, and the signal index must fit an int32; anything else counts in
 * *n_bad (device int) and yields NaN (idx_out -1).  b2cnn_parse_decimal is the same parser compiled for the host (tests; status 0 ok, 1 malformed,
 * 2 out of range). */
int b2cnn_decode_sample_messages(const void *bytes, const int64_t *offsets, int64_t n_msgs, int32_t *idx_out, double *val_out,
                                 const int64_t *row_of_msg, double *frame, int64_t frame_rows, int32_t n_sig, int32_t *n_bad,
                                 void *stream);
int b2cnn_decode_array_messages(const void *bytes, const int64_t *offsets, int64_t n_msgs, int32_t max_vals, double *vals_out,
                                int32_t *counts_out, int32_t *n_bad, void *stream);
double b2cnn_parse_decimal(const char *s, int64_t len, int32_t *status);

/* The B200-native alternative to one JSON message per (sample, signal): ONE binary frame per trigger for all patients.
 *   header (32 bytes, little-endian)  |  int32 subject_id[n_patients]  |  pad to 8 bytes  |  samples[n_patients][n_new][n_sig]
 * `kind` = B2CNN_SAMPLES_ADC16 (int16), _F64 or _GRID (fp64): the payload is exactly the array b2cnn_ring_push takes, so
 * "decoding" is one H2D copy.  b2cnn_frame_check validates a HOST buffer and returns the byte offsets of the two arrays. */
#define B2CNN_FRAME_MAGIC 0x46573242u /* "B2WF" */
typedef struct b2cnn_frame_header {
    uint32_t magic;              /* B2CNN_FRAME_MAGIC */
    uint16_t version;            /* 1 */
    uint16_t kind;               /* B2CNN_SAMPLES_* */
    uint32_t n_patients, n_new, n_sig;
    uint32_t reserved;
    uint64_t first_index;        /* index of the frame's first sample (grid point) in the stream: gaps are detectable */
} b2cnn_frame_header;
int b2cnn_frame_check(const void *frame, int64_t bytes, b2cnn_frame_header *header_out, int64_t *ids_offset, int64_t *samples_offset);

const char *b2cnn_last_error(void);
const char *b2cnn_version(void);

/* ---- One training step on the device (SURVEY.md section 8, row f4) ----
 * Replaces the body of the reference's training loop (bin/utils.py:200-208):
 *     optimizer.zero_grad(); output = model(input, age); loss = criterion(output, target); loss.backward(); optimizer.step()
 * with criterion = nn.BCEWithLogitsLoss() and torch.optim.Adam (bin/explore_torch.ipynb:3204-3205; no amsgrad, no weight decay), for the model in train() mode: B2CNN_MODE_SEQUENCE is what model(input_batch, age)
 * computes (the LSTM scans the batch axis, bin/models.py:29-30), B2CNN_MODE_INDEPENDENT treats every window as its own
 * sequence.  All pointers are DEVICE pointers, everything is fp32:
 *   params          the packed blob of b2cnn_weight_count() floats (no affine), updated in place when apply_update != 0
 *   adam_m, adam_v  optimizer state, same size (zero before step 1); grads: same size, receives d loss / d params
 *   step            1-based count of optimizer steps (bias correction)
 *   x [B][C][W], age [B], target [B] (0 / 1)
 *   mask1 [B][4][P1], mask2 [B][L_out]: the two nn.Dropout(0.1) masks of bin/models.py:25,28 ALREADY scaled by 1/(1-p)
 *                   (torch's Philox stream cannot be reproduced here, so the caller draws them); NULL = no dropout
 *   loss_out        one float: the mean BCE-with-logits loss of this batch (before the update)
 * The call allocates nothing and is asynchronous on `stream`.  Like every training call it checks all its arguments
 * before any CUDA call, then runs on cfg->device (the current device for -1) and restores the caller's device.
 * workspace: b2cnn_train_workspace_bytes(cfg, B) bytes; a smaller one is B2CNN_ESTATE before any launch.  The conv
 * layers run on position tiles of 128 window features that recompute the conv backward in shared memory, so the
 * workspace holds f, d f, the LSTM records and one region of partial sums (about 2 * 4 * B * L_out bytes plus the
 * per-window records).  The gradients are the same bits from run to run.  A geometry whose conv tile does not fit
 * shared memory (hundreds of input channels at W = 120, 83 or more from L_out = 128 on for the MyCNN5 layer stack)
 * is B2CNN_EINVAL. */
typedef struct b2cnn_adam {
    float lr, beta1, beta2, eps;   /* torch defaults: 1e-3, 0.9, 0.999, 1e-8 */
} b2cnn_adam;
int64_t b2cnn_train_workspace_bytes(const b2cnn_config *cfg, int64_t B);
int b2cnn_train_step(const b2cnn_config *cfg, float *params, float *adam_m, float *adam_v, float *grads, int64_t step,
                     const b2cnn_adam *opt, int apply_update, const float *x, int64_t B, const float *age, const float *target,
                     int mode, const float *mask1, const float *mask2, float *loss_out, void *workspace, int64_t workspace_bytes,
                     void *stream);
/* The same step with the class weight of the reference's training cell (bin/explore_torch.ipynb:3170,3204):
 * criterion = nn.BCEWithLogitsLoss(pos_weight=pos_weight), pos_weight = num_negatives / num_positives (> 0, finite);
 * loss_out is mean_b( (1-y) z + (1 + (pos_weight-1) y) (log1p(exp(-|z|)) + max(-z, 0)) ). */
int b2cnn_train_step_weighted(const b2cnn_config *cfg, float *params, float *adam_m, float *adam_v, float *grads, int64_t step,
                              const b2cnn_adam *opt, int apply_update, const float *x, int64_t B, const float *age,
                              const float *target, float pos_weight, int mode, const float *mask1, const float *mask2,
                              float *loss_out, void *workspace, int64_t workspace_bytes, void *stream);

/* ---- The model in train() mode as a differentiable function, for torch autograd (any loss, any optimizer) ----
 * Same pointers, modes and masks as b2cnn_train_step; neither call allocates, both are asynchronous on `stream`. */
/* forward in train() mode; the activations the backward pass needs stay in `workspace`
 * (b2cnn_train_workspace_bytes(cfg, B) bytes).  z_out[B]: logits (bin/models.py:34). */
int b2cnn_train_forward(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age,
                        int mode, const float *mask1, const float *mask2, float *z_out,
                        void *workspace, int64_t workspace_bytes, void *stream);
/* backward from an upstream gradient dz[B] = d loss / d z.  `workspace` must be the one the matching
 * forward filled, unchanged since.  grads: overwritten (not accumulated), b2cnn_weight_count() floats.
 * dx [B][C][W] and dage [B] may be NULL (not computed). */
int b2cnn_train_backward(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age,
                         int mode, const float *mask1, const float *mask2, const float *dz, float *grads,
                         float *dx, float *dage, void *workspace, int64_t workspace_bytes, void *stream);
/* b2cnn_train_backward with flags (0 = b2cnn_train_backward).  B2CNN_TRAIN_FROZEN_CONV: neither conv1 / conv2 nor the
 * input needs a gradient (fine-tuning the LSTM head on a fixed front end): d f and the whole convolutional backward
 * are skipped, the conv entries of grads are zero, and dx must be NULL. */
#define B2CNN_TRAIN_FROZEN_CONV 1
int b2cnn_train_backward_ex(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age,
                            int mode, const float *mask1, const float *mask2, const float *dz, float *grads,
                            float *dx, float *dage, int flags, void *workspace, int64_t workspace_bytes, void *stream);

/* ---- Many patients' window sequences in one training call ----
 * The _seq variants take a HOST array of sequence lengths in place of `mode`: the batch is n_seq consecutive sequences
 * of seq_lengths[0], ..., seq_lengths[n_seq - 1] windows (every length >= 1, the lengths add up to B), each scanned by
 * the LSTM from the zero state, no state crossing a sequence boundary.  The logits are those of one model(x_s, age_s)
 * call per sequence, concatenated; the loss is the mean over all B windows, as in b2cnn_train_step.  {B} is
 * B2CNN_MODE_SEQUENCE (the same bits) and {1, ..., 1} is B2CNN_MODE_INDEPENDENT.  Bad lengths (NULL, n_seq < 1, a
 * length below 1, a sum other than B) are B2CNN_EINVAL before any CUDA call.  The workspace is
 * b2cnn_train_workspace_bytes_seq() bytes: the call copies the sequence offsets into it (from the host array, on
 * `stream`), and one sized by b2cnn_train_workspace_bytes() is B2CNN_ESTATE before any launch.  Up to 256 sequences
 * are scanned one CTA each; beyond that a CTA scans ceil(n_seq / 256) consecutive sequences, a grouping taken from
 * (B, n_seq) alone.  Each CTA writes its head-gradient and loss partials as one row, and the rows are summed in
 * sequence order (no atomics): the gradients are the same bits from run to run.  With one sequence no row is
 * written and nothing is summed.
 * b2cnn_train_step_seq: b2cnn_train_step, or with pos_weight != NULL (one host float, > 0 and finite)
 * b2cnn_train_step_weighted.  b2cnn_train_forward_seq / b2cnn_train_backward_seq: the autograd pair, the backward with
 * the flags of b2cnn_train_backward_ex; the backward takes the lengths its forward took. */
int64_t b2cnn_train_workspace_bytes_seq(const b2cnn_config *cfg, int64_t B, const int64_t *seq_lengths, int64_t n_seq);
int b2cnn_train_step_seq(const b2cnn_config *cfg, float *params, float *adam_m, float *adam_v, float *grads, int64_t step,
                         const b2cnn_adam *opt, int apply_update, const float *x, int64_t B, const float *age, const float *target,
                         const float *pos_weight, const int64_t *seq_lengths, int64_t n_seq, const float *mask1, const float *mask2,
                         float *loss_out, void *workspace, int64_t workspace_bytes, void *stream);
int b2cnn_train_forward_seq(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age,
                            const int64_t *seq_lengths, int64_t n_seq, const float *mask1, const float *mask2, float *z_out,
                            void *workspace, int64_t workspace_bytes, void *stream);
int b2cnn_train_backward_seq(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age,
                             const int64_t *seq_lengths, int64_t n_seq, const float *mask1, const float *mask2, const float *dz,
                             float *grads, float *dx, float *dage, int flags, void *workspace, int64_t workspace_bytes,
                             void *stream);

/* ---- Training on whole recordings ----
 * The _record variants take `records` [B][C][N] (contiguous fp32, N >= the window W) in place of windows, a window
 * stride `stride` S (a positive multiple of the feature stride pool_s^2) and a HOST array window_counts[B]: recording b
 * contributes its windows w = 0 .. window_counts[b] - 1, window w being samples [w S, w S + W).  Every count lies in
 * [0, n_w], n_w = (N - W) / S + 1 (0 when N < W), and the counts add up to M >= 1.  The M windows are the rows, in
 * recording-major, window order: age[M], target[M], z_out[M], dz[M] and dage[M] are per window.
 * mode B2CNN_MODE_SEQUENCE: each recording's windows are one sequence, the LSTM starting from the zero state (the _seq
 * calls with the non-zero counts as lengths); B2CNN_MODE_INDEPENDENT: every window alone.  The dropout masks belong to
 * the recording: mask1 [B][4][P1(N)] and mask2 [B][L(N)], the geometry of a window of N samples, and window w uses
 * mask1[b][:][w S / pool_s + i] and mask2[b][w S / pool_s^2 + j], so a feature two windows share is dropped in both or
 * in neither.  The logits, the loss and the LSTM / Linear gradients (W_ih_l0 included) are the bits of the _seq /
 * independent call on the windows cut out of the recordings with their masks cut the same way; the conv gradients and
 * d_records sum each shared feature's gradient over its windows before the conv backward, so they match those sums up
 * to rounding.  Samples no counted window reads (a recording's tail, the gaps when S > W, a recording with count 0)
 * change nothing: NaN or inf there gives the bits that zeros give, and d_records[B][C][N] (or NULL) is 0 there.
 * Bad strides, counts or lengths are B2CNN_EINVAL before any CUDA call; the workspace is
 * b2cnn_train_workspace_bytes_record() bytes (a smaller one is B2CNN_ESTATE before any launch), and the calls copy the
 * counts' offsets into it on `stream`.  b2cnn_train_step_record: pos_weight NULL or one host float (> 0 and finite).
 * b2cnn_train_backward_record takes the arguments its forward took and the flags of b2cnn_train_backward_ex. */
int64_t b2cnn_train_workspace_bytes_record(const b2cnn_config *cfg, int64_t B, int64_t N, int64_t stride, const int64_t *window_counts,
                                           int mode);
int b2cnn_train_step_record(const b2cnn_config *cfg, float *params, float *adam_m, float *adam_v, float *grads, int64_t step,
                            const b2cnn_adam *opt, int apply_update, const float *records, int64_t B, int64_t N, int64_t stride,
                            const int64_t *window_counts, int mode, const float *age, const float *target, const float *pos_weight,
                            const float *mask1, const float *mask2, float *loss_out, void *workspace, int64_t workspace_bytes,
                            void *stream);
int b2cnn_train_forward_record(const b2cnn_config *cfg, const float *params, const float *records, int64_t B, int64_t N, int64_t stride,
                               const int64_t *window_counts, int mode, const float *age, const float *mask1, const float *mask2,
                               float *z_out, void *workspace, int64_t workspace_bytes, void *stream);
int b2cnn_train_backward_record(const b2cnn_config *cfg, const float *params, const float *records, int64_t B, int64_t N, int64_t stride,
                                const int64_t *window_counts, int mode, const float *age, const float *mask1, const float *mask2,
                                const float *dz, float *grads, float *d_records, float *dage, int flags, void *workspace,
                                int64_t workspace_bytes, void *stream);

/* Training on chunks of recordings (DESIGN.md §8, state across calls): the _record calls in sequence mode with each
 * recording's LSTM state, DEVICE float [B][64] = h0 | c0 | h1 | c1 (16 units each; b2cnn_score_record_state's layout).
 * mode must be B2CNN_MODE_SEQUENCE (else B2CNN_EINVAL); every argument is checked before any CUDA call, and the workspace
 * is b2cnn_train_workspace_bytes_record()'s for the same arguments (the states live in the caller's memory).  Every
 * state pointer may be NULL: a NULL state_in is the zero state, and with every state NULL each call computes what its
 * _record counterpart computes.  No two of a call's state arrays may overlap (B2CNN_EINVAL): the step's backward reads
 * state_in after its forward has written state_out, so a TBPTT loop carries the state in two buffers, swapped per call.
 *   b2cnn_train_forward_record_state  recording b's scan starts from state_in[b]; state_out[b] receives its state after
 *                        its last counted window.  A recording with window_counts[b] == 0 passes it through: state_out[b]
 *                        = state_in[b] (zeros for a NULL state_in).
 *   b2cnn_train_backward_record_state  the forward's arguments (state_in included), dz, and d_state_out: the gradient
 *                        of the loss at state_out (NULL: none).  Writes grads, d_records, dage as
 *                        b2cnn_train_backward_record does, and d_state_in [B][64]: the gradient at state_in (d_state_out[b]
 *                        for a recording without windows).  Chaining two forwards through the state and running the
 *                        backwards in reverse order, d_state_in of the second as d_state_out of the first, gives the
 *                        gradients of one call over the whole recordings.
 *   b2cnn_train_step_record_state  b2cnn_train_step_record from state_in, writing state_out: truncated back-propagation
 *                        through time (no gradient enters through state_out). */
int b2cnn_train_step_record_state(const b2cnn_config *cfg, float *params, float *adam_m, float *adam_v, float *grads, int64_t step,
                                  const b2cnn_adam *opt, int apply_update, const float *records, int64_t B, int64_t N, int64_t stride,
                                  const int64_t *window_counts, int mode, const float *age, const float *target, const float *pos_weight,
                                  const float *mask1, const float *mask2, const float *state_in, float *state_out, float *loss_out,
                                  void *workspace, int64_t workspace_bytes, void *stream);
int b2cnn_train_forward_record_state(const b2cnn_config *cfg, const float *params, const float *records, int64_t B, int64_t N,
                                     int64_t stride, const int64_t *window_counts, int mode, const float *age, const float *mask1,
                                     const float *mask2, const float *state_in, float *state_out, float *z_out, void *workspace,
                                     int64_t workspace_bytes, void *stream);
int b2cnn_train_backward_record_state(const b2cnn_config *cfg, const float *params, const float *records, int64_t B, int64_t N,
                                      int64_t stride, const int64_t *window_counts, int mode, const float *age, const float *mask1,
                                      const float *mask2, const float *state_in, const float *dz, const float *d_state_out, float *grads,
                                      float *d_records, float *dage, float *d_state_in, int flags, void *workspace, int64_t workspace_bytes,
                                      void *stream);


/* ---- Candidate heads on one frozen front end (DESIGN.md §8, training candidate heads) ----
 * One fused training step for n_heads in [1, B2CNN_SLIDE_MAX_HEADS] models that share conv1 / conv2: the conv forward
 * runs once on `frontend` (a packed blob of b2cnn_weight_count() floats, read for its conv entries only), and each head
 * trains its own LSTM and Linear entries (blob entries from W_ih_l0 on) with its own Adam state.  Nothing back-propagates
 * into the front end.  params, adam_m, adam_v and grads are HOST arrays of n_heads DEVICE pointers, each a full packed
 * blob; only entries from W_ih_l0 on are written, and the conv entries of grads are set to zero.  lr is a HOST array of
 * n_heads learning rates; opt gives beta1, beta2 and eps for every head (opt->lr is not read).  loss_out is a DEVICE array
 * of n_heads floats.  Every other argument is b2cnn_train_step_seq's / b2cnn_train_step_record's, shared by all heads:
 * the batch, the mode, the masks and pos_weight (NULL or one host float).  b2cnn_train_heads_step takes mode and, when
 * seq_lengths != NULL, the sequence lengths (mode must then be B2CNN_MODE_SEQUENCE).
 * Head h's loss and gradients are the bits b2cnn_train_step_seq / _weighted / _record computes on params[h] with the same
 * arguments, and its updated blob the bits of that call with apply_update.  The launch list does not depend on n_heads.
 * B2CNN_EINVAL before any CUDA call: n_heads outside [1, 8], a NULL pointer (adam_m / adam_v only with apply_update), two
 * heads sharing or overlapping a blob (params, grads and, with apply_update, adam_m / adam_v: none may overlap another),
 * and whatever the single-model calls refuse.  A workspace smaller than b2cnn_train_heads_workspace_bytes[_record]() is
 * B2CNN_ESTATE before any launch.  The call allocates nothing and is asynchronous on `stream`. */
int64_t b2cnn_train_heads_workspace_bytes(const b2cnn_config *cfg, int32_t n_heads, int64_t B, const int64_t *seq_lengths, int64_t n_seq);
int b2cnn_train_heads_step(const b2cnn_config *cfg, const float *frontend, int32_t n_heads, float *const *params, float *const *adam_m,
                           float *const *adam_v, float *const *grads, const float *lr, int64_t step, const b2cnn_adam *opt,
                           int apply_update, const float *x, int64_t B, const float *age, const float *target, const float *pos_weight,
                           int mode, const int64_t *seq_lengths, int64_t n_seq, const float *mask1, const float *mask2, float *loss_out,
                           void *workspace, int64_t workspace_bytes, void *stream);
int64_t b2cnn_train_heads_workspace_bytes_record(const b2cnn_config *cfg, int32_t n_heads, int64_t B, int64_t N, int64_t stride,
                                                 const int64_t *window_counts, int mode);
int b2cnn_train_heads_step_record(const b2cnn_config *cfg, const float *frontend, int32_t n_heads, float *const *params,
                                  float *const *adam_m, float *const *adam_v, float *const *grads, const float *lr, int64_t step,
                                  const b2cnn_adam *opt, int apply_update, const float *records, int64_t B, int64_t N, int64_t stride,
                                  const int64_t *window_counts, int mode, const float *age, const float *target, const float *pos_weight,
                                  const float *mask1, const float *mask2, float *loss_out, void *workspace, int64_t workspace_bytes,
                                  void *stream);

#ifdef __cplusplus
}
#endif
#endif /* B2CNN_H_ */

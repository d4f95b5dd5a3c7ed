// b2cnn_api.cu -- the extern "C" boundary declared in include/b2cnn.h.
// Replaces the reference's `model = torch.load(...); model.eval()` (bin/predictStream.py:36-37)
// and `output = model(x, age)` (bin/predictStream.py:157) with plain-pointer entry points.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "b2cnn_internal.cuh"
#include "b2cnn_proj_tc.cuh"
#include "b2cnn_slide.cuh"
#include "b2cnn_tc.cuh"

using namespace b2cnn;

static thread_local std::string g_err;

static int fail(int code, const std::string &msg) {
    g_err = msg;
    return code;
}
static int cuda_fail(cudaError_t e, const char *what) {
    g_err = std::string(what) + ": " + cudaGetErrorString(e);
    return B2CNN_ECUDA;
}
// rc, with the internal call's message under the entry point's name when rc is an error
static int finish(const char *fn, int rc, const char *err) {
    return rc == B2CNN_OK ? rc : fail(rc, std::string(fn) + ": " + err);
}
#define CU_TRY(expr)                                         \
    do {                                                     \
        cudaError_t e__ = (expr);                            \
        if (e__ != cudaSuccess) return cuda_fail(e__, #expr); \
    } while (0)

// Every entry point that touches the handle's device switches to it for the duration of the call only (DeviceGuard).
#define DEVICE_GUARD(dev)                   \
    DeviceGuard guard__(dev);               \
    if (guard__.err != cudaSuccess) return cuda_fail(guard__.err, "cudaSetDevice")

struct b2cnn_handle {
    b2cnn_config cfg;
    Dims d;
    int device = 0;
    int num_sms = 132;
    bool weights_set = false;
    uint64_t weight_gen = 0;    // bumped by every b2cnn_set_weights: a sliding-window scorer's features go stale
    ConvWeights cw;
    HeadWeights hw;
    float *d_blob = nullptr;    // packed blob as given
    float *d_wih0T = nullptr;   // [L][64]
    int64_t n_weights = 0;
    int64_t opt_path = B2CNN_PATH_AUTO;
    int64_t opt_tc_fused = 1;    // bf16 windows: conv + projection fused in the streaming kernel (C <= 3)
    int64_t opt_tc_splits = 3;   // bf16 pieces per conv1 weight in the fused kernels
    int64_t last_launches = 0;
    int last_path = 0;
    int64_t opt_profile = 0;
    int64_t opt_small = 1;      // single-launch kernel for short windows / small batches
    cudaEvent_t ev_stage[3] = {nullptr, nullptr, nullptr};   // start, after front end, after head
    bool ev_valid = false;
    TcState tc;                 // tensor-core path state (b2cnn_tc.cu)
    // ---- host-path staging (b2cnn_forward_host only)
    void *st_x[2] = {nullptr, nullptr};
    size_t st_x_bytes = 0;
    float *st_age = nullptr, *st_out = nullptr;
    void *st_ws = nullptr;
    size_t st_ws_bytes = 0, st_vec_elems = 0;
    cudaStream_t s_copy = nullptr, s_comp = nullptr;
    cudaEvent_t ev_copied[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr};
};

static int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

extern "C" int64_t b2cnn_l_out(const b2cnn_config *cfg) {
    Dims d;
    if (!cfg || !derive_dims(*cfg, d)) return -1;
    return d.L;
}

extern "C" int64_t b2cnn_weight_count(const b2cnn_config *cfg) {
    Dims d;
    if (!cfg || !derive_dims(*cfg, d)) return -1;
    return blob_offsets(d).total;
}

extern "C" const char *b2cnn_last_error(void) { return g_err.c_str(); }

// ---- one training step (b2cnn_train.cu) ----
static constexpr SeqLengths kNoSeq{false, nullptr, 0};

extern "C" int64_t b2cnn_train_workspace_bytes(const b2cnn_config *cfg, int64_t B) {
    const int64_t n = train_workspace_bytes(cfg, B, kNoSeq);
    if (n < 0) fail(B2CNN_EINVAL, "b2cnn_train_workspace_bytes: bad configuration / batch");
    return n;
}
extern "C" int64_t b2cnn_train_workspace_bytes_seq(const b2cnn_config *cfg, int64_t B, const int64_t *seq_lengths, int64_t n_seq) {
    const int64_t n = train_workspace_bytes(cfg, B, SeqLengths{true, seq_lengths, n_seq});
    if (n < 0) fail(B2CNN_EINVAL, "b2cnn_train_workspace_bytes_seq: bad configuration / batch / sequence lengths");
    return n;
}
static int train_step_api(const char *name, const b2cnn_config *cfg, float *params, float *adam_m, float *adam_v, float *grads,
                          int64_t step, const b2cnn_adam *opt, int apply_update, const float *x, int64_t B, const float *age,
                          const float *target, int weighted, float pos_weight, int mode, const SeqLengths &sl, const float *mask1,
                          const float *mask2, float *loss_out, void *workspace, int64_t workspace_bytes, void *stream) {
    if (!cfg || !opt) return fail(B2CNN_EINVAL, std::string(name) + ": null configuration");
    const char *err = "";
    const int rc = train_step(cfg, params, adam_m, adam_v, grads, step, opt->lr, opt->beta1, opt->beta2, opt->eps, apply_update, x, B, age,
                              target, weighted, pos_weight, mode, sl, mask1, mask2, loss_out, workspace, workspace_bytes,
                              reinterpret_cast<cudaStream_t>(stream), &err);
    return finish(name, rc, err);
}
extern "C" int b2cnn_train_step(const b2cnn_config *cfg, float *params, float *adam_m, float *adam_v, float *grads, int64_t step,
                                const b2cnn_adam *opt, int apply_update, const float *x, int64_t B, const float *age,
                                const float *target, int mode, const float *mask1, const float *mask2, float *loss_out,
                                void *workspace, int64_t workspace_bytes, void *stream) {
    return train_step_api("b2cnn_train_step", cfg, params, adam_m, adam_v, grads, step, opt, apply_update, x, B, age, target, 0, 1.f, mode,
                          kNoSeq, mask1, mask2, loss_out, workspace, workspace_bytes, stream);
}
extern "C" int b2cnn_train_step_weighted(const b2cnn_config *cfg, float *params, float *adam_m, float *adam_v, float *grads, int64_t step,
                                         const b2cnn_adam *opt, int apply_update, const float *x, int64_t B, const float *age,
                                         const float *target, float pos_weight, int mode, const float *mask1, const float *mask2,
                                         float *loss_out, void *workspace, int64_t workspace_bytes, void *stream) {
    return train_step_api("b2cnn_train_step_weighted", cfg, params, adam_m, adam_v, grads, step, opt, apply_update, x, B, age, target, 1,
                          pos_weight, mode, kNoSeq, mask1, mask2, loss_out, workspace, workspace_bytes, stream);
}
extern "C" int b2cnn_train_step_seq(const b2cnn_config *cfg, float *params, float *adam_m, float *adam_v, float *grads, int64_t step,
                                    const b2cnn_adam *opt, int apply_update, const float *x, int64_t B, const float *age,
                                    const float *target, const float *pos_weight, const int64_t *seq_lengths, int64_t n_seq,
                                    const float *mask1, const float *mask2, float *loss_out, void *workspace, int64_t workspace_bytes,
                                    void *stream) {
    return train_step_api("b2cnn_train_step_seq", cfg, params, adam_m, adam_v, grads, step, opt, apply_update, x, B, age, target,
                          pos_weight ? 1 : 0, pos_weight ? *pos_weight : 1.f, B2CNN_MODE_SEQUENCE, SeqLengths{true, seq_lengths, n_seq},
                          mask1, mask2, loss_out, workspace, workspace_bytes, stream);
}
extern "C" int b2cnn_train_forward(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age, int mode,
                                   const float *mask1, const float *mask2, float *z_out, void *workspace, int64_t workspace_bytes,
                                   void *stream) {
    const char *err = "";
    const int rc = train_forward(cfg, params, x, B, age, mode, kNoSeq, mask1, mask2, z_out, workspace, workspace_bytes,
                                 reinterpret_cast<cudaStream_t>(stream), &err);
    return finish("b2cnn_train_forward", rc, err);
}
extern "C" int b2cnn_train_forward_seq(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age,
                                       const int64_t *seq_lengths, int64_t n_seq, const float *mask1, const float *mask2, float *z_out,
                                       void *workspace, int64_t workspace_bytes, void *stream) {
    const char *err = "";
    const int rc = train_forward(cfg, params, x, B, age, B2CNN_MODE_SEQUENCE, SeqLengths{true, seq_lengths, n_seq}, mask1, mask2, z_out,
                                 workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream), &err);
    return finish("b2cnn_train_forward_seq", rc, err);
}
extern "C" int b2cnn_train_backward_ex(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age, int mode,
                                       const float *mask1, const float *mask2, const float *dz, float *grads, float *dx, float *dage,
                                       int flags, void *workspace, int64_t workspace_bytes, void *stream) {
    const char *err = "";
    const int rc = train_backward(cfg, params, x, B, age, mode, kNoSeq, mask1, mask2, dz, grads, dx, dage, flags, workspace, workspace_bytes,
                                  reinterpret_cast<cudaStream_t>(stream), &err);
    return finish("b2cnn_train_backward", rc, err);
}
extern "C" int b2cnn_train_backward(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age, int mode,
                                    const float *mask1, const float *mask2, const float *dz, float *grads, float *dx, float *dage,
                                    void *workspace, int64_t workspace_bytes, void *stream) {
    return b2cnn_train_backward_ex(cfg, params, x, B, age, mode, mask1, mask2, dz, grads, dx, dage, 0, workspace, workspace_bytes, stream);
}
extern "C" int b2cnn_train_backward_seq(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age,
                                        const int64_t *seq_lengths, int64_t n_seq, const float *mask1, const float *mask2, const float *dz,
                                        float *grads, float *dx, float *dage, int flags, void *workspace, int64_t workspace_bytes,
                                        void *stream) {
    const char *err = "";
    const int rc = train_backward(cfg, params, x, B, age, B2CNN_MODE_SEQUENCE, SeqLengths{true, seq_lengths, n_seq}, mask1, mask2, dz, grads,
                                  dx, dage, flags, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream), &err);
    return finish("b2cnn_train_backward_seq", rc, err);
}

// ---- preprocessing + window assembly (b2cnn_prep.cu) ----
extern "C" int64_t b2cnn_prep_window_count(int64_t n_samples, double fs, const b2cnn_prep_config *cfg) {
    const int64_t n = prep_window_count(n_samples, fs, cfg);
    if (n < 0) fail(B2CNN_EINVAL, "b2cnn_prep_window_count: bad record shape / configuration");
    return n;
}
extern "C" int64_t b2cnn_prep_workspace_bytes(int64_t n_samples, double fs, int32_t n_sel, const b2cnn_prep_config *cfg) {
    const int64_t n = prep_workspace_bytes(n_samples, fs, n_sel, cfg);
    if (n < 0) fail(B2CNN_EINVAL, "b2cnn_prep_workspace_bytes: bad record shape / configuration");
    return n;
}
extern "C" int b2cnn_prep_windows(const int16_t *raw, int64_t n_samples, int32_t n_sig, const int32_t *sel, int32_t n_sel,
                                  const double *gains, const double *baselines, double fs, const b2cnn_prep_config *cfg,
                                  void *x_out, int dtype, double *t0_out, void *workspace, int64_t workspace_bytes, void *stream) {
    const char *err = "";
    const int rc = prep_windows(raw, n_samples, n_sig, sel, n_sel, gains, baselines, fs, cfg, x_out, dtype, t0_out, workspace,
                                workspace_bytes, reinterpret_cast<cudaStream_t>(stream), &err);
    return finish("b2cnn_prep_windows", rc, err);
}
// ---- streaming form: per-patient device ring buffers (b2cnn_prep.cu) ----
struct b2cnn_ring { Ring *r; int device; };

extern "C" int b2cnn_ring_create(const b2cnn_prep_config *cfg, int32_t n_patients, int32_t n_sig, double fs, int32_t device,
                                 b2cnn_ring **out) {
    if (!cfg || !out) return fail(B2CNN_EINVAL, "b2cnn_ring_create: null argument");
    *out = nullptr;
    int dev = device;
    if (dev < 0) CU_TRY(cudaGetDevice(&dev));
    DEVICE_GUARD(dev);
    const char *err = "";
    Ring *r = nullptr;
    const int rc = ring_create(cfg, n_patients, n_sig, fs, dev, &r, &err);
    if (rc != B2CNN_OK) return finish("b2cnn_ring_create", rc, err);
    b2cnn_ring *h = new (std::nothrow) b2cnn_ring{r, dev};
    if (!h) { ring_destroy(r); return fail(B2CNN_ESTATE, "out of host memory"); }
    *out = h;
    return B2CNN_OK;
}
extern "C" void b2cnn_ring_destroy(b2cnn_ring *h) {
    if (!h) return;
    DeviceGuard guard(h->device);
    ring_destroy(h->r);
    delete h;
}
extern "C" int b2cnn_ring_reset(b2cnn_ring *h, void *stream) {
    if (!h) return fail(B2CNN_EINVAL, "b2cnn_ring_reset: null argument");
    DEVICE_GUARD(h->device);
    const char *err = "";
    const int rc = ring_reset(h->r, reinterpret_cast<cudaStream_t>(stream), &err);
    return finish("b2cnn_ring_reset", rc, err);
}
extern "C" int b2cnn_ring_set_signals(b2cnn_ring *h, int32_t patient, const int32_t *sel, int32_t n_sel, const double *gains,
                                      const double *baselines, void *stream) {
    if (!h) return fail(B2CNN_EINVAL, "b2cnn_ring_set_signals: null argument");
    DEVICE_GUARD(h->device);
    const char *err = "";
    const int rc = ring_set_signals(h->r, patient, sel, n_sel, gains, baselines, reinterpret_cast<cudaStream_t>(stream), &err);
    return finish("b2cnn_ring_set_signals", rc, err);
}
extern "C" int b2cnn_ring_push(b2cnn_ring *h, const void *new_samples, int sample_kind, int64_t n_new, void *x_out, int dtype,
                               int32_t *emitted, int64_t *window_index, double *t0_seconds, void *stream) {
    if (!h) return fail(B2CNN_EINVAL, "b2cnn_ring_push: null argument");
    if (sample_kind != B2CNN_SAMPLES_ADC16 && sample_kind != B2CNN_SAMPLES_F64 && sample_kind != B2CNN_SAMPLES_GRID)
        return fail(B2CNN_EINVAL, "b2cnn_ring_push: sample_kind must be B2CNN_SAMPLES_ADC16, _F64 or _GRID");
    DEVICE_GUARD(h->device);
    const char *err = "";
    int em = 0;
    const int rc = ring_push(h->r, new_samples, sample_kind, n_new, x_out, dtype, &em, window_index,
                             t0_seconds, reinterpret_cast<cudaStream_t>(stream), &err);
    if (rc != B2CNN_OK) return finish("b2cnn_ring_push", rc, err);
    if (emitted) *emitted = em;
    return B2CNN_OK;
}

// ---- wire formats (b2cnn_wire.cu) ----
extern "C" int b2cnn_decode_sample_messages(const void *bytes, const int64_t *offsets, int64_t n_msgs, int32_t *idx_out, double *val_out,
                                            const int64_t *row_of_msg, double *frame, int64_t frame_rows, int32_t n_sig, int32_t *n_bad,
                                            void *stream) {
    const char *err = "";
    const int rc = wire_decode_pairs(reinterpret_cast<const uint8_t *>(bytes), offsets, n_msgs, idx_out, val_out, row_of_msg, frame,
                                     frame_rows, n_sig, n_bad, reinterpret_cast<cudaStream_t>(stream), &err);
    return finish("b2cnn_decode_sample_messages", rc, err);
}
extern "C" int b2cnn_decode_array_messages(const void *bytes, const int64_t *offsets, int64_t n_msgs, int32_t max_vals, double *vals_out,
                                           int32_t *counts_out, int32_t *n_bad, void *stream) {
    const char *err = "";
    const int rc = wire_decode_arrays(reinterpret_cast<const uint8_t *>(bytes), offsets, n_msgs, max_vals, vals_out, counts_out, n_bad,
                                      reinterpret_cast<cudaStream_t>(stream), &err);
    return finish("b2cnn_decode_array_messages", rc, err);
}
extern "C" int b2cnn_frame_check(const void *frame, int64_t bytes, b2cnn_frame_header *header_out, int64_t *ids_offset,
                                 int64_t *samples_offset) {
    if (!frame || bytes < (int64_t)sizeof(b2cnn_frame_header)) return fail(B2CNN_EINVAL, "b2cnn_frame_check: buffer shorter than a header");
    b2cnn_frame_header hd;
    memcpy(&hd, frame, sizeof hd);
    if (hd.magic != B2CNN_FRAME_MAGIC || hd.version != 1) return fail(B2CNN_EINVAL, "b2cnn_frame_check: bad magic / version");
    if (hd.kind > B2CNN_SAMPLES_GRID || hd.n_patients < 1 || hd.n_new < 1 || hd.n_sig < 1 || hd.n_sig > 64)
        return fail(B2CNN_EINVAL, "b2cnn_frame_check: bad kind / shape");
    const int64_t esz = hd.kind == B2CNN_SAMPLES_ADC16 ? 2 : 8;
    const int64_t ids = sizeof hd, smp = (ids + 4ll * hd.n_patients + 7) / 8 * 8;
    // the header is untrusted input: three 32-bit counts can wrap a 64-bit product, so the size is formed in 128 bits
    const unsigned __int128 need128 = (unsigned __int128)smp + (unsigned __int128)esz * hd.n_patients * hd.n_new * hd.n_sig;
    const int64_t need = need128 > (unsigned __int128)INT64_MAX ? INT64_MAX : (int64_t)need128;
    if (bytes != need) {
        char buf[128];
        snprintf(buf, sizeof buf, "b2cnn_frame_check: frame is %lld bytes, its header describes %lld", (long long)bytes, (long long)need);
        return fail(B2CNN_EINVAL, buf);
    }
    if (header_out) *header_out = hd;
    if (ids_offset) *ids_offset = ids;
    if (samples_offset) *samples_offset = smp;
    return B2CNN_OK;
}
extern "C" double b2cnn_parse_decimal(const char *s, int64_t len, int32_t *status) {
    int st = 0;
    const double v = wire_parse_decimal_host(s, len, &st);
    if (status) *status = st;
    return v;
}

extern "C" const char *b2cnn_version(void) { return "b2cnn 0.4 (sm_90a; wgmma fused bf16 path, fp32 streaming path, generic path, device preprocessing + patient ring buffers)"; }

extern "C" int b2cnn_create(const b2cnn_config *cfg, b2cnn_handle **out) {
    if (!cfg || !out) return fail(B2CNN_EINVAL, "b2cnn_create: null argument");
    *out = nullptr;
    Dims d;
    if (!derive_dims(*cfg, d)) return fail(B2CNN_EINVAL, "b2cnn_create: window too short for this conv/pool stack");
    if (cfg->c_mid != kCMid || cfg->hidden != kHidden || cfg->layers != 2)
        return fail(B2CNN_EARCH, "b2cnn_create: only conv1 out_channels=4, LSTM hidden=16, layers=2 (bin/models.py:10,16) are supported");
    if (kCMid * d.C * d.K1 > kMaxW1) return fail(B2CNN_EARCH, "b2cnn_create: in_channels*k1 > 200 not supported");
    if (d.K2 > kMaxK2) return fail(B2CNN_EARCH, "b2cnn_create: k2 > 8 not supported");
    if (d.C > 16) return fail(B2CNN_EARCH, "b2cnn_create: in_channels > 16 not supported");
    if (cfg->act < 0 || cfg->act > 2) return fail(B2CNN_EINVAL, "b2cnn_create: bad activation");
    if (cfg->lstm_input != d.L) {
        char buf[256];
        snprintf(buf, sizeof buf,
                 "b2cnn_create: L_out(window=%d)=%d != lstm_input=%d: x.view(-1, MAGICNUM) would straddle windows (bin/models.py:29)",
                 d.W, d.L, cfg->lstm_input);
        return fail(B2CNN_EVIEW, buf);
    }
    int dev = cfg->device;
    if (dev < 0) CU_TRY(cudaGetDevice(&dev));
    DEVICE_GUARD(dev);
    b2cnn_handle *h = new (std::nothrow) b2cnn_handle();
    if (!h) return fail(B2CNN_ESTATE, "out of host memory");
    h->cfg = *cfg; h->d = d; h->device = dev;
    cudaError_t e = cudaDeviceGetAttribute(&h->num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) { delete h; return cuda_fail(e, "cudaDeviceGetAttribute"); }
    h->n_weights = b2cnn_weight_count(cfg);
    e = cudaMalloc(&h->d_blob, sizeof(float) * h->n_weights);
    if (e == cudaSuccess) e = cudaMalloc(&h->d_wih0T, sizeof(float) * (size_t)d.L * kGates);
    if (e != cudaSuccess) { b2cnn_destroy(h); return cuda_fail(e, "cudaMalloc(weights)"); }
    *out = h;
    return B2CNN_OK;
}

extern "C" void b2cnn_destroy(b2cnn_handle *h) {
    if (!h) return;
    DeviceGuard guard(h->device);
    tc_release(h->tc);
    cudaFree(h->d_blob); cudaFree(h->d_wih0T);
    for (int i = 0; i < 3; ++i)
        if (h->ev_stage[i]) cudaEventDestroy(h->ev_stage[i]);
    for (int i = 0; i < 2; ++i) {
        cudaFree(h->st_x[i]);
        if (h->ev_copied[i]) cudaEventDestroy(h->ev_copied[i]);
        if (h->ev_done[i]) cudaEventDestroy(h->ev_done[i]);
    }
    cudaFree(h->st_age); cudaFree(h->st_out); cudaFree(h->st_ws);
    if (h->s_copy) cudaStreamDestroy(h->s_copy);
    if (h->s_comp) cudaStreamDestroy(h->s_comp);
    delete h;
}

extern "C" int b2cnn_set_weights(b2cnn_handle *h, const float *blob, int64_t n, int on_device, void *stream) {
    if (!h || !blob) return fail(B2CNN_EINVAL, "b2cnn_set_weights: null argument");
    if (n != h->n_weights) {
        char buf[160];
        snprintf(buf, sizeof buf, "b2cnn_set_weights: expected %lld floats, got %lld", (long long)h->n_weights, (long long)n);
        return fail(B2CNN_EINVAL, buf);
    }
    cudaStream_t st = (cudaStream_t)stream;
    DEVICE_GUARD(h->device);
    const Dims &d = h->d;
    ++h->weight_gen;
    CU_TRY(cudaMemcpyAsync(h->d_blob, blob, sizeof(float) * n, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    // conv weights + affine -> host copy for the kernel-parameter constant bank
    const BlobOff off = blob_offsets(d);
    std::vector<float> conv(off.wih0), aff(2 * kCMid + 2, 0.f);
    if (on_device) {
        CU_TRY(cudaMemcpyAsync(conv.data(), blob, sizeof(float) * conv.size(), cudaMemcpyDeviceToHost, st));
        if (d.has_affine) CU_TRY(cudaMemcpyAsync(aff.data(), blob + off.affine, sizeof(float) * aff.size(), cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaStreamSynchronize(st));
    } else {
        memcpy(conv.data(), blob, sizeof(float) * conv.size());
        if (d.has_affine) memcpy(aff.data(), blob + off.affine, sizeof(float) * aff.size());
    }
    ConvWeights &cw = h->cw;
    memset(&cw, 0, sizeof cw);
    const float *w1 = conv.data() + off.w1, *b1 = conv.data() + off.b1, *w2 = conv.data() + off.w2, *b2 = conv.data() + off.b2;
    for (int o = 0; o < kCMid; ++o)
        for (int c = 0; c < d.C; ++c)
            for (int k = 0; k < d.K1; ++k) cw.w1[(c * d.K1 + k) * kCMid + o] = w1[((int64_t)o * d.C + c) * d.K1 + k];
    for (int o = 0; o < kCMid; ++o) cw.b1[o] = b1[o];
    for (int i = 0; i < kCMid * d.K2; ++i) cw.w2[i] = w2[i];
    cw.b2 = b2[0];
    for (int o = 0; o < kCMid; ++o) { cw.s1[o] = d.has_affine ? aff[o] : 1.f; cw.t1[o] = d.has_affine ? aff[kCMid + o] : 0.f; }
    cw.s2 = d.has_affine ? aff[2 * kCMid] : 1.f;
    cw.t2 = d.has_affine ? aff[2 * kCMid + 1] : 0.f;
    // head pointers into the device blob
    const float *p = h->d_blob, *wih0 = p + off.wih0;
    h->hw = HeadWeights{h->d_wih0T, p + off.whh0, p + off.bih0, p + off.bhh0, p + off.wih1, p + off.whh1, p + off.bih1, p + off.bhh1,
                        p + off.wo, p + off.bo};
    launch_transpose_wih(wih0, h->d_wih0T, d.L, st);
    CU_TRY(cudaGetLastError());
    int rc = tc_prepare(h->tc, d, cw, wih0, (int)h->opt_tc_splits, st);
    if (rc != 0) return fail(B2CNN_ECUDA, std::string("tc_prepare: ") + tc_error());
    h->weights_set = true;
    return B2CNN_OK;
}

// ---- which kernels a forward call runs: DESIGN.md §2 is the table this code implements ----
// The front end turns the windows into layer-0 gate partials (Stream, Fused) or feature rows (TcUnfused, Generic).
// A short-window kernel, where one applies, runs the whole call instead; the workspace stays that of the front end,
// so a size taken once serves every batch size and option.
enum class Front { Stream, Fused, TcUnfused, Generic };
enum class Short { None, Batch, Small };
struct Route { Front front; Short short_kernel; };

static Front front_end(const b2cnn_handle *h, const Dims &d, int dtype) {
    if (h->opt_path == B2CNN_PATH_GENERIC) return Front::Generic;
    if (dtype == B2CNN_DTYPE_F32) return h->tc.fused && d.XP % 4 == 0 ? Front::Stream : Front::Generic;   // TMA: 16-byte rows
    if (h->tc.fused && h->opt_tc_fused) return Front::Fused;
    return h->tc.features ? Front::TcUnfused : Front::Generic;
}

static Route route(const b2cnn_handle *h, const Dims &d, int dtype, int64_t B, int mode) {
    Route r{front_end(h, d, dtype), Short::None};
    if (h->opt_path == B2CNN_PATH_TENSORCORE || !h->opt_small) return r;
    const bool indep = mode == B2CNN_MODE_INDEPENDENT;
    // many short windows ([P,10,120], all patients of a trigger): one launch, one warp per window
    if (indep && B >= 8 && batch_supported(d)) r.short_kernel = Short::Batch;
    // few short windows (the production call is [1,10,120]): one launch does everything
    else if ((indep || B == 1) && B <= 256 && (int64_t)d.C * d.W <= 8192 && small_supported(d)) r.short_kernel = Short::Small;
    return r;
}

// Scratch of one call, in this order: feature rows [B][L] | range partials [slices][B][64] | gates [B][64] | the
// tensor-core region: NaN flags, then the pitch-aligned bf16 copy of x.
struct WsLayout { int64_t feats, partial, gates, tc, total; };

static WsLayout ws_layout(const b2cnn_handle *h, int64_t B, bool feats, bool stage) {
    const Dims &d = h->d;
    const int ks = choose_ksplit(d.L), ranges = h->tc.fused ? h->tc.n_ranges : 0;
    WsLayout w;
    w.feats = feats ? align_up(B * d.L * 4, 256) : 0;
    w.partial = align_up((int64_t)(ranges > ks ? ranges : ks) * B * kGates * 4, 256);
    w.gates = align_up(B * kGates * 4, 256);
    w.tc = h->tc.features || h->tc.fused ? tc_flags_bytes(B) + (stage ? tc_stage_bytes(d, B) : 0) : 0;
    w.total = w.feats + w.partial + w.gates + w.tc;
    return w;
}

// Only the unfused tensor-core and the generic front ends round-trip feature rows through HBM.  The bf16 tensor-core
// front ends copy x into the staging rows when its pitch is not a multiple of 8 samples; the staging region is also
// reserved whenever W is not, which is what b2cnn_workspace_bytes_for has always returned for such windows.
static WsLayout call_layout(const b2cnn_handle *h, const Dims &d, int64_t B, Front f) {
    const bool tc_bf16 = f == Front::Fused || f == Front::TcUnfused;
    return ws_layout(h, B, f == Front::TcUnfused || f == Front::Generic, d.W % 8 != 0 || (tc_bf16 && d.XP % 8 != 0));
}

// dtype-blind size: enough for whatever route a call of any dtype and row pitch may take
extern "C" int64_t b2cnn_workspace_bytes(b2cnn_handle *h, int64_t B, int mode) {
    (void)mode;
    if (!h || B < 1) return -1;
    return ws_layout(h, B, true, true).total;
}

// exact size for contiguous windows of `dtype`: 307 MB smaller at [4096,3,75000] bf16, where the features never leave the SM
extern "C" int64_t b2cnn_workspace_bytes_for(b2cnn_handle *h, int64_t B, int mode, int dtype) {
    (void)mode;
    if (!h || B < 1 || (dtype != B2CNN_DTYPE_F32 && dtype != B2CNN_DTYPE_BF16)) return -1;
    return call_layout(h, h->d, B, front_end(h, h->d, dtype)).total;
}

// the events b2cnn_last_stage_ms reads, created by the first profiled call
static int create_stage_events(b2cnn_handle *h) {
    for (int i = 0; i < 3; ++i)
        if (!h->ev_stage[i]) CU_TRY(cudaEventCreate(&h->ev_stage[i]));
    return B2CNN_OK;
}

// seq_off / n_seq: b2cnn_forward_seq's sequences (device memory, n_seq + 1 offsets; mode is B2CNN_MODE_SEQUENCE), else NULL / 0
static int forward_device(b2cnn_handle *h, const void *x, int dtype, int64_t B, int64_t xpitch, const float *age, int64_t n_age,
                          int mode, int apply_sigmoid, float *out, void *ws, int64_t ws_bytes, cudaStream_t st,
                          const int64_t *seq_off = nullptr, int64_t n_seq = 0) {
    Dims d = h->d;
    if (xpitch < d.W || xpitch > 0x7fffffff) return fail(B2CNN_EINVAL, "b2cnn_forward: x_pitch must be >= window");
    d.XP = (int)xpitch;
    const Route r = route(h, d, dtype, B, mode);
    const WsLayout wl = call_layout(h, d, B, r.front);
    if (!ws || ws_bytes < wl.total)
        return fail(B2CNN_ESTATE, "b2cnn_forward: workspace missing or smaller than b2cnn_workspace_bytes_for(); rows whose pitch is not "
                                  "a multiple of 16 bytes may need more: pad the rows, or size the workspace with b2cnn_workspace_bytes()");
    if (h->opt_path == B2CNN_PATH_TENSORCORE && r.front == Front::Generic)
        return fail(B2CNN_EARCH, "path=tensorcore requested but this shape/dtype/mode is not supported by the tensor-core kernel");
    char *base = (char *)ws;
    float *feats = (float *)base; base += wl.feats;
    float *partial = (float *)base; base += wl.partial;
    float *gates = (float *)base; base += wl.gates;
    void *tc_ws = base;
    const bool prof = h->opt_profile != 0;
    if (prof) {
        if (int rc = create_stage_events(h)) return rc;
        CU_TRY(cudaEventRecord(h->ev_stage[0], st));
    }
    // stage 0: the front end, or the short-window kernel that does the whole call
    const bool indep = mode == B2CNN_MODE_INDEPENDENT;
    const bool to_gates = r.front == Front::Stream || r.front == Front::Fused;   // the streaming kernels: features never leave the SM
    // feature layout: the generic kernel writes rows [B][L]; the tensor-core kernel's threads are windows, so it
    // writes the transpose [L][B] (coalesced across lanes)
    int64_t sB = d.L, sP = 1;
    const char *err = "", *what;
    int n;
    if (r.short_kernel == Short::Batch) {
        what = "short-window batch kernel";
        n = launch_short_batch(d, h->cw, h->hw, x, dtype, B, age, n_age, apply_sigmoid, out, h->num_sms, st, &err);
    } else if (r.short_kernel == Short::Small) {
        what = "small-window kernel";
        n = launch_small_forward(d, h->cw, h->hw, x, dtype, B, age, n_age, apply_sigmoid, out, st, &err);
    } else if (to_gates) {
        what = r.front == Front::Stream ? "fp32 stream kernel" : "tensor-core fused kernel";
        n = tc_gates(h->tc, d, h->cw, h->hw, x, dtype, B, partial, gates, tc_ws, h->num_sms, st, &err, !indep);
    } else if (r.front == Front::TcUnfused) {
        what = "tensor-core front end";
        sB = 1; sP = B;
        n = tc_frontend(h->tc, d, h->cw, x, B, feats, sB, sP, tc_ws, h->num_sms, st, &err);
    } else {
        what = "front end";
        n = launch_frontend_generic(d, h->cw, x, dtype, B, feats, sB, sP, st, h->num_sms, &err);
    }
    if (n < 0) return fail(n == kLaunchArch ? B2CNN_EARCH : B2CNN_ECUDA, std::string(what) + ": " + err);
    int launches = n;
    if (prof) CU_TRY(cudaEventRecord(h->ev_stage[1], st));
    // stage 1: projection + LSTM head
    if (r.short_kernel == Short::None) {
        // the head kernel is the last reader of the call's exception list: it also puts the handle's flag state back to zero
        const bool cleans = to_gates && indep && h->tc.cur_own;
        if (!to_gates)
            n = launch_head(d, h->hw, feats, sB, sP, B, age, n_age, mode, apply_sigmoid, out, gates, partial, choose_ksplit(d.L), st, &err,
                            seq_off, n_seq);
        else if (indep)
            n = launch_reduce_lstm_head(d, h->hw, partial, h->tc.n_ranges, B, age, n_age, apply_sigmoid, out, st, &err,
                                        cleans ? h->tc.cur_count : nullptr, h->tc.cur_flags, h->tc.cur_list);
        else
            n = launch_lstm_head(d, h->hw, gates, B, age, n_age, mode, apply_sigmoid, out, st, &err, seq_off, n_seq);
        if (n < 0) return fail(B2CNN_ECUDA, std::string("head: ") + err);
        if (cleans) h->tc.flags_clean = true;
        launches += n;
    }
    if (prof) { CU_TRY(cudaEventRecord(h->ev_stage[2], st)); h->ev_valid = true; }
    h->last_launches = launches;
    h->last_path = r.short_kernel != Short::None || r.front == Front::Generic ? B2CNN_PATH_GENERIC
                   : r.front == Front::Stream                               ? B2CNN_PATH_STREAM
                                                                            : B2CNN_PATH_TENSORCORE;
    return B2CNN_OK;
}

// the arguments every call on B windows of `dtype` shares (the forward calls also take age and mode)
static int check_windows(const char *fn, b2cnn_handle *h, const void *x, int dtype, int64_t B, const float *out) {
    if (!h || !x || !out) return fail(B2CNN_EINVAL, std::string(fn) + ": null argument");
    if (!h->weights_set) return fail(B2CNN_ESTATE, std::string(fn) + ": weights not set (call b2cnn_set_weights)");
    if (B < 1 || B > (int64_t)0x7fffffff / 64) return fail(B2CNN_EINVAL, std::string(fn) + ": batch size out of range");
    if (dtype != B2CNN_DTYPE_F32 && dtype != B2CNN_DTYPE_BF16) return fail(B2CNN_EINVAL, std::string(fn) + ": dtype must be f32 (0) or bf16 (1)");
    return B2CNN_OK;
}

static int check_call(b2cnn_handle *h, const void *x, int dtype, int64_t B, const float *age, int64_t n_age, int mode, float *out) {
    if (!age) return fail(B2CNN_EINVAL, "b2cnn_forward: null argument");
    if (int rc = check_windows("b2cnn_forward", h, x, dtype, B, out)) return rc;
    if (mode != B2CNN_MODE_INDEPENDENT && mode != B2CNN_MODE_SEQUENCE) return fail(B2CNN_EINVAL, "b2cnn_forward: bad mode");
    if (n_age != 1 && n_age != B) return fail(B2CNN_EINVAL, "b2cnn_forward: age must have 1 or B elements");
    return B2CNN_OK;
}

extern "C" int b2cnn_forward(b2cnn_handle *h, const void *x, int dtype, int64_t B, const float *age, int64_t n_age,
                             int mode, int apply_sigmoid, float *out, void *workspace, int64_t workspace_bytes, void *stream) {
    return b2cnn_forward_pitched(h, x, dtype, B, h ? h->d.W : 0, age, n_age, mode, apply_sigmoid, out, workspace, workspace_bytes,
                                 stream);
}

extern "C" int b2cnn_forward_pitched(b2cnn_handle *h, const void *x, int dtype, int64_t B, int64_t x_pitch, const float *age,
                                     int64_t n_age, int mode, int apply_sigmoid, float *out, void *workspace,
                                     int64_t workspace_bytes, void *stream) {
    int rc = check_call(h, x, dtype, B, age, n_age, mode, out);
    if (rc) return rc;
    DEVICE_GUARD(h->device);
    return forward_device(h, x, dtype, B, x_pitch, age, n_age, mode, apply_sigmoid, out, workspace, workspace_bytes, (cudaStream_t)stream);
}

// The sequence offsets of b2cnn_forward_seq sit after what b2cnn_workspace_bytes(h, B) covers.
static int64_t seq_ws_base(b2cnn_handle *h, int64_t B) { return ws_layout(h, B, true, true).total; }

extern "C" int64_t b2cnn_workspace_bytes_seq(b2cnn_handle *h, int64_t B, const int64_t *seq_lengths, int64_t n_seq) {
    std::vector<int64_t> off;
    const char *err = "";
    if (!h || B < 1) { fail(B2CNN_EINVAL, "b2cnn_workspace_bytes_seq: null handle / bad batch"); return -1; }
    if (!seq_offsets(SeqLengths{true, seq_lengths, n_seq}, B, off, &err)) {
        fail(B2CNN_EINVAL, std::string("b2cnn_workspace_bytes_seq: ") + err);
        return -1;
    }
    return seq_ws_base(h, B) + align_up(8 * (n_seq + 1), 256);
}

extern "C" int b2cnn_forward_seq(b2cnn_handle *h, const void *x, int dtype, int64_t B, int64_t x_pitch, const float *age, int64_t n_age,
                                 const int64_t *seq_lengths, int64_t n_seq, int apply_sigmoid, float *out, void *workspace,
                                 int64_t workspace_bytes, void *stream) {
    int rc = check_call(h, x, dtype, B, age, n_age, B2CNN_MODE_SEQUENCE, out);
    if (rc) return rc;
    std::vector<int64_t> off;
    const char *err = "";
    if (!seq_offsets(SeqLengths{true, seq_lengths, n_seq}, B, off, &err)) return fail(B2CNN_EINVAL, std::string("b2cnn_forward_seq: ") + err);
    const int64_t base = seq_ws_base(h, B);
    if (!workspace || workspace_bytes < base + align_up(8 * (n_seq + 1), 256))
        return fail(B2CNN_ESTATE, "b2cnn_forward_seq: workspace missing or smaller than b2cnn_workspace_bytes_seq()");
    DEVICE_GUARD(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    int64_t *doff = reinterpret_cast<int64_t *>((char *)workspace + base);
    CU_TRY(cudaMemcpyAsync(doff, off.data(), sizeof(int64_t) * off.size(), cudaMemcpyHostToDevice, st));
    return forward_device(h, x, dtype, B, x_pitch, age, n_age, B2CNN_MODE_SEQUENCE, apply_sigmoid, out, workspace, base, st, doff, n_seq);
}

extern "C" int b2cnn_features(b2cnn_handle *h, const void *x, int dtype, int64_t B, float *feats, void *stream) {
    int rc = check_windows("b2cnn_features", h, x, dtype, B, feats);
    if (rc) return rc;
    DEVICE_GUARD(h->device);
    const char *err = "";
    int n;
    if (h->opt_path != B2CNN_PATH_GENERIC && dtype == B2CNN_DTYPE_BF16 && h->tc.features) {
        n = tc_features(h->tc, h->d, h->cw, x, B, feats, h->num_sms, (cudaStream_t)stream, &err);
        h->last_path = B2CNN_PATH_TENSORCORE;
    } else {
        if (h->opt_path == B2CNN_PATH_TENSORCORE) return fail(B2CNN_EARCH, "b2cnn_features: tensor-core path unavailable for this shape");
        n = launch_frontend_generic(h->d, h->cw, x, dtype, B, feats, h->d.L, 1, (cudaStream_t)stream, h->num_sms, &err);
        h->last_path = B2CNN_PATH_GENERIC;
    }
    if (n < 0) return fail(n == kLaunchArch ? B2CNN_EARCH : B2CNN_ECUDA, std::string("front end: ") + err);
    h->last_launches = n;
    return B2CNN_OK;
}

// ---- sliding-window scorer over a per-patient feature ring (b2cnn_slide.cu) ----
// digest: the front-end digest of the handle's weights at the last reset (what every extra head must have)
struct b2cnn_slide { Slide *s; b2cnn_handle *h; uint64_t gen; uint64_t digest; };

static uint64_t weights_digest(const Slide *s, const ConvWeights &cw) {
    b2cnn_slide_state_header hdr;
    slide_describe_state(s, cw, &hdr);
    return hdr.frontend_digest;
}

// B2CNN_ESTATE when the handle's weights changed since the scorer's last reset, else B2CNN_OK
static int check_fresh(const char *fn, const b2cnn_slide *o,
                       const char *why = "the handle's weights changed since the scorer's last reset (stored features are stale)") {
    return o->gen == o->h->weight_gen ? B2CNN_OK : fail(B2CNN_ESTATE, std::string(fn) + ": " + why);
}

// B2CNN_EINVAL unless path is B2CNN_PATH_AUTO, B2CNN_PATH_GENERIC or B2CNN_PATH_TENSORCORE
static int check_path(const char *fn, int path) {
    if (path == B2CNN_PATH_TENSORCORE || path == B2CNN_PATH_GENERIC || path == B2CNN_PATH_AUTO) return B2CNN_OK;
    return fail(B2CNN_EINVAL, std::string(fn) + ": path must be B2CNN_PATH_AUTO, B2CNN_PATH_GENERIC or B2CNN_PATH_TENSORCORE");
}

static int slide_create_on(const char *fn, b2cnn_handle *h, int32_t n_patients, int32_t stride, int dtype, int path, int mode,
                           b2cnn_slide **out) {
    if (!h || !out) return fail(B2CNN_EINVAL, std::string(fn) + ": null argument");
    *out = nullptr;
    if (int rc = check_path(fn, path)) return rc;
    if (mode != B2CNN_MODE_INDEPENDENT && mode != B2CNN_MODE_SEQUENCE)
        return fail(B2CNN_EINVAL, std::string(fn) + ": mode must be B2CNN_MODE_INDEPENDENT or B2CNN_MODE_SEQUENCE");
    if (!h->weights_set) return fail(B2CNN_ESTATE, std::string(fn) + ": weights not set (call b2cnn_set_weights)");
    DEVICE_GUARD(h->device);
    const char *err = "";
    Slide *s = nullptr;
    // auto: the tensor-core path where it holds the model (slide_create refuses everything else with B2CNN_EARCH; its
    // geometries have F = 4, so a stride it refuses the generic path refuses too), else the generic path
    const bool tc = path == B2CNN_PATH_TENSORCORE || (path == B2CNN_PATH_AUTO && h->tc.fused);
    const int rc = slide_create(h->d, h->tc, tc ? B2CNN_PATH_TENSORCORE : B2CNN_PATH_GENERIC, mode, n_patients, stride, dtype,
                                h->device, h->num_sms, &s, &err);
    if (rc != B2CNN_OK) return finish(fn, rc, err);
    b2cnn_slide *o = new (std::nothrow) b2cnn_slide{s, h, h->weight_gen, weights_digest(s, h->cw)};
    if (!o) { slide_destroy(s); return fail(B2CNN_ESTATE, "out of host memory"); }
    if (slide_reset(s, nullptr, &err) != B2CNN_OK || cudaStreamSynchronize(nullptr) != cudaSuccess) {
        b2cnn_slide_destroy(o);
        return fail(B2CNN_ECUDA, std::string(fn) + ": initial reset");
    }
    *out = o;
    return B2CNN_OK;
}
extern "C" int b2cnn_slide_create(b2cnn_handle *h, int32_t n_patients, int32_t stride, int dtype, b2cnn_slide **out) {
    return slide_create_on("b2cnn_slide_create", h, n_patients, stride, dtype, B2CNN_PATH_TENSORCORE, B2CNN_MODE_INDEPENDENT, out);
}
extern "C" int b2cnn_slide_create_path(b2cnn_handle *h, int32_t n_patients, int32_t stride, int dtype, int path, b2cnn_slide **out) {
    return slide_create_on("b2cnn_slide_create_path", h, n_patients, stride, dtype, path, B2CNN_MODE_INDEPENDENT, out);
}
extern "C" int b2cnn_slide_create_ex(b2cnn_handle *h, int32_t n_patients, int32_t stride, int dtype, int path, int mode, b2cnn_slide **out) {
    return slide_create_on("b2cnn_slide_create_ex", h, n_patients, stride, dtype, path, mode, out);
}
extern "C" int b2cnn_slide_path(const b2cnn_slide *o) { return o ? slide_path(o->s) : -1; }
extern "C" int b2cnn_slide_mode(const b2cnn_slide *o) { return o ? slide_mode(o->s) : -1; }
extern "C" void b2cnn_slide_destroy(b2cnn_slide *o) {
    if (!o) return;
    DeviceGuard guard(slide_device(o->s));
    slide_destroy(o->s);
    delete o;
}
extern "C" int b2cnn_slide_reset(b2cnn_slide *o, void *stream) {
    if (!o) return fail(B2CNN_EINVAL, "b2cnn_slide_reset: null argument");
    DEVICE_GUARD(slide_device(o->s));
    const char *err = "";
    const int rc = slide_reset(o->s, reinterpret_cast<cudaStream_t>(stream), &err);
    if (rc != B2CNN_OK) return finish("b2cnn_slide_reset", rc, err);
    o->gen = o->h->weight_gen;
    o->digest = weights_digest(o->s, o->h->cw);
    return B2CNN_OK;
}
static int slide_push_api(const char *fn, b2cnn_slide *o, const void *new_samples, int64_t pitch, const float *age, int64_t n_age,
                          int apply_sigmoid, float *out, bool heads, int32_t *emitted, int64_t *window_index, void *stream) {
    if (!o || !new_samples || !age || !out || !emitted || !window_index) return fail(B2CNN_EINVAL, std::string(fn) + ": null argument");
    b2cnn_handle *h = o->h;
    if (int rc = check_fresh(fn, o)) return rc;
    const int stale = heads ? slide_stale_head(o->s, o->digest) : -1;
    if (stale >= 0)
        return fail(B2CNN_ESTATE, std::string(fn) + ": head " + std::to_string(stale) +
                                      " has other front-end weights than the scorer (its conv weights changed at the last reset)");
    DEVICE_GUARD(h->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    cudaEvent_t *ev = nullptr;
    if (h->opt_profile) {
        if (int rc = create_stage_events(h)) return rc;
        ev = h->ev_stage;
    }
    const char *err = "";
    int em = 0;
    int64_t widx = -1;
    const int rc = slide_push(o->s, h->cw, h->hw, h->tc, new_samples, pitch, age, n_age, apply_sigmoid, out, heads, &em, &widx, ev, st,
                              &err);
    if (rc != B2CNN_OK) return finish(fn, rc, err);
    h->ev_valid = ev != nullptr;
    *emitted = em;
    if (em) *window_index = widx;
    return B2CNN_OK;
}
extern "C" int b2cnn_slide_push(b2cnn_slide *o, const void *new_samples, int64_t pitch, const float *age, int64_t n_age,
                                int apply_sigmoid, float *out, int32_t *emitted, int64_t *window_index, void *stream) {
    return slide_push_api("b2cnn_slide_push", o, new_samples, pitch, age, n_age, apply_sigmoid, out, false, emitted, window_index, stream);
}
extern "C" int b2cnn_slide_push_heads(b2cnn_slide *o, const void *new_samples, int64_t pitch, const float *age, int64_t n_age,
                                      int apply_sigmoid, float *out, int32_t *emitted, int64_t *window_index, void *stream) {
    return slide_push_api("b2cnn_slide_push_heads", o, new_samples, pitch, age, n_age, apply_sigmoid, out, true, emitted, window_index,
                          stream);
}
extern "C" int b2cnn_slide_n_heads(const b2cnn_slide *o) { return o ? slide_n_heads(o->s) : -1; }
static int slide_set_heads_api(const char *fn, b2cnn_slide *o, b2cnn_handle *const *heads, int32_t n, int32_t flags, void *stream) {
    const std::string pre = std::string(fn) + ": ";
    if (!o || (n > 0 && !heads)) return fail(B2CNN_EINVAL, pre + "null argument");
    if (flags & ~B2CNN_SLIDE_HEADS_SHORTER_WINDOWS) return fail(B2CNN_EINVAL, pre + "unknown flag bits");
    if (n < 0 || n > B2CNN_SLIDE_MAX_HEADS)
        return fail(B2CNN_EINVAL, pre + "n must be in [0, " + std::to_string(B2CNN_SLIDE_MAX_HEADS) + "]");
    if (n > 0 && slide_mode(o->s) == B2CNN_MODE_SEQUENCE)
        return fail(B2CNN_EINVAL, pre + "a sequence-mode scorer takes no extra heads");
    const b2cnn_handle *h = o->h;
    const b2cnn_config &c = h->cfg;
    const bool shorter = flags & B2CNN_SLIDE_HEADS_SHORTER_WINDOWS;
    const int F = h->d.feature_stride(), R = h->d.receptive_field();
    std::vector<SlideHeadSource> src((size_t)n);
    for (int i = 0; i < n; ++i) {
        const b2cnn_handle *x = heads[i];
        const std::string which = "head " + std::to_string(i) + ": ";
        if (!x) return fail(B2CNN_EINVAL, pre + which + "null handle");
        if (!x->weights_set) return fail(B2CNN_EINVAL, pre + which + "weights not set (call b2cnn_set_weights)");
        if (x->device != h->device) return fail(B2CNN_EINVAL, pre + which + "on another device than the scorer");
        const b2cnn_config &e = x->cfg;
        if (e.in_channels != c.in_channels || e.k1 != c.k1 || e.c_mid != c.c_mid || e.k2 != c.k2 || e.pool_k != c.pool_k ||
            e.pool_s != c.pool_s || e.hidden != c.hidden || e.layers != c.layers || e.act != c.act || e.flags != c.flags ||
            (!shorter && (e.window != c.window || e.lstm_input != c.lstm_input)))
            return fail(B2CNN_EARCH, pre + which + (shorter ? "another architecture than the scorer's model (only window, lstm_input and age_coef may differ)"
                                                            : "another architecture than the scorer's model (only age_coef may differ)"));
        if (e.window > c.window) return fail(B2CNN_EARCH, pre + which + "a longer window than the scorer's");
        if ((c.window - e.window) % F != 0)
            return fail(B2CNN_EARCH, pre + which + "the scorer's window minus the head's is not a multiple of the feature stride " +
                                          std::to_string(F) + " (another feature lattice)");
        if (e.window < R || e.lstm_input != (e.window - R) / F + 1)
            return fail(B2CNN_EARCH, pre + which + "lstm_input is not the feature count of the head's window");
        if (slide_path(o->s) == B2CNN_PATH_TENSORCORE &&
            (!x->tc.fused || (e.window == c.window && (x->tc.n_ranges != h->tc.n_ranges || x->tc.chunks_per_cta != h->tc.chunks_per_cta))))
            return fail(B2CNN_EARCH, pre + which + (e.window == c.window ? "no packed W_ih chunks of the scorer's layout"
                                                                         : "no packed W_ih chunks of the streaming kernels for its window"));
        src[i] = SlideHeadSource{x->hw, &x->tc, x->d.age_coef, weights_digest(o->s, x->cw), e.window, e.lstm_input};
    }
    if (int rc = check_fresh(fn, o, "the scorer's handle's weights changed since its last reset (call reset first)")) return rc;
    for (int i = 0; i < n; ++i)
        if (src[i].digest != o->digest)
            return fail(B2CNN_ESTATE, pre + ("head " + std::to_string(i)) + ": other front-end (conv / affine) weights than the scorer's");
    DEVICE_GUARD(h->device);
    const char *err = "";
    const int rc = slide_set_heads(o->s, src.data(), n, reinterpret_cast<cudaStream_t>(stream), &err);
    return finish(fn, rc, err);
}
extern "C" int b2cnn_slide_set_heads(b2cnn_slide *o, b2cnn_handle *const *heads, int32_t n, void *stream) {
    return slide_set_heads_api("b2cnn_slide_set_heads", o, heads, n, 0, stream);
}
extern "C" int b2cnn_slide_set_heads_ex(b2cnn_slide *o, b2cnn_handle *const *heads, int32_t n, int32_t flags, void *stream) {
    return slide_set_heads_api("b2cnn_slide_set_heads_ex", o, heads, n, flags, stream);
}
extern "C" int b2cnn_slide_features(b2cnn_slide *o, float *feats, void *stream) {
    if (!o || !feats) return fail(B2CNN_EINVAL, "b2cnn_slide_features: null argument");
    if (int rc = check_fresh("b2cnn_slide_features", o)) return rc;
    DEVICE_GUARD(slide_device(o->s));
    const char *err = "";
    const int rc = slide_features(o->s, feats, reinterpret_cast<cudaStream_t>(stream), &err);
    return finish("b2cnn_slide_features", rc, err);
}

extern "C" int64_t b2cnn_slide_admit_workspace_bytes(b2cnn_slide *o, int32_t n, int64_t history_len) {
    return o ? slide_admit_workspace_bytes(o->s, n, history_len) : -1;
}
extern "C" int b2cnn_slide_admit(b2cnn_slide *o, const int32_t *patients, int32_t n, const void *history, int64_t history_len,
                                 int64_t pitch, int dtype, void *workspace, int64_t workspace_bytes, void *stream) {
    if (!o) return fail(B2CNN_EINVAL, "b2cnn_slide_admit: null argument");
    if (dtype != slide_dtype(o->s)) return fail(B2CNN_EINVAL, "b2cnn_slide_admit: the history's dtype is not the scorer's");
    if (int rc = check_fresh("b2cnn_slide_admit", o)) return rc;
    b2cnn_handle *h = o->h;
    DEVICE_GUARD(h->device);
    const char *err = "";
    const int rc = slide_admit(o->s, h->cw, h->tc, patients, n, history, history_len, pitch, workspace, workspace_bytes,
                               reinterpret_cast<cudaStream_t>(stream), &err);
    return finish("b2cnn_slide_admit", rc, err);
}
extern "C" int b2cnn_slide_discharge(b2cnn_slide *o, const int32_t *patients, int32_t n, void *stream) {
    if (!o) return fail(B2CNN_EINVAL, "b2cnn_slide_discharge: null argument");
    DEVICE_GUARD(slide_device(o->s));
    const char *err = "";
    const int rc = slide_discharge(o->s, patients, n, reinterpret_cast<cudaStream_t>(stream), &err);
    return finish("b2cnn_slide_discharge", rc, err);
}
extern "C" int b2cnn_slide_samples_seen(b2cnn_slide *o, int64_t *seen, void *stream) {
    if (!o || !seen) return fail(B2CNN_EINVAL, "b2cnn_slide_samples_seen: null argument");
    DEVICE_GUARD(slide_device(o->s));
    const char *err = "";
    const int rc = slide_samples_seen(o->s, seen, reinterpret_cast<cudaStream_t>(stream), &err);
    return finish("b2cnn_slide_samples_seen", rc, err);
}
extern "C" int b2cnn_slide_describe_state(b2cnn_slide *o, b2cnn_slide_state_header *out) {
    if (!o || !out) return fail(B2CNN_EINVAL, "b2cnn_slide_describe_state: null argument");
    slide_describe_state(o->s, o->h->cw, out);
    return B2CNN_OK;
}
extern "C" int64_t b2cnn_slide_state_workspace_bytes(b2cnn_slide *o, int32_t n) {
    return o ? slide_state_workspace_bytes(o->s, n) : -1;
}
static int slide_export_api(const char *fn, b2cnn_slide *o, const int32_t *patients, int32_t n, float *features, float *tails,
                            int64_t *seen_host, float *lstm, b2cnn_slide_state_header *header, void *workspace, int64_t workspace_bytes,
                            void *stream) {
    if (!o || !header) return fail(B2CNN_EINVAL, std::string(fn) + ": null argument");
    if (int rc = check_fresh(fn, o)) return rc;
    DEVICE_GUARD(slide_device(o->s));
    const char *err = "";
    const int rc = slide_export(o->s, o->h->cw, patients, n, features, tails, seen_host, lstm, header, workspace, workspace_bytes,
                                reinterpret_cast<cudaStream_t>(stream), &err);
    return finish(fn, rc, err);
}
static int slide_import_api(const char *fn, b2cnn_slide *o, const int32_t *patients, int32_t n, const b2cnn_slide_state_header *header,
                            const float *features, const float *tails, const int64_t *seen_host, const float *lstm, void *workspace,
                            int64_t workspace_bytes, void *stream) {
    if (!o || !header) return fail(B2CNN_EINVAL, std::string(fn) + ": null argument");
    if (int rc = check_fresh(fn, o)) return rc;
    DEVICE_GUARD(slide_device(o->s));
    const char *err = "";
    const int rc = slide_import(o->s, o->h->cw, patients, n, *header, features, tails, seen_host, lstm, workspace, workspace_bytes,
                                reinterpret_cast<cudaStream_t>(stream), &err);
    return finish(fn, rc, err);
}
extern "C" int b2cnn_slide_export(b2cnn_slide *o, const int32_t *patients, int32_t n, float *features, float *tails, int64_t *seen_host,
                                  b2cnn_slide_state_header *header, void *workspace, int64_t workspace_bytes, void *stream) {
    return slide_export_api("b2cnn_slide_export", o, patients, n, features, tails, seen_host, nullptr, header, workspace, workspace_bytes,
                            stream);
}
extern "C" int b2cnn_slide_export_ex(b2cnn_slide *o, const int32_t *patients, int32_t n, float *features, float *tails, int64_t *seen_host,
                                     float *lstm, b2cnn_slide_state_header *header, void *workspace, int64_t workspace_bytes, void *stream) {
    return slide_export_api("b2cnn_slide_export_ex", o, patients, n, features, tails, seen_host, lstm, header, workspace, workspace_bytes,
                            stream);
}
extern "C" int b2cnn_slide_import(b2cnn_slide *o, const int32_t *patients, int32_t n, const b2cnn_slide_state_header *header,
                                  const float *features, const float *tails, const int64_t *seen_host, void *workspace,
                                  int64_t workspace_bytes, void *stream) {
    return slide_import_api("b2cnn_slide_import", o, patients, n, header, features, tails, seen_host, nullptr, workspace, workspace_bytes,
                            stream);
}
extern "C" int b2cnn_slide_import_ex(b2cnn_slide *o, const int32_t *patients, int32_t n, const b2cnn_slide_state_header *header,
                                     const float *features, const float *tails, const int64_t *seen_host, const float *lstm, void *workspace,
                                     int64_t workspace_bytes, void *stream) {
    return slide_import_api("b2cnn_slide_import_ex", o, patients, n, header, features, tails, seen_host, lstm, workspace, workspace_bytes,
                            stream);
}

// ---- every sliding window of whole recordings (b2cnn_slide.cu) ----
// the path of a record call (B2CNN_OK) or the error: auto takes the tensor-core path where it holds the model, as a scorer
static int record_path(const char *fn, const b2cnn_handle *h, int dtype, int path, bool *use_tc) {
    if (!h) return fail(B2CNN_EINVAL, std::string(fn) + ": null argument");
    if (!h->weights_set) return fail(B2CNN_ESTATE, std::string(fn) + ": weights not set (call b2cnn_set_weights)");
    if (dtype != B2CNN_DTYPE_F32 && dtype != B2CNN_DTYPE_BF16) return fail(B2CNN_EINVAL, std::string(fn) + ": dtype must be f32 (0) or bf16 (1)");
    if (int rc = check_path(fn, path)) return rc;
    if (path == B2CNN_PATH_TENSORCORE && !h->tc.fused)
        return fail(B2CNN_EARCH, std::string(fn) + ": the tensor-core path covers the streaming tensor-core geometries only (MyCNN5 or "
                                                   "MyCNN2/3/4 conv/pool, 1 to 3 channels, tanh, no affine)");
    *use_tc = path == B2CNN_PATH_TENSORCORE || (path == B2CNN_PATH_AUTO && h->tc.fused);
    return B2CNN_OK;
}

static int64_t record_workspace(const char *fn, b2cnn_handle *h, int64_t B, int64_t N, int64_t pitch, int64_t stride, int dtype, int path,
                                int mode) {
    bool tc = false;
    if (record_path(fn, h, dtype, path, &tc) != B2CNN_OK) return -1;
    if (pitch < N) { fail(B2CNN_EINVAL, std::string(fn) + ": pitch must be >= the recording length"); return -1; }
    const char *err = "";
    const int64_t n = record_workspace_bytes(h->d, h->tc, tc, B, N, stride, dtype, mode, &err);
    if (n < 0) fail(B2CNN_EINVAL, std::string(fn) + ": " + err);
    return n;
}

extern "C" int64_t b2cnn_record_workspace_bytes(b2cnn_handle *h, int64_t B, int64_t N, int64_t pitch, int64_t stride, int dtype, int path) {
    return record_workspace("b2cnn_record_workspace_bytes", h, B, N, pitch, stride, dtype, path, B2CNN_MODE_INDEPENDENT);
}

extern "C" int64_t b2cnn_record_workspace_bytes_ex(b2cnn_handle *h, int64_t B, int64_t N, int64_t pitch, int64_t stride, int dtype, int path,
                                                   int mode) {
    return record_workspace("b2cnn_record_workspace_bytes_ex", h, B, N, pitch, stride, dtype, path, mode);
}

static int record_score(const char *fn, b2cnn_handle *h, const void *x, int dtype, int64_t B, int64_t N, int64_t pitch, int64_t stride,
                        int path, int mode, const float *age, int64_t n_age, int apply_sigmoid, float *out, void *workspace,
                        int64_t workspace_bytes, void *stream) {
    bool tc = false;
    if (int rc = record_path(fn, h, dtype, path, &tc)) return rc;
    if (!x || !age || !out) return fail(B2CNN_EINVAL, std::string(fn) + ": null argument");
    DEVICE_GUARD(h->device);
    const char *err = "";
    const int rc = score_record(h->d, h->cw, h->hw, h->tc, tc, h->num_sms, x, dtype, B, N, pitch, stride, mode, age, n_age, apply_sigmoid,
                                out, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream), &err);
    if (rc != B2CNN_OK) return finish(fn, rc, err);
    h->last_path = tc ? B2CNN_PATH_TENSORCORE : B2CNN_PATH_GENERIC;
    return B2CNN_OK;
}

extern "C" int b2cnn_score_record(b2cnn_handle *h, const void *x, int dtype, int64_t B, int64_t N, int64_t pitch, int64_t stride, int path,
                                  const float *age, int64_t n_age, int apply_sigmoid, float *out, void *workspace, int64_t workspace_bytes,
                                  void *stream) {
    return record_score("b2cnn_score_record", h, x, dtype, B, N, pitch, stride, path, B2CNN_MODE_INDEPENDENT, age, n_age, apply_sigmoid,
                        out, workspace, workspace_bytes, stream);
}

extern "C" int b2cnn_score_record_ex(b2cnn_handle *h, const void *x, int dtype, int64_t B, int64_t N, int64_t pitch, int64_t stride, int path,
                                     int mode, const float *age, int64_t n_age, int apply_sigmoid, float *out, void *workspace,
                                     int64_t workspace_bytes, void *stream) {
    return record_score("b2cnn_score_record_ex", h, x, dtype, B, N, pitch, stride, path, mode, age, n_age, apply_sigmoid, out, workspace,
                        workspace_bytes, stream);
}

// ---- host-pointer entry: chunked H2D overlapped with compute -----------------------------
static int ensure_host_staging(b2cnn_handle *h, size_t x_chunk_bytes, int64_t B, size_t ws_bytes) {
    if (!h->s_copy) {
        CU_TRY(cudaStreamCreateWithFlags(&h->s_copy, cudaStreamNonBlocking));
        CU_TRY(cudaStreamCreateWithFlags(&h->s_comp, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            CU_TRY(cudaEventCreateWithFlags(&h->ev_copied[i], cudaEventDisableTiming));
            CU_TRY(cudaEventCreateWithFlags(&h->ev_done[i], cudaEventDisableTiming));
        }
    }
    if (x_chunk_bytes > h->st_x_bytes) {
        for (int i = 0; i < 2; ++i) { cudaFree(h->st_x[i]); h->st_x[i] = nullptr; CU_TRY(cudaMalloc(&h->st_x[i], x_chunk_bytes)); }
        h->st_x_bytes = x_chunk_bytes;
    }
    if ((size_t)B > h->st_vec_elems) {
        cudaFree(h->st_age); cudaFree(h->st_out); h->st_age = h->st_out = nullptr;
        CU_TRY(cudaMalloc(&h->st_age, sizeof(float) * B));
        CU_TRY(cudaMalloc(&h->st_out, sizeof(float) * B));
        h->st_vec_elems = (size_t)B;
    }
    if (ws_bytes > h->st_ws_bytes) {
        cudaFree(h->st_ws); h->st_ws = nullptr;
        CU_TRY(cudaMalloc(&h->st_ws, ws_bytes));
        h->st_ws_bytes = ws_bytes;
    }
    return B2CNN_OK;
}

extern "C" int b2cnn_forward_host(b2cnn_handle *h, const void *x_host, int dtype, int64_t B, const float *age_host,
                                  int64_t n_age, int mode, int apply_sigmoid, float *out_host) {
    int rc = check_call(h, x_host, dtype, B, age_host, n_age, mode, out_host);
    if (rc) return rc;
    DEVICE_GUARD(h->device);
    const Dims &d = h->d;
    const size_t esz = dtype == B2CNN_DTYPE_BF16 ? 2 : 4;
    const size_t win_bytes = (size_t)d.C * d.W * esz;
    // independent windows: stream in chunks of ~64 MiB; a sequence scan needs the whole batch.
    int64_t chunk = B;
    if (mode == B2CNN_MODE_INDEPENDENT) {
        chunk = (int64_t)((64u << 20) / win_bytes);
        if (chunk < 1) chunk = 1;
        if (chunk > B) chunk = B;
    }
    const int64_t ws_bytes = b2cnn_workspace_bytes_for(h, chunk, mode, dtype);
    rc = ensure_host_staging(h, (size_t)chunk * win_bytes, B, (size_t)ws_bytes);
    if (rc) return rc;
    CU_TRY(cudaMemcpyAsync(h->st_age, age_host, sizeof(float) * n_age, cudaMemcpyHostToDevice, h->s_copy));
    int64_t launches = 0;
    int idx = 0;
    for (int64_t b0 = 0; b0 < B; b0 += chunk, ++idx) {
        const int64_t nb = (B - b0 < chunk) ? (B - b0) : chunk;
        const int s = idx & 1;
        if (idx >= 2) CU_TRY(cudaStreamWaitEvent(h->s_copy, h->ev_done[s], 0));
        CU_TRY(cudaMemcpyAsync(h->st_x[s], (const char *)x_host + (size_t)b0 * win_bytes, (size_t)nb * win_bytes,
                               cudaMemcpyHostToDevice, h->s_copy));
        CU_TRY(cudaEventRecord(h->ev_copied[s], h->s_copy));
        CU_TRY(cudaStreamWaitEvent(h->s_comp, h->ev_copied[s], 0));
        rc = forward_device(h, h->st_x[s], dtype, nb, d.W, n_age == 1 ? h->st_age : h->st_age + b0, n_age == 1 ? 1 : nb, mode,
                            apply_sigmoid, h->st_out + b0, h->st_ws, ws_bytes, h->s_comp);
        if (rc) return rc;
        launches += h->last_launches;
        CU_TRY(cudaEventRecord(h->ev_done[s], h->s_comp));
    }
    CU_TRY(cudaMemcpyAsync(out_host, h->st_out, sizeof(float) * B, cudaMemcpyDeviceToHost, h->s_comp));
    CU_TRY(cudaStreamSynchronize(h->s_comp));
    CU_TRY(cudaStreamSynchronize(h->s_copy));
    h->last_launches = launches;
    return B2CNN_OK;
}

extern "C" int b2cnn_set_option(b2cnn_handle *h, const char *key, int64_t value) {
    if (!h || !key) return fail(B2CNN_EINVAL, "b2cnn_set_option: null argument");
    if (!strcmp(key, "path")) {
        if (value < 0 || value > 2) return fail(B2CNN_EINVAL, "path must be 0 (auto), 1 (generic) or 2 (tensorcore)");
        h->opt_path = value;
        return B2CNN_OK;
    }
    if (!strcmp(key, "small_kernel")) { h->opt_small = value ? 1 : 0; return B2CNN_OK; }
    if (!strcmp(key, "tc_fused")) { h->opt_tc_fused = value ? 1 : 0; return B2CNN_OK; }
    if (!strcmp(key, "profile")) { h->opt_profile = value ? 1 : 0; h->ev_valid = false; return B2CNN_OK; }
    if (!strcmp(key, "tc_splits")) {
        if (value != 2 && value != 3) return fail(B2CNN_EINVAL, "tc_splits must be 2 or 3");
        if (h->weights_set && value != h->opt_tc_splits) return fail(B2CNN_ESTATE, "set tc_splits before b2cnn_set_weights");
        h->opt_tc_splits = value;
        return B2CNN_OK;
    }
    return fail(B2CNN_EINVAL, std::string("unknown option: ") + key);
}

extern "C" int64_t b2cnn_get_option(b2cnn_handle *h, const char *key) {
    if (!h || !key) return -1;
    if (!strcmp(key, "path")) return h->opt_path;
    if (!strcmp(key, "tc_splits")) return h->opt_tc_splits;
    if (!strcmp(key, "num_sms")) return h->num_sms;
    if (!strcmp(key, "profile")) return h->opt_profile;
    if (!strcmp(key, "tc_available")) return h->tc.features || (h->tc.fused && h->opt_tc_fused) ? 1 : 0;   // for bf16 windows
    return -1;
}

extern "C" int64_t b2cnn_last_launch_count(b2cnn_handle *h) { return h ? h->last_launches : -1; }
extern "C" int b2cnn_last_path(b2cnn_handle *h) { return h ? h->last_path : -1; }

extern "C" double b2cnn_last_stage_ms(b2cnn_handle *h, int stage) {
    if (!h || !h->ev_valid || stage < 0 || stage > 1) return -1.0;
    if (cudaEventSynchronize(h->ev_stage[stage + 1]) != cudaSuccess) return -1.0;
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, h->ev_stage[stage], h->ev_stage[stage + 1]) != cudaSuccess) return -1.0;
    return (double)ms;
}

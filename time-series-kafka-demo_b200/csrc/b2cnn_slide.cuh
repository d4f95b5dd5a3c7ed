// b2cnn_slide.cuh -- interface of the sliding-window scorer, b2cnn_slide.cu (b2cnn_slide_* in include/b2cnn.h).
#pragma once
#include "b2cnn_tc.cuh"

namespace b2cnn {

struct Slide;
// `d`: the model's geometry; the scorer keeps a copy.  Checks stride and geometry, allocates all device state.  path:
// B2CNN_PATH_TENSORCORE (the geometries `tc` holds in its streaming kernels, else B2CNN_EARCH) or B2CNN_PATH_GENERIC
// (exact CUDA-core kernels for any geometry b2cnn_create accepts; B2CNN_EARCH, before allocating anything, where the
// generic front end's tile does not fit shared memory, with num_sms sizing its grid); stride % pool_s^2 == 0
// mode: B2CNN_MODE_INDEPENDENT, or B2CNN_MODE_SEQUENCE (each patient's LSTM state [64] fp32 on the device, carried
// from push to push; zeroed at reset, admit, discharge and an import without state); anything else B2CNN_EINVAL
int slide_create(const Dims &d, const TcState &tc, int path, int mode, int n_patients, int stride, int dtype, int device, int num_sms,
                 Slide **out, const char **err);
int slide_path(const Slide *s);   // B2CNN_PATH_TENSORCORE or B2CNN_PATH_GENERIC
int slide_mode(const Slide *s);   // B2CNN_MODE_INDEPENDENT or B2CNN_MODE_SEQUENCE
void slide_destroy(Slide *s);
int slide_device(const Slide *s);
int slide_reset(Slide *s, cudaStream_t st, const char **err);
// ev: nullptr, or three events recorded at the start, after the front end and after the head (profiling).
// heads: out is [1 + slide_n_heads][P], row 0 the model's logits as without, row i those of head i - 1.
int slide_push(Slide *s, const ConvWeights &cw, const HeadWeights &hw, const TcState &tc, const void *x, int64_t pitch,
               const float *age, int64_t n_age, int apply_sigmoid, float *out, bool heads, int *emitted, int64_t *window_index,
               cudaEvent_t *ev, cudaStream_t st, const char **err);
// extra heads (b2cnn_slide_set_heads): what a head is copied from -- a handle of the same architecture and front end,
// its window W <= the scorer's with (scorer W - W) % F == 0 and L = L_out(W) (checked by the caller)
struct SlideHeadSource {
    HeadWeights hw;                  // the handle's pointers into its blob and its W_ih^T [L][64]
    const TcState *tc;               // its packed W_ih chunks (tensor-core path)
    float age_coef;
    uint64_t digest;                 // its front-end digest
    int W, L;                        // its window and feature count
};
// replaces the heads with copies of src[0 .. n) (allocated and copied here, the stream synchronised); on failure the
// previous heads stay
int slide_set_heads(Slide *s, const SlideHeadSource *src, int n, cudaStream_t st, const char **err);
int slide_n_heads(const Slide *s);
int slide_stale_head(const Slide *s, uint64_t digest);
int slide_features(const Slide *s, float *feats, cudaStream_t st, const char **err);
// per-patient lifecycle: `patients` host indices; `hist` [k][C][pitch] device samples in the scorer's dtype
int64_t slide_admit_workspace_bytes(const Slide *s, int64_t k, int64_t H);
// lstm: nullptr (a sequence-mode scorer's LSTM state rows of the patients are zeroed) or [k][64] device fp32 rows they
// start from (sequence mode only, else B2CNN_EINVAL)
int slide_admit(Slide *s, const ConvWeights &cw, const TcState &tc, const int *patients, int64_t k, const void *hist, int64_t H,
                int64_t pitch, const float *lstm, void *ws, int64_t ws_bytes, cudaStream_t st, const char **err);
int slide_discharge(Slide *s, const int *patients, int64_t k, cudaStream_t st, const char **err);
int slide_samples_seen(Slide *s, int64_t *out, cudaStream_t st, const char **err);
int slide_dtype(const Slide *s);
// export / import of patients (b2cnn_slide_export / _import): `cw` the handle's current conv weights (the digest);
// lstm: nullptr or [k][64] device fp32 LSTM state rows (sequence mode only, else B2CNN_EINVAL); an import into a
// sequence-mode scorer without them zeroes the patients' rows
void slide_describe_state(const Slide *s, const ConvWeights &cw, b2cnn_slide_state_header *out);
int64_t slide_state_workspace_bytes(const Slide *s, int64_t k);
int slide_export(const Slide *s, const ConvWeights &cw, const int *patients, int64_t k, float *feats, float *tails, int64_t *seen_host,
                 float *lstm, b2cnn_slide_state_header *hdr, void *ws, int64_t ws_bytes, cudaStream_t st, const char **err);
int slide_import(Slide *s, const ConvWeights &cw, const int *patients, int64_t k, const b2cnn_slide_state_header &hdr, const float *feats,
                 const float *tails, const int64_t *seen_host, const float *lstm, void *ws, int64_t ws_bytes, cudaStream_t st,
                 const char **err);

}  // namespace b2cnn

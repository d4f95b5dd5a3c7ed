// b2cnn_slide.cuh -- interface of the sliding-window scorer, b2cnn_slide.cu (b2cnn_slide_* in include/b2cnn.h).
#pragma once
#include "b2cnn_tc.cuh"

namespace b2cnn {

struct Slide;
// `d`: the model's geometry; the scorer keeps a copy.  Checks stride and geometry, allocates all device state.
int slide_create(const Dims &d, const TcState &tc, int n_patients, int stride, int dtype, int device, Slide **out,
                 const char **err);
// the generic path: exact CUDA-core kernels for any geometry b2cnn_create accepts (B2CNN_EARCH, before allocating
// anything, where the generic front end's tile does not fit shared memory); stride % pool_s^2 == 0
int slide_create_generic(const Dims &d, int n_patients, int stride, int dtype, int device, int num_sms, Slide **out,
                         const char **err);
int slide_path(const Slide *s);   // B2CNN_PATH_TENSORCORE or B2CNN_PATH_GENERIC
void slide_destroy(Slide *s);
int slide_device(const Slide *s);
int slide_reset(Slide *s, cudaStream_t st, const char **err);
// ev: nullptr, or three events recorded at the start, after the front end and after the head (profiling)
int slide_push(Slide *s, const ConvWeights &cw, const HeadWeights &hw, const TcState &tc, const void *x, int64_t pitch,
               const float *age, int64_t n_age, int apply_sigmoid, float *out, int *emitted, int64_t *window_index,
               cudaEvent_t *ev, cudaStream_t st, const char **err);
int slide_features(const Slide *s, float *feats, cudaStream_t st, const char **err);
// per-patient lifecycle: `patients` host indices; `hist` [k][C][pitch] device samples in the scorer's dtype
int64_t slide_admit_workspace_bytes(const Slide *s, int64_t k, int64_t H);
int slide_admit(Slide *s, const ConvWeights &cw, const TcState &tc, const int *patients, int64_t k, const void *hist, int64_t H,
                int64_t pitch, void *ws, int64_t ws_bytes, cudaStream_t st, const char **err);
int slide_discharge(Slide *s, const int *patients, int64_t k, cudaStream_t st, const char **err);
int slide_samples_seen(Slide *s, int64_t *out, cudaStream_t st, const char **err);
int slide_dtype(const Slide *s);

}  // namespace b2cnn

// b2cnn_prep.cu -- the two steps in FRONT of the model call, on the device (SURVEY.md section 8, f2 + f1):
//
//   f2  bin/processStream.py:196-208  per (patient, signal): mean of the samples of a 180 s window that
//                                     slides by 5 s (Spark `window(...)` + avg: nulls are skipped)
//       bin/processStream.py:62-123   forward-fill, back-fill, then 0-fill of that 5-second grid
//   f1  bin/predictStream.py:245-259  600 s windows sliding by 60 s -> 120 grid points per signal
//       bin/predictStream.py:105-139  x_arr[0, signal_index, :] = the 120 points, absent signals = zeros
//
// Input is one WFDB format-16 numerics record as it lies on disk (interleaved little-endian int16,
// -32768 == missing; physical = (adc - baseline) / gain, bin/sendStream.py:46 via wfdb.rdrecord), output
// is the [n_windows, n_channels, 120] batch the model consumes, written in f32 or bf16 straight into the
// tensor that b2cnn_forward reads -- the Kafka/Spark hop and the per-row numpy assembly disappear for replay.
// All sums are fp64 like Spark's avg, taken directly over the window's samples in time order.  The checker is
// oracle/stream_np.py, itself pinned against pandas (oracle/stream_pandas.py: the reference notebook's own
// resample('5S').first() / rolling('3min').mean(), bin/explore_torch.ipynb:402,405).
//
// Time base and window edges: sample i sits at i * round(1e9 / fs) nanoseconds (integers: edges compare exactly).
// Grid point k (label tau = k * 5 s) is Spark's half-open window [windowStart, windowStart + 180 s) with
// windowStart = tau - 175 s: it averages the valid samples with time in [tau - 175 s, tau + 5 s).  On the 5-second
// lattice (every MIMIC numerics record) that is the sample set of pandas' right-closed (tau - 180 s, tau].
//
// Two forms of the same arithmetic:
//   b2cnn_prep_windows   a whole record at once (replay)
//   b2cnn_ring_*         the streaming form: per-patient device ring buffers; every trigger appends the new samples
//                        of ALL patients, finalises the grid points whose window is complete, and emits one
//                        [n_patients, 10, 120] batch for ONE predict() call (bin/predictStream.py:70-157 is a Python
//                        loop with B = 1 per patient row).  Trigger-by-trigger output == whole-record output bit-for-bit.
// This is byte shuffling around a few thousand samples per signal: launch-latency work, not a roofline kernel.
#include <cuda_bf16.h>

#include <cmath>

#include "b2cnn_internal.cuh"

namespace b2cnn {

constexpr int kPrepThreads = 1024;

struct PrepDims {
    int64_t n_samples, n_grid, n_windows;
    int n_sig, n_sel, n_channels, window_points, step;
    int64_t period_ns, grid_ns, smooth_ns;
    double grid_s;
};

struct PrepSignals {            // per selected signal: column in the record, gain, baseline
    int col[16];
    double gain[16], baseline[16];
};

__device__ __forceinline__ double phys_value(const int16_t *raw, int64_t i, int n_sig, int col, double gain, double base,
                                             bool *ok) {
    const int16_t a = raw[i * n_sig + col];
    *ok = a != (int16_t)-32768;
    return ((double)a - base) / gain;
}

// number of sample times t_i = i * period_ns (0 <= i < n) that are < v_ns  (numpy.searchsorted(t, v, side="left"))
__host__ __device__ __forceinline__ int64_t count_lt(int64_t n, int64_t period_ns, int64_t v_ns) {
    if (v_ns <= 0) return 0;
    const int64_t c = (v_ns + period_ns - 1) / period_ns;
    return c < n ? c : n;
}

// grid value k of signal ch: mean of the valid samples with time in [tau - smooth + grid, tau + grid), tau = k * grid.
// The window's samples are summed directly, in time order (what Spark's avg over the window rows does); a
// prefix-sum difference would leave cancellation residue (1e-12 instead of an exact 0 for an all-zero window).
__global__ void prep_grid_kernel(const int16_t *__restrict__ raw, PrepDims d, PrepSignals sg, double *__restrict__ grid) {
    const int ch = blockIdx.y;
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= d.n_grid) return;
    const int64_t tau = k * d.grid_ns;
    const int64_t lo = count_lt(d.n_samples, d.period_ns, tau - d.smooth_ns + d.grid_ns);
    const int64_t hi = count_lt(d.n_samples, d.period_ns, tau + d.grid_ns);
    const int col = sg.col[ch];
    const double gain = sg.gain[ch], base = sg.baseline[ch];
    double s = 0.0; int cnt = 0;
    for (int64_t i = lo; i < hi; ++i) {
        bool ok;
        const double v = phys_value(raw, i, d.n_sig, col, gain, base, &ok);
        if (ok) { s += v; ++cnt; }
    }
    grid[(int64_t)ch * d.n_grid + k] = cnt > 0 ? s / (double)cnt : nan("");
}

// one CTA per signal: forward fill (last valid value), back fill of the leading gap, zeros if nothing is valid
__global__ void __launch_bounds__(kPrepThreads)
prep_fill_kernel(PrepDims d, double *__restrict__ grid) {
    __shared__ long long sh_last[kPrepThreads];
    __shared__ long long sh_first;                                // first valid index of the signal (n_grid: none)
    const int ch = blockIdx.x, tid = threadIdx.x;
    double *g = grid + (int64_t)ch * d.n_grid;
    const int64_t per = (d.n_grid + kPrepThreads - 1) / kPrepThreads;
    const int64_t k0 = (int64_t)tid * per, k1 = min(k0 + per, d.n_grid);
    if (tid == 0) sh_first = (long long)d.n_grid;
    __syncthreads();
    long long last = -1, first_here = (long long)d.n_grid;
    for (int64_t k = k0; k < k1; ++k)
        if (g[k] == g[k]) { last = k; if (first_here > k) first_here = k; }
    sh_last[tid] = last;
    if (first_here < (long long)d.n_grid) atomicMin(&sh_first, first_here);
    __syncthreads();
    for (int off = 1; off < kPrepThreads; off <<= 1) {           // inclusive max-scan of the chunk results
        long long v = -1;
        if (tid >= off) v = sh_last[tid - off];
        __syncthreads();
        if (tid >= off && v > sh_last[tid]) sh_last[tid] = v;
        __syncthreads();
    }
    long long carry = tid > 0 ? sh_last[tid - 1] : -1;            // last valid index before this chunk
    const long long first = sh_first;
    const double first_val = first < (long long)d.n_grid ? g[first] : 0.0;
    // Values are read before any thread of this chunk overwrites them: a chunk only writes its own range and
    // reads g[carry] from an EARLIER chunk's last valid entry, which that chunk leaves unchanged (valid stays).
    const double carry_val = carry >= 0 ? g[carry] : 0.0;
    __syncthreads();
    double cur = carry_val; bool have = carry >= 0;
    for (int64_t k = k0; k < k1; ++k) {
        const double v = g[k];
        if (v == v) { cur = v; have = true; }
        else g[k] = have ? cur : first_val;                      // leading gap: back fill (or 0 when all missing)
    }
}

template <typename Tout>
__device__ __forceinline__ Tout cast_out(double v);
template <>
__device__ __forceinline__ float cast_out<float>(double v) { return (float)v; }                   // predictStream.py:155 .float()
template <>
__device__ __forceinline__ __nv_bfloat16 cast_out<__nv_bfloat16>(double v) { return __float2bfloat16_rn((float)v); }

// x[w][c][p] = grid[c][w * step + p] for the signals the record has, zeros for the rest (predictStream.py:131)
template <typename Tout>
__global__ void prep_assemble_kernel(PrepDims d, const double *__restrict__ grid, Tout *__restrict__ x, double *__restrict__ t0) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t per_w = (int64_t)d.n_channels * d.window_points;
    if (e >= d.n_windows * per_w) return;
    const int64_t w = e / per_w;
    const int r = (int)(e - w * per_w);
    const int c = r / d.window_points, pnt = r - c * d.window_points;
    double v = 0.0;
    if (c < d.n_sel) v = grid[(int64_t)c * d.n_grid + w * d.step + pnt];
    x[e] = cast_out<Tout>(v);
    if (t0 && r == 0) t0[w] = (double)(w * d.step) * d.grid_s;
}

static bool prep_dims(int64_t n_samples, int n_sig, int n_sel, double fs, const b2cnn_prep_config *cfg, PrepDims *d, const char **err) {
    if (!cfg || n_samples < 1 || n_sig < 1 || n_sig > 64 || n_sel < 0 || n_sel > 16 || !(fs > 0.0)) { *err = "bad record shape"; return false; }
    if (cfg->n_channels < 1 || cfg->n_channels > 16 || n_sel > cfg->n_channels || cfg->window_points < 1 || cfg->grid_s < 1 ||
        cfg->smooth_s < 1 || cfg->stride_s < cfg->grid_s || cfg->stride_s % cfg->grid_s) { *err = "bad preprocessing configuration"; return false; }
    d->n_samples = n_samples; d->n_sig = n_sig; d->n_sel = n_sel;
    d->n_channels = cfg->n_channels; d->window_points = cfg->window_points; d->step = cfg->stride_s / cfg->grid_s;
    d->period_ns = llround(1e9 / fs); d->grid_s = (double)cfg->grid_s;
    d->grid_ns = (int64_t)cfg->grid_s * 1000000000ll; d->smooth_ns = (int64_t)cfg->smooth_s * 1000000000ll;
    if (d->period_ns < 1 || cfg->smooth_s < cfg->grid_s) { *err = "bad sampling rate / smoothing window"; return false; }
    d->n_grid = ((n_samples - 1) * d->period_ns) / d->grid_ns + 1;
    const int64_t span = d->n_grid - d->window_points + 1;
    d->n_windows = span > 0 ? (span + d->step - 1) / d->step : 0;
    return true;
}

int64_t prep_window_count(int64_t n_samples, double fs, const b2cnn_prep_config *cfg) {
    PrepDims d; const char *e = "";
    if (!prep_dims(n_samples, 1, 0, fs, cfg, &d, &e)) return -1;
    return d.n_windows;
}

static int64_t align256(int64_t v) { return (v + 255) / 256 * 256; }

int64_t prep_workspace_bytes(int64_t n_samples, double fs, int n_sel, const b2cnn_prep_config *cfg) {
    PrepDims d; const char *e = "";
    if (!prep_dims(n_samples, 1, n_sel, fs, cfg, &d, &e)) return -1;
    const int64_t ns = n_sel > 0 ? n_sel : 1;
    return align256(ns * d.n_grid * 8);                        // the 5-second grid of every selected signal, fp64
}

int prep_windows(const int16_t *raw, int64_t n_samples, int n_sig, const int *sel, int n_sel, const double *gains,
                 const double *baselines, double fs, const b2cnn_prep_config *cfg, void *x_out, int dtype, double *t0_out,
                 void *workspace, int64_t ws_bytes, cudaStream_t st, const char **err) {
    PrepDims d;
    if (!prep_dims(n_samples, n_sig, n_sel, fs, cfg, &d, err)) return B2CNN_EINVAL;
    if (!raw || !x_out || (n_sel > 0 && (!sel || !gains || !baselines))) { *err = "null pointer"; return B2CNN_EINVAL; }
    if (dtype != B2CNN_DTYPE_F32 && dtype != B2CNN_DTYPE_BF16) { *err = "dtype must be f32 or bf16"; return B2CNN_EINVAL; }
    if (ws_bytes < prep_workspace_bytes(n_samples, fs, n_sel, cfg) || !workspace) { *err = "workspace too small (b2cnn_prep_workspace_bytes)"; return B2CNN_ESTATE; }
    if (d.n_windows == 0) return B2CNN_OK;
    PrepSignals sg;
    for (int i = 0; i < n_sel; ++i) {
        if (sel[i] < 0 || sel[i] >= n_sig || !(gains[sel[i]] != 0.0)) { *err = "bad signal selection / zero gain"; return B2CNN_EINVAL; }
        sg.col[i] = sel[i]; sg.gain[i] = gains[sel[i]]; sg.baseline[i] = baselines[sel[i]];
    }
    double *grid = reinterpret_cast<double *>(workspace);
    if (n_sel > 0) {
        dim3 gg((unsigned)((d.n_grid + 255) / 256), n_sel);
        prep_grid_kernel<<<gg, 256, 0, st>>>(raw, d, sg, grid);
        prep_fill_kernel<<<n_sel, kPrepThreads, 0, st>>>(d, grid);
    }
    const int64_t total = d.n_windows * d.n_channels * d.window_points;
    const unsigned nb = (unsigned)((total + 255) / 256);
    if (dtype == B2CNN_DTYPE_F32)
        prep_assemble_kernel<float><<<nb, 256, 0, st>>>(d, grid, reinterpret_cast<float *>(x_out), t0_out);
    else
        prep_assemble_kernel<__nv_bfloat16><<<nb, 256, 0, st>>>(d, grid, reinterpret_cast<__nv_bfloat16 *>(x_out), t0_out);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return B2CNN_ECUDA; }
    return B2CNN_OK;
}

// ------------------------------------------------------------------------------------------------------------
// Streaming form: per-patient device ring buffers (SURVEY.md section 8, row f1 as written).
//
// State per patient (device memory, owned by the ring):
//   samples  [R][n_sig] fp64 physical values (NaN = missing), a circular buffer over the absolute sample index:
//            the last ~185 s + one trigger of samples, i.e. everything a not-yet-final grid point can still need
//   grid     [n_channels][G] fp64, circular over the absolute grid index k: forward-filled values; the leading gap
//            (nothing valid yet) is kept as NaN and resolved at emit time
//   last / first [n_channels]: forward-fill carry and the first valid value (back-fill of the leading gap)
// A grid point is FINAL once no future sample can fall into its window: tau + 5 s <= t_next (the time of the next,
// not yet received sample).  Window w = grid points 12w .. 12w + 119 is emitted by the push that finalises its last
// point.  All patients of a ring share the sampling rate and receive the same number of samples per push, so the
// bookkeeping (counts, indices) is host-side scalar arithmetic; the device holds data only.
// Differences from a whole-record pass are confined to what a causal stream cannot know: a leading gap longer than
// the first window is emitted as zeros (the reference's per-micro-batch fillna(0), bin/processStream.py:123) instead
// of being back-filled from the future.
// ------------------------------------------------------------------------------------------------------------
constexpr int kRingMaxNewPts = 64;      // grid points one push may finalise (a trigger finalises 12)
constexpr int kRingGrid = 256;          // grid ring capacity (>= window_points + kRingMaxNewPts)

struct RingPush {
    double *samples, *grid, *last, *first;      // ring state (see above)
    const int *col; const double *gain, *base; const int *n_sel;   // [P][16] signal selection per patient
    const void *in;                             // new samples [P][n_new][n_sig]: int16 ADC units or fp64 physical,
    int in_is_adc, in_is_grid;                  // or (in_is_grid) fp64 grid points that are already smoothed and filled
    int64_t N0, n_new, R;                       // samples before this push, new samples, sample-ring capacity
    int64_t k0; int n_pts;                      // first new grid index, number of grid points finalised by this push
    int64_t period_ns, grid_ns, smooth_ns;
    int n_sig, n_channels, window_points;
    int64_t emit_k;                             // first grid index of the window to emit, or -1
    void *x_out; int out_bf16;                  // [P][n_channels][window_points]
};

__global__ void __launch_bounds__(256)
ring_push_kernel(RingPush a) {
    __shared__ double s_pts[16][kRingMaxNewPts];
    const int p = blockIdx.x, tid = threadIdx.x;
    double *smp = a.samples + (int64_t)p * a.R * a.n_sig;
    double *grid = a.grid + (int64_t)p * a.n_channels * kRingGrid;
    const int nsel = a.n_sel[p];
    if (a.in_is_grid) {
        // bin/processStream.py already did the smoothing and the fills: the points go straight into the grid ring
        const double *in = reinterpret_cast<const double *>(a.in) + (int64_t)p * a.n_new * a.n_sig;
        for (int e = tid; e < nsel * a.n_pts; e += blockDim.x) {
            const int c = e / a.n_pts, q = e - c * a.n_pts;
            grid[c * kRingGrid + (int)((a.k0 + q) % kRingGrid)] = in[(int64_t)q * a.n_sig + a.col[p * 16 + c]];
        }
        __syncthreads();
    }
    // ---- 1. the new samples -> physical values -> sample ring
    if (!a.in_is_grid)
    for (int64_t e = tid; e < a.n_new * a.n_sig; e += blockDim.x) {
        const int64_t i = e / a.n_sig; const int sg = (int)(e - i * a.n_sig);
        double v;
        if (a.in_is_adc) {
            const int16_t adc = reinterpret_cast<const int16_t *>(a.in)[((int64_t)p * a.n_new + i) * a.n_sig + sg];
            v = (double)adc;                                          // converted per selected channel below (gain / baseline)
            if (adc == (int16_t)-32768) v = nan("");
        } else {
            v = reinterpret_cast<const double *>(a.in)[((int64_t)p * a.n_new + i) * a.n_sig + sg];
        }
        smp[((a.N0 + i) % a.R) * a.n_sig + sg] = v;
    }
    __syncthreads();
    // ---- 2. the grid points this push finalises: direct window sums in time order (as prep_grid_kernel)
    const int64_t N1 = a.N0 + a.n_new;
    if (!a.in_is_grid)
    for (int e = tid; e < nsel * a.n_pts; e += blockDim.x) {
        const int c = e / a.n_pts, q = e - c * a.n_pts;
        const int64_t tau = (a.k0 + q) * a.grid_ns;
        const int64_t lo = count_lt(N1, a.period_ns, tau - a.smooth_ns + a.grid_ns);
        const int64_t hi = count_lt(N1, a.period_ns, tau + a.grid_ns);
        const int col = a.col[p * 16 + c];
        const double gain = a.gain[p * 16 + c], base = a.base[p * 16 + c];
        double sum = 0.0; int cnt = 0;
        for (int64_t i = lo; i < hi; ++i) {
            double v = smp[(i % a.R) * a.n_sig + col];
            if (v == v) { if (a.in_is_adc) v = (v - base) / gain; sum += v; ++cnt; }
        }
        s_pts[c][q] = cnt > 0 ? sum / (double)cnt : nan("");
    }
    __syncthreads();
    // ---- 3. forward fill across pushes (one thread per channel, sequential over <= 64 points)
    if (!a.in_is_grid && tid < nsel) {
        double last = a.last[p * 16 + tid], first = a.first[p * 16 + tid];
        for (int q = 0; q < a.n_pts; ++q) {
            double v = s_pts[tid][q];
            if (v == v) { last = v; if (first != first) first = v; } else v = last;
            grid[tid * kRingGrid + (int)((a.k0 + q) % kRingGrid)] = v;
        }
        a.last[p * 16 + tid] = last; a.first[p * 16 + tid] = first;
    }
    __syncthreads();
    // ---- 4. the 600 s window that just completed -> x_out[p] (absent signals: zeros, predictStream.py:131)
    if (a.emit_k >= 0) {
        const int per = a.n_channels * a.window_points;
        for (int e = tid; e < per; e += blockDim.x) {
            const int c = e / a.window_points, j = e - c * a.window_points;
            double v = 0.0;
            if (c < nsel) {
                v = grid[c * kRingGrid + (int)((a.emit_k + j) % kRingGrid)];
                if (v != v) { const double f = a.first[p * 16 + c]; v = f == f ? f : 0.0; }   // leading gap: back fill, else 0
            }
            const int64_t o = (int64_t)p * per + e;
            if (a.out_bf16) reinterpret_cast<__nv_bfloat16 *>(a.x_out)[o] = cast_out<__nv_bfloat16>(v);
            else reinterpret_cast<float *>(a.x_out)[o] = cast_out<float>(v);
        }
    }
}

__global__ void ring_fill_nan_kernel(double *p, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = nan("");
}

struct Ring {
    b2cnn_prep_config cfg;
    int n_patients = 0, n_sig = 0, device = 0;
    int64_t period_ns = 0, grid_ns = 0, smooth_ns = 0, R = 0;
    int64_t n_samples = 0, k_done = 0, w_next = 0;
    double *d_samples = nullptr, *d_grid = nullptr, *d_last = nullptr, *d_first = nullptr, *d_gain = nullptr, *d_base = nullptr;
    int *d_col = nullptr, *d_nsel = nullptr;
};

int ring_create(const b2cnn_prep_config *cfg, int n_patients, int n_sig, double fs, int device, Ring **out, const char **err) {
    PrepDims d;
    if (!prep_dims(1, n_sig, 0, fs, cfg, &d, err)) return B2CNN_EINVAL;
    if (n_patients < 1 || n_patients > (1 << 20)) { *err = "n_patients out of range"; return B2CNN_EINVAL; }
    if (cfg->window_points + kRingMaxNewPts > kRingGrid) { *err = "window_points too large for the grid ring"; return B2CNN_EINVAL; }
    const int64_t stride_ns = (int64_t)cfg->stride_s * 1000000000ll;
    // a single sample must not complete two windows, or no push schedule could keep to one window per push
    if (d.period_ns > stride_ns) { *err = "sampling period longer than the stride"; return B2CNN_EINVAL; }
    Ring *r = new Ring();
    r->cfg = *cfg; r->n_patients = n_patients; r->n_sig = n_sig; r->device = device;
    r->period_ns = d.period_ns; r->grid_ns = d.grid_ns; r->smooth_ns = d.smooth_ns;
    const int64_t max_new = stride_ns / d.period_ns + 2;
    r->R = (d.smooth_ns + 2 * d.grid_ns) / d.period_ns + max_new + 4;
    const int64_t P = n_patients;
    cudaError_t e = cudaMalloc(&r->d_samples, sizeof(double) * P * r->R * n_sig);
    if (e == cudaSuccess) e = cudaMalloc(&r->d_grid, sizeof(double) * P * cfg->n_channels * kRingGrid);
    if (e == cudaSuccess) e = cudaMalloc(&r->d_last, sizeof(double) * P * 16);
    if (e == cudaSuccess) e = cudaMalloc(&r->d_first, sizeof(double) * P * 16);
    if (e == cudaSuccess) e = cudaMalloc(&r->d_gain, sizeof(double) * P * 16);
    if (e == cudaSuccess) e = cudaMalloc(&r->d_base, sizeof(double) * P * 16);
    if (e == cudaSuccess) e = cudaMalloc(&r->d_col, sizeof(int) * P * 16);
    if (e == cudaSuccess) e = cudaMalloc(&r->d_nsel, sizeof(int) * P);
    if (e == cudaSuccess) e = cudaMemset(r->d_nsel, 0, sizeof(int) * P);
    if (e == cudaSuccess) e = cudaMemset(r->d_col, 0, sizeof(int) * P * 16);
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); ring_destroy(r); return B2CNN_ECUDA; }
    *out = r;
    return ring_reset(r, nullptr, err);
}

void ring_destroy(Ring *r) {
    if (!r) return;
    cudaFree(r->d_samples); cudaFree(r->d_grid); cudaFree(r->d_last); cudaFree(r->d_first);
    cudaFree(r->d_gain); cudaFree(r->d_base); cudaFree(r->d_col); cudaFree(r->d_nsel);
    delete r;
}

int ring_device(const Ring *r) { return r->device; }

int ring_reset(Ring *r, cudaStream_t st, const char **err) {
    r->n_samples = r->k_done = r->w_next = 0;
    const int64_t n = (int64_t)r->n_patients * 16;
    ring_fill_nan_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(r->d_last, n);
    ring_fill_nan_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(r->d_first, n);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return B2CNN_ECUDA; }
    return B2CNN_OK;
}

int ring_set_signals(Ring *r, int patient, const int *sel, int n_sel, const double *gains, const double *baselines,
                     cudaStream_t st, const char **err) {
    if (patient < 0 || patient >= r->n_patients || n_sel < 0 || n_sel > 16 || n_sel > r->cfg.n_channels ||
        (n_sel > 0 && !sel)) { *err = "bad patient index / signal selection"; return B2CNN_EINVAL; }
    int col[16] = {0}; double gain[16], base[16];
    for (int i = 0; i < 16; ++i) { gain[i] = 1.0; base[i] = 0.0; }
    for (int i = 0; i < n_sel; ++i) {
        if (sel[i] < 0 || sel[i] >= r->n_sig) { *err = "signal column out of range"; return B2CNN_EINVAL; }
        col[i] = sel[i];
        if (gains) { if (!(gains[sel[i]] != 0.0)) { *err = "zero gain"; return B2CNN_EINVAL; } gain[i] = gains[sel[i]]; }
        if (baselines) base[i] = baselines[sel[i]];
    }
    cudaError_t e = cudaMemcpyAsync(r->d_col + patient * 16, col, sizeof col, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(r->d_gain + patient * 16, gain, sizeof gain, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(r->d_base + patient * 16, base, sizeof base, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(r->d_nsel + patient, &n_sel, sizeof(int), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);           // the host arrays above are stack memory
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return B2CNN_ECUDA; }
    return B2CNN_OK;
}

// One trigger.  Returns B2CNN_OK; *emitted = 1 when x_out[n_patients][n_channels][window_points] was written (window index
// *window_out, start time *t0_out seconds), 0 while the first 600 s are still filling.
int ring_push(Ring *r, const void *new_samples, int sample_kind, int64_t n_new, void *x_out, int dtype, int *emitted,
              int64_t *window_out, double *t0_out, cudaStream_t st, const char **err) {
    if (!new_samples || !x_out || !emitted || n_new < 1) { *err = "null pointer / n_new < 1"; return B2CNN_EINVAL; }
    if (dtype != B2CNN_DTYPE_F32 && dtype != B2CNN_DTYPE_BF16) { *err = "dtype must be f32 or bf16"; return B2CNN_EINVAL; }
    const bool is_grid = sample_kind == B2CNN_SAMPLES_GRID;
    const int in_is_adc = sample_kind == B2CNN_SAMPLES_ADC16;
    const int64_t N1 = is_grid ? r->n_samples : r->n_samples + n_new;
    const int64_t t_next = N1 * r->period_ns;                        // time of the first sample NOT yet received
    const int64_t k_end = is_grid ? r->k_done + n_new : t_next / r->grid_ns;   // grid points 0 .. k_end-1 are final
    const int64_t n_pts = k_end - r->k_done;
    const int step = r->cfg.stride_s / r->cfg.grid_s;
    if (n_pts > kRingMaxNewPts || (is_grid && n_new > step) ||
        (!is_grid && n_new * r->period_ns > (int64_t)r->cfg.stride_s * 1000000000ll + r->period_ns)) {
        *err = "one push may carry at most stride_s seconds of samples / grid points"; return B2CNN_EINVAL;
    }
    // One push emits at most one window.  A push that would also complete the window after the one it emits would leave
    // a backlog, and a backlog that outgrows the grid ring is read back from overwritten slots: refuse it, state unchanged.
    const int64_t w_last_k = r->w_next * step + r->cfg.window_points - 1;
    if (w_last_k + step <= k_end - 1) {
        *err = "push would complete two windows: one push may finalise at most one window (cut pushes at stride boundaries)";
        return B2CNN_EINVAL;
    }
    const bool emit = w_last_k <= k_end - 1;
    RingPush a;
    a.samples = r->d_samples; a.grid = r->d_grid; a.last = r->d_last; a.first = r->d_first;
    a.col = r->d_col; a.gain = r->d_gain; a.base = r->d_base; a.n_sel = r->d_nsel;
    a.in = new_samples; a.in_is_adc = in_is_adc; a.in_is_grid = is_grid ? 1 : 0; a.N0 = r->n_samples; a.n_new = n_new; a.R = r->R;
    a.k0 = r->k_done; a.n_pts = (int)n_pts;
    a.period_ns = r->period_ns; a.grid_ns = r->grid_ns; a.smooth_ns = r->smooth_ns;
    a.n_sig = r->n_sig; a.n_channels = r->cfg.n_channels; a.window_points = r->cfg.window_points;
    a.emit_k = emit ? r->w_next * step : -1;
    a.x_out = x_out; a.out_bf16 = dtype == B2CNN_DTYPE_BF16;
    ring_push_kernel<<<r->n_patients, 256, 0, st>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return B2CNN_ECUDA; }
    *emitted = emit ? 1 : 0;
    if (emit) {
        if (window_out) *window_out = r->w_next;
        if (t0_out) *t0_out = (double)(r->w_next * step) * (double)r->cfg.grid_s;
        ++r->w_next;
    }
    r->n_samples = N1; r->k_done = k_end;
    return B2CNN_OK;
}

}  // namespace b2cnn

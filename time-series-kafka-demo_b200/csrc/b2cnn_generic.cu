// b2cnn_generic.cu -- exact-fp32 CUDA-core front end:
//   conv1 + act + pool -> conv2 + act + pool -> feature rows   (bin/models.py:23-29)
// for any (C, K1, K2, pool_k, pool_s, W) and f32 or bf16 input.  This is the path every shape
// can take (production [1,10,120], the older checkpoints, fp32 inputs, odd window lengths)
// and the exact re-computation path behind the tensor-core kernel (b2cnn_tc.cu).
//
// Work decomposition: CTA = (tile of `tile_p` final positions) x (strided loop over windows).
// Per window-tile, three block-synchronous stages through shared memory:
//   1. stage the C x ni input samples of the tile's receptive field as fp32
//   2. conv1 in registers: each thread owns RUN consecutive pooled outputs x 4 channels, i.e.
//      NT1 = PS*(RUN-1)+PK conv1 positions slid over a register window of the input; pooling
//      happens BEFORE the activation (max commutes with +bias and with monotone tanh/relu),
//      halving the transcendental count; NaNs propagate (max.NaN) like ATen's max_pool1d
//   3. conv2 + pool + act, two final positions per thread, written straight to global
// Shared-memory rows use padi() (one pad word per 32) so that "thread r reads a window at
// stride 4 or 8" is bank-conflict free.
#include "b2cnn_internal.cuh"

namespace b2cnn {

template <typename T>
__device__ __forceinline__ float ld_in(const T *p);
template <>
__device__ __forceinline__ float ld_in<float>(const float *p) {
    return __ldg(p);
}
template <>
__device__ __forceinline__ float ld_in<__nv_bfloat16>(const __nv_bfloat16 *p) {
    return __bfloat162float(__ldg(p));
}

__device__ __forceinline__ float conv_epilogue(float v, float bias, float s, float t, int has_affine) {
    v += bias;
    return has_affine ? fmaf(v, s, t) : v;
}

// ------------------------------------------------------------------------------------------
// Templated kernel: K1/K2/PK/PS (and optionally C) are compile-time so the FMA loops unroll and
// the conv weights become constant-bank immediates.
// ------------------------------------------------------------------------------------------
template <int CT, int K1, int K2, int PK, int PS, int RUN, typename Tin>
__global__ void __launch_bounds__(256, 2) frontend_kernel(const __grid_constant__ FrontParams p) {
    extern __shared__ float smem[];
    const int C = CT > 0 ? CT : p.d.C;
    float *xs = smem;
    float *a1 = smem + C * p.xs_stride;
    constexpr int NT1 = PS * (RUN - 1) + PK;   // conv1 positions per thread-run
    constexpr int NX = NT1 + K1 - 1;           // input samples per thread-run and channel
    constexpr int NQ = PS + PK;                // conv2 outputs for two final positions
    constexpr int NA = NQ + K2 - 1;
    const int tid = threadIdx.x;
    const int act = p.d.act, aff = p.d.has_affine;
    const bool gate_mode = p.gate_part != nullptr;
    __shared__ float gred[4][kGates];
    const int tile_lo = gate_mode ? blockIdx.x * p.tiles_per_slice : blockIdx.x;
    const int tile_hi = gate_mode ? min(p.n_tiles, tile_lo + p.tiles_per_slice) : tile_lo + 1;

    const int nwin = p.win_count ? *p.win_count : p.B;
    for (int wi = blockIdx.y; wi < nwin; wi += gridDim.y) {
        const int b = p.win_list ? p.win_list[wi] : wi;
        float gacc = 0.f;                      // gate mode: thread (gate g = tid & 63, position slice tid >> 6)
      for (int tile = tile_lo; tile < tile_hi; ++tile) {
        const int p0 = tile * p.tile_p;
        const int tp = min(p.tile_p, p.d.L - p0);
        const int nq = (tp - 1) * PS + PK;
        const int nj = nq + K2 - 1;
        const int nt = (nj - 1) * PS + PK;
        const int ni = nt + K1 - 1;
        const int i0 = p0 * PS * PS;           // first input sample of the receptive field
        const int n_runs = (nj + RUN - 1) / RUN;
        const int n_runs2 = (tp + 1) / 2;
        // ---- stage 1: input tile -> smem (fp32) ------------------------------------------
        const Tin *xb = reinterpret_cast<const Tin *>(p.x) + (int64_t)b * C * p.d.XP + i0;
        for (int c = 0; c < C; ++c) {
            const Tin *row = xb + (int64_t)c * p.d.XP;
            float *dst = xs + c * p.xs_stride;
            for (int i = tid; i < ni; i += 256) dst[padi(i)] = ld_in<Tin>(row + i);
        }
        __syncthreads();

        // ---- stage 2: conv1 -> pool -> act --------------------------------------------------
        for (int r = tid; r < n_runs; r += 256) {
            float acc[kCMid][NT1];
#pragma unroll
            for (int o = 0; o < kCMid; ++o)
#pragma unroll
                for (int i = 0; i < NT1; ++i) acc[o][i] = 0.f;
            const int base = PS * RUN * r;
            auto channel = [&](int c) {
                float xv[NX];
                const float *src = xs + c * p.xs_stride;
#pragma unroll
                for (int i = 0; i < NX; ++i) xv[i] = src[padi(base + i)];
#pragma unroll
                for (int k = 0; k < K1; ++k)
#pragma unroll
                    for (int i = 0; i < NT1; ++i)
#pragma unroll
                        for (int o = 0; o < kCMid; ++o)
                            acc[o][i] = fmaf(p.cw.w1[(c * K1 + k) * kCMid + o], xv[i + k], acc[o][i]);
            };
            if constexpr (CT > 0) {
#pragma unroll
                for (int c = 0; c < CT; ++c) channel(c);
            } else {
#pragma unroll 1
                for (int c = 0; c < C; ++c) channel(c);
            }
#pragma unroll
            for (int jj = 0; jj < RUN; ++jj) {
                const int j = RUN * r + jj;
                if (j < nj) {
#pragma unroll
                    for (int o = 0; o < kCMid; ++o) {
                        float v;
                        if (!aff) {   // pool first, then bias + activation (monotone)
                            float m = acc[o][PS * jj];
#pragma unroll
                            for (int u = 1; u < PK; ++u) m = max_nan(m, acc[o][PS * jj + u]);
                            v = apply_act(m + p.cw.b1[o], act);
                        } else {      // affine scale may be negative: activation first
                            v = apply_act(conv_epilogue(acc[o][PS * jj], p.cw.b1[o], p.cw.s1[o], p.cw.t1[o], 1), act);
#pragma unroll
                            for (int u = 1; u < PK; ++u)
                                v = max_nan(v, apply_act(conv_epilogue(acc[o][PS * jj + u], p.cw.b1[o],
                                                                        p.cw.s1[o], p.cw.t1[o], 1), act));
                        }
                        a1[o * p.a1_stride + padi(j)] = v;
                    }
                }
            }
        }
        __syncthreads();

        // ---- stage 3: conv2 -> pool -> act -> features ----------------------------------
        for (int r = tid; r < n_runs2; r += 256) {
            float acc2[NQ];
#pragma unroll
            for (int i = 0; i < NQ; ++i) acc2[i] = 0.f;
            const int qb = PS * 2 * r;
#pragma unroll
            for (int c = 0; c < kCMid; ++c) {
                float av[NA];
                const float *src = a1 + c * p.a1_stride;
#pragma unroll
                for (int i = 0; i < NA; ++i) av[i] = src[padi(qb + i)];
#pragma unroll
                for (int k = 0; k < K2; ++k)
#pragma unroll
                    for (int i = 0; i < NQ; ++i) acc2[i] = fmaf(p.cw.w2[c * K2 + k], av[i + k], acc2[i]);
            }
#pragma unroll
            for (int pp = 0; pp < 2; ++pp) {
                const int pl = 2 * r + pp;
                if (pl < tp) {
                    float v;
                    if (!aff) {
                        float m = acc2[PS * pp];
#pragma unroll
                        for (int u = 1; u < PK; ++u) m = max_nan(m, acc2[PS * pp + u]);
                        v = apply_act(m + p.cw.b2, act);
                    } else {
                        v = apply_act(conv_epilogue(acc2[PS * pp], p.cw.b2, p.cw.s2, p.cw.t2, 1), act);
#pragma unroll
                        for (int u = 1; u < PK; ++u)
                            v = max_nan(v, apply_act(conv_epilogue(acc2[PS * pp + u], p.cw.b2, p.cw.s2, p.cw.t2, 1), act));
                    }
                    if (gate_mode) xs[pl] = v;     // xs is free after stage 2: the tile's features stay on chip
                    else p.feats[(int64_t)b * p.sB + (int64_t)(p0 + pl) * p.sP] = v;
                }
            }
        }
        // no barrier needed here in feature mode: the next iteration's stage 1 only writes xs (whose readers
        // all passed the stage-2 barrier) and its own barrier orders a1 reuse.
        if (gate_mode) {
            __syncthreads();
            const int g = tid & 63;
            for (int pl = tid >> 6; pl < tp; pl += 4) gacc = fmaf(xs[pl], __ldg(p.wih0T + (int64_t)(p0 + pl) * kGates + g), gacc);
            __syncthreads();                   // xs is rewritten by the next tile's stage 1
        }
      }
        if (gate_mode) {                       // fixed-order sum of the four position slices -> gate_part[slice][b][g]
            gred[tid >> 6][tid & 63] = gacc;
            __syncthreads();
            if (tid < kGates)
                p.gate_part[((int64_t)blockIdx.x * p.B + b) * kGates + tid] =
                    tile_lo < tile_hi ? (gred[0][tid] + gred[1][tid]) + (gred[2][tid] + gred[3][tid]) : 0.f;
            __syncthreads();
        }
    }
}

// ------------------------------------------------------------------------------------------
// Fully runtime-parameterised kernel (any K1/K2/pool): one pooled output per thread.
// ------------------------------------------------------------------------------------------
template <typename Tin>
__global__ void __launch_bounds__(256) frontend_any_kernel(const __grid_constant__ FrontParams p) {
    extern __shared__ float smem[];
    const Dims &d = p.d;
    const int C = d.C, K1 = d.K1, K2 = d.K2, PK = d.PK, PS = d.PS;
    float *xs = smem;
    float *a1 = smem + C * p.xs_stride;
    const int tid = threadIdx.x;
    const int p0 = blockIdx.x * p.tile_p;
    const int tp = min(p.tile_p, d.L - p0);
    const int nq = (tp - 1) * PS + PK;
    const int nj = nq + K2 - 1;
    const int nt = (nj - 1) * PS + PK;
    const int ni = nt + K1 - 1;
    const int i0 = p0 * PS * PS;
    const int nwin = p.win_count ? *p.win_count : p.B;
    for (int wi = blockIdx.y; wi < nwin; wi += gridDim.y) {
        const int b = p.win_list ? p.win_list[wi] : wi;
        const Tin *xb = reinterpret_cast<const Tin *>(p.x) + (int64_t)b * C * d.XP + i0;
        for (int c = 0; c < C; ++c)
            for (int i = tid; i < ni; i += 256) xs[c * p.xs_stride + padi(i)] = ld_in<Tin>(xb + (int64_t)c * d.XP + i);
        __syncthreads();
        for (int e = tid; e < nj * kCMid; e += 256) {
            const int j = e >> 2, o = e & 3;
            float best = 0.f;
            for (int u = 0; u < PK; ++u) {
                const int t = PS * j + u;
                float s = 0.f;
                for (int c = 0; c < C; ++c)
                    for (int k = 0; k < K1; ++k)
                        s = fmaf(p.cw.w1[(c * K1 + k) * kCMid + o], xs[c * p.xs_stride + padi(t + k)], s);
                const float v = apply_act(conv_epilogue(s, p.cw.b1[o], p.cw.s1[o], p.cw.t1[o], d.has_affine), d.act);
                best = (u == 0) ? v : max_nan(best, v);
            }
            a1[o * p.a1_stride + padi(j)] = best;
        }
        __syncthreads();
        for (int pl = tid; pl < tp; pl += 256) {
            float best = 0.f;
            for (int u = 0; u < PK; ++u) {
                const int q = PS * pl + u;
                float s = 0.f;
                for (int c = 0; c < kCMid; ++c)
                    for (int k = 0; k < K2; ++k) s = fmaf(p.cw.w2[c * K2 + k], a1[c * p.a1_stride + padi(q + k)], s);
                const float v = apply_act(conv_epilogue(s, p.cw.b2, p.cw.s2, p.cw.t2, d.has_affine), d.act);
                best = (u == 0) ? v : max_nan(best, v);
            }
            p.feats[(int64_t)b * p.sB + (int64_t)(p0 + pl) * p.sP] = best;
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------
// Host-side dispatch
// ------------------------------------------------------------------------------------------
template <typename K>
static int launch_one(K kernel, const FrontParams &p, dim3 grid, size_t smem, cudaStream_t st,
                      const char **err) {
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    }
    kernel<<<grid, 256, smem, st>>>(p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return 1;
}

template <int CT, int K1, int K2, int PK, int PS>
static int launch_variant(const FrontParams &p, int run, int dtype, dim3 grid, size_t smem,
                          cudaStream_t st, const char **err) {
    if (dtype == B2CNN_DTYPE_F32) {
        if (run == 4) return launch_one(frontend_kernel<CT, K1, K2, PK, PS, 4, float>, p, grid, smem, st, err);
        return launch_one(frontend_kernel<CT, K1, K2, PK, PS, 1, float>, p, grid, smem, st, err);
    }
    if (run == 4) return launch_one(frontend_kernel<CT, K1, K2, PK, PS, 4, __nv_bfloat16>, p, grid, smem, st, err);
    return launch_one(frontend_kernel<CT, K1, K2, PK, PS, 1, __nv_bfloat16>, p, grid, smem, st, err);
}

int launch_frontend_generic(const Dims &d, const ConvWeights &cw, const void *x, int dtype,
                            int64_t B, float *feats, int64_t sB, int64_t sP, cudaStream_t st,
                            int num_sms, const char **err) {
    return launch_frontend_generic_listed(d, cw, x, dtype, B, feats, sB, sP, nullptr, nullptr, st, num_sms, err);
}

static int launch_frontend_impl(const Dims &d, const ConvWeights &cw, const void *x, int dtype, int64_t B, float *feats,
                                int64_t sB, int64_t sP, const int *win_list, const int *win_count, const float *wih0T,
                                float *gate_part, int gate_slices, cudaStream_t st, int num_sms, const char **err);

// win_list / win_count (device memory, may be null): recompute only the listed windows; the
// count is read on the device, so an empty list costs one almost-empty launch and no host sync.
int launch_frontend_generic_listed(const Dims &d, const ConvWeights &cw, const void *x, int dtype,
                                   int64_t B, float *feats, int64_t sB, int64_t sP, const int *win_list,
                                   const int *win_count, cudaStream_t st, int num_sms, const char **err) {
    return launch_frontend_impl(d, cw, x, dtype, B, feats, sB, sP, win_list, win_count, nullptr, nullptr, 0, st, num_sms, err);
}

// The exception path of the streaming tensor-core kernels in ONE launch and without a feature buffer: for every
// listed window the exact features of a slice of positions are multiplied by W_ih_l0^T on the spot and written as
// gate_part[slice][b][64] -- the very rows of the range-partial buffer the head kernel sums (the streaming kernel's
// rows for these windows hold NaN garbage and are overwritten; unused slices are zero-filled).
int launch_frontend_generic_gates_listed(const Dims &d, const ConvWeights &cw, const void *x, int dtype, int64_t B,
                                         const float *wih0T, float *gate_part, int gate_slices, const int *win_list,
                                         const int *win_count, cudaStream_t st, int num_sms, const char **err) {
    if (!gate_part || !wih0T || gate_slices < 1 || !win_list || !win_count) { *err = "gate mode: null argument"; return -1; }
    return launch_frontend_impl(d, cw, x, dtype, B, nullptr, 0, 0, win_list, win_count, wih0T, gate_part, gate_slices, st, num_sms, err);
}

static int launch_frontend_impl(const Dims &d, const ConvWeights &cw, const void *x, int dtype, int64_t B, float *feats,
                                int64_t sB, int64_t sP, const int *win_list, const int *win_count, const float *wih0T,
                                float *gate_part, int gate_slices, cudaStream_t st, int num_sms, const char **err) {
    FrontParams p;
    p.x = x; p.feats = feats; p.sB = sB; p.sP = sP; p.B = (int)B; p.d = d; p.cw = cw;
    p.win_list = win_list; p.win_count = win_count;
    p.gate_part = gate_part; p.wih0T = wih0T; p.gate_slices = gate_slices; p.tiles_per_slice = 1;
    // 508 final positions -> <= 256 thread-runs of 4 pooled outputs in stage 2 (see header).
    const int kTile = 508;
    p.tile_p = d.L < kTile ? d.L : kTile;
    p.n_tiles = (d.L + p.tile_p - 1) / p.tile_p;
    const int run = (p.tile_p >= 96) ? 4 : 1;   // tiny windows: spread conv1 over more threads
    const int nq = (p.tile_p - 1) * d.PS + d.PK, nj = nq + d.K2 - 1;
    const int nt = (nj - 1) * d.PS + d.PK, ni = nt + d.K1 - 1;
    p.xs_stride = padi(ni + d.PS * 4 + d.PK + d.K1 + 8) + 1;
    p.a1_stride = padi(nj + d.PS * 2 + d.PK + d.K2 + 8) + 1;
    const size_t smem = (size_t)(d.C * p.xs_stride + kCMid * p.a1_stride) * sizeof(float);
    if (smem > 220 * 1024) {
        *err = "the generic front end's tile does not fit shared memory (in_channels * pool_s^2 too large for this window length)";
        return kLaunchArch;
    }
    int gx = p.n_tiles;
    if (gate_part) {                            // every slice of the partial buffer gets a CTA (empty ones write zeros)
        p.tiles_per_slice = (p.n_tiles + gate_slices - 1) / gate_slices;
        gx = gate_slices;
    }
    int gy = (2 * num_sms + gx - 1) / gx;
    if (gy > B) gy = (int)B;
    if (win_list && gy > 16) gy = 16;          // the exception path: few windows expected
    if (gate_part && gy > 4) gy = 4;           // ... and its (normally empty) launch sits on the critical path of every forward
    if (gy < 1) gy = 1;
    if (gy > 65535) gy = 65535;
    dim3 grid(gx, gy);

#define B2_TRY(CT, K1_, K2_, PK_, PS_)                                                         \
    if ((CT == 0 || d.C == CT) && d.K1 == K1_ && d.K2 == K2_ && d.PK == PK_ && d.PS == PS_)   \
        return launch_variant<CT, K1_, K2_, PK_, PS_>(p, run, dtype, grid, smem, st, err);
    // MyCNN5 architecture (bin/models.py) at the synthetic C=3 and the production C=10
    B2_TRY(3, 10, 5, 3, 2)
    B2_TRY(10, 10, 5, 3, 2)
    // MyCNN2/3/4 architecture (bin/explore_torch copy.ipynb:189-277)
    B2_TRY(3, 5, 5, 2, 2)
    B2_TRY(7, 5, 5, 2, 2)
    B2_TRY(10, 5, 5, 2, 2)
    // same kernel shapes, any channel count
    B2_TRY(0, 10, 5, 3, 2)
    B2_TRY(0, 5, 5, 2, 2)
#undef B2_TRY
    if (gate_part) { *err = "gate mode needs a templated conv geometry"; return -1; }
    if (dtype == B2CNN_DTYPE_F32) return launch_one(frontend_any_kernel<float>, p, grid, smem, st, err);
    return launch_one(frontend_any_kernel<__nv_bfloat16>, p, grid, smem, st, err);
}

}  // namespace b2cnn

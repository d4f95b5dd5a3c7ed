// b2cnn_batch.cu -- MANY short windows per launch: the production shape of the reference, [P, 10, 120]
// (bin/predictStream.py:105: one row per patient and trigger; config.cfg:23 WINDOWSIZE = 120), scored as ONE batch
// instead of P python-level model() calls.
//
// One WARP owns a window from the first sample to the logit; nothing but __syncwarp() between the stages
// (bin/models.py:23-34):
//   stage 0  the window's C x W samples -> the warp's shared-memory rows (16-byte loads, fp32 or bf16 input)
//   stage 1  conv1: lane l owns conv positions 4l .. 4l+3 x 4 output channels = 8 float2 accumulators;
//            per input channel 4 LDS.128 of samples, per tap one broadcast LDS.128 of the 4 channel weights and
//            8 FFMA pairs.  pool1 BEFORE the activation (max commutes with +bias and monotone tanh / relu; max.NaN
//            propagates NaNs like ATen's max_pool1d); the one pooled position that straddles two lanes comes by shuffle
//   stage 2  conv2 + pool2 + activation: lane l owns feature l (L_out <= 32)
//   stage 3  LSTM layer 0 from the zero state: lane l owns gate rows l and l + 32 (W_ih_l0^T in shared memory,
//            CTA-wide), cell by shuffles, layer 1 the same way, Linear(16 -> 1), age scale
// CTA = 8 warps, grid-strided over the batch; the LSTM / Linear weights are staged once per CTA.
// Independent-window semantics only (a batch-as-sequence scan goes through the general path).
#include "b2cnn_internal.cuh"

namespace b2cnn {

constexpr int kBtWarps = 8;
constexpr int kBtXS = 144;          // padded sample row: W <= 128 plus the zero tail conv1's register window may touch
constexpr int kBtMaxL = 32;

struct BatchParams {
    const void *x;
    const float *age;
    float *out;
    int64_t n_age;
    int B, apply_sigmoid;
    Dims d;
    HeadWeights hw;
    ConvWeights cw;
};

__device__ __forceinline__ float2 bt_fma2(float2 a, float2 b, float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
__device__ __forceinline__ float bt_age_scale(float age, float coef) {
    float s = __fadd_rn(__fmul_rn(age, coef), 1.0f);      // models.py:32: separate multiply and add
    return (s > 0.f || s != s) ? s : 0.f;
}

template <int C, int K1, int PK, typename Tin>
__global__ void __launch_bounds__(kBtWarps * 32)
short_batch_kernel(const __grid_constant__ BatchParams p) {
    constexpr int K2 = 5, PS = 2;
    extern __shared__ __align__(16) float bsm[];
    const Dims &d = p.d;
    const int W = d.W, P1 = d.P1, L = d.L;
    // CTA-wide: conv1 weights as float4 per (c, k), W_ih_l0^T [L][64], W_ih_l1^T [16][64], biases, Linear
    float4 *sw1 = reinterpret_cast<float4 *>(bsm);                 // [C * K1]
    float *swih0 = bsm + 4 * C * K1;                               // [kBtMaxL][64]
    float *swih1 = swih0 + kBtMaxL * kGates;                       // [16][64]   swih1[k * 64 + row]
    float *sbias = swih1 + kHidden * kGates;                       // bih0 | bhh0 | bih1 | bhh1 | wo[16] | bo
    float *warp_base = sbias + 4 * kGates + kHidden + 16;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float *xs = warp_base + warp * (C * kBtXS + kCMid * 64 + 32);  // [C][kBtXS]
    float *a1 = xs + C * kBtXS;                                    // [4][64]
    float *fs = a1 + kCMid * 64;                                   // [32]

    for (int i = threadIdx.x; i < C * K1; i += blockDim.x)
        sw1[i] = make_float4(p.cw.w1[i * 4 + 0], p.cw.w1[i * 4 + 1], p.cw.w1[i * 4 + 2], p.cw.w1[i * 4 + 3]);
    for (int i = threadIdx.x; i < L * kGates; i += blockDim.x) swih0[i] = __ldg(p.hw.wih0T + i);
    for (int i = threadIdx.x; i < kGates * kHidden; i += blockDim.x) swih1[(i & 15) * kGates + (i >> 4)] = __ldg(p.hw.wih1 + i);
    for (int i = threadIdx.x; i < kGates; i += blockDim.x) {
        sbias[i] = __ldg(p.hw.bih0 + i); sbias[kGates + i] = __ldg(p.hw.bhh0 + i);
        sbias[2 * kGates + i] = __ldg(p.hw.bih1 + i); sbias[3 * kGates + i] = __ldg(p.hw.bhh1 + i);
    }
    if (threadIdx.x < kHidden) sbias[4 * kGates + threadIdx.x] = __ldg(p.hw.wo + threadIdx.x);
    if (threadIdx.x == 0) sbias[4 * kGates + kHidden] = __ldg(p.hw.bo);
    for (int i = lane; i < C * kBtXS; i += 32) xs[i] = 0.f;        // the zero tail of every row stays zero
    __syncthreads();

    const int act = d.act;
    const int64_t win_elems = (int64_t)C * d.XP;
    constexpr int VEC = 16 / (int)sizeof(Tin);                     // elements per 16-byte load
    const bool vec_ok = (d.XP % VEC) == 0 && (W % VEC) == 0 && (reinterpret_cast<uintptr_t>(p.x) & 15) == 0;
    for (int b = blockIdx.x * kBtWarps + warp; b < p.B; b += gridDim.x * kBtWarps) {
        // ---- stage 0: samples -> shared memory (fp32)
        const Tin *xb = reinterpret_cast<const Tin *>(p.x) + (int64_t)b * win_elems;
        if (vec_ok) {
            const int per_row = W / VEC;
#pragma unroll
            for (int c = 0; c < C; ++c) {
                if (lane < per_row) {
                    const uint4 v = __ldg(reinterpret_cast<const uint4 *>(xb + (int64_t)c * d.XP) + lane);
                    float *dst = xs + c * kBtXS + lane * VEC;
                    if constexpr (sizeof(Tin) == 4) {
                        *reinterpret_cast<uint4 *>(dst) = v;
                    } else {
                        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
                        float f[8];
#pragma unroll
                        for (int q = 0; q < 4; ++q) { f[2 * q] = __uint_as_float(u[q] << 16); f[2 * q + 1] = __uint_as_float(u[q] & 0xffff0000u); }
                        *reinterpret_cast<float4 *>(dst) = make_float4(f[0], f[1], f[2], f[3]);
                        *reinterpret_cast<float4 *>(dst + 4) = make_float4(f[4], f[5], f[6], f[7]);
                    }
                }
            }
        } else {
            for (int c = 0; c < C; ++c)
                for (int i = lane; i < W; i += 32) {
                    float v;
                    if constexpr (sizeof(Tin) == 4) v = __ldg(reinterpret_cast<const float *>(xb) + (int64_t)c * d.XP + i);
                    else v = __bfloat162float(__ldg(reinterpret_cast<const __nv_bfloat16 *>(xb) + (int64_t)c * d.XP + i));
                    xs[c * kBtXS + i] = v;
                }
        }
        __syncwarp();
        // ---- stage 1: conv1 (positions 4 lane .. 4 lane + 3) -> pool1 -> activation -> a1
        float2 acc[4][2];
#pragma unroll
        for (int i = 0; i < 4; ++i) { acc[i][0] = make_float2(0.f, 0.f); acc[i][1] = make_float2(0.f, 0.f); }
#pragma unroll
        for (int c = 0; c < C; ++c) {
            float xv[16];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float4 v = *reinterpret_cast<const float4 *>(xs + c * kBtXS + 4 * lane + 4 * q);
                xv[4 * q] = v.x; xv[4 * q + 1] = v.y; xv[4 * q + 2] = v.z; xv[4 * q + 3] = v.w;
            }
#pragma unroll
            for (int k = 0; k < K1; ++k) {
                const float4 w = sw1[c * K1 + k];
                const float2 w01 = make_float2(w.x, w.y), w23 = make_float2(w.z, w.w);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float2 xx = make_float2(xv[i + k], xv[i + k]);
                    acc[i][0] = bt_fma2(w01, xx, acc[i][0]);
                    acc[i][1] = bt_fma2(w23, xx, acc[i][1]);
                }
            }
        }
        {
            float pj[2][kCMid];                                    // pooled positions 2 lane, 2 lane + 1
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float v0[2] = {acc[0][h].x, acc[0][h].y}, v1[2] = {acc[1][h].x, acc[1][h].y};
                const float v2[2] = {acc[2][h].x, acc[2][h].y}, v3[2] = {acc[3][h].x, acc[3][h].y};
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int o = 2 * h + e;
                    if (PK == 3) {
                        const float nxt = __shfl_down_sync(0xffffffffu, v0[e], 1);      // conv position 4 (lane + 1)
                        pj[0][o] = max_nan(max_nan(v0[e], v1[e]), v2[e]);
                        pj[1][o] = max_nan(max_nan(v2[e], v3[e]), nxt);
                    } else {
                        pj[0][o] = max_nan(v0[e], v1[e]);
                        pj[1][o] = max_nan(v2[e], v3[e]);
                    }
                }
            }
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
                const int j = 2 * lane + jj;
                if (j < P1) {
#pragma unroll
                    for (int o = 0; o < kCMid; ++o) a1[o * 64 + j] = apply_act(pj[jj][o] + p.cw.b1[o], act);
                }
            }
        }
        __syncwarp();
        // ---- stage 2: conv2 -> pool2 -> activation: feature `lane`
        if (lane < L) {
            float best = 0.f;
#pragma unroll
            for (int u = 0; u < PK; ++u) {
                const int q = PS * lane + u;
                float s = 0.f;
#pragma unroll
                for (int c = 0; c < kCMid; ++c)
#pragma unroll
                    for (int k = 0; k < K2; ++k) s = fmaf(p.cw.w2[c * K2 + k], a1[c * 64 + q + k], s);
                best = (u == 0) ? s : max_nan(best, s);
            }
            fs[lane] = apply_act(best + p.cw.b2, act);
        }
        __syncwarp();
        // ---- stage 3: LSTM layer 0 (zero state) -> layer 1 -> Linear -> age scale (models.py:30-34)
        const int u = lane & 15;
        const bool lo = lane < 16;
        float ga = 0.f, gb = 0.f;
        for (int pp = 0; pp < L; ++pp) {
            const float f = fs[pp];
            ga = fmaf(f, swih0[pp * kGates + lane], ga);
            gb = fmaf(f, swih0[pp * kGates + lane + 32], gb);
        }
        ga = (ga + sbias[lane]) + sbias[kGates + lane];
        gb = (gb + sbias[lane + 32]) + sbias[kGates + lane + 32];
        float A = sigmoid_acc(ga);                                 // lanes < 16: i ; lanes >= 16: f
        float Bv = lo ? tanhf(gb) : sigmoid_acc(gb);               // lanes < 16: g ; lanes >= 16: o
        float ig = __shfl_sync(0xffffffffu, A, u), fg = __shfl_sync(0xffffffffu, A, u + 16);
        float gg = __shfl_sync(0xffffffffu, Bv, u), og = __shfl_sync(0xffffffffu, Bv, u + 16);
        const float c0 = fg * 0.f + ig * gg;
        const float h0 = og * tanhf(c0);
        ga = 0.f; gb = 0.f;
#pragma unroll
        for (int k = 0; k < kHidden; ++k) {
            const float hk = __shfl_sync(0xffffffffu, h0, k);
            ga = fmaf(swih1[k * kGates + lane], hk, ga);
            gb = fmaf(swih1[k * kGates + lane + 32], hk, gb);
        }
        ga = (ga + sbias[2 * kGates + lane]) + sbias[3 * kGates + lane];
        gb = (gb + sbias[2 * kGates + lane + 32]) + sbias[3 * kGates + lane + 32];
        A = sigmoid_acc(ga);
        Bv = lo ? tanhf(gb) : sigmoid_acc(gb);
        ig = __shfl_sync(0xffffffffu, A, u); fg = __shfl_sync(0xffffffffu, A, u + 16);
        gg = __shfl_sync(0xffffffffu, Bv, u); og = __shfl_sync(0xffffffffu, Bv, u + 16);
        const float c1 = fg * 0.f + ig * gg;
        const float h1 = og * tanhf(c1);
        float y = 0.f;
#pragma unroll
        for (int k = 0; k < kHidden; ++k) y = fmaf(sbias[4 * kGates + k], __shfl_sync(0xffffffffu, h1, k), y);
        if (lane == 0) {
            y += sbias[4 * kGates + kHidden];
            y *= bt_age_scale(p.age[p.n_age == 1 ? 0 : b], d.age_coef);
            p.out[b] = p.apply_sigmoid ? sigmoid_acc(y) : y;
        }
        __syncwarp();                                              // xs / a1 / fs are rewritten by the next window
    }
}

static size_t batch_smem_bytes(int C, int K1) {
    return sizeof(float) * ((size_t)4 * C * K1 + kBtMaxL * kGates + kHidden * kGates + 4 * kGates + kHidden + 16 +
                            (size_t)kBtWarps * (C * kBtXS + kCMid * 64 + 32));
}

bool batch_supported(const Dims &d) {
    const bool geom = (d.K1 == 10 && d.PK == 3) || (d.K1 == 5 && d.PK == 2);
    const bool chan = d.C == 10 || d.C == 7 || d.C == 3;
    return geom && chan && d.K2 == 5 && d.PS == 2 && !d.has_affine && d.W <= 128 && d.L1 <= 124 && d.L >= 1 && d.L <= kBtMaxL &&
           d.P1 <= 64;
}

int launch_short_batch(const Dims &d, const ConvWeights &cw, const HeadWeights &hw, const void *x, int dtype, int64_t B,
                       const float *age, int64_t n_age, int apply_sigmoid, float *out, int num_sms, cudaStream_t st, const char **err) {
    BatchParams p;
    p.x = x; p.age = age; p.out = out; p.n_age = n_age; p.B = (int)B; p.apply_sigmoid = apply_sigmoid;
    p.d = d; p.hw = hw; p.cw = cw;
    const size_t smem = batch_smem_bytes(d.C, d.K1);
    int ctas = (int)((B + kBtWarps - 1) / kBtWarps);
    const int per_sm = smem <= 72 * 1024 ? 3 : (smem <= 110 * 1024 ? 2 : 1);
    if (ctas > num_sms * per_sm) ctas = num_sms * per_sm;
    cudaError_t e = cudaErrorInvalidValue;
#define BT_LAUNCH(CC, KK, PP)                                                                                          \
    if (d.C == CC && d.K1 == KK && d.PK == PP) {                                                                       \
        if (dtype == B2CNN_DTYPE_F32) {                                                                                \
            e = cudaFuncSetAttribute(short_batch_kernel<CC, KK, PP, float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
            if (e == cudaSuccess) short_batch_kernel<CC, KK, PP, float><<<ctas, kBtWarps * 32, smem, st>>>(p);         \
        } else {                                                                                                       \
            e = cudaFuncSetAttribute(short_batch_kernel<CC, KK, PP, __nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
            if (e == cudaSuccess) short_batch_kernel<CC, KK, PP, __nv_bfloat16><<<ctas, kBtWarps * 32, smem, st>>>(p); \
        }                                                                                                              \
    }
    BT_LAUNCH(10, 10, 3) BT_LAUNCH(10, 5, 2) BT_LAUNCH(7, 5, 2) BT_LAUNCH(7, 10, 3) BT_LAUNCH(3, 10, 3) BT_LAUNCH(3, 5, 2)
#undef BT_LAUNCH
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return 1;
}

}  // namespace b2cnn

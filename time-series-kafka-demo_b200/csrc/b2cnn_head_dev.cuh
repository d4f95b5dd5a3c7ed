// b2cnn_head_dev.cuh -- the LSTM head of ONE independent window on 16 lanes (lane u = hidden unit u), shared by
// head_reduce_independent_kernel (b2cnn_head.cu) (one place for the arithmetic; a version fused into the
// streaming kernel was built and removed: its registers spilled the streaming loop, see DESIGN.md).  bin/models.py:30-34 from the zero state:
//   gates0[g] = (sum_k partial[k][b][g] + b_ih[g]) + b_hh[g]      slices summed in FIXED order
//   layer 0, layer 1 (W_hh * h and f * c vanish but are kept as written), Linear(16 -> 1), age scale, optional sigmoid
// and (seq_step, below) one step of the LSTM carried across windows, on a whole warp.
#pragma once
#include "b2cnn_internal.cuh"

namespace b2cnn {

__device__ __forceinline__ float head_age_scale(float age, float coef) {
    // models.py:32: relu(age * coef + 1) -- a separate multiply and add in the reference
    float s = __fadd_rn(__fmul_rn(age, coef), 1.0f);
    return (s > 0.f || s != s) ? s : 0.f;
}

// All 32 lanes of the warp must call this together (full-mask shuffles); lanes (lane & 16) .. +15 work on one window.
//   row:          this window's row of slice 0, as float4 (lane u reads gates 4u .. 4u+3 of every slice: one coalesced
//                 256-byte read per slice and window); dead lanes pass any valid window's row
//   slice_stride: distance between slices in float4 units
//   s_w1:         W_ih_l1 transposed in shared memory, s_w1[k * 64 + row]
// Returns the window's logit (or probability) in every lane of its half-warp; the caller stores it from lane u == 0.
template <bool kCacheGlobal, int kInFlight>
__device__ __forceinline__ float head_window16(const float4 *__restrict__ row, int64_t slice_stride, int slices, const HeadWeights &hw,
                                               const float *__restrict__ s_w1, float age, float coef, int apply_sigmoid, int lane) {
    const int u = lane & 15;
    float g4[4];
    {
        // every gate is summed in slice order, 8 x 16-byte loads in flight per lane
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        int k = 0;
        for (; k + kInFlight <= slices; k += kInFlight) {
            float4 v[kInFlight];
#pragma unroll
            for (int j = 0; j < kInFlight; ++j) v[j] = kCacheGlobal ? __ldg(row + (int64_t)(k + j) * slice_stride) : __ldcg(row + (int64_t)(k + j) * slice_stride);
#pragma unroll
            for (int j = 0; j < kInFlight; ++j) { s.x += v[j].x; s.y += v[j].y; s.z += v[j].z; s.w += v[j].w; }
        }
        for (; k < slices; ++k) {
            const float4 v = kCacheGlobal ? __ldg(row + (int64_t)k * slice_stride) : __ldcg(row + (int64_t)k * slice_stride);
            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
        // redistribute: unit u needs gates u, 16+u, 32+u, 48+u, which sit in lanes (q*16+u)/4 at component (q*16+u)%4 = u%4
        const int base16 = lane & 16, comp = u & 3;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int src = base16 + ((q * kHidden + u) >> 2);
            const float a = __shfl_sync(0xffffffffu, s.x, src), b2 = __shfl_sync(0xffffffffu, s.y, src);
            const float c = __shfl_sync(0xffffffffu, s.z, src), d2 = __shfl_sync(0xffffffffu, s.w, src);
            const float sum = comp == 0 ? a : comp == 1 ? b2 : comp == 2 ? c : d2;
            g4[q] = (sum + __ldg(hw.bih0 + q * kHidden + u)) + __ldg(hw.bhh0 + q * kHidden + u);
        }
    }
    // layer 0 from the zero state
    const float c0 = sigmoid_acc(g4[1]) * 0.f + sigmoid_acc(g4[0]) * tanhf(g4[2]);
    const float h0 = sigmoid_acc(g4[3]) * tanhf(c0);
    // layer 1: gi[q] = (sum_k W_ih_l1[q*16+u][k] h0[k] + b_ih) + b_hh, k ascending
    float gi[4] = {0.f, 0.f, 0.f, 0.f};
    const int base = lane & 16;
#pragma unroll
    for (int k = 0; k < kHidden; ++k) {
        const float hk = __shfl_sync(0xffffffffu, h0, base + k);
#pragma unroll
        for (int q = 0; q < 4; ++q) gi[q] = fmaf(s_w1[k * kGates + q * kHidden + u], hk, gi[q]);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) gi[q] = (gi[q] + __ldg(hw.bih1 + q * kHidden + u)) + __ldg(hw.bhh1 + q * kHidden + u);
    const float c1 = sigmoid_acc(gi[1]) * 0.f + sigmoid_acc(gi[0]) * tanhf(gi[2]);
    const float h1 = sigmoid_acc(gi[3]) * tanhf(c1);
    // Linear(16 -> 1): y = fma(wo[u], h1[u], y) for u ascending
    float y = 0.f;
#pragma unroll
    for (int k = 0; k < kHidden; ++k) {
        const float hk = __shfl_sync(0xffffffffu, h1, base + k);
        y = fmaf(__ldg(hw.wo + k), hk, y);
    }
    y += __ldg(hw.bo);
    y *= head_age_scale(age, coef);
    return apply_sigmoid ? sigmoid_acc(y) : y;
}

// ---- one step of the LSTM carried from window to window (sequence mode), one warp per sequence ----
// Shared by head_sequence_kernel (a scan over consecutive rows) and slide_seq_step_kernel (one step per patient of a
// sliding scorer from its stored state), so that both run the same instructions.  Lane l owns gate rows l and l + 32
// of every weight matrix (registers); units' (h, c) are held twice, by lanes u and u + 16.
struct SeqLaneWeights {
    float whh0a[kHidden], whh0b[kHidden], wih1a[kHidden], wih1b[kHidden], whh1a[kHidden], whh1b[kHidden];
    float bih1a, bih1b, bhh1a, bhh1b, wo, bo;
};

__device__ __forceinline__ void seq_load_weights(const HeadWeights &hw, int l, SeqLaneWeights &w) {
#pragma unroll
    for (int k = 0; k < kHidden; ++k) {
        w.whh0a[k] = hw.whh0[l * kHidden + k]; w.whh0b[k] = hw.whh0[(l + 32) * kHidden + k];
        w.wih1a[k] = hw.wih1[l * kHidden + k]; w.wih1b[k] = hw.wih1[(l + 32) * kHidden + k];
        w.whh1a[k] = hw.whh1[l * kHidden + k]; w.whh1b[k] = hw.whh1[(l + 32) * kHidden + k];
    }
    w.bih1a = hw.bih1[l]; w.bih1b = hw.bih1[l + 32]; w.bhh1a = hw.bhh1[l]; w.bhh1b = hw.bhh1[l + 32];
    w.wo = hw.wo[l & 15]; w.bo = hw.bo[0];
}

struct SeqState { float h0, c0, h1, c1; };   // lane l: unit l & 15

// All 32 lanes call this together (full-mask shuffles).  ga, gb: the window's layer-0 pre-activations (W_ih x + b_ih)
// + b_hh of gate rows l and l + 32.  Advances s by one window (bin/models.py:30); lane 0 then reads *age and writes
// *out = (Linear(h1) + b) * relu(age coef + 1), or its sigmoid (models.py:31-34).
__device__ __forceinline__ void seq_step(const SeqLaneWeights &w, SeqState &s, float ga, float gb, int l, const float *age, float coef,
                                         int apply_sigmoid, float *out) {
    const int u = l & 15;
    const bool lo = l < 16;
    // ---- layer 0: add W_hh h_{t-1}
    float ra = 0.f, rb = 0.f;
#pragma unroll
    for (int k = 0; k < kHidden; ++k) {
        const float hk = __shfl_sync(0xffffffffu, s.h0, k);
        ra = fmaf(w.whh0a[k], hk, ra); rb = fmaf(w.whh0b[k], hk, rb);
    }
    ga += ra; gb += rb;
    float A = sigmoid_acc(ga);                         // lanes <16: i ; lanes >=16: f
    float Bv = lo ? tanhf(gb) : sigmoid_acc(gb);       // lanes <16: g ; lanes >=16: o
    float ig = __shfl_sync(0xffffffffu, A, u), fg = __shfl_sync(0xffffffffu, A, u + 16);
    float gg = __shfl_sync(0xffffffffu, Bv, u), og = __shfl_sync(0xffffffffu, Bv, u + 16);
    s.c0 = fg * s.c0 + ig * gg;
    s.h0 = og * tanhf(s.c0);
    // ---- layer 1: input h0 (new), recurrent h1 (old)
    float sa = 0.f, sb = 0.f; ra = 0.f; rb = 0.f;
#pragma unroll
    for (int k = 0; k < kHidden; ++k) {
        const float xk = __shfl_sync(0xffffffffu, s.h0, k);
        const float hk = __shfl_sync(0xffffffffu, s.h1, k);
        sa = fmaf(w.wih1a[k], xk, sa); sb = fmaf(w.wih1b[k], xk, sb);
        ra = fmaf(w.whh1a[k], hk, ra); rb = fmaf(w.whh1b[k], hk, rb);
    }
    ga = (sa + w.bih1a) + (ra + w.bhh1a);
    gb = (sb + w.bih1b) + (rb + w.bhh1b);
    A = sigmoid_acc(ga);
    Bv = lo ? tanhf(gb) : sigmoid_acc(gb);
    ig = __shfl_sync(0xffffffffu, A, u); fg = __shfl_sync(0xffffffffu, A, u + 16);
    gg = __shfl_sync(0xffffffffu, Bv, u); og = __shfl_sync(0xffffffffu, Bv, u + 16);
    s.c1 = fg * s.c1 + ig * gg;
    s.h1 = og * tanhf(s.c1);
    // ---- Linear(16->1) + age scale
    float y = lo ? w.wo * s.h1 : 0.f;
#pragma unroll
    for (int off = 8; off >= 1; off >>= 1) y += __shfl_xor_sync(0xffffffffu, y, off);
    if (l == 0) {
        y = (y + w.bo) * head_age_scale(*age, coef);
        *out = apply_sigmoid ? sigmoid_acc(y) : y;
    }
}

}  // namespace b2cnn

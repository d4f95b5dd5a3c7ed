// b2cnn_head.cu -- everything after x.view(-1, MAGICNUM) (bin/models.py:29):
//   LSTM layer-0 input projection (features x weight_ih_l0^T), the 2-layer LSTM cell
//   (models.py:30), Linear(16->1) (models.py:31) and the age scale (models.py:32-34).
//
//   proj_kernel          [B x L] x [L x 64] fp32 tiled GEMM with split-K partials
//   reduce_gates_kernel  sums the split-K partials in fixed order (deterministic) + biases
//   head_independent     one thread per window, LSTM from the zero state (predictStream.py:157)
//   head_sequence        one warp per segment scans its rows carrying (h, c) -- the reference's
//                        model(x_batch) semantics for B > 1 (models.py:29-30, utils.py:249), over
//                        the whole batch, over each sequence of b2cnn_forward_seq or over each
//                        recording's windows (utils.py:671-692)
#include "b2cnn_internal.cuh"
#include "b2cnn_head_dev.cuh"

#ifndef B2CNN_HEAD_INFLIGHT
#define B2CNN_HEAD_INFLIGHT 8                    // 16-byte loads of range partials in flight per lane
#endif

namespace b2cnn {

// ---------------------------------------------------------------------------------------
__global__ void transpose_wih_kernel(const float *__restrict__ w, float *__restrict__ wT, int L) {
    // w: [64][L] -> wT: [L][64]
    __shared__ float tile[32][33];
    const int p0 = blockIdx.x * 32, g0 = blockIdx.y * 32;
    const int tx = threadIdx.x, ty = threadIdx.y;   // 32 x 8
    for (int i = ty; i < 32; i += 8) {
        const int g = g0 + i, pp = p0 + tx;
        tile[i][tx] = (pp < L) ? w[(int64_t)g * L + pp] : 0.f;
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
        const int pp = p0 + i, g = g0 + tx;
        if (pp < L) wT[(int64_t)pp * kGates + g] = tile[tx][i];
    }
}

void launch_transpose_wih(const float *wih0, float *wih0T, int L, cudaStream_t st) {
    dim3 grid((L + 31) / 32, kGates / 32), block(32, 8);
    transpose_wih_kernel<<<grid, block, 0, st>>>(wih0, wih0T, L);
}

// ---------------------------------------------------------------------------------------
// gates0 partial[ks][b][g] = sum_{p in split ks} F[b][p] * WT[p][g]
// CTA tile: 64 windows x 64 gates, K-chunks of 32, 4x4 register tile per thread.
// ---------------------------------------------------------------------------------------
constexpr int kPM = 64, kPK = 32, kFsStride = 68;

// kProjRing: F is a sliding scorer's position-major feature ring (sB = 1, sP = its row pitch) whose cap >= L slots hold
// window position k in slot (head + k) mod cap; kProjRecord: row b is window w = b mod n_w of recording r = b / n_w,
// position k at F[r sB + w step + k] (sP = 1: a recording's features, record-major); otherwise (kProjRows) position k of
// window b is F[b sB + k sP].  The tiles, the zero padding and the summation order are the same in every mode.
constexpr int kProjRows = 0, kProjRing = 1, kProjRecord = 2;
template <int kMode>
__device__ __forceinline__ void proj_body(const float *__restrict__ F, int64_t sB, int64_t sP, int head, int cap,
                                          const float *__restrict__ WT, float *__restrict__ part, int B, int L, int k_per_split,
                                          int n_w = 1, int64_t step = 0) {
    constexpr bool kRing = kMode == kProjRing;
    __shared__ __align__(16) float Fs[kPK][kFsStride];
    __shared__ __align__(16) float Ws[kPK][kGates];
    const int tid = threadIdx.x;
    const int tm = tid >> 4, tn = tid & 15;
    const int b0 = blockIdx.x * kPM;
    const int ks = blockIdx.y;
    const int kbeg = ks * k_per_split;
    const int kend = min(L, kbeg + k_per_split);
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = kbeg; k0 < kend; k0 += kPK) {
#pragma unroll
        for (int it = 0; it < (kPM * kPK) / 256; ++it) {
            const int e = tid + it * 256;
            int m, kk;
            if (sP == 1) { m = e >> 5; kk = e & 31; } else { m = e & 63; kk = e >> 6; }
            const int b = b0 + m, k = k0 + kk;
            int slot = k;
            if (kRing) {
                slot = head + k;
                if (slot >= cap) slot -= cap;
            }
            int64_t row_off;
            if constexpr (kMode == kProjRecord) {
                const int r = b / n_w;
                row_off = (int64_t)r * sB + (int64_t)(b - r * n_w) * step;
            } else {
                row_off = (int64_t)b * sB;
            }
            Fs[kk][m] = (b < B && k < kend) ? __ldg(F + row_off + (int64_t)slot * sP) : 0.f;
        }
#pragma unroll
        for (int it = 0; it < (kPK * kGates) / 256; ++it) {
            const int e = tid + it * 256;
            const int kk = e >> 6, g = e & 63;
            const int k = k0 + kk;
            Ws[kk][g] = (k < kend) ? __ldg(WT + (int64_t)k * kGates + g) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kPK; ++kk) {
            const float4 a = *reinterpret_cast<const float4 *>(&Fs[kk][4 * tm]);
            const float4 w = *reinterpret_cast<const float4 *>(&Ws[kk][4 * tn]);
            const float av[4] = {a.x, a.y, a.z, a.w};
            const float wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int b = b0 + 4 * tm + i;
        if (b < B) {
            float4 v = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
            *reinterpret_cast<float4 *>(part + ((int64_t)ks * B + b) * kGates + 4 * tn) = v;
        }
    }
}

__global__ void __launch_bounds__(256)
proj_kernel(const float *__restrict__ F, int64_t sB, int64_t sP, const float *__restrict__ WT,
            float *__restrict__ part, int B, int L, int k_per_split) {
    proj_body<kProjRows>(F, sB, sP, 0, L, WT, part, B, L, k_per_split);
}

// the sliding scorer's projection over its feature ring of cap slots (b2cnn_slide.cu, generic path): head in [0, cap),
// L <= cap window positions
__global__ void __launch_bounds__(256)
ring_proj_kernel(const float *__restrict__ ring, int64_t pitch, int head, int cap, const float *__restrict__ WT,
                 float *__restrict__ part, int B, int L, int k_per_split) {
    proj_body<kProjRing>(ring, 1, pitch, head, cap, WT, part, B, L, k_per_split);
}

// whole recordings (b2cnn_record.cu, b2cnn_score_record): row b = window b mod n_w of recording b / n_w, whose features
// start at feats[(b / n_w) rec_pitch + (b mod n_w) step]
__global__ void __launch_bounds__(256)
record_proj_kernel(const float *__restrict__ feats, int64_t rec_pitch, int n_w, int64_t step, const float *__restrict__ WT,
                   float *__restrict__ part, int B, int L, int k_per_split) {
    proj_body<kProjRecord>(feats, rec_pitch, 1, 0, L, WT, part, B, L, k_per_split, n_w, step);
}

// gates[b][g] = (sum_ks partial[ks][b][g] + b_ih[g]) + b_hh[g]
__global__ void reduce_gates_kernel(const float *__restrict__ part, int ksplit, int64_t B,
                                    const float *__restrict__ bih, const float *__restrict__ bhh,
                                    float *__restrict__ gates) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= B * kGates) return;
    const int g = (int)(e & 63);
    float s = 0.f;
    for (int k = 0; k < ksplit; ++k) s += part[(int64_t)k * B * kGates + e];
    gates[e] = (s + __ldg(bih + g)) + __ldg(bhh + g);
}

// ---------------------------------------------------------------------------------------
__device__ __forceinline__ float age_scale(float age, float coef) { return head_age_scale(age, coef); }

// One thread per window; zero initial state so W_hh * h and f * c vanish (kept as written).
__global__ void __launch_bounds__(128)
head_independent_kernel(const float *__restrict__ gates0, HeadWeights hw, const float *__restrict__ age,
                        int64_t n_age, float coef, int apply_sigmoid, float *__restrict__ out, int64_t B) {
    __shared__ float s_wih1[kGates * kHidden];
    __shared__ float s_b1a[kGates], s_b1b[kGates], s_wo[kHidden + 1];
    for (int i = threadIdx.x; i < kGates * kHidden; i += blockDim.x) s_wih1[i] = hw.wih1[i];
    for (int i = threadIdx.x; i < kGates; i += blockDim.x) { s_b1a[i] = hw.bih1[i]; s_b1b[i] = hw.bhh1[i]; }
    for (int i = threadIdx.x; i < kHidden; i += blockDim.x) s_wo[i] = hw.wo[i];
    if (threadIdx.x == 0) s_wo[kHidden] = hw.bo[0];
    __syncthreads();
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float *g = gates0 + b * kGates;
    float h0[kHidden];
#pragma unroll
    for (int u = 0; u < kHidden; ++u) {
        const float ig = sigmoid_acc(g[u]), fg = sigmoid_acc(g[kHidden + u]);
        const float gg = tanhf(g[2 * kHidden + u]), og = sigmoid_acc(g[3 * kHidden + u]);
        const float c = fg * 0.f + ig * gg;
        h0[u] = og * tanhf(c);
    }
    float y = 0.f;
#pragma unroll 1
    for (int u = 0; u < kHidden; ++u) {
        float gi[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int r = q * kHidden + u;
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < kHidden; ++k) s = fmaf(s_wih1[r * kHidden + k], h0[k], s);
            gi[q] = (s + s_b1a[r]) + s_b1b[r];
        }
        const float c = sigmoid_acc(gi[1]) * 0.f + sigmoid_acc(gi[0]) * tanhf(gi[2]);
        const float h1 = sigmoid_acc(gi[3]) * tanhf(c);
        y = fmaf(s_wo[u], h1, y);
    }
    y += s_wo[kHidden];
    y *= age_scale(age[n_age == 1 ? 0 : b], coef);
    out[b] = apply_sigmoid ? sigmoid_acc(y) : y;
}

// Independent windows, reduction fused in: 16 lanes per window (lane u = hidden unit u), 16 windows per CTA.
// gates0[b][g] = (sum_k partial[k][b][g] + b_ih[g]) + b_hh[g] in the same fixed order as reduce_gates_kernel
// (windows a tensor-core front end flagged had their partial rows overwritten by the exact re-computation before
// this kernel runs).  The arithmetic per window is head_window16 (b2cnn_head_dev.cuh), which the fused streaming
// kernel runs too; it equals head_independent_kernel term for term.
// win_list / win_count (device memory, may be null): only the listed windows -- the exception path of the fused kernel.
__global__ void __launch_bounds__(256)
head_reduce_independent_kernel(const float *__restrict__ part, int slices, HeadWeights hw, const float *__restrict__ age,
                               int64_t n_age, float coef, int apply_sigmoid, float *__restrict__ out, int64_t B,
                               const int *__restrict__ win_list, const int *__restrict__ win_count,
                               int *__restrict__ clean_count, int *__restrict__ clean_flags, const int *__restrict__ clean_list) {
    __shared__ float s_w1[kHidden * kGates];               // W_ih_l1 transposed: s_w1[k * 64 + row], conflict-free per k
    // Last consumer of the call's exception list (the re-computation that read it ran before this kernel): put the
    // handle's flag state back to all-zero -- exactly the flags the streaming kernel set, and the count -- so the next
    // call needs no memset.  Nothing in this kernel reads them.
    if (clean_count != nullptr && blockIdx.x == 0) {
        const int n = *clean_count;
        for (int i = threadIdx.x; i < n; i += blockDim.x) clean_flags[clean_list[i]] = 0;
        __syncthreads();
        if (threadIdx.x == 0) *clean_count = 0;
    }
    for (int i = threadIdx.x; i < kGates * kHidden; i += blockDim.x) s_w1[(i & 15) * kGates + (i >> 4)] = __ldg(hw.wih1 + i);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int64_t nwin = win_count ? *win_count : B;
    const int64_t per_pass = (int64_t)gridDim.x * (blockDim.x >> 4);
    const int64_t passes = (nwin + per_pass - 1) / per_pass;                 // the same for every thread: shuffles stay full-warp
    for (int64_t it = 0; it < passes; ++it) {
        const int64_t wi = it * per_pass + (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4);
        const bool live = wi < nwin;
        const int64_t wl = live ? wi : nwin - 1;            // dead lanes shadow the last window
        const int64_t b = win_list ? win_list[wl] : wl;
        const float y = head_window16<true, B2CNN_HEAD_INFLIGHT>(reinterpret_cast<const float4 *>(part + b * kGates) + (lane & 15), B * (kGates / 4), slices, hw,
                                            s_w1, age[n_age == 1 ? 0 : b], coef, apply_sigmoid, lane);
        if (live && (lane & 15) == 0) out[b] = y;
    }
}

// One warp (one CTA) per segment: CTA s scans rows s seg_len .. s seg_len + seg_len - 1 of gates0, age (n_age > 1) and
// out sequentially from the zero state, or with seg_off rows seg_off[s] .. seg_off[s + 1] - 1.  forward's sequence mode
// is one segment of B rows, or one per sequence of b2cnn_forward_seq; b2cnn_score_record's is one segment per recording,
// of its n_w windows.  Each row is one seq_step (b2cnn_head_dev.cuh).
__global__ void __launch_bounds__(32)
head_sequence_kernel(const float *__restrict__ gates0, HeadWeights hw, const float *__restrict__ age,
                     int64_t n_age, float coef, int apply_sigmoid, float *__restrict__ out, int64_t seg_len,
                     const int64_t *__restrict__ seg_off) {
    const int l = threadIdx.x;
    const int64_t row0 = seg_off ? seg_off[blockIdx.x] : (int64_t)blockIdx.x * seg_len;
    const int64_t B = seg_off ? seg_off[blockIdx.x + 1] - row0 : seg_len;
    gates0 += row0 * kGates;
    out += row0;
    if (n_age != 1) age += row0;
    SeqLaneWeights w;
    seq_load_weights(hw, l, w);
    SeqState s = {0.f, 0.f, 0.f, 0.f};
    float na = gates0[l], nb = gates0[l + 32];
    for (int64_t t = 0; t < B; ++t) {
        const float ga = na, gb = nb;                      // (W_ih x + b_ih) + b_hh
        if (t + 1 < B) { na = gates0[(t + 1) * kGates + l]; nb = gates0[(t + 1) * kGates + l + 32]; }
        seq_step(w, s, ga, gb, l, age + (n_age == 1 ? 0 : t), coef, apply_sigmoid, out + t);
    }
}

// A sequence-mode sliding scorer's head (b2cnn_slide.cu): one seq_step per live patient from its stored state
// state[p] = {h0, c0, h1, c1} (16 units each), written back.  Its layer-0 pre-activations are summed from the range
// partials [slices][P][64] in reduce_gates_kernel's order, (sum_k part[k][p][g] + b_ih[g]) + b_hh[g], so that a
// patient's steps are those of head_sequence_kernel over its windows.  Warp w takes patients w, w + warps, ...: the
// weights are loaded once per warp.  seen: nullptr (every patient live) or the counts before the push advances them;
// patient p is live when seen[p] >= 0 && seen[p] + S >= W, and the state of any other patient is left as it is.
constexpr int kSeqStepThreads = 128, kSeqStepPerWarp = 4;
__global__ void __launch_bounds__(kSeqStepThreads)
slide_seq_step_kernel(const float *__restrict__ part, int slices, int64_t P, HeadWeights hw, const float *__restrict__ age,
                      int64_t n_age, float coef, int apply_sigmoid, float *__restrict__ out, float *__restrict__ state,
                      const int64_t *__restrict__ seen, int64_t S, int64_t W) {
    constexpr int kIn = B2CNN_HEAD_INFLIGHT;
    const int l = threadIdx.x & 31, u = l & 15;
    SeqLaneWeights w;
    seq_load_weights(hw, l, w);
    const float bih0a = hw.bih0[l], bih0b = hw.bih0[l + 32], bhh0a = hw.bhh0[l], bhh0b = hw.bhh0[l + 32];
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5), slice = P * kGates;
    for (int64_t p = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < P; p += warps) {
        if (seen) {
            const int64_t v = seen[p];
            if (v < 0 || v + S < W) continue;                      // warp-uniform
        }
        const float *row = part + p * kGates + l;
        float sa = 0.f, sb = 0.f;
        int k = 0;
        for (; k + kIn <= slices; k += kIn) {
            float va[kIn], vb[kIn];
#pragma unroll
            for (int j = 0; j < kIn; ++j) { va[j] = __ldcg(row + (k + j) * slice); vb[j] = __ldcg(row + (k + j) * slice + 32); }
#pragma unroll
            for (int j = 0; j < kIn; ++j) { sa += va[j]; sb += vb[j]; }
        }
        for (; k < slices; ++k) { sa += __ldcg(row + k * slice); sb += __ldcg(row + k * slice + 32); }
        float *st = state + p * kGates;
        SeqState s = {st[u], st[kHidden + u], st[2 * kHidden + u], st[3 * kHidden + u]};
        seq_step(w, s, (sa + bih0a) + bhh0a, (sb + bih0b) + bhh0b, l, age + (n_age == 1 ? 0 : p), coef, apply_sigmoid, out + p);
        if (l < kHidden) { st[u] = s.h0; st[kHidden + u] = s.c0; st[2 * kHidden + u] = s.h1; st[3 * kHidden + u] = s.c1; }
    }
}

// ---------------------------------------------------------------------------------------
int choose_ksplit(int L) {
    // Depends on L only: the summation order of a window's projection must not change with the
    // batch it arrives in (prefix / chunking consistency is tested bit-for-bit).
    int ks = (L + 2047) / 2048;
    return ks < 1 ? 1 : ks;
}

// positions per split-K slice (whole K-chunks) and the number of slices the projection writes
static int proj_split(int L, int ksplit, int *ks_eff) {
    int kps = (L + ksplit - 1) / ksplit;
    kps = ((kps + kPK - 1) / kPK) * kPK;           // whole K-chunks per split
    *ks_eff = (L + kps - 1) / kps;
    return kps;
}

int proj_slices(int L) {
    int ks_eff;
    proj_split(L, choose_ksplit(L), &ks_eff);
    return ks_eff;
}

int launch_head(const Dims &d, const HeadWeights &hw, const float *feats, int64_t sB, int64_t sP,
                int64_t B, const float *age, int64_t n_age, int mode, int apply_sigmoid,
                float *out, float *gates_ws, float *partial_ws, int ksplit, cudaStream_t st,
                const char **err, const int64_t *seq_off, int64_t n_seq) {
    int launches = 0;
    int ks_eff;
    const int kps = proj_split(d.L, ksplit, &ks_eff);
    dim3 grid((unsigned)((B + kPM - 1) / kPM), ks_eff);
    proj_kernel<<<grid, 256, 0, st>>>(feats, sB, sP, hw.wih0T, partial_ws, (int)B, d.L, kps);
    ++launches;
    int n = launch_reduce_gates(partial_ws, ks_eff, B, hw, gates_ws, st, err);
    if (n < 0) return -1;
    launches += n;
    n = launch_lstm_head(d, hw, gates_ws, B, age, n_age, mode, apply_sigmoid, out, st, err, seq_off, n_seq);
    if (n < 0) return -1;
    return launches + n;
}

// launch_head of independent windows over a feature ring: window b's position k in ring[((head + k) mod cap) pitch + b]
int launch_ring_proj(const Dims &d, const HeadWeights &hw, const float *ring, int64_t pitch, int cap, int head, int64_t B, float *partial_ws,
                     cudaStream_t st, const char **err) {
    int ks_eff;
    const int kps = proj_split(d.L, choose_ksplit(d.L), &ks_eff);
    ring_proj_kernel<<<dim3((unsigned)((B + kPM - 1) / kPM), ks_eff), 256, 0, st>>>(ring, pitch, head, cap, hw.wih0T, partial_ws, (int)B,
                                                                                    d.L, kps);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return ks_eff;
}

int launch_ring_head(const Dims &d, const HeadWeights &hw, const float *ring, int64_t pitch, int cap, int head, int64_t B,
                     const float *age, int64_t n_age, int apply_sigmoid, float *out, float *gates_ws, float *partial_ws,
                     cudaStream_t st, const char **err) {
    const int ks_eff = launch_ring_proj(d, hw, ring, pitch, cap, head, B, partial_ws, st, err);
    if (ks_eff < 0) return -1;
    int n = launch_reduce_gates(partial_ws, ks_eff, B, hw, gates_ws, st, err);
    if (n < 0) return -1;
    n = launch_lstm_head(d, hw, gates_ws, B, age, n_age, B2CNN_MODE_INDEPENDENT, apply_sigmoid, out, st, err);
    return n < 0 ? -1 : 3;
}

// launch_head of the windows of whole recordings: window w of recording r is row r n_w + w of out and of age; in
// sequence mode each recording's n_w rows are one LSTM scan
int launch_record_head(const Dims &d, const HeadWeights &hw, const float *feats, int64_t rec_pitch, int n_w, int64_t step, int64_t rows,
                       const float *age, int64_t n_age, int mode, int apply_sigmoid, float *out, float *gates_ws, float *partial_ws,
                       cudaStream_t st, const char **err) {
    int ks_eff;
    const int kps = proj_split(d.L, choose_ksplit(d.L), &ks_eff);
    record_proj_kernel<<<dim3((unsigned)((rows + kPM - 1) / kPM), ks_eff), 256, 0, st>>>(feats, rec_pitch, n_w, step, hw.wih0T,
                                                                                        partial_ws, (int)rows, d.L, kps);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    int n = launch_reduce_gates(partial_ws, ks_eff, rows, hw, gates_ws, st, err);
    if (n < 0) return -1;
    n = mode == B2CNN_MODE_SEQUENCE
            ? launch_sequence_segments(d, hw, gates_ws, rows / n_w, n_w, age, n_age, apply_sigmoid, out, st, err)
            : launch_lstm_head(d, hw, gates_ws, rows, age, n_age, B2CNN_MODE_INDEPENDENT, apply_sigmoid, out, st, err);
    return n < 0 ? -1 : 3;
}

// gates[b][g] = (sum over `slices` partial[s][b][g] + b_ih[g]) + b_hh[g], fixed summation order
int launch_reduce_gates(const float *partial, int slices, int64_t B, const HeadWeights &hw, float *gates,
                        cudaStream_t st, const char **err) {
    const int64_t n = B * kGates;
    reduce_gates_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(partial, slices, B, hw.bih0, hw.bhh0, gates);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return 1;
}

// independent windows: slice reduction + LSTM cells + Linear + age scale in one launch
int launch_reduce_lstm_head(const Dims &d, const HeadWeights &hw, const float *partial, int slices, int64_t B,
                            const float *age, int64_t n_age, int apply_sigmoid, float *out, cudaStream_t st, const char **err,
                            int *clean_count, int *clean_flags, const int *clean_list) {
    head_reduce_independent_kernel<<<(unsigned)((B * 16 + 255) / 256), 256, 0, st>>>(partial, slices, hw, age, n_age, d.age_coef,
                                                                                  apply_sigmoid, out, B, nullptr, nullptr,
                                                                                  clean_count, clean_flags, clean_list);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return 1;
}

// LSTM cells + Linear + age scale from layer-0 gate pre-activations (bin/models.py:30-34)
int launch_lstm_head(const Dims &d, const HeadWeights &hw, const float *gates, int64_t B, const float *age,
                     int64_t n_age, int mode, int apply_sigmoid, float *out, cudaStream_t st, const char **err,
                     const int64_t *seq_off, int64_t n_seq) {
    if (mode == B2CNN_MODE_INDEPENDENT) {
        head_independent_kernel<<<(unsigned)((B + 127) / 128), 128, 0, st>>>(gates, hw, age, n_age, d.age_coef,
                                                                             apply_sigmoid, out, B);
    } else {
        return seq_off ? launch_sequence_segments(d, hw, gates, n_seq, 0, age, n_age, apply_sigmoid, out, st, err, seq_off)
                       : launch_sequence_segments(d, hw, gates, 1, B, age, n_age, apply_sigmoid, out, st, err);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return 1;
}

// n_seg independent LSTM scans of seg_len consecutive rows each, one warp per segment
int launch_sequence_segments(const Dims &d, const HeadWeights &hw, const float *gates, int64_t n_seg, int64_t seg_len, const float *age,
                             int64_t n_age, int apply_sigmoid, float *out, cudaStream_t st, const char **err, const int64_t *seg_off) {
    head_sequence_kernel<<<(unsigned)n_seg, 32, 0, st>>>(gates, hw, age, n_age, d.age_coef, apply_sigmoid, out, seg_len, seg_off);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return 1;
}

// one LSTM step per live patient of a sequence-mode scorer from its range partials and state (slide_seq_step_kernel)
int launch_seq_step(const Dims &d, const HeadWeights &hw, const float *partial, int slices, int64_t P, const float *age, int64_t n_age,
                    int apply_sigmoid, float *out, float *state, const int64_t *seen, int64_t S, cudaStream_t st, const char **err) {
    constexpr int64_t per_cta = (kSeqStepThreads / 32) * kSeqStepPerWarp;
    slide_seq_step_kernel<<<(unsigned)((P + per_cta - 1) / per_cta), kSeqStepThreads, 0, st>>>(partial, slices, P, hw, age, n_age, d.age_coef,
                                                                                            apply_sigmoid, out, state, seen, S, d.W);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return 1;
}

}  // namespace b2cnn

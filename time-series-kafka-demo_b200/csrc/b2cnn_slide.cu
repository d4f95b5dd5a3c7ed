// b2cnn_slide.cu -- sliding-window scorer: P patient streams scored every S samples with the last W samples as the
// window (the reference's 600 s window sliding by 60 s, bin/predictStream.py:248-252), computing only the features the
// new samples complete.
//
// The front end (conv1 -> pool -> tanh -> conv2 -> pool -> tanh) is translation-equivariant: window feature i of a
// window starting at sample s reads samples s + 4i .. s + 4i + R - 1 (R = 24 for MyCNN5, 16 for MyCNN2/3/4 geometry).
// With S % 4 == 0 every window's features lie on one stream lattice: stream feature g starts at sample 4g + phi,
// phi = (-W) mod 4, and window n (samples [nS - W, nS)) is stream features G_n .. G_n + L - 1, G_n = (nS - W - phi) / 4.
// Exactly the last L features computed so far, so the ring has L slots, stream feature g in slot g mod L, laid out
// position-major [slot][P] (rows padded to 4 patients; thread == patient stores coalesce).
//
// Per push (segment = samples [(n-1)S, nS) of every patient):
//   * main features, those whose samples all lie in the segment: tc_stream_kernel's ring store mode (b2cnn_tc.cu)
//     reading the segment straight from the caller's buffer (first feature at segment sample phi; a segment with
//     phi != 0 or rows not 16-byte aligned is first copied, shifted by phi, into the scorer's staging rows);
//   * windows the tensor-core kernel flagged (a NaN / inf sample turns a whole block NaN there) get these features
//     recomputed by slide_exact_kernel, the generic kernel's fp32 arithmetic term for term;
//   * seam features, whose receptive field starts in the previous push: slide_exact_kernel again, reading the
//     last 24 samples of each patient's stream (kept per patient, fp32) in front of the segment;
//   * once n S >= W: slide_ring_proj_kernel, [P x L] . [L x 64] over the ring on wgmma with window feature j in slot
//     (G_n + j) mod L, split-K over the streaming kernels' position ranges (they depend on L only) ->
//     partial[range][P][64]; then the head kernel of the independent forward sums the ranges in fixed order and runs
//     the LSTM cells, Linear, age scale and sigmoid.  Extra heads (b2cnn_slide_set_heads_ex) may have a shorter window
//     W_k ending at nS: window positions d .. L - 1 of the scorer's, d = (W - W_k) / F, with their own ranges.
//     In sequence mode (slide_create with B2CNN_MODE_SEQUENCE) slide_seq_step_kernel takes the head's place: one LSTM
//     step per live patient from its state in `lstm`, carried from push to push (utils.run_model over its windows).
//
// Per-patient lifecycle (b2cnn_slide_admit / _discharge): seen[p] counts patient p's samples since its admission (-1:
// discharged); its window after a push is the last W samples of (history | pushes since admission), defined once
// seen[p] >= W.  An admission with history is a push of the listed patients aimed at a k-patient scratch ring (the same
// tensor-core / exact kernels), scattered into their ring columns, plus their tail.  Pushes then run unchanged for all
// P patients; slide_live_kernel advances seen and writes NaN for patients without a complete window.  None of this
// runs for a scorer that never admitted or discharged a patient since its last reset.
//
// All of the above is the tensor-core path.  The generic path (slide_create with B2CNN_PATH_GENERIC, "generic path"
// below) runs the same ring and lifecycle for every geometry on exact CUDA-core kernels, with F = pool_s^2 in place of
// 4.  slide_push and slide_admit are shared; only the step that computes the features differs between the paths.
#include <algorithm>
#include <cstring>
#include <new>
#include <type_traits>
#include <vector>

#include "b2cnn_proj_tc.cuh"
#include "b2cnn_slide.cuh"

namespace b2cnn {

constexpr int kSlideTail = 24;       // stream samples kept per patient and channel: the largest receptive field

// An extra head scored from the scorer's ring (b2cnn_slide_set_heads): a snapshot of a model's LSTM / Linear weights,
// W_ih^T, age coefficient and (tensor-core path) packed W_ih chunks, with its range partials, in one allocation.  Its
// window W_k <= W ends where the scorer's does (b2cnn_slide_set_heads_ex): its L_k features are the last L_k of the
// scorer's window, window positions d .. L - 1 with d = (W - W_k) / F = L - L_k.
struct SlideHead {
    HeadWeights hw;                  // into mem
    float age_coef = 0.f;
    uint64_t digest = 0;             // the model's front-end digest when it was attached
    int W = 0, L = 0;                // its window and feature count
    int ranges = 0, feats_per_cta = 0, chunks_per_cta = 0;   // tensor-core path: its handle's TcState (from L_k only)
    const uint8_t *wpack = nullptr;  // tensor-core path: [n_ranges][chunks_per_cta][6 KB], into mem
    float *partial = nullptr;        // tensor-core path: [n_ranges][P][64], into mem
    void *mem = nullptr;
};

struct Slide {
    int device;
    Dims d;
    int P, S, dtype, R, phi;
    int path = B2CNN_PATH_TENSORCORE;  // or B2CNN_PATH_GENERIC: exact CUDA-core kernels for any geometry (below)
    int F = 4;                       // feature stride pool_s^2 in samples
    int T = kSlideTail;              // tail samples kept per patient and channel: kSlideTail, R - 1 on the generic path
    int num_sms = 0;                 // generic path: sizes the generic front end's grid
    int ranges;                      // projection split-K: the streaming kernels' position ranges (TcState, from L only)
    int64_t n = 0;                   // pushes since the last reset
    int64_t g_done = -1;             // last stream feature computed (-1: none)
    int tail_cur = 0;                // which of the two tail buffers holds the current tail
    float *ring = nullptr;           // [L][ring_pitch]
    int64_t ring_pitch = 0;          // P rounded up to 4: 16-byte rows for the projection's TMA boxes
    float *tail = nullptr;           // [2][P][C][T]
    float *partial = nullptr;        // [ranges][P][64]
    float *gates = nullptr;          // generic path: [P][64] layer-0 gate pre-activations
    int *flags = nullptr;            // flags [P] | list [P] | count
    void *stage = nullptr;           // [P][C][Sp] in the window dtype; generic path: fp32 seam rows [P][C][Sp]
    int64_t Sp = 0;
    bool lifecycle = false;          // set by the first admit / discharge since the last reset
    int64_t *seen = nullptr;         // [P] on the device: samples since admission, -1: discharged (while lifecycle)
    std::vector<int64_t> seen_h;     // its host mirror, equal to it in stream order
    int mode = B2CNN_MODE_INDEPENDENT;   // or B2CNN_MODE_SEQUENCE: each patient's LSTM state carried from push to push
    float *lstm = nullptr;           // sequence mode: [P][64] fp32 on the device, h0 | c0 | h1 | c1 of 16 units each
    int *lidx = nullptr;             // sequence mode: [P] device indices of a discharge's patients (their rows zeroed)
    std::vector<SlideHead> heads;    // extra heads, rows 1.. of a push with heads
};

static int64_t fdiv(int64_t a, int64_t m) { return a >= 0 ? a / m : -((-a + m - 1) / m); }
// a mod m in [0, m): stream features before sample 0 (negative g) exist once a patient is admitted with history
__host__ __device__ __forceinline__ int64_t mod_nn(int64_t a, int64_t m) {
    const int64_t r = a % m;
    return r < 0 ? r + m : r;
}

template <typename T>
__device__ __forceinline__ float ld_sample(const T *p);
template <>
__device__ __forceinline__ float ld_sample<float>(const float *p) { return __ldg(p); }
template <>
__device__ __forceinline__ float ld_sample<__nv_bfloat16>(const __nv_bfloat16 *p) { return __bfloat162float(__ldg(p)); }

struct SlideExactParams {
    const void *x;                   // the segment, [P][C][pitch]
    int64_t pitch;
    const float *tail;               // [P][C][kSlideTail]: the stream samples just before the segment
    float *ring;
    int64_t ring_pitch;
    int cap, P;
    int64_t g0;                      // first stream feature of the launch
    int ng;                          // features
    int64_t seg0;                    // stream index of the segment's first sample
    int phi;
    const int *list, *count;         // listed form: only these patients (count read on the device)
    ConvWeights cw;
};

// One feature, exact fp32, in the generic kernel's order (b2cnn_generic.cu): conv1 sums channel-major then tap,
// pooling before bias + tanh with max.NaN, conv2 over the 4 channels then taps.
template <int C, int K1, int PK, typename Tin>
__device__ float exact_feature(const SlideExactParams &p, int b, int64_t g) {
    constexpr int K2 = 5, PS = 2, NA = PK + K2 - 1, NT = PS * (NA - 1) + PK, NX = NT + K1 - 1;
    const int64_t s0 = 4 * g + p.phi - p.seg0;           // first sample relative to the segment; < 0: in the tail
    const Tin *xb = reinterpret_cast<const Tin *>(p.x) + (int64_t)b * C * p.pitch;
    const float *tb = p.tail + (int64_t)b * C * kSlideTail;
    float xs[C][NX];
#pragma unroll
    for (int c = 0; c < C; ++c)
#pragma unroll
        for (int i = 0; i < NX; ++i) {
            const int64_t r = s0 + i;
            xs[c][i] = r >= 0 ? ld_sample<Tin>(xb + c * p.pitch + r) : tb[c * kSlideTail + kSlideTail + r];
        }
    float a1[kCMid][NA];
#pragma unroll
    for (int j = 0; j < NA; ++j)
#pragma unroll
        for (int o = 0; o < kCMid; ++o) {
            float m = 0.f;
#pragma unroll
            for (int u = 0; u < PK; ++u) {
                const int t = PS * j + u;
                float s = 0.f;
#pragma unroll
                for (int c = 0; c < C; ++c)
#pragma unroll
                    for (int k = 0; k < K1; ++k) s = fmaf(p.cw.w1[(c * K1 + k) * kCMid + o], xs[c][t + k], s);
                m = u == 0 ? s : max_nan(m, s);
            }
            a1[o][j] = tanhf(m + p.cw.b1[o]);
        }
    float best = 0.f;
#pragma unroll
    for (int u = 0; u < PK; ++u) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < kCMid; ++c)
#pragma unroll
            for (int k = 0; k < K2; ++k) s = fmaf(p.cw.w2[c * K2 + k], a1[c][u + k], s);
        best = u == 0 ? s : max_nan(best, s);
    }
    return tanhf(best + p.cw.b2);
}

// all patients: thread x = patient, blockIdx.y = feature; listed: thread x = feature, blockIdx.y strides the list
template <int C, int K1, int PK, typename Tin>
__global__ void __launch_bounds__(128) slide_exact_kernel(const __grid_constant__ SlideExactParams p) {
    auto store = [&](int b, int gi) {
        const int64_t g = p.g0 + gi;
        p.ring[mod_nn(g, p.cap) * p.ring_pitch + b] = exact_feature<C, K1, PK, Tin>(p, b, g);
    };
    if (!p.list) {
        const int b = blockIdx.x * blockDim.x + threadIdx.x;
        if (b < p.P) store(b, blockIdx.y);
        return;
    }
    const int gi = blockIdx.x * blockDim.x + threadIdx.x;
    const int nwin = *p.count;
    if (gi >= p.ng) return;
    for (int wi = blockIdx.y; wi < nwin; wi += gridDim.y) store(p.list[wi], gi);
}

// segment rows shifted by phi into 16-byte aligned rows of Sp samples (tail zero-filled)
template <typename T>
__global__ void slide_stage_kernel(const T *__restrict__ src, int64_t sp, int phi, int n, T *__restrict__ dst, int64_t dp,
                                   int64_t rows) {
    const int64_t total = rows * dp;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / dp, i = e - r * dp;
        dst[e] = i < n ? src[r * sp + i + phi] : T(0);
    }
}

// ---- projection over the ring on the tensor cores -----------------------------------------------------------------
// The split-K ranges and 16-position chunks are those of the streaming kernels (TcState: feats_per_cta, chunks_per_cta,
// n_ranges, all from L only), so the packed W_ih chunks of tc_prepare serve unchanged: chunk m of range r holds the
// weights of window positions r F + 16 m - foff + k (k < 16), zero outside the range.  A row's window (L positions,
// its first in slot `head`) may be a suffix of the ring's (cap >= L slots): a head with a shorter window.
// CTA = (128 patients, range), the chunk arithmetic of b2cnn_proj_tc.cuh:
//   warp 4: TMA producer -- per chunk one {128 patients x 16 slots} fp32 box of the ring at the chunk's first slot and,
//           when the 16 slots wrap past cap, a second box at slot 0; plus the 6 KB W_ih chunk (bulk copy); two stages;
//   warps 0-3: thread == patient, its features read from the ring boxes.
constexpr int kRpBox = 16 * kRpM * 4;                // one TMA box: 16 slots x 128 patients fp32
// HP: heads per CTA, each with its own W_ih chunk slot per stage (HP = 1: the scorer's own model alone)
template <int HP>
constexpr size_t kRpSmemHP = 1024 + 2 * 2 * kRpBox + 2 * HP * kRpWChunk + 3 * kRpPiece + 64;
constexpr size_t kRpSmem = kRpSmemHP<1>;

struct RingProjParams {
    const uint8_t *wpack;            // [n_ranges][chunks_per_cta][kRpWChunk]
    float *partial;                  // [n_ranges][P][64]
    int P, L, cap, head, feats_per_cta, chunks_per_cta, foff;   // L: the row's window positions; cap: the ring's slots
};

// A push with heads: rows 0 (the scorer's model) .. K (its heads) of the output, HP rows per CTA.  CTA x = tile * pairs
// + pair, so that the pairs of one (patient tile, range) are neighbours in launch order and may find its ring box in L2.
constexpr int kRpMaxRows = 1 + B2CNN_SLIDE_MAX_HEADS;
struct RingProjHeads {
    RingProjParams p;                         // its wpack / partial are not read
    const uint8_t *wpack[kRpMaxRows + 1];     // row r's packed W_ih chunks
    float *partial[kRpMaxRows + 1];           // row r's [n_ranges][P][64]; nullptr: a padding row, computed, not stored
    int pairs;                                // CTAs per (patient tile, range)
};
template <int HP>
using RingProjArgs = std::conditional_t<HP == 1, RingProjParams, RingProjHeads>;
__device__ __forceinline__ const RingProjParams &rp_base(const RingProjParams &a) { return a; }
__device__ __forceinline__ const RingProjParams &rp_base(const RingProjHeads &a) { return a.p; }

// Per head the instructions are those of HP = 1: the same A pieces, the same 12 MMAs per chunk in the same order, the
// same chunk order.  So each head's partials are bit-identical to those of a scorer of its model.
template <int HP>
__global__ void __launch_bounds__(kRpThreads, 1)
slide_ring_proj_kernel(const __grid_constant__ CUtensorMap tm, const __grid_constant__ RingProjArgs<HP> args) {
    const RingProjParams &p = rp_base(args);
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    float *sF = reinterpret_cast<float *>(smem);                  // [2 stages][2 boxes][16][128]
    uint8_t *sW = smem + 2 * 2 * kRpBox;                           // [2 stages][HP][6 KB]
    uint8_t *sPc = sW + 2 * HP * kRpWChunk;                        // [3 pieces][4 KB]
    uint64_t *bars = reinterpret_cast<uint64_t *>(sPc + 3 * kRpPiece);
    const uint32_t bar_full = smem_u32(bars + 0), bar_empty = smem_u32(bars + 2);
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
    const int lane = threadIdx.x & 31;
    int tile = blockIdx.x, row0 = 0;
    if constexpr (HP > 1) { tile = blockIdx.x / args.pairs; row0 = HP * (blockIdx.x - tile * args.pairs); }
    auto wpack_of = [&](int j) {
        if constexpr (HP == 1) return p.wpack;
        else return args.wpack[row0 + j];
    };
    auto partial_of = [&](int j) {
        if constexpr (HP == 1) return p.partial;
        else return args.partial[row0 + j];
    };
    const int b0 = tile * kRpM;
    const int lo = blockIdx.y * p.feats_per_cta, hi = min(p.L, lo + p.feats_per_cta);
    const int nch = p.chunks_per_cta;
    if (threadIdx.x == 0) {
        for (int i = 0; i < 2; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // ring slot of the chunk's first window position (which may lie before 0 or past L: those features are masked)
    auto first_slot = [&](int m) {
        int s = (p.head + lo + 16 * m - p.foff) % p.cap;
        return s < 0 ? s + p.cap : s;
    };
    if (warp == 4) {
        if (lane == 0) {
            for (int m = 0; m < nch; ++m) {
                const int u = m & 1;
                mbar_wait(bar_empty + 8 * u, ((m >> 1) & 1) ^ 1);
                const int s0 = first_slot(m);
                const bool wraps = s0 + 16 > p.cap;
                mbar_expect_tx(bar_full + 8 * u, (wraps ? 2 : 1) * kRpBox + HP * kRpWChunk);
                const uint32_t dst = smem_u32(sF + (size_t)u * 2 * 16 * kRpM);
                tma_load_2d(dst, &tm, b0, s0, bar_full + 8 * u);
                if (wraps) tma_load_2d(dst + kRpBox, &tm, b0, 0, bar_full + 8 * u);
#pragma unroll
                for (int j = 0; j < HP; ++j)
                    bulk_load_1d(smem_u32(sW + (u * HP + j) * kRpWChunk), wpack_of(j) + ((size_t)blockIdx.y * nch + m) * kRpWChunk,
                                 kRpWChunk, bar_full + 8 * u);
            }
        }
        return;
    }
    const int row = threadIdx.x;
    float gacc[HP][2][32];
#pragma unroll
    for (int j = 0; j < HP; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 32; ++i) gacc[j][h][i] = 0.f;
    uint8_t *arow = sPc + (row >> 3) * 256 + (row & 7) * 16;
#pragma unroll 1
    for (int m = 0; m < nch; ++m) {
        const int u = m & 1;
        mbar_wait(bar_full + 8 * u, (m >> 1) & 1);
        const int s0 = first_slot(m), q0 = lo + 16 * m - p.foff;
        const float *fa = sF + (size_t)u * 2 * 16 * kRpM, *fb = fa + 16 * kRpM;
        rp_split_row(arow, [&](int k) {
            const int q = q0 + k;
            if (q < lo || q >= hi) return 0.f;
            return s0 + k < p.cap ? fa[k * kRpM + row] : fb[(s0 + k - p.cap) * kRpM + row];
        });
        fence_proxy_async();
        wg_bar();
        const uint32_t pa = smem_u32(sPc);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < HP; ++j) rp_mma_chunk(gacc[j], pa, smem_u32(sW + (u * HP + j) * kRpWChunk));
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * u);
        wg_bar();                                                  // A tile free for the next chunk
    }
#pragma unroll
    for (int j = 0; j < HP; ++j) {
        float *const part = partial_of(j);
        if (HP > 1 && !part) continue;
        rp_store_partial(part, blockIdx.y, p.P, b0, warp, lane, gacc[j]);
    }
}

// feats[b][j] = ring[(head + j) mod cap][b]
__global__ void slide_gather_kernel(const float *__restrict__ ring, int64_t pitch, int cap, int P, int head, int L,
                                    float *__restrict__ feats) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= P) return;
    for (int j = blockIdx.y; j < L; j += gridDim.y) feats[(int64_t)b * L + j] = ring[(int64_t)((head + j) % cap) * pitch + b];
}

// ---- lifecycle kernels ------------------------------------------------------------------------------------------
// ring[(g mod L)][idx[j]] = scratch[(g mod cap)][j], g in [g0, g0 + ng): an admission's features into the ring
__global__ void slide_scatter_kernel(const float *__restrict__ scratch, int64_t spitch, int cap, const int *__restrict__ idx, int k,
                                     int64_t g0, int ng, float *__restrict__ ring, int64_t rpitch, int L) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    const int q = idx[j];
    for (int i = blockIdx.y; i < ng; i += gridDim.y) {
        const int64_t g = g0 + i;
        ring[mod_nn(g, L) * rpitch + q] = scratch[mod_nn(g, cap) * spitch + j];
    }
}

// seen[b] += adv for admitted patients (seen >= 0); then row b of x [P][len] = NaN unless seen[b] >= W.
// adv != 0 only with gridDim.y == 1 (one thread per patient reads and writes seen).
__global__ void slide_live_kernel(int64_t *__restrict__ seen, int P, int64_t adv, int64_t W, float *__restrict__ x, int64_t len) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= P) return;
    int64_t v = seen[b];
    if (adv != 0 && v >= 0) seen[b] = v += adv;
    if (!x || v >= W) return;
    for (int64_t j = blockIdx.y; j < len; j += gridDim.y) x[b * len + j] = __int_as_float(0x7fc00000);
}

// rows idx[j] (j < k) of dst [P][ct] = 0: the LSTM state of a sequence-mode scorer's admitted or discharged patients
__global__ void slide_zero_rows_kernel(float *__restrict__ dst, const int *__restrict__ idx, int64_t k, int64_t ct) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= k * ct) return;
    const int64_t j = e / ct;
    dst[(int64_t)idx[j] * ct + (e - j * ct)] = 0.f;
}

// out[r][P] = NaN for every row r with bit r of `rows` set (blockIdx.y = r): the rows of a push with heads whose window
// no patient has complete yet (a scorer without lifecycle calls; with them slide_live_kernel masks those rows whole)
__global__ void slide_nan_rows_kernel(float *__restrict__ out, int P, unsigned rows) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < P && ((rows >> blockIdx.y) & 1u)) out[(int64_t)blockIdx.y * P + b] = __int_as_float(0x7fc00000);
}

// ---- tails of T samples per patient and channel (T = kSlideTail on the tensor-core path, R - 1 on the generic one) ----
// new tail = the last T samples of (old tail | segment)
template <typename Tin>
__global__ void slide_shift_tail_kernel(const Tin *__restrict__ x, int64_t pitch, int S, int T, const float *__restrict__ tin,
                                        float *__restrict__ tout, int64_t rows) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= rows * T) return;
    const int64_t r = e / T;
    const int64_t u = S + e % T;
    tout[e] = u < T ? tin[r * T + u] : ld_sample<Tin>(x + r * pitch + (u - T));
}

// tail rows of the admitted patients = the last T samples of their history [k][C][pitch] (zeros in front of a shorter
// one: they only reach features that start before the history, which no valid window holds)
template <typename Tin>
__global__ void slide_seed_tail_kernel(const Tin *__restrict__ h, int64_t pitch, int64_t H, const int *__restrict__ idx, int k,
                                       int C, int T, float *__restrict__ tail) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)k * C * T) return;
    const int64_t r = e / T;                               // history row j * C + c
    const int64_t u = e % T;
    const int64_t t = H - T + u;
    tail[((int64_t)idx[r / C] * C + r % C) * T + u] = t >= 0 ? ld_sample<Tin>(h + r * pitch + t) : 0.f;
}

// seam rows [rows][T + n] fp32 (generic path): the tail's T samples, then the segment's first n
template <typename Tin>
__global__ void slide_seam_rows_kernel(const Tin *__restrict__ x, int64_t pitch, const float *__restrict__ tail, int T, int n,
                                       float *__restrict__ dst, int64_t rows) {
    const int64_t w = T + n, total = rows * w;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / w, i = e - r * w;
        dst[e] = i < T ? tail[r * T + i] : ld_sample<Tin>(x + r * pitch + (i - T));
    }
}

// ------------------------------------------------------------------------------------------
template <int C, int K1, int PK>
static void launch_exact_t(const SlideExactParams &p, int dtype, dim3 grid, cudaStream_t st) {
    if (dtype == B2CNN_DTYPE_F32) slide_exact_kernel<C, K1, PK, float><<<grid, 128, 0, st>>>(p);
    else slide_exact_kernel<C, K1, PK, __nv_bfloat16><<<grid, 128, 0, st>>>(p);
}

// features [p.g0, p.g0 + ng) exactly into p.ring: of every one of its p.P rows (p.list == nullptr) or of the listed ones
static int launch_exact_p(SlideExactParams p, const Slide &s, int64_t ng, cudaStream_t st, const char **err) {
    if (ng <= 0) return 0;
    p.ng = (int)ng;
    const dim3 grid = p.list ? dim3((unsigned)((ng + 127) / 128), 16) : dim3((unsigned)((p.P + 127) / 128), (unsigned)ng);
    const int key = s.d.C * 10 + (s.d.K1 == 10 ? 0 : 1);
    switch (key) {
        case 10: launch_exact_t<1, 10, 3>(p, s.dtype, grid, st); break;
        case 20: launch_exact_t<2, 10, 3>(p, s.dtype, grid, st); break;
        case 30: launch_exact_t<3, 10, 3>(p, s.dtype, grid, st); break;
        case 11: launch_exact_t<1, 5, 2>(p, s.dtype, grid, st); break;
        case 21: launch_exact_t<2, 5, 2>(p, s.dtype, grid, st); break;
        case 31: launch_exact_t<3, 5, 2>(p, s.dtype, grid, st); break;
        default: *err = "no exact feature kernel for this geometry"; return -1;
    }
    if (cudaGetLastError() != cudaSuccess) { *err = "exact feature kernel launch"; return -1; }
    return 1;
}

// ---- generic path: every geometry, exact fp32 on CUDA cores --------------------------------------------------------
// Lattice of a conv/pool geometry: feature stride F = pool_s^2, receptive field R (Dims::receptive_field; L = (W - R) /
// F + 1), phase phi = (-W) mod F; stream feature g reads samples F g + phi .. F g + phi + R - 1.
// Every feature comes from the generic front end predict() runs on whole windows (launch_frontend_generic: the
// templated frontend_kernel or frontend_any_kernel, the same arithmetic term for term), pointed at the first feature's
// sample with the window's row pitch and writing straight into ring slots:
//   * main features (samples all in the segment): the pushed segment, read in place (any pitch, any alignment);
//   * seam features: fp32 seam rows = the patient's last T = R - 1 samples | the segment's first min(S, T);
//   * an admission's features: the history rows, read in place, into a scratch ring (then slide_scatter_kernel).
// The projection is launch_head's proj_kernel tiles and order reading the ring with its rotation (ring_proj_kernel),
// then launch_head's reduction and LSTM head.

static int64_t window_head(const Slide &s, int64_t n);

// features [g0, g0 + ng) of B windows into dst, feature g of window b at dst[(g mod cap) dpitch + b]; feature g0's first
// sample at sample x0 of each channel row (rows `pitch` samples apart, windows C pitch apart).  One front-end launch per
// run of consecutive slots: two when the range wraps.  ng <= cap.
static int ring_front(const Slide &s, const ConvWeights &cw, const void *x, int dtype, int64_t pitch, int64_t B, int64_t x0,
                      int64_t g0, int64_t ng, float *dst, int64_t dpitch, int64_t cap, cudaStream_t st, const char **err) {
    const int64_t esz = dtype == B2CNN_DTYPE_BF16 ? 2 : 4;
    while (ng > 0) {
        const int64_t slot = mod_nn(g0, cap), n = std::min(ng, cap - slot);
        Dims d = s.d;
        d.L = (int)n; d.W = (int)((n - 1) * s.F + s.R); d.XP = (int)pitch;
        const int rc = launch_frontend_generic(d, cw, static_cast<const char *>(x) + x0 * esz, dtype, B, dst + slot * dpitch, 1, dpitch,
                                               st, s.num_sms, err);
        if (rc < 0) return rc;
        g0 += n; ng -= n; x0 += n * s.F;
    }
    return 1;
}

// ---- the per-path step of a push: ring slots [g_lo, g_hi] -------------------------------------------------------
// Tensor-core path: features [p.g0, p.g0 + Q) of p.P rows [p.P][C][p.pitch] holding stream samples [p.seg0, p.seg0 +
// len) into p.ring, slot g mod p.cap.  From Q >= 32 on, tc_ring_features from the rows (first copied into `stage` rows
// of sp samples, shifted to start at feature p.g0, where it does not start them or they are not 16-byte aligned), then
// the rows it flagged in `flags` [2 p.P + 1] exactly; below that every row exactly.
static int tc_ring_block(const Slide &s, const TcState &tc, SlideExactParams p, int64_t Q, int64_t len, void *stage, int64_t sp,
                         int *flags, cudaStream_t st, const char **err) {
    if (Q >= 32) {
        const int64_t esz = s.dtype == B2CNN_DTYPE_BF16 ? 2 : 4, rows = (int64_t)p.P * s.d.C;
        const int64_t off = s.F * p.g0 + p.phi - p.seg0;               // the row sample feature p.g0 starts at
        const void *xin = p.x;
        int64_t xp = p.pitch;
        if (off != 0 || p.pitch % (16 / esz) != 0 || (reinterpret_cast<uintptr_t>(p.x) & 15) != 0) {
            const unsigned blocks = (unsigned)std::min<int64_t>((rows * sp + 255) / 256, 65536);
            if (esz == 2)
                slide_stage_kernel<uint16_t><<<blocks, 256, 0, st>>>(static_cast<const uint16_t *>(p.x), p.pitch, (int)off, (int)(len - off),
                                                                     static_cast<uint16_t *>(stage), sp, rows);
            else
                slide_stage_kernel<float><<<blocks, 256, 0, st>>>(static_cast<const float *>(p.x), p.pitch, (int)off, (int)(len - off),
                                                                  static_cast<float *>(stage), sp, rows);
            if (cudaGetLastError() != cudaSuccess) { *err = "staging launch"; return -1; }
            xin = stage; xp = sp;
        }
        Dims dseg = s.d;
        dseg.W = (int)(len - off); dseg.L = (int)Q; dseg.XP = (int)xp;
        if (cudaMemsetAsync(flags, 0, sizeof(int) * (size_t)(2 * p.P + 1), st) != cudaSuccess) { *err = "memset flags"; return -1; }
        if (tc_ring_features(tc, dseg, p.cw, xin, xp, s.dtype, p.P, p.ring, p.ring_pitch, p.cap, (int)mod_nn(p.g0, p.cap), flags, st,
                             err) < 0)
            return -1;
        p.list = flags + p.P; p.count = flags + 2 * p.P;
    }
    return launch_exact_p(p, s, Q, st, err);
}

// tensor-core path: main features [g_m0, g_hi] from the segment (tc_ring_block), seam features [g_lo, min(g_hi, g_m0 -
// 1)] exactly, their receptive field starting in the tail
static int push_features_tc(Slide *s, const ConvWeights &cw, const TcState &tc, const void *x, int64_t pitch, const float *tail_in,
                            int64_t g_lo, int64_t g_m0, int64_t g_hi, cudaStream_t st, const char **err) {
    SlideExactParams p;
    memset(&p, 0, sizeof p);
    p.x = x; p.pitch = pitch; p.tail = tail_in; p.ring = s->ring; p.ring_pitch = s->ring_pitch; p.cap = s->d.L; p.P = s->P;
    p.g0 = g_m0; p.seg0 = s->n * s->S; p.phi = s->phi; p.cw = cw;
    if (tc_ring_block(*s, tc, p, g_hi - g_m0 + 1, s->S, s->stage, s->Sp, s->flags, st, err) < 0) return -1;
    p.g0 = g_lo;
    return launch_exact_p(p, *s, std::min(g_hi, g_m0 - 1) - g_lo + 1, st, err);
}

// generic path: main features [g_m0, g_hi] straight from the segment (feature g_m0 starts at its sample phi), seam
// features [g_lo, min(g_hi, g_m0 - 1)] from seam rows: they start in the last T samples before the segment and end in
// its first min(S, T) (F g_lo + phi >= seg0 - T: g_lo - 1 is at most the last feature complete before this push)
static int push_features_generic(Slide *s, const ConvWeights &cw, const void *x, int64_t pitch, const float *tail_in, int64_t g_lo,
                                 int64_t g_m0, int64_t g_hi, cudaStream_t st, const char **err) {
    const int64_t P = s->P, T = s->T, seg0 = s->n * s->S;
    if (g_hi >= g_m0 &&
        ring_front(*s, cw, x, s->dtype, pitch, P, s->phi, g_m0, g_hi - g_m0 + 1, s->ring, s->ring_pitch, s->d.L, st, err) < 0)
        return -1;
    const int64_t seam_hi = std::min(g_hi, g_m0 - 1);
    if (seam_hi < g_lo) return 1;
    const int64_t rows = P * s->d.C, total = rows * s->Sp;
    const unsigned blocks = (unsigned)std::min<int64_t>((total + 255) / 256, 65536);
    const int nseg = (int)(s->Sp - T);
    if (s->dtype == B2CNN_DTYPE_BF16)
        slide_seam_rows_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16 *>(x), pitch, tail_in, (int)T,
                                                                      nseg, reinterpret_cast<float *>(s->stage), rows);
    else
        slide_seam_rows_kernel<float><<<blocks, 256, 0, st>>>(reinterpret_cast<const float *>(x), pitch, tail_in, (int)T, nseg,
                                                              reinterpret_cast<float *>(s->stage), rows);
    if (cudaGetLastError() != cudaSuccess) { *err = "seam rows launch"; return -1; }
    return ring_front(*s, cw, s->stage, B2CNN_DTYPE_F32, s->Sp, P, s->F * g_lo + s->phi - seg0 + T, g_lo, seam_hi - g_lo + 1, s->ring,
                      s->ring_pitch, s->d.L, st, err);
}

int slide_create(const Dims &d, const TcState &tc, int path, int mode, int n_patients, int stride, int dtype, int device, int num_sms,
                 Slide **out, const char **err) {
    *out = nullptr;
    const bool tcp = path == B2CNN_PATH_TENSORCORE;
    if (mode != B2CNN_MODE_INDEPENDENT && mode != B2CNN_MODE_SEQUENCE) {
        *err = "mode must be B2CNN_MODE_INDEPENDENT (0) or B2CNN_MODE_SEQUENCE (1)"; return B2CNN_EINVAL;
    }
    if (dtype != B2CNN_DTYPE_F32 && dtype != B2CNN_DTYPE_BF16) { *err = "dtype must be f32 (0) or bf16 (1)"; return B2CNN_EINVAL; }
    if (n_patients < 1 || n_patients > (1 << 24)) { *err = "n_patients out of range"; return B2CNN_EINVAL; }
    if (stride < 1 || stride > d.W) { *err = "stride must be in [1, window]"; return B2CNN_EINVAL; }
    const int F = d.feature_stride(), R = d.receptive_field();
    if (stride % F != 0) {
        *err = tcp ? "stride must be a multiple of the feature stride (4 samples)"
                   : "stride must be a multiple of the feature stride (pool_s^2 samples)";
        return B2CNN_EINVAL;
    }
    if (tcp && !tc.fused) {
        *err = "the sliding-window scorer covers the streaming tensor-core geometries only (MyCNN5 or MyCNN2/3/4 conv/pool, "
               "1 to 3 channels, tanh, no affine)";
        return B2CNN_EARCH;
    }
    if (d.W < R || d.L != (d.W - R) / F + 1) { *err = "the feature lattice does not match the window's feature count"; return B2CNN_EARCH; }
    if (!tcp && !frontend_generic_fits(d)) {
        *err = "the generic front end's tile does not fit shared memory (in_channels * pool_s^2 too large for this window length)";
        return B2CNN_EARCH;
    }
    Slide *s = new (std::nothrow) Slide();
    if (!s) { *err = "out of host memory"; return B2CNN_ESTATE; }
    s->device = device; s->d = d; s->P = n_patients; s->S = stride; s->dtype = dtype; s->num_sms = num_sms;
    s->path = tcp ? B2CNN_PATH_TENSORCORE : B2CNN_PATH_GENERIC; s->F = F; s->R = R;
    s->T = tcp ? kSlideTail : std::max(R - 1, 1);
    s->phi = (F - d.W % F) % F;
    s->ranges = tcp ? tc.n_ranges : proj_slices(d.L);
    s->ring_pitch = (n_patients + 3) & ~3;
    // staging rows: tensor-core path, the segment shifted by phi in the window dtype; generic path, fp32 seam rows
    s->Sp = tcp ? (stride + 7) & ~7 : s->T + std::min(stride, s->T);
    const int64_t P = n_patients, esz = tcp && dtype == B2CNN_DTYPE_BF16 ? 2 : 4;
    bool ok = cudaMalloc(&s->ring, sizeof(float) * (size_t)d.L * s->ring_pitch) == cudaSuccess &&
              cudaMalloc(&s->tail, sizeof(float) * (size_t)2 * P * d.C * s->T) == cudaSuccess &&
              cudaMalloc(&s->partial, sizeof(float) * (size_t)s->ranges * P * kGates) == cudaSuccess &&
              (tcp ? cudaMalloc(&s->flags, sizeof(int) * (size_t)(2 * P + 1)) : cudaMalloc(&s->gates, sizeof(float) * (size_t)P * kGates)) ==
                  cudaSuccess &&
              cudaMalloc(&s->stage, (size_t)(P * d.C * s->Sp * esz)) == cudaSuccess &&
              cudaMalloc(&s->seen, sizeof(int64_t) * (size_t)P) == cudaSuccess;
    s->mode = mode;
    if (ok && mode == B2CNN_MODE_SEQUENCE)
        ok = cudaMalloc(&s->lstm, sizeof(float) * (size_t)P * kGates) == cudaSuccess &&
             cudaMalloc(&s->lidx, sizeof(int) * (size_t)P) == cudaSuccess;
    if (!ok) { (void)cudaGetLastError(); slide_destroy(s); *err = "cudaMalloc(scorer state)"; return B2CNN_ECUDA; }
    *out = s;
    return B2CNN_OK;
}

void slide_destroy(Slide *s) {
    if (!s) return;
    cudaFree(s->ring); cudaFree(s->tail); cudaFree(s->partial); cudaFree(s->gates); cudaFree(s->flags); cudaFree(s->stage);
    cudaFree(s->seen); cudaFree(s->lstm); cudaFree(s->lidx);
    for (SlideHead &hd : s->heads) cudaFree(hd.mem);
    delete s;
}

int slide_device(const Slide *s) { return s->device; }
int slide_dtype(const Slide *s) { return s->dtype; }
int slide_path(const Slide *s) { return s->path; }
int slide_mode(const Slide *s) { return s->mode; }

int slide_reset(Slide *s, cudaStream_t st, const char **err) {
    s->n = 0; s->g_done = -1; s->tail_cur = 0; s->lifecycle = false;
    if (cudaMemsetAsync(s->tail, 0, sizeof(float) * (size_t)2 * s->P * s->d.C * s->T, st) != cudaSuccess) {
        *err = "memset tail"; return B2CNN_ECUDA;
    }
    if (s->lstm && cudaMemsetAsync(s->lstm, 0, sizeof(float) * (size_t)s->P * kGates, st) != cudaSuccess) {
        *err = "memset LSTM state"; return B2CNN_ECUDA;
    }
    return B2CNN_OK;
}

template <bool kExport>
__global__ void slide_state_tail_kernel(const float *__restrict__ src, float *__restrict__ dst, const int *__restrict__ idx, int64_t k,
                                        int64_t ct);

// a sequence-mode scorer: the LSTM state rows of the k patients whose device indices are idx = 0, or = src [k][64]
// (device) when src is not null (else nothing)
static int set_lstm_rows(const Slide &s, const int *idx, int64_t k, const float *src, cudaStream_t st, const char **err) {
    if (!s.lstm || k == 0) return B2CNN_OK;
    const unsigned blocks = (unsigned)((k * kGates + 255) / 256);
    if (src) slide_state_tail_kernel<false><<<blocks, 256, 0, st>>>(src, s.lstm, idx, k, kGates);
    else slide_zero_rows_kernel<<<blocks, 256, 0, st>>>(s.lstm, idx, k, kGates);
    if (cudaGetLastError() != cudaSuccess) { *err = "LSTM state launch"; return B2CNN_ECUDA; }
    return B2CNN_OK;
}

static int64_t window_head(const Slide &s, int64_t n) { return fdiv(n * s.S - s.d.W - s.phi, s.F); }

// slide_live_kernel over the P patients: seen += adv, then NaN rows of x [P][len] without a complete window of W samples
static int launch_live(const Slide &s, int64_t adv, int64_t W, float *x, int64_t len, cudaStream_t st, const char **err) {
    const unsigned gy = adv != 0 || len <= 1 ? 1u : (unsigned)std::min<int64_t>(len, 64);
    slide_live_kernel<<<dim3((unsigned)((s.P + 127) / 128), gy), 128, 0, st>>>(s.seen, s.P, adv, W, x, len);
    if (cudaGetLastError() != cudaSuccess) { *err = "lifecycle mask launch"; return -1; }
    return 1;
}

// a push's lifecycle step: the device counts advance by S (and out[P] gets its NaNs), then the host mirror -- only once
// the launch went out, so that the two never disagree
static int advance_seen(Slide *s, float *out, cudaStream_t st, const char **err) {
    if (launch_live(*s, s->S, s->d.W, out, 1, st, err) < 0) return -1;
    for (int64_t &v : s->seen_h)
        if (v >= 0) v += s->S;
    return 1;
}


static int score_windows(Slide *s, const HeadWeights &hw, const TcState *tc, const float *age, int64_t n_age, int apply_sigmoid,
                         float *out, bool heads, int *emitted, int64_t *window_index, cudaEvent_t *ev, cudaStream_t st, const char **err);

int slide_push(Slide *s, const ConvWeights &cw, const HeadWeights &hw, const TcState &tc, const void *x, int64_t pitch,
               const float *age, int64_t n_age, int apply_sigmoid, float *out, bool heads, int *emitted, int64_t *window_index,
               cudaEvent_t *ev, cudaStream_t st, const char **err) {
    const Dims &d = s->d;
    const bool tcp = s->path == B2CNN_PATH_TENSORCORE;
    const int64_t P = s->P, S = s->S, T = s->T;
    if (pitch < S || pitch > 0x7fffffff) { *err = "pitch must be in [stride, 2^31)"; return B2CNN_EINVAL; }
    if (n_age != 1 && n_age != P) { *err = "age must have 1 or n_patients elements"; return B2CNN_EINVAL; }
    if (tcp && tc.n_ranges != s->ranges) { *err = "the handle's position ranges changed since create"; return B2CNN_ESTATE; }
    const int64_t n1 = s->n + 1;
    const int64_t g_hi = fdiv(n1 * S - s->R - s->phi, s->F);   // last feature whose samples have all arrived
    const int64_t g_m0 = s->n * S / s->F;                       // first feature that starts inside the segment
    const int64_t g_lo = std::max(s->g_done + 1, window_head(*s, n1));   // earlier features never enter a window
    const float *tail_in = s->tail + (size_t)s->tail_cur * P * d.C * T;
    float *tail_out = s->tail + (size_t)(s->tail_cur ^ 1) * P * d.C * T;
    if (ev && cudaEventRecord(ev[0], st) != cudaSuccess) { *err = "cudaEventRecord"; return B2CNN_ECUDA; }
    const int rc = tcp ? push_features_tc(s, cw, tc, x, pitch, tail_in, g_lo, g_m0, g_hi, st, err)
                       : push_features_generic(s, cw, x, pitch, tail_in, g_lo, g_m0, g_hi, st, err);
    if (rc < 0) return B2CNN_ECUDA;
    const int64_t rows = P * d.C, blocks = (rows * T + 255) / 256;
    if (s->dtype == B2CNN_DTYPE_BF16)
        slide_shift_tail_kernel<__nv_bfloat16><<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16 *>(x), pitch, (int)S,
                                                                                 (int)T, tail_in, tail_out, rows);
    else
        slide_shift_tail_kernel<float><<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const float *>(x), pitch, (int)S, (int)T, tail_in,
                                                                         tail_out, rows);
    if (cudaGetLastError() != cudaSuccess) { *err = "tail launch"; return B2CNN_ECUDA; }
    if (ev && cudaEventRecord(ev[1], st) != cudaSuccess) { *err = "cudaEventRecord"; return B2CNN_ECUDA; }
    s->n = n1;
    if (g_hi >= g_lo) s->g_done = g_hi;
    s->tail_cur ^= 1;
    return score_windows(s, hw, tcp ? &tc : nullptr, age, n_age, apply_sigmoid, out, heads, emitted, window_index, ev, st, err);
}

// one row of a push: the scorer's model (row 0) or head r - 1, with what its projection and head need
struct ScoreRow {
    const HeadWeights *hw;
    Dims d;                          // the model's Dims with the row's window, feature count and age coefficient
    int ranges, feats_per_cta, chunks_per_cta;   // split-K slices of its partials (tensor-core path: its TcState)
    const uint8_t *wpack;            // tensor-core path: its packed W_ih chunks
    float *partial;
    int head;                        // ring slot of its window position 0
};

// the end of push n = s->n: projection over the ring + head for every row whose window is complete (every patient's,
// or with the lifecycle on, one); on tensor cores with `tc`, else (generic path) on CUDA cores.  With `heads`, out is
// [1 + K][P]: row 0 the scorer's model as without, row i head i - 1 from the same ring.  A head with window W_k < W
// reads the last L_k positions of the scorer's window: its position 0 is the scorer's position d = (W - W_k) / F.
static int score_windows(Slide *s, const HeadWeights &hw, const TcState *tc, const float *age, int64_t n_age, int apply_sigmoid,
                         float *out, bool heads, int *emitted, int64_t *window_index, cudaEvent_t *ev, cudaStream_t st,
                         const char **err) {
    const Dims &d = s->d;
    const int64_t P = s->P, S = s->S, n1 = s->n;
    const int rows = 1 + (heads ? (int)s->heads.size() : 0);
    auto complete = [&](int64_t Wr) {
        if (!s->lifecycle) return n1 * S >= Wr;
        return std::any_of(s->seen_h.begin(), s->seen_h.end(), [&](int64_t v) { return v >= 0 && v + S >= Wr; });
    };
    const int64_t G = window_head(*s, n1);
    ScoreRow row[kRpMaxRows];
    unsigned live = 0;                                             // bit r: row r is scored
    for (int r = 0; r < rows; ++r) {
        ScoreRow &w = row[r];
        w.d = d;
        if (r == 0) {
            w.hw = &hw; w.ranges = s->ranges; w.partial = s->partial;
            w.feats_per_cta = tc ? tc->feats_per_cta : 0; w.chunks_per_cta = tc ? tc->chunks_per_cta : 0;
            w.wpack = tc ? reinterpret_cast<const uint8_t *>(tc->d_wpack) : nullptr;
        } else {
            const SlideHead &hd = s->heads[r - 1];
            w.hw = &hd.hw; w.d.W = hd.W; w.d.L = hd.L; w.d.age_coef = hd.age_coef;
            w.ranges = hd.ranges; w.feats_per_cta = hd.feats_per_cta; w.chunks_per_cta = hd.chunks_per_cta;
            w.wpack = hd.wpack; w.partial = tc ? hd.partial : s->partial;   // generic path: one after another on the scorer's
        }
        w.head = (int)mod_nn(G + (d.W - w.d.W) / s->F, d.L);
        if (complete(w.d.W)) live |= 1u << r;
    }
    *emitted = 0;
    if (!live) {
        if (s->lifecycle && advance_seen(s, nullptr, st, err) < 0) return B2CNN_ECUDA;
        if (ev && cudaEventRecord(ev[2], st) != cudaSuccess) { *err = "cudaEventRecord"; return B2CNN_ECUDA; }
        return B2CNN_OK;
    }
    // sequence mode (no heads): row 0's head is one LSTM step per live patient from its state, before seen advances
    const bool seq = s->mode == B2CNN_MODE_SEQUENCE;
    const int64_t *seen_now = s->lifecycle ? s->seen : nullptr;
    if (!tc) {
        // each row: the same kernels over the same ring with its own W_ih^T, LSTM, Linear and age coefficient
        for (int r = 0; r < rows; ++r) {
            if (!((live >> r) & 1u)) continue;
            if (r == 0 && seq) {
                const int slices = launch_ring_proj(d, hw, s->ring, s->ring_pitch, d.L, row[0].head, P, s->partial, st, err);
                if (slices < 0 ||
                    launch_seq_step(d, hw, s->partial, slices, P, age, n_age, apply_sigmoid, out, s->lstm, seen_now, S, st, err) < 0)
                    return B2CNN_ECUDA;
                continue;
            }
            if (launch_ring_head(row[r].d, *row[r].hw, s->ring, s->ring_pitch, d.L, row[r].head, P, age, n_age, apply_sigmoid, out + r * P,
                                 s->gates, s->partial, st, err) < 0)
                return B2CNN_ECUDA;
        }
    } else {
        CUtensorMap tm;
        if (tc_ring_tmap(s->ring, P, s->ring_pitch, d.L, &tm, err) != 0) return B2CNN_ECUDA;
        const unsigned tiles = (unsigned)((P + kRpM - 1) / kRpM);
        // rows of one window share its ranges, chunks and A pieces: they run in pairs (HP = 2; an odd count pads the last
        // pair with a copy of its row that is not stored); a row whose window no other scored row has runs alone (HP = 1)
        for (unsigned todo = live; todo;) {
            const int r0 = __builtin_ctz(todo);
            const ScoreRow &w0 = row[r0];
            int grp[kRpMaxRows], g = 0;
            for (int r = r0; r < rows; ++r)
                if (((todo >> r) & 1u) && row[r].d.W == w0.d.W && row[r].ranges == w0.ranges &&
                    row[r].feats_per_cta == w0.feats_per_cta && row[r].chunks_per_cta == w0.chunks_per_cta) {
                    grp[g++] = r;
                    todo &= ~(1u << r);
                }
            RingProjParams rp;
            rp.wpack = w0.wpack; rp.partial = w0.partial;
            rp.P = (int)P; rp.L = w0.d.L; rp.cap = d.L; rp.head = w0.head;
            rp.feats_per_cta = w0.feats_per_cta; rp.chunks_per_cta = w0.chunks_per_cta; rp.foff = d.K1 == 10 ? 3 : 2;
            if (g == 1) {
                if (cudaFuncSetAttribute(slide_ring_proj_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRpSmem) != cudaSuccess) {
                    *err = "projection smem attribute"; return B2CNN_ECUDA;
                }
                slide_ring_proj_kernel<1><<<dim3(tiles, (unsigned)w0.ranges), kRpThreads, kRpSmem, st>>>(tm, rp);
            } else {
                RingProjHeads a;
                memset(&a, 0, sizeof a);
                a.p = rp;
                for (int j = 0; j < g; ++j) { a.wpack[j] = row[grp[j]].wpack; a.partial[j] = row[grp[j]].partial; }
                a.pairs = (g + 1) / 2;
                if (g % 2) a.wpack[g] = a.wpack[g - 1];                 // partial[g] stays nullptr
                if (cudaFuncSetAttribute(slide_ring_proj_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRpSmemHP<2>) !=
                    cudaSuccess) {
                    *err = "projection smem attribute"; return B2CNN_ECUDA;
                }
                slide_ring_proj_kernel<2><<<dim3(tiles * (unsigned)a.pairs, (unsigned)w0.ranges), kRpThreads, kRpSmemHP<2>, st>>>(tm, a);
            }
            if (cudaGetLastError() != cudaSuccess) { *err = "projection launch"; return B2CNN_ECUDA; }
        }
        for (int r = 0; r < rows; ++r) {
            if (!((live >> r) & 1u)) continue;
            if (r == 0 && seq) {
                if (launch_seq_step(d, hw, s->partial, s->ranges, P, age, n_age, apply_sigmoid, out, s->lstm, seen_now, S, st, err) < 0)
                    return B2CNN_ECUDA;
                continue;
            }
            if (launch_reduce_lstm_head(row[r].d, *row[r].hw, row[r].partial, row[r].ranges, P, age, n_age, apply_sigmoid, out + r * P, st,
                                        err) < 0)
                return B2CNN_ECUDA;
        }
    }
    // rows no patient has a complete window for yet: NaN (with the lifecycle on, the masks below write them whole)
    const unsigned all = (1u << rows) - 1u;
    if (!s->lifecycle && live != all) {
        slide_nan_rows_kernel<<<dim3((unsigned)((P + 127) / 128), (unsigned)rows), 128, 0, st>>>(out, (int)P, all & ~live);
        if (cudaGetLastError() != cudaSuccess) { *err = "NaN rows launch"; return B2CNN_ECUDA; }
    }
    // row 0 is masked as without heads, and seen advances once; rows 1..K take the mask of their own windows from the
    // advanced counts
    if (s->lifecycle && advance_seen(s, out, st, err) < 0) return B2CNN_ECUDA;
    for (int r = 1; s->lifecycle && r < rows; ++r)
        if (launch_live(*s, 0, row[r].d.W, out + r * P, 1, st, err) < 0) return B2CNN_ECUDA;
    if (ev && cudaEventRecord(ev[2], st) != cudaSuccess) { *err = "cudaEventRecord"; return B2CNN_ECUDA; }
    *emitted = 1;
    *window_index = n1 - (d.W + S - 1) / S;
    return B2CNN_OK;
}

int slide_features(const Slide *s, float *feats, cudaStream_t st, const char **err) {
    bool live = s->n * s->S >= s->d.W;
    if (s->lifecycle) live = std::any_of(s->seen_h.begin(), s->seen_h.end(), [&](int64_t v) { return v >= s->d.W; });
    if (!live) { *err = "no window yet: no patient's window is complete"; return B2CNN_ESTATE; }
    const int head = (int)mod_nn(window_head(*s, s->n), s->d.L);
    slide_gather_kernel<<<dim3((unsigned)((s->P + 127) / 128), 64), 128, 0, st>>>(s->ring, s->ring_pitch, s->d.L, s->P, head, s->d.L, feats);
    if (cudaGetLastError() != cudaSuccess) { *err = "gather launch"; return B2CNN_ECUDA; }
    if (s->lifecycle && launch_live(*s, 0, s->d.W, feats, s->d.L, st, err) < 0) return B2CNN_ECUDA;
    return B2CNN_OK;
}

// ---- per-patient lifecycle ----------------------------------------------------------------------------------------
static int check_patients(const Slide &s, const int *patients, int64_t k, const char **err) {
    if (k < 0 || k > s.P) { *err = "patient count must be in [0, n_patients]"; return B2CNN_EINVAL; }
    if (k > 0 && !patients) { *err = "null patient indices"; return B2CNN_EINVAL; }
    std::vector<char> hit((size_t)s.P, 0);
    for (int64_t j = 0; j < k; ++j) {
        const int q = patients[j];
        if (q < 0 || q >= s.P) { *err = "patient index out of range"; return B2CNN_EINVAL; }
        if (hit[q]) { *err = "patient index listed twice"; return B2CNN_EINVAL; }
        hit[q] = 1;
    }
    return B2CNN_OK;
}

// the counts after a lifecycle call: before the first one every patient has seen the whole stream
static std::vector<int64_t> next_seen(const Slide &s, const int *patients, int64_t k, int64_t value) {
    std::vector<int64_t> v = s.lifecycle ? s.seen_h : std::vector<int64_t>((size_t)s.P, s.n * s.S);
    for (int64_t j = 0; j < k; ++j) v[patients[j]] = value;
    return v;
}

// uploads `next` (pageable: the driver has copied it when the call returns) and makes it the host mirror; called after
// every other launch of the lifecycle call succeeded, so a failed call leaves the lifecycle state as it was
static int commit_seen(Slide *s, std::vector<int64_t> &next, cudaStream_t st, const char **err) {
    if (cudaMemcpyAsync(s->seen, next.data(), sizeof(int64_t) * (size_t)s->P, cudaMemcpyHostToDevice, st) != cudaSuccess) {
        *err = "copy of the sample counts"; return B2CNN_ECUDA;
    }
    s->seen_h.swap(next);
    s->lifecycle = true;
    return B2CNN_OK;
}

// workspace of an admission of k patients with H history samples: scratch ring [cap][round_up(k, 4)] fp32 (cap: the
// features that fit in H samples, at most L) | flags [k] + list [k] + count | indices [k] | staging rows
// [k][C][round_up(H, 8)] in the window dtype (always counted: an unaligned or phase-shifted history is copied there)
struct AdmitLayout {
    int64_t kp, cap, hp;
    size_t scratch, flags, idx, stage, total;
};
static AdmitLayout admit_layout(const Slide &s, int64_t k, int64_t H) {
    AdmitLayout a;
    const int64_t esz = s.dtype == B2CNN_DTYPE_BF16 ? 2 : 4;
    a.kp = (k + 3) & ~3;
    a.cap = H >= s.R ? std::min<int64_t>((H - s.R) / s.F + 1, s.d.L) : 0;
    a.hp = (H + 7) & ~7;
    a.scratch = al256(sizeof(float) * (size_t)(a.cap * a.kp));
    a.flags = al256(sizeof(int) * (size_t)(2 * k + 1));
    a.idx = al256(sizeof(int) * (size_t)k);
    // the generic path reads the history in place, whatever its alignment
    a.stage = s.path == B2CNN_PATH_GENERIC ? 0 : al256((size_t)(k * s.d.C * a.hp * esz));
    a.total = a.scratch + a.flags + a.idx + a.stage;
    return a;
}

int64_t slide_admit_workspace_bytes(const Slide *s, int64_t k, int64_t H) {
    if (k < 0 || k > s->P || H < 0 || H > s->d.W) return -1;
    return (int64_t)admit_layout(*s, k, H).total;
}

int slide_admit(Slide *s, const ConvWeights &cw, const TcState &tc, const int *patients, int64_t k, const void *hist, int64_t H,
                int64_t pitch, const float *lstm, void *ws, int64_t ws_bytes, cudaStream_t st, const char **err) {
    const Dims &d = s->d;
    int rc = check_patients(*s, patients, k, err);
    if (rc != B2CNN_OK) return rc;
    if (lstm && s->mode != B2CNN_MODE_SEQUENCE) { *err = "an LSTM state array for an independent-mode scorer"; return B2CNN_EINVAL; }
    if (H < 0 || H > d.W) { *err = "history length must be in [0, window]"; return B2CNN_EINVAL; }
    if (H > 0 && !hist) { *err = "null history with a positive length"; return B2CNN_EINVAL; }
    if (H > 0 && pitch < H) { *err = "history pitch must be >= its length"; return B2CNN_EINVAL; }
    if (H > 0 && pitch > 0x7fffffff) { *err = "history pitch must be < 2^31"; return B2CNN_EINVAL; }
    if (k == 0) return B2CNN_OK;
    const AdmitLayout a = admit_layout(*s, k, H);
    if (!ws || ws_bytes < (int64_t)a.total) {
        *err = "workspace missing or smaller than b2cnn_slide_admit_workspace_bytes()"; return B2CNN_ESTATE;
    }
    char *base = static_cast<char *>(ws);
    float *scratch = reinterpret_cast<float *>(base);
    int *flags = reinterpret_cast<int *>(base + a.scratch);
    int *idx = reinterpret_cast<int *>(base + a.scratch + a.flags);
    void *stage = base + a.scratch + a.flags + a.idx;

    if (cudaMemcpyAsync(idx, patients, sizeof(int) * (size_t)k, cudaMemcpyHostToDevice, st) != cudaSuccess) {
        *err = "copy of the patient indices"; return B2CNN_ECUDA;
    }
    // the history is stream samples [nS - H, nS): the features wholly inside it that lie in the current window n
    // (features() may read it before the next push) or can still enter a later one
    const int64_t nS = s->n * s->S;
    const int64_t g_lo = std::max(-fdiv(-(nS - H - s->phi), s->F), window_head(*s, s->n));
    const int64_t g_hi = fdiv(nS - s->R - s->phi, s->F);
    const int64_t Q = g_hi - g_lo + 1;
    if (H > 0 && Q > 0 && s->path == B2CNN_PATH_GENERIC) {
        // the generic front end straight from the history rows into the scratch ring, slot g mod Q
        const int rc2 = ring_front(*s, cw, hist, s->dtype, pitch, k, s->F * g_lo + s->phi - (nS - H), g_lo, Q, scratch, a.kp, Q, st, err);
        if (rc2 < 0) return rc2 == kLaunchArch ? B2CNN_EARCH : B2CNN_ECUDA;
    } else if (H > 0 && Q > 0) {
        SlideExactParams p;                                            // into the scratch ring, slot g mod Q (Q <= a.cap)
        memset(&p, 0, sizeof p);
        p.x = hist; p.pitch = pitch; p.tail = s->tail; p.ring = scratch; p.ring_pitch = a.kp; p.cap = (int)Q; p.P = (int)k;
        p.g0 = g_lo; p.seg0 = nS - H; p.phi = s->phi; p.cw = cw;
        if (tc_ring_block(*s, tc, p, Q, H, stage, a.hp, flags, st, err) < 0) return B2CNN_ECUDA;
    }
    if (H > 0 && Q > 0) {
        const unsigned gy = (unsigned)std::min<int64_t>(Q, 1024);
        slide_scatter_kernel<<<dim3((unsigned)((k + 127) / 128), gy), 128, 0, st>>>(scratch, a.kp, (int)Q, idx, (int)k, g_lo, (int)Q,
                                                                                   s->ring, s->ring_pitch, d.L);
        if (cudaGetLastError() != cudaSuccess) { *err = "scatter launch"; return B2CNN_ECUDA; }
    }
    // the next push's seam features read the history's last samples from the current tail
    float *tail = s->tail + (size_t)s->tail_cur * s->P * d.C * s->T;
    const int64_t blocks = (k * d.C * s->T + 255) / 256;
    if (s->dtype == B2CNN_DTYPE_BF16)
        slide_seed_tail_kernel<__nv_bfloat16><<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16 *>(hist), pitch, H, idx,
                                                                                (int)k, d.C, s->T, tail);
    else
        slide_seed_tail_kernel<float><<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const float *>(hist), pitch, H, idx, (int)k, d.C,
                                                                        s->T, tail);
    if (cudaGetLastError() != cudaSuccess) { *err = "tail launch"; return B2CNN_ECUDA; }
    // sequence mode: the LSTM starts again, from zero or from the caller's rows
    if ((rc = set_lstm_rows(*s, idx, k, lstm, st, err)) != B2CNN_OK) return rc;
    std::vector<int64_t> next = next_seen(*s, patients, k, H);
    if ((rc = commit_seen(s, next, st, err)) != B2CNN_OK) return rc;
    // features from the history's last complete one on are seam features of the next push, for every patient (before
    // sample 0 of the stream they have negative indices: the other patients' copies of them are never read)
    if (H > 0 && g_hi < s->g_done) s->g_done = g_hi;
    return B2CNN_OK;
}

int slide_discharge(Slide *s, const int *patients, int64_t k, cudaStream_t st, const char **err) {
    int rc = check_patients(*s, patients, k, err);
    if (rc != B2CNN_OK || k == 0) return rc;
    if (s->lstm) {
        if (cudaMemcpyAsync(s->lidx, patients, sizeof(int) * (size_t)k, cudaMemcpyHostToDevice, st) != cudaSuccess) {
            *err = "copy of the patient indices"; return B2CNN_ECUDA;
        }
        if ((rc = set_lstm_rows(*s, s->lidx, k, nullptr, st, err)) != B2CNN_OK) return rc;
    }
    std::vector<int64_t> next = next_seen(*s, patients, k, -1);
    return commit_seen(s, next, st, err);
}

int slide_samples_seen(Slide *s, int64_t *out, cudaStream_t st, const char **err) {
    const size_t bytes = sizeof(int64_t) * (size_t)s->P;
    cudaError_t e;
    if (s->lifecycle) {
        e = cudaMemcpyAsync(out, s->seen, bytes, cudaMemcpyDeviceToDevice, st);
    } else {
        s->seen_h.assign((size_t)s->P, s->n * s->S);
        e = cudaMemcpyAsync(out, s->seen_h.data(), bytes, cudaMemcpyHostToDevice, st);
    }
    if (e != cudaSuccess) { *err = "copy of the sample counts"; return B2CNN_ECUDA; }
    return B2CNN_OK;
}

// ---- export / import of patients ----------------------------------------------------------------------------------
// A patient's state is its current window in window order (features [L], position j from ring slot (G_n + j) mod L),
// its tail [C][T] and its count.  Window position j is stream feature G_n + j, which starts at sample F (G_n + j) + phi
// = nS - W + F j: F j samples into the window, for any scorer with the same W and F.  So the state does not depend on
// the ring's rotation, P, the slot, the push count or the stride, and an import is an admission with a full history
// whose features come from the state instead of the front end.

// rows[j][i] <-> ring[(head + i) mod L][idx[j]] (i < L, j < k) through a 32 x 32 shared-memory tile, so that both the
// position-major ring side (consecutive patient columns of one slot) and the patient-major row side (consecutive
// positions of one patient) move in whole 128-byte lines.  kExport: src = ring, dst = rows; else src = rows, dst = ring.
constexpr int kStTile = 32, kStRows = 8;
template <bool kExport>
__global__ void __launch_bounds__(kStTile * kStRows)
slide_state_kernel(const float *__restrict__ src, float *__restrict__ dst, int64_t ring_pitch, int L, int head,
                   const int *__restrict__ idx, int k) {
    __shared__ float tile[kStTile][kStTile + 1];                   // [position][patient]
    const int tx = threadIdx.x, ty = threadIdx.y, j0 = blockIdx.x * kStTile;
    const bool col_ok = j0 + tx < k;                               // ring side: lane = patient
    const int64_t col = col_ok ? idx[j0 + tx] : 0;
    for (int i0 = blockIdx.y * kStTile; i0 < L; i0 += gridDim.y * kStTile) {
#pragma unroll
        for (int r = ty; r < kStTile; r += kStRows) {
            const int i = i0 + r, j = j0 + r;
            if constexpr (kExport) {
                if (col_ok && i < L) tile[r][tx] = src[(int64_t)(head + i - (head + i >= L ? L : 0)) * ring_pitch + col];
            } else {
                if (j < k && i0 + tx < L) tile[tx][r] = src[(int64_t)j * L + i0 + tx];
            }
        }
        __syncthreads();
#pragma unroll
        for (int r = ty; r < kStTile; r += kStRows) {
            const int i = i0 + r, j = j0 + r;
            if constexpr (kExport) {
                if (j < k && i0 + tx < L) dst[(int64_t)j * L + i0 + tx] = tile[tx][r];
            } else {
                if (col_ok && i < L) dst[(int64_t)(head + i - (head + i >= L ? L : 0)) * ring_pitch + col] = tile[r][tx];
            }
        }
        __syncthreads();
    }
}

// tails[j][c][t] <-> tail[idx[j]][c][t]: one contiguous row of ct = C T floats per patient.  kExport: src = the
// scorer's tail, dst = tails; else the reverse.
template <bool kExport>
__global__ void slide_state_tail_kernel(const float *__restrict__ src, float *__restrict__ dst, const int *__restrict__ idx, int64_t k,
                                        int64_t ct) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= k * ct) return;
    const int64_t j = e / ct, own = (int64_t)idx[j] * ct + (e - j * ct);
    if constexpr (kExport) dst[e] = src[own];
    else dst[own] = src[e];
}

static uint64_t fnv1a(uint64_t h, const void *p, size_t n) {
    const unsigned char *b = static_cast<const unsigned char *>(p);
    for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 0x100000001b3ull; }
    return h;
}

uint64_t frontend_digest(const Dims &d, const ConvWeights &cw) {
    const int32_t geo[7] = {d.C, d.K1, d.K2, d.PK, d.PS, d.act, d.has_affine};
    uint64_t h = fnv1a(0xcbf29ce484222325ull, geo, sizeof geo);
    h = fnv1a(h, cw.w1, sizeof(float) * (size_t)d.C * d.K1 * kCMid);
    h = fnv1a(h, cw.b1, sizeof cw.b1);
    h = fnv1a(h, cw.w2, sizeof(float) * (size_t)kCMid * d.K2);
    h = fnv1a(h, &cw.b2, sizeof cw.b2);
    if (d.has_affine) {
        h = fnv1a(h, cw.s1, sizeof cw.s1);
        h = fnv1a(h, cw.t1, sizeof cw.t1);
        h = fnv1a(h, &cw.s2, sizeof cw.s2);
        h = fnv1a(h, &cw.t2, sizeof cw.t2);
    }
    return h;
}

// ---- extra heads --------------------------------------------------------------------------------------------------
// One allocation per head: the blob's LSTM / Linear part (whh0 .. bo, contiguous in b2cnn_set_weights' blob) | W_ih^T
// [L_k][64] | tensor-core path: the packed W_ih chunks | the range partials [n_ranges][P][64], both of the head's own
// TcState (L_k).  The generic path's heads run one after another on the scorer's own partials and gates
// (proj_slices(L_k) <= proj_slices(L) for L_k <= L: it is ceil(L / 2048) for every L below 2^24).
struct HeadLayout {
    size_t lstm, wih0T, wpack, partial, total;
    int64_t n_lstm;
};
static HeadLayout head_layout(const Slide &s, const SlideHeadSource &src) {
    HeadLayout a;
    a.n_lstm = src.hw.bo + 1 - src.hw.whh0;
    a.lstm = al256(sizeof(float) * (size_t)a.n_lstm);
    a.wih0T = al256(sizeof(float) * (size_t)src.L * kGates);
    const bool tcp = s.path == B2CNN_PATH_TENSORCORE;
    a.wpack = tcp ? al256((size_t)src.tc->n_ranges * src.tc->chunks_per_cta * kRpWChunk) : 0;
    a.partial = tcp ? al256(sizeof(float) * (size_t)src.tc->n_ranges * s.P * kGates) : 0;
    a.total = a.lstm + a.wih0T + a.wpack + a.partial;
    return a;
}

static const float *rebase(const float *p, const float *from, float *to) { return to + (p - from); }

int slide_set_heads(Slide *s, const SlideHeadSource *src, int n, cudaStream_t st, const char **err) {
    std::vector<SlideHead> next((size_t)n);
    auto drop = [&](const char *what) {
        (void)cudaGetLastError();
        for (SlideHead &hd : next) cudaFree(hd.mem);
        *err = what;
        return B2CNN_ECUDA;
    };
    for (int i = 0; i < n; ++i) {
        const HeadWeights &w = src[i].hw;
        const HeadLayout a = head_layout(*s, src[i]);
        SlideHead &hd = next[i];
        if (cudaMalloc(&hd.mem, a.total) != cudaSuccess) return drop("cudaMalloc(head weights)");
        char *base = static_cast<char *>(hd.mem);
        float *lstm = reinterpret_cast<float *>(base), *wih0T = reinterpret_cast<float *>(base + a.lstm);
        if (cudaMemcpyAsync(lstm, w.whh0, sizeof(float) * (size_t)a.n_lstm, cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
            cudaMemcpyAsync(wih0T, w.wih0T, sizeof(float) * (size_t)src[i].L * kGates, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
            return drop("copy of the head weights");
        hd.hw.wih0T = wih0T;
        hd.hw.whh0 = rebase(w.whh0, w.whh0, lstm); hd.hw.bih0 = rebase(w.bih0, w.whh0, lstm); hd.hw.bhh0 = rebase(w.bhh0, w.whh0, lstm);
        hd.hw.wih1 = rebase(w.wih1, w.whh0, lstm); hd.hw.whh1 = rebase(w.whh1, w.whh0, lstm);
        hd.hw.bih1 = rebase(w.bih1, w.whh0, lstm); hd.hw.bhh1 = rebase(w.bhh1, w.whh0, lstm);
        hd.hw.wo = rebase(w.wo, w.whh0, lstm); hd.hw.bo = rebase(w.bo, w.whh0, lstm);
        hd.age_coef = src[i].age_coef;
        hd.digest = src[i].digest;
        hd.W = src[i].W; hd.L = src[i].L;
        hd.ranges = proj_slices(hd.L);
        if (s->path == B2CNN_PATH_TENSORCORE) {
            hd.ranges = src[i].tc->n_ranges;
            hd.feats_per_cta = src[i].tc->feats_per_cta; hd.chunks_per_cta = src[i].tc->chunks_per_cta;
            uint8_t *wp = reinterpret_cast<uint8_t *>(base + a.lstm + a.wih0T);
            if (cudaMemcpyAsync(wp, src[i].tc->d_wpack, (size_t)src[i].tc->n_ranges * src[i].tc->chunks_per_cta * kRpWChunk,
                                cudaMemcpyDeviceToDevice, st) != cudaSuccess)
                return drop("copy of the packed W_ih chunks");
            hd.wpack = wp;
            hd.partial = reinterpret_cast<float *>(base + a.lstm + a.wih0T + a.wpack);
        }
    }
    // the snapshot is complete when the call returns: later weight changes of the models cannot reach it
    if (cudaStreamSynchronize(st) != cudaSuccess) return drop("copy of the head weights");
    for (SlideHead &hd : s->heads) cudaFree(hd.mem);
    s->heads.swap(next);
    return B2CNN_OK;
}

int slide_n_heads(const Slide *s) { return (int)s->heads.size(); }

// the first head whose front-end digest is not `digest`, or -1
int slide_stale_head(const Slide *s, uint64_t digest) {
    for (size_t i = 0; i < s->heads.size(); ++i)
        if (s->heads[i].digest != digest) return (int)i;
    return -1;
}

void slide_describe_state(const Slide *s, const ConvWeights &cw, b2cnn_slide_state_header *o) {
    memset(o, 0, sizeof *o);
    o->magic = B2CNN_SLIDE_STATE_MAGIC; o->version = B2CNN_SLIDE_STATE_VERSION; o->path = (uint16_t)s->path;
    o->dtype = s->dtype; o->in_channels = s->d.C; o->window = s->d.W; o->lstm_input = s->d.L;
    o->feature_stride = s->F; o->tail_len = s->T;
    o->frontend_digest = frontend_digest(s->d, cw);
}

// the workspace holds the k device indices
int64_t slide_state_workspace_bytes(const Slide *s, int64_t k) {
    if (k < 0 || k > s->P) return -1;
    return (int64_t)al256(sizeof(int) * (size_t)k);
}

// the indices into the workspace, then the feature tile kernel and the tail kernel in one direction; a sequence-mode
// scorer's LSTM state rows [k][64] too: exported into dst_lstm when it is given, imported from src_lstm, or zeroed (an
// import without them starts the patients' LSTM again, as an admission does)
template <bool kExport>
static int launch_state(const Slide &s, const int *patients, int64_t k, const float *src_rows, float *dst_rows, const float *src_tails,
                        float *dst_tails, const float *src_lstm, float *dst_lstm, void *ws, cudaStream_t st, const char **err) {
    int *idx = static_cast<int *>(ws);
    if (cudaMemcpyAsync(idx, patients, sizeof(int) * (size_t)k, cudaMemcpyHostToDevice, st) != cudaSuccess) {
        *err = "copy of the patient indices"; return B2CNN_ECUDA;
    }
    const int L = s.d.L, head = (int)mod_nn(window_head(s, s.n), L);
    const dim3 grid((unsigned)((k + kStTile - 1) / kStTile), (unsigned)std::min<int64_t>((L + kStTile - 1) / kStTile, 65535));
    if constexpr (kExport) slide_state_kernel<true><<<grid, dim3(kStTile, kStRows), 0, st>>>(s.ring, dst_rows, s.ring_pitch, L, head, idx, (int)k);
    else slide_state_kernel<false><<<grid, dim3(kStTile, kStRows), 0, st>>>(src_rows, s.ring, s.ring_pitch, L, head, idx, (int)k);
    if (cudaGetLastError() != cudaSuccess) { *err = "state feature launch"; return B2CNN_ECUDA; }
    float *tail = s.tail + (size_t)s.tail_cur * s.P * s.d.C * s.T;
    const int64_t ct = (int64_t)s.d.C * s.T, blocks = (k * ct + 255) / 256;
    if constexpr (kExport) slide_state_tail_kernel<true><<<(unsigned)blocks, 256, 0, st>>>(tail, dst_tails, idx, k, ct);
    else slide_state_tail_kernel<false><<<(unsigned)blocks, 256, 0, st>>>(src_tails, tail, idx, k, ct);
    if (cudaGetLastError() != cudaSuccess) { *err = "state tail launch"; return B2CNN_ECUDA; }
    const unsigned lblocks = (unsigned)((k * kGates + 255) / 256);
    if constexpr (kExport) {
        if (dst_lstm) slide_state_tail_kernel<true><<<lblocks, 256, 0, st>>>(s.lstm, dst_lstm, idx, k, kGates);
    } else {
        if (set_lstm_rows(s, idx, k, src_lstm, st, err) != B2CNN_OK) return B2CNN_ECUDA;
    }
    if (cudaGetLastError() != cudaSuccess) { *err = "LSTM state launch"; return B2CNN_ECUDA; }
    return B2CNN_OK;
}

static int check_state_args(const Slide &s, const int *patients, int64_t k, const void *feats, const void *tails, const void *seen,
                            const void *lstm, void *ws, int64_t ws_bytes, const char **err) {
    const int rc = check_patients(s, patients, k, err);
    if (rc != B2CNN_OK) return rc;
    if (lstm && s.mode != B2CNN_MODE_SEQUENCE) { *err = "an LSTM state array for an independent-mode scorer"; return B2CNN_EINVAL; }
    if (k > 0 && (!feats || !tails || !seen)) { *err = "null feature, tail or count array with patients listed"; return B2CNN_EINVAL; }
    if (k > 0 && (!ws || ws_bytes < slide_state_workspace_bytes(&s, k))) {
        *err = "workspace missing or smaller than b2cnn_slide_state_workspace_bytes()"; return B2CNN_ESTATE;
    }
    return B2CNN_OK;
}

int slide_export(const Slide *s, const ConvWeights &cw, const int *patients, int64_t k, float *feats, float *tails, int64_t *seen_host,
                 float *lstm, b2cnn_slide_state_header *hdr, void *ws, int64_t ws_bytes, cudaStream_t st, const char **err) {
    int rc = check_state_args(*s, patients, k, feats, tails, seen_host, lstm, ws, ws_bytes, err);
    if (rc != B2CNN_OK) return rc;
    if (k > 0 && (rc = launch_state<true>(*s, patients, k, nullptr, feats, nullptr, tails, nullptr, lstm, ws, st, err)) != B2CNN_OK)
        return rc;
    // the host mirror: the counts need no device read (before any lifecycle call every patient has seen n S samples)
    for (int64_t j = 0; j < k; ++j) seen_host[j] = s->lifecycle ? s->seen_h[patients[j]] : s->n * s->S;
    slide_describe_state(s, cw, hdr);
    return B2CNN_OK;
}

int slide_import(Slide *s, const ConvWeights &cw, const int *patients, int64_t k, const b2cnn_slide_state_header &hdr, const float *feats,
                 const float *tails, const int64_t *seen_host, const float *lstm, void *ws, int64_t ws_bytes, cudaStream_t st,
                 const char **err) {
    if (hdr.magic != B2CNN_SLIDE_STATE_MAGIC || hdr.version != B2CNN_SLIDE_STATE_VERSION) {
        *err = "not a scorer state header of this version (magic, version)"; return B2CNN_EINVAL;
    }
    b2cnn_slide_state_header mine;
    slide_describe_state(s, cw, &mine);
    if (hdr.path != mine.path || hdr.dtype != mine.dtype || hdr.in_channels != mine.in_channels || hdr.window != mine.window ||
        hdr.lstm_input != mine.lstm_input || hdr.feature_stride != mine.feature_stride || hdr.tail_len != mine.tail_len) {
        *err = "the state's path, dtype, in_channels, window, lstm_input, feature stride or tail length is not the scorer's";
        return B2CNN_EINVAL;
    }
    if (hdr.frontend_digest != mine.frontend_digest) {
        *err = "the state's features come from other front-end weights than the handle's (conv / affine digest differs)";
        return B2CNN_ESTATE;
    }
    int rc = check_state_args(*s, patients, k, feats, tails, seen_host, lstm, ws, ws_bytes, err);
    if (rc != B2CNN_OK) return rc;
    for (int64_t j = 0; j < k; ++j)
        if (seen_host[j] < -1) { *err = "a sample count below -1"; return B2CNN_EINVAL; }
    if (k == 0) return B2CNN_OK;
    if ((rc = launch_state<false>(*s, patients, k, feats, nullptr, tails, nullptr, lstm, nullptr, ws, st, err)) != B2CNN_OK) return rc;
    std::vector<int64_t> next = next_seen(*s, patients, 0, 0);
    for (int64_t j = 0; j < k; ++j) next[patients[j]] = seen_host[j];
    if ((rc = commit_seen(s, next, st, err)) != B2CNN_OK) return rc;
    // as after an admission with a full history: the next push computes the seam features from the window's last one on
    const int64_t g_hi = fdiv(s->n * s->S - s->R - s->phi, s->F);
    if (g_hi < s->g_done) s->g_done = g_hi;
    return B2CNN_OK;
}

}  // namespace b2cnn

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
//     the LSTM cells, Linear, age scale and sigmoid.
//
// Per-patient lifecycle (b2cnn_slide_admit / _discharge): seen[p] counts patient p's samples since its admission (-1:
// discharged); its window after a push is the last W samples of (history | pushes since admission), defined once
// seen[p] >= W.  An admission with history is a push of the listed patients aimed at a k-patient scratch ring (the same
// tensor-core / exact kernels), scattered into their ring columns, plus their tail.  Pushes then run unchanged for all
// P patients; slide_live_kernel advances seen and writes NaN for patients without a complete window.  None of this
// runs for a scorer that never admitted or discharged a patient since its last reset.
//
// All of the above is the tensor-core path.  The generic path (slide_create_generic, "generic path" below) runs the
// same ring and lifecycle for every geometry on exact CUDA-core kernels, with F = pool_s^2 in place of 4.
#include <algorithm>
#include <cstring>
#include <new>
#include <vector>

#include "b2cnn_slide.cuh"
#include "b2cnn_tc_ptx.cuh"

namespace b2cnn {

constexpr int kSlideTail = 24;       // stream samples kept per patient and channel: the largest receptive field

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
};

static int64_t fdiv4(int64_t a) { return a >= 0 ? a / 4 : -((-a + 3) / 4); }
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

// new tail = the last kSlideTail samples of (old tail | segment)
template <typename Tin>
__global__ void slide_tail_kernel(const Tin *__restrict__ x, int64_t pitch, int S, const float *__restrict__ tin,
                                  float *__restrict__ tout, int64_t rows) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= rows * kSlideTail) return;
    const int64_t r = e / kSlideTail;
    const int u = S + (int)(e % kSlideTail);
    tout[e] = u < kSlideTail ? tin[r * kSlideTail + u] : ld_sample<Tin>(x + r * pitch + (u - kSlideTail));
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
// weights of window positions r F + 16 m - foff + k (k < 16), zero outside the range.  CTA = (128 patients, range):
//   warp 4: TMA producer -- per chunk one {128 patients x 16 slots} fp32 box of the ring at the chunk's first slot and,
//           when the 16 slots wrap past L, a second box at slot 0; plus the 6 KB W_ih chunk (bulk copy); two stages;
//   warps 0-3: thread == patient: the chunk's 16 features (0 outside the range) split into three bf16 pieces written
//           as the K-major A tile, then 2 row halves x 6 m64n64k16 piece pairs (hh hm mh hl lh mm, fp32-equivalent
//           products, as the fused kernel) accumulating partial[range][patient][64] in registers.
constexpr int kRpThreads = 160;
constexpr int kRpM = 128;                            // patients per CTA
constexpr int kRpBox = 16 * kRpM * 4;                // one TMA box: 16 slots x 128 patients fp32
constexpr int kRpWChunk = 3 * 64 * 16 * 2;           // a packed W_ih chunk (tc_pack_wih_kernel, kFuWChunkBytes)
constexpr int kRpPiece = kRpM * 16 * 2;              // one bf16 piece of the A tile
constexpr size_t kRpSmem = 1024 + 2 * 2 * kRpBox + 2 * kRpWChunk + 3 * kRpPiece + 64;

struct RingProjParams {
    const uint8_t *wpack;            // [n_ranges][chunks_per_cta][kRpWChunk]
    float *partial;                  // [n_ranges][P][64]
    int P, L, head, feats_per_cta, chunks_per_cta, foff;
};

__global__ void __launch_bounds__(kRpThreads, 1)
slide_ring_proj_kernel(const __grid_constant__ CUtensorMap tm, const __grid_constant__ RingProjParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    float *sF = reinterpret_cast<float *>(smem);                  // [2 stages][2 boxes][16][128]
    uint8_t *sW = smem + 2 * 2 * kRpBox;                           // [2 stages][6 KB]
    uint8_t *sPc = sW + 2 * kRpWChunk;                             // [3 pieces][4 KB]
    uint64_t *bars = reinterpret_cast<uint64_t *>(sPc + 3 * kRpPiece);
    const uint32_t bar_full = smem_u32(bars + 0), bar_empty = smem_u32(bars + 2);
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
    const int lane = threadIdx.x & 31;
    const int b0 = blockIdx.x * kRpM;
    const int lo = blockIdx.y * p.feats_per_cta, hi = min(p.L, lo + p.feats_per_cta);
    const int nch = p.chunks_per_cta;
    if (threadIdx.x == 0) {
        for (int i = 0; i < 2; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // ring slot of the chunk's first window position (which may lie before 0 or past L: those features are masked)
    auto first_slot = [&](int m) {
        int s = (p.head + lo + 16 * m - p.foff) % p.L;
        return s < 0 ? s + p.L : s;
    };
    if (warp == 4) {
        if (lane == 0) {
            for (int m = 0; m < nch; ++m) {
                const int u = m & 1;
                mbar_wait(bar_empty + 8 * u, ((m >> 1) & 1) ^ 1);
                const int s0 = first_slot(m);
                const bool wraps = s0 + 16 > p.L;
                mbar_expect_tx(bar_full + 8 * u, (wraps ? 2 : 1) * kRpBox + kRpWChunk);
                const uint32_t dst = smem_u32(sF + (size_t)u * 2 * 16 * kRpM);
                tma_load_2d(dst, &tm, b0, s0, bar_full + 8 * u);
                if (wraps) tma_load_2d(dst + kRpBox, &tm, b0, 0, bar_full + 8 * u);
                bulk_load_1d(smem_u32(sW + u * kRpWChunk), p.wpack + ((size_t)blockIdx.y * nch + m) * kRpWChunk, kRpWChunk,
                             bar_full + 8 * u);
            }
        }
        return;
    }
    const int row = threadIdx.x;
    float gacc[2][32];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 32; ++i) gacc[h][i] = 0.f;
    uint8_t *arow = sPc + (row >> 3) * 256 + (row & 7) * 16;
#pragma unroll 1
    for (int m = 0; m < nch; ++m) {
        const int u = m & 1;
        mbar_wait(bar_full + 8 * u, (m >> 1) & 1);
        const int s0 = first_slot(m), q0 = lo + 16 * m - p.foff;
        const float *fa = sF + (size_t)u * 2 * 16 * kRpM, *fb = fa + 16 * kRpM;
        auto feat = [&](int k) {
            const int q = q0 + k;
            if (q < lo || q >= hi) return 0.f;
            return s0 + k < p.L ? fa[k * kRpM + row] : fb[(s0 + k - p.L) * kRpM + row];
        };
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
            const float f0 = feat(2 * kk), f1 = feat(2 * kk + 1);
            const uint32_t h = pack_bf16x2(f0, f1);
            const float r1x = f0 - __uint_as_float(h << 16), r1y = f1 - __uint_as_float(h & 0xffff0000u);
            const uint32_t md = pack_bf16x2(r1x, r1y);
            const uint32_t lw = pack_bf16x2(r1x - __uint_as_float(md << 16), r1y - __uint_as_float(md & 0xffff0000u));
            const int off = (kk >> 2) * 128 + (kk & 3) * 4;
            *reinterpret_cast<uint32_t *>(arow + off) = h;
            *reinterpret_cast<uint32_t *>(arow + kRpPiece + off) = md;
            *reinterpret_cast<uint32_t *>(arow + 2 * kRpPiece + off) = lw;
        }
        fence_proxy_async();
        wg_bar();
        const uint32_t pa = smem_u32(sPc), pw = smem_u32(sW + u * kRpWChunk);
        wgmma_fence();
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            constexpr int kAp[6] = {0, 0, 1, 0, 2, 1}, kWp[6] = {0, 1, 0, 2, 0, 1};
#pragma unroll
            for (int q = 0; q < 6; ++q)
                wgmma_m64n64(gacc[hh], gdesc_none_kmajor(pa + kAp[q] * kRpPiece + hh * 2048, 128, 256),
                             gdesc_none_kmajor(pw + kWp[q] * 2048, 128, 256));
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * u);
        wg_bar();                                                  // A tile free for the next chunk
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) {
            const int bb = b0 + 64 * hh + 16 * warp + (lane >> 2) + 8 * e2;
            if (bb < p.P) {
                float *dst = p.partial + ((int64_t)blockIdx.y * p.P + bb) * kGates + 2 * (lane & 3);
#pragma unroll
                for (int e = 2 * e2; e < 32; e += 4)
                    *reinterpret_cast<float2 *>(dst + 8 * (e >> 2)) = make_float2(gacc[hh][e], gacc[hh][e + 1]);
            }
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

// tail rows of the admitted patients = the last kSlideTail samples of their history [k][C][pitch] (zeros in front of
// a shorter one: they only reach features that start before the history, which no valid window holds)
template <typename Tin>
__global__ void slide_admit_tail_kernel(const Tin *__restrict__ h, int64_t pitch, int64_t H, const int *__restrict__ idx, int k,
                                        int C, float *__restrict__ tail) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)k * C * kSlideTail) return;
    const int64_t r = e / kSlideTail;                     // history row j * C + c
    const int u = (int)(e % kSlideTail);
    const int64_t t = H - kSlideTail + u;
    tail[((int64_t)idx[r / C] * C + r % C) * kSlideTail + u] = t >= 0 ? ld_sample<Tin>(h + r * pitch + t) : 0.f;
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

// ---- generic path kernels: tails of any length T ------------------------------------------------------------------
// new tail = the last T samples of (old tail | segment)
template <typename Tin>
__global__ void slide_gtail_kernel(const Tin *__restrict__ x, int64_t pitch, int S, int T, const float *__restrict__ tin,
                                   float *__restrict__ tout, int64_t rows) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= rows * T) return;
    const int64_t r = e / T;
    const int64_t u = S + e % T;
    tout[e] = u < T ? tin[r * T + u] : ld_sample<Tin>(x + r * pitch + (u - T));
}

// seam rows [rows][T + n] fp32: the tail's T samples, then the segment's first n
template <typename Tin>
__global__ void slide_seam_rows_kernel(const Tin *__restrict__ x, int64_t pitch, const float *__restrict__ tail, int T, int n,
                                       float *__restrict__ dst, int64_t rows) {
    const int64_t w = T + n, total = rows * w;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / w, i = e - r * w;
        dst[e] = i < T ? tail[r * T + i] : ld_sample<Tin>(x + r * pitch + (i - T));
    }
}

// tail rows of the admitted patients = the last T samples of their history (zeros in front of a shorter one)
template <typename Tin>
__global__ void slide_admit_gtail_kernel(const Tin *__restrict__ h, int64_t pitch, int64_t H, const int *__restrict__ idx, int k,
                                         int C, int T, float *__restrict__ tail) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)k * C * T) return;
    const int64_t r = e / T;                               // history row j * C + c
    const int64_t u = e % T;
    const int64_t t = H - T + u;
    tail[((int64_t)idx[r / C] * C + r % C) * T + u] = t >= 0 ? ld_sample<Tin>(h + r * pitch + t) : 0.f;
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

// features [g0, g0 + ng) of the pushed segment exactly into the scorer's ring: of every patient (list == nullptr) or
// of the listed ones
static int launch_exact(const Slide &s, const ConvWeights &cw, const void *x, int64_t pitch, const float *tail, int64_t g0,
                        int64_t ng, const int *list, const int *count, cudaStream_t st, const char **err) {
    SlideExactParams p;
    memset(&p, 0, sizeof p);
    p.x = x; p.pitch = pitch; p.tail = tail; p.ring = s.ring; p.ring_pitch = s.ring_pitch; p.cap = s.d.L; p.P = s.P;
    p.g0 = g0; p.seg0 = s.n * s.S; p.phi = s.phi; p.list = list; p.count = count; p.cw = cw;
    return launch_exact_p(p, s, ng, st, err);
}

// ---- generic path: every geometry, exact fp32 on CUDA cores --------------------------------------------------------
// Lattice of a conv/pool geometry: feature stride F = pool_s^2, receptive field R = pool_s (pool_k + k2 - 2) + pool_k +
// k1 - 1 (L = (W - R) / F + 1), phase phi = (-W) mod F; stream feature g reads samples F g + phi .. F g + phi + R - 1.
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

int slide_create_generic(const Dims &d, int n_patients, int stride, int dtype, int device, int num_sms, Slide **out,
                         const char **err) {
    *out = nullptr;
    if (dtype != B2CNN_DTYPE_F32 && dtype != B2CNN_DTYPE_BF16) { *err = "dtype must be f32 (0) or bf16 (1)"; return B2CNN_EINVAL; }
    if (n_patients < 1 || n_patients > (1 << 24)) { *err = "n_patients out of range"; return B2CNN_EINVAL; }
    if (stride < 1 || stride > d.W) { *err = "stride must be in [1, window]"; return B2CNN_EINVAL; }
    const int F = d.PS * d.PS, R = d.PS * (d.PK + d.K2 - 2) + d.PK + d.K1 - 1;
    if (stride % F != 0) { *err = "stride must be a multiple of the feature stride (pool_s^2 samples)"; return B2CNN_EINVAL; }
    if (d.W < R || d.L != (d.W - R) / F + 1) { *err = "the feature lattice does not match the window's feature count"; return B2CNN_EARCH; }
    if (!frontend_generic_fits(d)) {
        *err = "the generic front end's tile does not fit shared memory (in_channels * pool_s^2 too large for this window length)";
        return B2CNN_EARCH;
    }
    Slide *s = new (std::nothrow) Slide();
    if (!s) { *err = "out of host memory"; return B2CNN_ESTATE; }
    s->device = device; s->d = d; s->P = n_patients; s->S = stride; s->dtype = dtype;
    s->path = B2CNN_PATH_GENERIC; s->F = F; s->R = R; s->T = std::max(R - 1, 1); s->num_sms = num_sms;
    s->phi = (F - d.W % F) % F;
    s->ranges = proj_slices(d.L);
    s->ring_pitch = (n_patients + 3) & ~3;
    s->Sp = s->T + std::min(stride, s->T);
    const int64_t P = n_patients;
    bool ok = cudaMalloc(&s->ring, sizeof(float) * (size_t)d.L * s->ring_pitch) == cudaSuccess &&
              cudaMalloc(&s->tail, sizeof(float) * (size_t)2 * P * d.C * s->T) == cudaSuccess &&
              cudaMalloc(&s->partial, sizeof(float) * (size_t)s->ranges * P * kGates) == cudaSuccess &&
              cudaMalloc(&s->gates, sizeof(float) * (size_t)P * kGates) == cudaSuccess &&
              cudaMalloc(&s->stage, sizeof(float) * (size_t)(P * d.C * s->Sp)) == cudaSuccess &&
              cudaMalloc(&s->seen, sizeof(int64_t) * (size_t)P) == cudaSuccess;
    if (!ok) { (void)cudaGetLastError(); slide_destroy(s); *err = "cudaMalloc(scorer state)"; return B2CNN_ECUDA; }
    *out = s;
    return B2CNN_OK;
}

static int score_windows(Slide *s, const HeadWeights &hw, const TcState *tc, const float *age, int64_t n_age, int apply_sigmoid,
                         float *out, int *emitted, int64_t *window_index, cudaEvent_t *ev, cudaStream_t st, const char **err);

static int slide_push_generic(Slide *s, const ConvWeights &cw, const HeadWeights &hw, const void *x, int64_t pitch, const float *age,
                              int64_t n_age, int apply_sigmoid, float *out, int *emitted, int64_t *window_index, cudaEvent_t *ev,
                              cudaStream_t st, const char **err) {
    const Dims &d = s->d;
    const int64_t P = s->P, S = s->S, T = s->T;
    if (pitch < S || pitch > 0x7fffffff) { *err = "pitch must be in [stride, 2^31)"; return B2CNN_EINVAL; }
    if (n_age != 1 && n_age != P) { *err = "age must have 1 or n_patients elements"; return B2CNN_EINVAL; }
    const int64_t n1 = s->n + 1, seg0 = s->n * S;
    const int64_t g_hi = fdiv(n1 * S - s->R - s->phi, s->F);   // last feature whose samples have all arrived
    const int64_t g_m0 = seg0 / s->F;                           // first feature that starts inside the segment
    const int64_t g_lo = std::max(s->g_done + 1, window_head(*s, n1));   // earlier features never enter a window
    const float *tail_in = s->tail + (size_t)s->tail_cur * P * d.C * T;
    float *tail_out = s->tail + (size_t)(s->tail_cur ^ 1) * P * d.C * T;
    if (ev && cudaEventRecord(ev[0], st) != cudaSuccess) { *err = "cudaEventRecord"; return B2CNN_ECUDA; }
    // ---- main features [g_m0, g_hi], straight from the segment (feature g_m0 starts at its sample phi)
    if (g_hi >= g_m0 &&
        ring_front(*s, cw, x, s->dtype, pitch, P, s->phi, g_m0, g_hi - g_m0 + 1, s->ring, s->ring_pitch, d.L, st, err) < 0)
        return B2CNN_ECUDA;
    // ---- seam features [g_lo, min(g_hi, g_m0 - 1)]: they start in the last T samples before the segment and end in its
    // first min(S, T) (F g_lo + phi >= seg0 - T: g_lo - 1 is at most the last feature complete before this push)
    const int64_t seam_hi = std::min(g_hi, g_m0 - 1);
    if (seam_hi >= g_lo) {
        const int64_t rows = P * d.C, total = rows * s->Sp;
        const unsigned blocks = (unsigned)std::min<int64_t>((total + 255) / 256, 65536);
        const int nseg = (int)(s->Sp - T);
        if (s->dtype == B2CNN_DTYPE_BF16)
            slide_seam_rows_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16 *>(x), pitch, tail_in,
                                                                          (int)T, nseg, reinterpret_cast<float *>(s->stage), rows);
        else
            slide_seam_rows_kernel<float><<<blocks, 256, 0, st>>>(reinterpret_cast<const float *>(x), pitch, tail_in, (int)T, nseg,
                                                                  reinterpret_cast<float *>(s->stage), rows);
        if (cudaGetLastError() != cudaSuccess) { *err = "seam rows launch"; return B2CNN_ECUDA; }
        if (ring_front(*s, cw, s->stage, B2CNN_DTYPE_F32, s->Sp, P, s->F * g_lo + s->phi - seg0 + T, g_lo, seam_hi - g_lo + 1, s->ring,
                       s->ring_pitch, d.L, st, err) < 0)
            return B2CNN_ECUDA;
    }
    {
        const int64_t rows = P * d.C, total = rows * T;
        if (s->dtype == B2CNN_DTYPE_BF16)
            slide_gtail_kernel<__nv_bfloat16><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
                reinterpret_cast<const __nv_bfloat16 *>(x), pitch, (int)S, (int)T, tail_in, tail_out, rows);
        else
            slide_gtail_kernel<float><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float *>(x), pitch, (int)S,
                                                                                     (int)T, tail_in, tail_out, rows);
        if (cudaGetLastError() != cudaSuccess) { *err = "tail launch"; return B2CNN_ECUDA; }
    }
    if (ev && cudaEventRecord(ev[1], st) != cudaSuccess) { *err = "cudaEventRecord"; return B2CNN_ECUDA; }
    s->n = n1;
    if (g_hi >= g_lo) s->g_done = g_hi;
    s->tail_cur ^= 1;
    return score_windows(s, hw, nullptr, age, n_age, apply_sigmoid, out, emitted, window_index, ev, st, err);
}

int slide_create(const Dims &d, const TcState &tc, int n_patients, int stride, int dtype, int device, Slide **out,
                 const char **err) {
    *out = nullptr;
    if (dtype != B2CNN_DTYPE_F32 && dtype != B2CNN_DTYPE_BF16) { *err = "dtype must be f32 (0) or bf16 (1)"; return B2CNN_EINVAL; }
    if (n_patients < 1 || n_patients > (1 << 24)) { *err = "n_patients out of range"; return B2CNN_EINVAL; }
    if (stride < 1 || stride > d.W) { *err = "stride must be in [1, window]"; return B2CNN_EINVAL; }
    if (stride % 4 != 0) { *err = "stride must be a multiple of the feature stride (4 samples)"; return B2CNN_EINVAL; }
    if (!tc.fused) {
        *err = "the sliding-window scorer covers the streaming tensor-core geometries only (MyCNN5 or MyCNN2/3/4 conv/pool, "
               "1 to 3 channels, tanh, no affine)";
        return B2CNN_EARCH;
    }
    Slide *s = new (std::nothrow) Slide();
    if (!s) { *err = "out of host memory"; return B2CNN_ESTATE; }
    s->device = device; s->d = d; s->P = n_patients; s->S = stride; s->dtype = dtype;
    s->R = d.K1 == 10 ? 24 : 16;
    s->phi = (4 - d.W % 4) % 4;
    s->ranges = tc.n_ranges;
    s->ring_pitch = (n_patients + 3) & ~3;
    s->Sp = (stride + 7) & ~7;
    const int64_t P = n_patients, esz = dtype == B2CNN_DTYPE_BF16 ? 2 : 4;
    bool ok = cudaMalloc(&s->ring, sizeof(float) * (size_t)d.L * s->ring_pitch) == cudaSuccess &&
              cudaMalloc(&s->tail, sizeof(float) * (size_t)2 * P * d.C * kSlideTail) == cudaSuccess &&
              cudaMalloc(&s->partial, sizeof(float) * (size_t)s->ranges * P * kGates) == cudaSuccess &&
              cudaMalloc(&s->flags, sizeof(int) * (size_t)(2 * P + 1)) == cudaSuccess &&
              cudaMalloc(&s->stage, (size_t)(P * d.C * s->Sp * esz)) == cudaSuccess &&
              cudaMalloc(&s->seen, sizeof(int64_t) * (size_t)P) == cudaSuccess;
    if (!ok) { (void)cudaGetLastError(); slide_destroy(s); *err = "cudaMalloc(scorer state)"; return B2CNN_ECUDA; }
    *out = s;
    return B2CNN_OK;
}

void slide_destroy(Slide *s) {
    if (!s) return;
    cudaFree(s->ring); cudaFree(s->tail); cudaFree(s->partial); cudaFree(s->gates); cudaFree(s->flags); cudaFree(s->stage);
    cudaFree(s->seen);
    delete s;
}

int slide_device(const Slide *s) { return s->device; }
int slide_dtype(const Slide *s) { return s->dtype; }
int slide_path(const Slide *s) { return s->path; }

int slide_reset(Slide *s, cudaStream_t st, const char **err) {
    s->n = 0; s->g_done = -1; s->tail_cur = 0; s->lifecycle = false;
    if (cudaMemsetAsync(s->tail, 0, sizeof(float) * (size_t)2 * s->P * s->d.C * s->T, st) != cudaSuccess) {
        *err = "memset tail"; return B2CNN_ECUDA;
    }
    return B2CNN_OK;
}

static int64_t window_head(const Slide &s, int64_t n) { return fdiv(n * s.S - s.d.W - s.phi, s.F); }

// slide_live_kernel over the P patients: seen += adv, then NaN rows of x [P][len] without a complete window
static int launch_live(const Slide &s, int64_t adv, float *x, int64_t len, cudaStream_t st, const char **err) {
    const unsigned gy = adv != 0 || len <= 1 ? 1u : (unsigned)std::min<int64_t>(len, 64);
    slide_live_kernel<<<dim3((unsigned)((s.P + 127) / 128), gy), 128, 0, st>>>(s.seen, s.P, adv, s.d.W, x, len);
    if (cudaGetLastError() != cudaSuccess) { *err = "lifecycle mask launch"; return -1; }
    return 1;
}

// a push's lifecycle step: the device counts advance by S (and out[P] gets its NaNs), then the host mirror -- only once
// the launch went out, so that the two never disagree
static int advance_seen(Slide *s, float *out, cudaStream_t st, const char **err) {
    if (launch_live(*s, s->S, out, 1, st, err) < 0) return -1;
    for (int64_t &v : s->seen_h)
        if (v >= 0) v += s->S;
    return 1;
}

int slide_push(Slide *s, const ConvWeights &cw, const HeadWeights &hw, const TcState &tc, const void *x, int64_t pitch,
               const float *age, int64_t n_age, int apply_sigmoid, float *out, int *emitted, int64_t *window_index,
               cudaEvent_t *ev, cudaStream_t st, const char **err) {
    if (s->path == B2CNN_PATH_GENERIC)
        return slide_push_generic(s, cw, hw, x, pitch, age, n_age, apply_sigmoid, out, emitted, window_index, ev, st, err);
    const Dims &d = s->d;
    const int64_t P = s->P, S = s->S, esz = s->dtype == B2CNN_DTYPE_BF16 ? 2 : 4;
    if (pitch < S) { *err = "pitch must be >= stride"; return B2CNN_EINVAL; }
    if (n_age != 1 && n_age != P) { *err = "age must have 1 or n_patients elements"; return B2CNN_EINVAL; }
    if (tc.n_ranges != s->ranges) { *err = "the handle's position ranges changed since create"; return B2CNN_ESTATE; }
    const int64_t n1 = s->n + 1;
    const int64_t g_hi = fdiv4(n1 * S - s->R - s->phi);      // last feature whose samples have all arrived
    const int64_t g_m0 = s->n * S / 4;                        // first feature that starts inside the segment
    int64_t g_lo = s->g_done + 1;
    const int64_t G = window_head(*s, n1);
    if (g_lo < G) g_lo = G;                                   // earlier features never enter a window
    const float *tail_in = s->tail + (size_t)s->tail_cur * P * d.C * kSlideTail;
    float *tail_out = s->tail + (size_t)(s->tail_cur ^ 1) * P * d.C * kSlideTail;
    if (ev && cudaEventRecord(ev[0], st) != cudaSuccess) { *err = "cudaEventRecord"; return B2CNN_ECUDA; }

    // ---- main features [g_m0, g_hi]: tensor cores from the segment, exact re-computation of flagged patients
    const int64_t Q = g_hi - g_m0 + 1;
    if (Q >= 32) {
        const int unit = 16 / (int)esz;
        const void *xin = x;
        int64_t xp = pitch;
        if (s->phi != 0 || pitch % unit != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0) {
            const int64_t rows = P * d.C;
            const unsigned blocks = (unsigned)((rows * s->Sp + 255) / 256 < 65536 ? (rows * s->Sp + 255) / 256 : 65536);
            if (esz == 2)
                slide_stage_kernel<uint16_t><<<blocks, 256, 0, st>>>(reinterpret_cast<const uint16_t *>(x), pitch, s->phi, (int)(S - s->phi),
                                                                     reinterpret_cast<uint16_t *>(s->stage), s->Sp, rows);
            else
                slide_stage_kernel<float><<<blocks, 256, 0, st>>>(reinterpret_cast<const float *>(x), pitch, s->phi, (int)(S - s->phi),
                                                                  reinterpret_cast<float *>(s->stage), s->Sp, rows);
            if (cudaGetLastError() != cudaSuccess) { *err = "staging launch"; return B2CNN_ECUDA; }
            xin = s->stage; xp = s->Sp;
        }
        Dims dseg = d;
        dseg.W = (int)(S - s->phi); dseg.L = (int)Q; dseg.XP = (int)xp;
        if (cudaMemsetAsync(s->flags, 0, sizeof(int) * (size_t)(2 * P + 1), st) != cudaSuccess) { *err = "memset flags"; return B2CNN_ECUDA; }
        if (tc_ring_features(tc, dseg, cw, xin, xp, s->dtype, P, s->ring, s->ring_pitch, d.L, (int)(g_m0 % d.L), s->flags, st, err) < 0)
            return B2CNN_ECUDA;
        if (launch_exact(*s, cw, x, pitch, tail_in, g_m0, Q, s->flags + P, s->flags + 2 * P, st, err) < 0) return B2CNN_ECUDA;
    } else if (launch_exact(*s, cw, x, pitch, tail_in, g_m0, Q, nullptr, nullptr, st, err) < 0) {
        return B2CNN_ECUDA;
    }
    // ---- seam features [g_lo, g_m0 - 1]: receptive field starts in the previous push
    const int64_t seam_hi = g_hi < g_m0 - 1 ? g_hi : g_m0 - 1;
    if (launch_exact(*s, cw, x, pitch, tail_in, g_lo, seam_hi - g_lo + 1, nullptr, nullptr, st, err) < 0) return B2CNN_ECUDA;
    {
        const int64_t rows = P * d.C, total = rows * kSlideTail;
        if (esz == 2)
            slide_tail_kernel<__nv_bfloat16><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
                reinterpret_cast<const __nv_bfloat16 *>(x), pitch, (int)S, tail_in, tail_out, rows);
        else
            slide_tail_kernel<float><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float *>(x), pitch, (int)S,
                                                                                    tail_in, tail_out, rows);
        if (cudaGetLastError() != cudaSuccess) { *err = "tail launch"; return B2CNN_ECUDA; }
    }
    if (ev && cudaEventRecord(ev[1], st) != cudaSuccess) { *err = "cudaEventRecord"; return B2CNN_ECUDA; }
    s->n = n1;
    if (g_hi >= g_lo) s->g_done = g_hi;
    s->tail_cur ^= 1;
    return score_windows(s, hw, &tc, age, n_age, apply_sigmoid, out, emitted, window_index, ev, st, err);
}

// the end of push n = s->n: projection over the ring + head, once a window is complete (every patient's, or with the
// lifecycle on, one); on tensor cores with `tc`, else (generic path) on CUDA cores
static int score_windows(Slide *s, const HeadWeights &hw, const TcState *tc, const float *age, int64_t n_age, int apply_sigmoid,
                         float *out, int *emitted, int64_t *window_index, cudaEvent_t *ev, cudaStream_t st, const char **err) {
    const Dims &d = s->d;
    const int64_t P = s->P, S = s->S, n1 = s->n;
    bool live = n1 * S >= d.W;
    if (s->lifecycle)
        live = std::any_of(s->seen_h.begin(), s->seen_h.end(), [&](int64_t v) { return v >= 0 && v + S >= d.W; });
    *emitted = 0;
    if (!live) {
        if (s->lifecycle && advance_seen(s, nullptr, st, err) < 0) return B2CNN_ECUDA;
        if (ev && cudaEventRecord(ev[2], st) != cudaSuccess) { *err = "cudaEventRecord"; return B2CNN_ECUDA; }
        return B2CNN_OK;
    }
    const int head = (int)mod_nn(window_head(*s, n1), d.L);
    if (!tc) {
        if (launch_ring_head(d, hw, s->ring, s->ring_pitch, head, P, age, n_age, apply_sigmoid, out, s->gates, s->partial, st, err) < 0)
            return B2CNN_ECUDA;
    } else {
        CUtensorMap tm;
        if (tc_ring_tmap(s->ring, P, s->ring_pitch, d.L, &tm, err) != 0) return B2CNN_ECUDA;
        RingProjParams rp;
        rp.wpack = reinterpret_cast<const uint8_t *>(tc->d_wpack); rp.partial = s->partial;
        rp.P = (int)P; rp.L = d.L; rp.head = head;
        rp.feats_per_cta = tc->feats_per_cta; rp.chunks_per_cta = tc->chunks_per_cta; rp.foff = d.K1 == 10 ? 3 : 2;
        if (cudaFuncSetAttribute(slide_ring_proj_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRpSmem) != cudaSuccess) {
            *err = "projection smem attribute"; return B2CNN_ECUDA;
        }
        slide_ring_proj_kernel<<<dim3((unsigned)((P + kRpM - 1) / kRpM), (unsigned)s->ranges), kRpThreads, kRpSmem, st>>>(tm, rp);
        if (cudaGetLastError() != cudaSuccess) { *err = "projection launch"; return B2CNN_ECUDA; }
        if (launch_reduce_lstm_head(d, hw, s->partial, s->ranges, P, age, n_age, apply_sigmoid, out, st, err) < 0) return B2CNN_ECUDA;
    }
    if (s->lifecycle && advance_seen(s, out, st, err) < 0) return B2CNN_ECUDA;
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
    if (s->lifecycle && launch_live(*s, 0, feats, s->d.L, st, err) < 0) return B2CNN_ECUDA;
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
static size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }
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
                int64_t pitch, void *ws, int64_t ws_bytes, cudaStream_t st, const char **err) {
    const Dims &d = s->d;
    int rc = check_patients(*s, patients, k, err);
    if (rc != B2CNN_OK) return rc;
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
    const int64_t esz = s->dtype == B2CNN_DTYPE_BF16 ? 2 : 4;
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
        const int cap = (int)Q;                                        // Q <= a.cap
        const int64_t off = 4 * g_lo + s->phi - (nS - H);               // (H - W) mod 4 + 4 (g_lo - first feature inside)
        SlideExactParams p;
        memset(&p, 0, sizeof p);
        p.x = hist; p.pitch = pitch; p.tail = s->tail; p.ring = scratch; p.ring_pitch = a.kp; p.cap = cap; p.P = (int)k;
        p.g0 = g_lo; p.seg0 = nS - H; p.phi = s->phi; p.cw = cw;
        if (Q >= 32) {
            const int unit = 16 / (int)esz;
            const void *xin = hist;
            int64_t xp = pitch;
            if (off != 0 || pitch % unit != 0 || (reinterpret_cast<uintptr_t>(hist) & 15) != 0) {
                const int64_t rows = k * d.C;
                const unsigned blocks = (unsigned)std::min<int64_t>((rows * a.hp + 255) / 256, 65536);
                if (esz == 2)
                    slide_stage_kernel<uint16_t><<<blocks, 256, 0, st>>>(reinterpret_cast<const uint16_t *>(hist), pitch, (int)off,
                                                                         (int)(H - off), reinterpret_cast<uint16_t *>(stage), a.hp, rows);
                else
                    slide_stage_kernel<float><<<blocks, 256, 0, st>>>(reinterpret_cast<const float *>(hist), pitch, (int)off,
                                                                      (int)(H - off), reinterpret_cast<float *>(stage), a.hp, rows);
                if (cudaGetLastError() != cudaSuccess) { *err = "staging launch"; return B2CNN_ECUDA; }
                xin = stage; xp = a.hp;
            }
            Dims dh = d;
            dh.W = (int)(H - off); dh.L = cap; dh.XP = (int)xp;
            if (cudaMemsetAsync(flags, 0, sizeof(int) * (size_t)(2 * k + 1), st) != cudaSuccess) { *err = "memset flags"; return B2CNN_ECUDA; }
            if (tc_ring_features(tc, dh, cw, xin, xp, s->dtype, k, scratch, a.kp, cap, (int)mod_nn(g_lo, cap), flags, st, err) < 0)
                return B2CNN_ECUDA;
            p.list = flags + k; p.count = flags + 2 * k;                // flagged histories: exact, over all Q features
        }
        if (launch_exact_p(p, *s, Q, st, err) < 0) return B2CNN_ECUDA;
    }
    if (H > 0 && Q > 0) {
        const unsigned gy = (unsigned)std::min<int64_t>(Q, 1024);
        slide_scatter_kernel<<<dim3((unsigned)((k + 127) / 128), gy), 128, 0, st>>>(scratch, a.kp, (int)Q, idx, (int)k, g_lo, (int)Q,
                                                                                   s->ring, s->ring_pitch, d.L);
        if (cudaGetLastError() != cudaSuccess) { *err = "scatter launch"; return B2CNN_ECUDA; }
    }
    // the next push's seam features read the history's last samples from the current tail
    float *tail = s->tail + (size_t)s->tail_cur * s->P * d.C * s->T;
    const int64_t total = k * d.C * s->T;
    if (s->path == B2CNN_PATH_GENERIC) {
        if (esz == 2)
            slide_admit_gtail_kernel<__nv_bfloat16><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
                reinterpret_cast<const __nv_bfloat16 *>(hist), pitch, H, idx, (int)k, d.C, s->T, tail);
        else
            slide_admit_gtail_kernel<float><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float *>(hist), pitch,
                                                                                             H, idx, (int)k, d.C, s->T, tail);
    } else if (esz == 2)
        slide_admit_tail_kernel<__nv_bfloat16><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
            reinterpret_cast<const __nv_bfloat16 *>(hist), pitch, H, idx, (int)k, d.C, tail);
    else
        slide_admit_tail_kernel<float><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float *>(hist), pitch, H,
                                                                                        idx, (int)k, d.C, tail);
    if (cudaGetLastError() != cudaSuccess) { *err = "tail launch"; return B2CNN_ECUDA; }
    std::vector<int64_t> next = next_seen(*s, patients, k, H);
    if ((rc = commit_seen(s, next, st, err)) != B2CNN_OK) return rc;
    // features from the history's last complete one on are seam features of the next push, for every patient (before
    // sample 0 of the stream they have negative indices: the other patients' copies of them are never read)
    if (H > 0 && g_hi < s->g_done) s->g_done = g_hi;
    return B2CNN_OK;
}

int slide_discharge(Slide *s, const int *patients, int64_t k, cudaStream_t st, const char **err) {
    const int rc = check_patients(*s, patients, k, err);
    if (rc != B2CNN_OK || k == 0) return rc;
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

}  // namespace b2cnn

// b2cnn_tc.cu -- wgmma / TMA front end for bf16 windows (sm_90a).
//
// conv1 (bin/models.py:23) is 82 % of the path's FLOPs at the headline shape [4096,3,75000]:
// 9.0 M MAC per window, which on the FP32 CUDA cores alone costs several times what the HBM
// roofline allows.  Here it runs on the tensor cores as a banded-Toeplitz GEMM whose M axis is
// the WINDOW index:
//
//   D[w, (s,o)] = sum_{c} sum_{k<16}  X_c[w, 8n+k] * T_c[k, (s,o)],   T_c[k,(s,o)] = w1[o][c][k-s]
//
//   * A = X_c: 128 windows x 32 consecutive samples of channel c, brought by ONE 3-D TMA box
//     {32 samples, 1 channel, 128 windows} into the canonical K-major SWIZZLE_64B layout; the
//     8-position block n of the tile uses the K=16 slice starting at 16-byte chunk n (descriptor
//     start address + 16n bytes), so one landed tile feeds 3 blocks = 24 conv1 positions
//     (tiles advance by 24 samples; the 8 overlapping samples are re-read from L2, not HBM).
//     The small tile keeps the kernel at about 100 KB of shared memory: two CTAs share an SM.
//   * B = T_c: the fp32 conv1 weights expanded to a 16 x 32 band matrix (8 output shifts s x 4
//     output channels o, column 8 (s/2) + 2 o + s%2, so that each lane of the accumulator fragment
//     holds every shift of one channel) and split into 2 or 3 bf16 pieces (hi/mid/lo) so that, the inputs
//     being exactly bf16, every product is exact and the fp32 accumulation carries the full
//     fp32 weight precision.  One wgmma m64n32k16 per (row half, block, channel, piece).
//   * The one tap that does not fit a 16-sample slice (s=7, k=9 -> sample 8n+16) is added by
//     the epilogue on the CUDA cores from the same shared-memory tile (12 FMA per block).
//   * Zero band entries turn an inf/NaN sample into NaN for its whole 8-position block, a
//     superset of the reference's NaNs: a window whose features contain a NaN is flagged and
//     recomputed by the exact generic kernel (b2cnn_generic.cu), still on the GPU.
// The kernel itself, its epilogue and the fused layer-0 projection are in b2cnn_tc_fused.cuh.
#include <cuda.h>

#include <cstdlib>
#include <cstring>
#include <vector>

#include "b2cnn_tc.cuh"
#include "b2cnn_tc_ptx.cuh"

namespace b2cnn {

static thread_local const char *g_tc_err = "";
const char *tc_error() { return g_tc_err; }

constexpr int64_t kOwnFlagCap = 65536;   // windows per call served by the handle's own flag state (512 KB); larger batches use the workspace copy
constexpr int kTcM = 128;          // windows per CTA (two wgmma m64 row halves)
constexpr int kTcAdv = 24;         // conv1 positions (= samples) a tile advances
constexpr int kTcBlocks = 3;       // 8-position blocks per 32-sample tile
constexpr int kTcARow = 64;        // bytes per window row of a bf16 tile (32 samples, SWIZZLE_64B)
constexpr int kTcF32ARow = 128;    // ... of an fp32 tile (32 samples, SWIZZLE_128B)
constexpr int kTcBBytes = 32 * 16 * 2;   // one band matrix piece: N=32 x K=16 bf16
constexpr int kTcMaxC = 4;

// windows flagged by the tensor-core kernel -> compact index list for the exact re-computation
__global__ void tc_compact_flags_kernel(int *flags, int B, int *list, int *count) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B && flags[b]) list[atomicAdd(count, 1)] = b;      // flags stay set: the head kernel picks the recomputed rows by them
}

}  // namespace b2cnn
#include "b2cnn_tc_fused.cuh"
namespace b2cnn {

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)ptr;
    }
    return fn;
}

static uint16_t bf16_rn(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
    u += 0x7fffu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
}
static float bf16_to_f(uint16_t h) {
    uint32_t u = (uint32_t)h << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}

// MyCNN2/3/4 geometry: fused kernel only (ARCH 1)
static bool arch1_ok(const Dims &d) {
    return d.K1 == 5 && d.K2 == 5 && d.PK == 2 && d.PS == 2 && d.C >= 1 && d.C <= 3 && d.act == B2CNN_ACT_TANH &&
           !d.has_affine && d.L >= 32;
}
static bool arch_ok(const Dims &d) {
    return d.K1 == 10 && d.K2 == 5 && d.PK == 3 && d.PS == 2 && d.C >= 1 && d.C <= kTcMaxC &&
           d.act == B2CNN_ACT_TANH && !d.has_affine && d.L >= 32;
}

static int tiles_per_cta_for(const Dims &d);

int tc_prepare(TcState &s, const Dims &d, const ConvWeights &cw, const float *d_wih0, int splits, cudaStream_t st) {
    s.features = s.fused = false;
    s.splits = splits;
    if (!arch_ok(d) && !arch1_ok(d)) return 0;   // not an error: this shape takes the generic path
    if (!get_encode()) return 0;
    if (!s.d_flagstate) {
        const int64_t cap = kOwnFlagCap;
        if (cudaMalloc(reinterpret_cast<void **>(&s.d_flagstate), sizeof(int) * (2 * cap + 16)) == cudaSuccess &&
            cudaMemset(s.d_flagstate, 0, sizeof(int) * (2 * cap + 16)) == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess) {
            s.flag_cap = cap; s.flags_clean = true;
        } else {
            cudaFree(s.d_flagstate); s.d_flagstate = nullptr; s.flag_cap = 0;    // not an error: the workspace copy is used
            (void)cudaGetLastError();
        }
    }
    // band matrices: piece sp of T_c[k][(s,o)] = w1[o][c][k-s], stored as GMMA K-major
    // no-swizzle core matrices: byte = (n/8)*256 + (k/8)*128 + (n%8)*16 + (k%8)*2, with column
    // n = 8 (s/2) + 2 o + s%2: lane l of the accumulator fragment, which holds columns 8 j + 2 (l%4) + {0, 1},
    // then holds all 8 shifts of out channel l%4 (see b2cnn_tc_fused.cuh).
    //   d_bmats   [C][3][1 KB]  three bf16 pieces (hi/mid/lo: the full 24-bit fp32 mantissa)
    //   d_bmats2  [C][2][1 KB]  the first two pieces only (16 mantissa bits; tc_splits=2, an option:
    //                           6 instead of 9 MMAs per block, weights rounded to 2^-17 relative)
    std::vector<uint16_t> host((size_t)d.C * 3 * 512, 0), host2((size_t)d.C * 2 * 512, 0);
    for (int c = 0; c < d.C; ++c)
        for (int sft = 0; sft < 8; ++sft)
            for (int o = 0; o < kCMid; ++o)
                for (int k = 0; k < 16; ++k) {
                    const int tap = k - sft;
                    if (tap < 0 || tap >= d.K1) continue;
                    float w = cw.w1[(c * d.K1 + tap) * kCMid + o];
                    const int n = 8 * (sft >> 1) + 2 * o + (sft & 1);   // column of (shift, out channel)
                    const size_t off = (size_t)(n / 8) * 128 + (k / 8) * 64 + (n % 8) * 8 + (k % 8);   // in bf16 units
                    for (int sp = 0; sp < 3; ++sp) {
                        const uint16_t piece = bf16_rn(w);
                        host[((size_t)c * 3 + sp) * 512 + off] = piece;
                        if (sp < 2) host2[((size_t)c * 2 + sp) * 512 + off] = piece;
                        w -= bf16_to_f(piece);
                    }
                }
    if (!s.d_bmats && cudaMalloc(&s.d_bmats, host.size() * 2 + 16) != cudaSuccess) { g_tc_err = "cudaMalloc(band matrices)"; return -1; }
    if (!s.d_bmats2 && cudaMalloc(&s.d_bmats2, host2.size() * 2 + 16) != cudaSuccess) { g_tc_err = "cudaMalloc(band matrices)"; return -1; }
    if (cudaMemcpyAsync(s.d_bmats, host.data(), host.size() * 2, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(s.d_bmats2, host2.data(), host2.size() * 2, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) { g_tc_err = "upload band matrices"; return -1; }
    s.features = arch_ok(d);
    // ---- fused kernels (bf16 and fp32 windows: the same 3-block tiles and ranges): W_ih_l0 packed per (range, chunk)
    s.tiles_per_cta = tiles_per_cta_for(d);
    s.feats_per_cta = 2 * kTcBlocks * s.tiles_per_cta - 4;   // even: every range starts 16-byte aligned (TMA)
    s.chunks_per_cta = (kTcBlocks * s.tiles_per_cta + 7) / 8;
    s.n_ranges = (d.L + s.feats_per_cta - 1) / s.feats_per_cta;
    if (d.C <= 3) {
        const size_t bytes = (size_t)s.n_ranges * s.chunks_per_cta * kFuWChunkBytes;
        cudaFree(s.d_wpack); s.d_wpack = nullptr;
        if (cudaMalloc(&s.d_wpack, bytes) != cudaSuccess) { g_tc_err = "cudaMalloc(packed W_ih)"; return -1; }
        const int64_t total = (int64_t)s.n_ranges * s.chunks_per_cta * 1024;
        tc_pack_wih_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(d_wih0, reinterpret_cast<uint8_t *>(s.d_wpack), d.L,
                                                                          s.feats_per_cta, s.chunks_per_cta, s.n_ranges, d.K1 == 10 ? 3 : 2);
        if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) { g_tc_err = "pack W_ih"; return -1; }
        s.fused = true;
    }
    return 0;
}

void tc_release(TcState &s) {
    cudaFree(s.d_flagstate);
    s.d_flagstate = nullptr; s.flag_cap = 0; s.flags_clean = false; s.owner_set = false;
    cudaFree(s.d_bmats);
    cudaFree(s.d_bmats2);
    cudaFree(s.d_wpack);
    s.d_bmats = nullptr;
    s.d_bmats2 = nullptr;
    s.d_wpack = nullptr;
    s.features = s.fused = false;
}

// A TMA tensor map needs a row pitch that is a multiple of 16 bytes.  bf16 windows whose pitch is not a
// multiple of 8 samples (contiguous 7500, 37500 ...) are copied once into a pitch-aligned scratch (costs one
// extra read + write of the input; W % 8 == 0, e.g. the headline 75000, streams straight from x).
static int64_t padded_w(const Dims &d) { return (d.W + 7) & ~7; }
int64_t tc_flags_bytes(int64_t B) { return ((2 * B + 64) * 4 + 255) / 256 * 256; }
int64_t tc_stage_bytes(const Dims &d, int64_t B) { return (B * d.C * padded_w(d) * 2 + 255) / 256 * 256; }

// rows of W samples, `sp` elements apart -> rows Wp (multiple of 8) apart, tail zero-filled.
// VEC 8: W % 4 == 0 and sp % 4 == 0: every row starts 8-byte aligned; one thread moves 16 output bytes with two
//        8-byte loads (a 16-byte load would be misaligned on every other row) and ONE 16-byte store.
// VEC 1: any W (2-byte accesses).
template <int VEC>
__global__ void tc_repack_rows_kernel(const uint16_t *__restrict__ src, uint16_t *__restrict__ dst, int64_t rows, int W, int64_t sp, int Wp) {
    const int per_row = Wp / VEC;
    for (int64_t r = blockIdx.y; r < rows; r += gridDim.y) {
        const uint16_t *in = src + r * sp;
        uint16_t *out = dst + r * Wp;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < per_row; i += gridDim.x * blockDim.x) {
            if (VEC == 8) {
                uint2 a = make_uint2(0u, 0u), b = make_uint2(0u, 0u);
                if (i * 8 < W) a = __ldg(reinterpret_cast<const uint2 *>(in + i * 8));
                if (i * 8 + 4 < W) b = __ldg(reinterpret_cast<const uint2 *>(in + i * 8 + 4));
                *reinterpret_cast<uint4 *>(out + i * 8) = make_uint4(a.x, a.y, b.x, b.y);
            } else {
                out[i] = i < W ? in[i] : (uint16_t)0;
            }
        }
    }
}

// returns the pointer / pitch the tensor map must describe (x itself when its rows are 16-byte aligned: W % 8 == 0
// for a contiguous tensor, or a producer that padded the row pitch -- b2cnn_forward_pitched)
static const void *tc_stage_input(const Dims &d, const void *x, int64_t B, void *scratch_after_flags, int64_t *pitch,
                                  int *launches, cudaStream_t st) {
    *pitch = d.XP;
    if ((d.XP % 8) == 0) return x;
    const int64_t rows = B * d.C;
    const int Wp = (int)padded_w(d);
    dim3 grid(4, (unsigned)(rows < 32768 ? rows : 32768));
    if (d.W % 4 == 0 && d.XP % 4 == 0)
        tc_repack_rows_kernel<8><<<grid, 256, 0, st>>>(reinterpret_cast<const uint16_t *>(x), reinterpret_cast<uint16_t *>(scratch_after_flags), rows, d.W, d.XP, Wp);
    else
        tc_repack_rows_kernel<1><<<grid, 256, 0, st>>>(reinterpret_cast<const uint16_t *>(x), reinterpret_cast<uint16_t *>(scratch_after_flags), rows, d.W, d.XP, Wp);
    *pitch = Wp;
    ++*launches;
    return scratch_after_flags;
}

static int tiles_per_cta_for(const Dims &d) {
    // About 33 position ranges per window whatever its length (depends on L only, so a window's
    // summation order never depends on the batch).  A CTA's stream emits 6*tiles - 4 features.
    // L=18745 -> 96 tiles (572 features) per CTA and 33 ranges x 32 window tiles = 1056 CTAs at B=4096:
    // 4 waves of the 264 bf16 CTAs resident on 132 SMs (two per SM), 8 waves of the fp32 kernel (one per
    // SM).  Shorter windows get proportionally shorter ranges so that small batches still fill the SMs.
    if (const char *e = getenv("B2CNN_TC_TILES")) { const int v = atoi(e); if (v >= 1 && v <= 16384) return v; }
    int nt = ((d.L + 32) / 33 + 4 + 2 * kTcBlocks - 1) / (2 * kTcBlocks);
    if (nt < 4) nt = 4;
    return nt;
}

// epilogue constants of tc_stream_kernel (conv2 consumes r = (1 - tanh)/2: sum w*(1 - 2r) = sum(w) + sum (-2w)*r)
static void fill_epilogue(TcFusedParams &p, const Dims &d, const ConvWeights &cw) {
    for (int o = 0; o < kCMid; ++o) {
        for (int c = 0; c < d.C; ++c) {
            for (int k = 0; k < d.K1; ++k) p.w1[c][k][o] = cw.w1[(c * d.K1 + k) * kCMid + o];
            p.w9[c][o] = d.K1 == 10 ? cw.w1[(c * d.K1 + 9) * kCMid + o] : 0.f;
        }
        p.b1s[o] = cw.b1[o] * k2Log2e;
        for (int k = 0; k < 5; ++k) p.w2n[o][k] = -2.f * cw.w2[o * d.K2 + k];
    }
    double sw = 0.0;
    for (int i = 0; i < kCMid * d.K2; ++i) sw += cw.w2[i];
    p.b2s = (float)((cw.b2 + sw) * (double)k2Log2e);
}

// one launch of tc_stream_kernel<C, SPLITS, ARCH, F32IN, OUT> over grid (window tiles, position ranges)
template <int C, int SPLITS, int ARCH, bool F32IN, int OUT>
static cudaError_t launch_stream(const CUtensorMap &tm, const TcFusedParams &p, dim3 grid, cudaStream_t st) {
    const size_t smem = hp_smem_bytes(C, SPLITS, F32IN, OUT);
    cudaError_t e = cudaFuncSetAttribute(tc_stream_kernel<C, SPLITS, ARCH, F32IN, OUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    tc_stream_kernel<C, SPLITS, ARCH, F32IN, OUT><<<grid, hp_threads(F32IN), smem, st>>>(tm, p);
    return cudaGetLastError();
}

static int make_tmap(const Dims &d, const void *x, int64_t pitch, int64_t B, bool f32, CUtensorMap *tm, const char **err) {
    if ((reinterpret_cast<uintptr_t>(x) & 15) != 0) { *err = "x must be 16-byte aligned for TMA"; return -1; }
    const int esz = f32 ? 4 : 2;
    cuuint64_t gdim[3] = {(cuuint64_t)d.W, (cuuint64_t)d.C, (cuuint64_t)B};
    cuuint64_t gstr[2] = {(cuuint64_t)pitch * esz, (cuuint64_t)d.C * pitch * esz};
    // 32 samples per window: one 64-byte SWIZZLE_64B row (bf16) or one 128-byte SWIZZLE_128B row (fp32)
    cuuint32_t box[3] = {32, 1, kTcM};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = get_encode()(tm, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(x),
                              gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, f32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { *err = "cuTensorMapEncodeTiled failed"; return -1; }
    return 0;
}

static int launch_tc_kernel(const TcState &s, const Dims &d, const ConvWeights &cw, const void *x, int64_t pitch, int64_t B,
                            float *feats, int64_t sB, int64_t sP, int *nanflag, cudaStream_t st, const char **err) {
    CUtensorMap tm;
    if (make_tmap(d, x, pitch, B, false, &tm, err) != 0) return -1;
    TcFusedParams p;
    memset(&p, 0, sizeof p);
    p.feats = feats; p.sB = sB; p.sP = sP; p.nanflag = nanflag;
    p.bmats = reinterpret_cast<const uint8_t *>(s.d_bmats);
    p.B = (int)B; p.W = d.W; p.L = d.L;
    // an EVEN feature count per range keeps every range's first sample (4 * p0 elements) 16-byte aligned:
    // an unaligned TMA box start faults
    p.tiles_per_cta = s.tiles_per_cta;
    p.feats_per_cta = s.feats_per_cta;
    fill_epilogue(p, d, cw);
    const int n_pr = (d.L + p.feats_per_cta - 1) / p.feats_per_cta;
    dim3 grid((unsigned)((B + kTcM - 1) / kTcM), n_pr);
    cudaError_t e;
    switch (d.C) {
        case 1: e = launch_stream<1, 3, 0, false, kOutFeatures>(tm, p, grid, st); break;
        case 2: e = launch_stream<2, 3, 0, false, kOutFeatures>(tm, p, grid, st); break;
        case 3: e = launch_stream<3, 3, 0, false, kOutFeatures>(tm, p, grid, st); break;
        case 4: e = launch_stream<4, 3, 0, false, kOutFeatures>(tm, p, grid, st); break;
        default: *err = "no tensor-core instantiation for this channel count"; return -1;
    }
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return 1;
}

// TMA/wgmma front end + NaN-flag compaction + exact re-computation of flagged windows.
// `ws`: 2*B+64 ints of scratch (flags, list, count); pass nullptr to allocate stream-ordered.
int tc_frontend(TcState &s, const Dims &d, const ConvWeights &cw, const void *x, int64_t B, float *feats,
                int64_t sB, int64_t sP, void *ws, int num_sms, cudaStream_t st, const char **err) {
    int *flags = reinterpret_cast<int *>(ws);
    const bool own = flags == nullptr;
    const int64_t own_bytes = tc_flags_bytes(B) + (d.XP % 8 ? tc_stage_bytes(d, B) : 0);
    if (own && cudaMallocAsync(&flags, (size_t)own_bytes, st) != cudaSuccess) { *err = "cudaMallocAsync"; return -1; }
    int *list = flags + B, *count = list + B;
    int launches = -1;
    if (cudaMemsetAsync(flags, 0, sizeof(int) * (2 * B + 1), st) != cudaSuccess) {
        *err = "memset flags";
    } else {
        int staged = 0;
        int64_t pitch = d.XP;
        const void *xin = tc_stage_input(d, x, B, reinterpret_cast<char *>(flags) + tc_flags_bytes(B), &pitch, &staged, st);
        int n = launch_tc_kernel(s, d, cw, xin, pitch, B, feats, sB, sP, flags, st, err);
        if (n >= 0) {
            tc_compact_flags_kernel<<<(unsigned)((B + 255) / 256), 256, 0, st>>>(flags, (int)B, list, count);
            int m = launch_frontend_generic_listed(d, cw, x, B2CNN_DTYPE_BF16, B, feats, sB, sP, list, count, st, num_sms, err);
            if (m >= 0) launches = staged + n + 1 + m;
        }
    }
    if (own) cudaFreeAsync(flags, st);
    return launches;
}

int tc_features(TcState &s, const Dims &d, const ConvWeights &cw, const void *x, int64_t B, float *feats,
                int num_sms, cudaStream_t st, const char **err) {
    // parity-test entry: row-major [B][L] features (uncoalesced stores; not a timed path)
    return tc_frontend(s, d, cw, x, B, feats, d.L, 1, nullptr, num_sms, st, err);
}

// Where this call keeps count | flags | list: the handle's own, already-zero copy (see TcState) or the head of the
// workspace, zeroed here.  count and flags are adjacent in both, the list needs no zeroing.
static int flag_bufs(TcState &s, void *ws, int64_t B, cudaStream_t st, bool cleaning_head_follows, const char **err) {
    bool own = false;
    if (s.d_flagstate && B <= s.flag_cap && cleaning_head_follows) {
        if (!s.owner_set) { s.owner_set = true; s.owner_stream = st; }
        own = s.owner_stream == st;
    }
    if (own) {
        s.cur_count = s.d_flagstate; s.cur_flags = s.cur_count + 16; s.cur_list = s.cur_flags + s.flag_cap;
        if (!s.flags_clean && cudaMemsetAsync(s.cur_count, 0, sizeof(int) * (s.flag_cap + 16), st) != cudaSuccess) { *err = "memset flags"; return -1; }
        s.flags_clean = false;                    // until the cleaning head kernel of this call has been launched
    } else {
        s.cur_count = reinterpret_cast<int *>(ws); s.cur_flags = s.cur_count + 16; s.cur_list = s.cur_flags + B;
        if (cudaMemsetAsync(s.cur_count, 0, sizeof(int) * (B + 16), st) != cudaSuccess) { *err = "memset flags"; return -1; }
    }
    s.cur_own = own;
    return 0;
}

// streaming front end + projection -> range partials (and gates[B][64]); flagged (NaN) windows are recomputed exactly.
int tc_gates(TcState &s, const Dims &d, const ConvWeights &cw, const HeadWeights &hw, const void *x, int dtype, int64_t B,
             float *partial, float *gates, void *ws, int num_sms, cudaStream_t st, const char **err, bool reduce_here) {
    const bool f32 = dtype == B2CNN_DTYPE_F32;
    // scratch ints: count | flags | list  (the handle's own zero-between-calls copy, or the head of the workspace)
    if (flag_bufs(s, ws, B, st, !reduce_here, err) != 0) return -1;
    int *count = s.cur_count, *flags = s.cur_flags, *list = s.cur_list;
    int staged = 0;
    int64_t pitch = d.XP;         // fp32 windows arrive with 16-byte rows (the caller routes any other pitch elsewhere)
    const void *xin = f32 ? x : tc_stage_input(d, x, B, reinterpret_cast<char *>(ws) + tc_flags_bytes(B), &pitch, &staged, st);
    CUtensorMap tm;
    if (make_tmap(d, xin, pitch, B, f32, &tm, err) != 0) return -1;
    TcFusedParams p;
    memset(&p, 0, sizeof p);
    p.partial = partial; p.nanflag = flags; p.list = list; p.count = count;
    p.wpack = reinterpret_cast<const uint8_t *>(s.d_wpack);
    p.B = (int)B; p.W = d.W; p.L = d.L;
    p.tiles_per_cta = s.tiles_per_cta; p.feats_per_cta = s.feats_per_cta; p.chunks_per_cta = s.chunks_per_cta;
    fill_epilogue(p, d, cw);
    // bf16 pieces per conv1 weight: 3 (fp32-equivalent) or 2; fp32 windows multiply the fp32 weights (key 1)
    const int sp = f32 ? 1 : s.splits;
    if (!f32) p.bmats = reinterpret_cast<const uint8_t *>(sp == 2 ? s.d_bmats2 : s.d_bmats);
    dim3 grid((unsigned)((B + kTcM - 1) / kTcM), s.n_ranges);
    const int key = d.C * 100 + sp * 10 + (d.K1 == 10 ? 0 : 1);
    cudaError_t le;
    switch (key) {
#define GATES_CASE(CC, SS, AA) case CC * 100 + SS * 10 + AA: le = launch_stream<CC, SS, AA, SS == 1, kOutGates>(tm, p, grid, st); break;
        GATES_CASE(1, 2, 0) GATES_CASE(2, 2, 0) GATES_CASE(3, 2, 0) GATES_CASE(1, 3, 0) GATES_CASE(2, 3, 0) GATES_CASE(3, 3, 0)
        GATES_CASE(1, 2, 1) GATES_CASE(2, 2, 1) GATES_CASE(3, 2, 1) GATES_CASE(1, 3, 1) GATES_CASE(2, 3, 1) GATES_CASE(3, 3, 1)
        GATES_CASE(1, 1, 0) GATES_CASE(2, 1, 0) GATES_CASE(3, 1, 0) GATES_CASE(1, 1, 1) GATES_CASE(2, 1, 1) GATES_CASE(3, 1, 1)
#undef GATES_CASE
        default: *err = "no streaming instantiation for this channel count / split"; return -1;
    }
    if (le != cudaSuccess) { *err = cudaGetErrorString(le); return -1; }
    int launches = 1 + staged;
    // the exception path: exact gate partials of the flagged windows, written over their rows of `partial`
    // (one launch; the list was compacted by the kernel itself, an empty list costs one almost-empty launch)
    int n = launch_frontend_generic_gates_listed(d, cw, x, dtype, B, hw.wih0T, partial, s.n_ranges, list, count, st, num_sms, err);
    if (n < 0) return -1;
    launches += n;
    // reduce_here == false: the caller's head kernel sums the range partials itself (independent windows)
    n = reduce_here ? launch_reduce_gates(partial, s.n_ranges, B, hw, gates, st, err) : 0;
    if (n < 0) return -1;
    return launches + n;
}

// 2-D map of a scorer's feature ring [L][pitch] fp32 (pitch % 4 == 0): boxes of 16 positions x 128 patients
int tc_ring_tmap(const float *ring, int64_t P, int64_t pitch, int L, CUtensorMap *tm, const char **err) {
    if (!get_encode()) { *err = "cuTensorMapEncodeTiled unavailable"; return -1; }
    cuuint64_t gdim[2] = {(cuuint64_t)P, (cuuint64_t)L};
    cuuint64_t gstr[1] = {(cuuint64_t)pitch * 4};
    cuuint32_t box[2] = {kTcM, 16};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = get_encode()(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(ring), gdim, gstr, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { *err = "cuTensorMapEncodeTiled(ring) failed"; return -1; }
    return 0;
}

// The new features of a sliding-window scorer (b2cnn_slide.cu) straight into its position-major ring.  `dseg`
// describes the segment from its first feature's first sample (W = samples, L = features, C); x: 16-byte aligned,
// `pitch` a multiple of 16 bytes.  flags [P] (zeroed by the caller) | list [P] | count: windows whose features
// may hold a tensor-core NaN, compacted for the exact re-computation.  Returns the launch count.
int tc_ring_features(const TcState &s, const Dims &dseg, const ConvWeights &cw, const void *x, int64_t pitch, int dtype,
                     int64_t P, float *ring, int64_t ring_pitch, int cap, int slot0, int *flags, cudaStream_t st, const char **err) {
    const bool f32 = dtype == B2CNN_DTYPE_F32;
    CUtensorMap tm;
    if (make_tmap(dseg, x, pitch, P, f32, &tm, err) != 0) return -1;
    TcFusedParams p;
    memset(&p, 0, sizeof p);
    p.feats = ring; p.sB = 1; p.sP = ring_pitch; p.nanflag = flags;
    p.ring_slot0 = slot0; p.ring_cap = cap;
    p.bmats = reinterpret_cast<const uint8_t *>(s.d_bmats);
    p.B = (int)P; p.W = dseg.W; p.L = dseg.L;
    p.tiles_per_cta = tiles_per_cta_for(dseg);
    p.feats_per_cta = 2 * kTcBlocks * p.tiles_per_cta - 4;
    fill_epilogue(p, dseg, cw);
    dim3 grid((unsigned)((P + kTcM - 1) / kTcM), (dseg.L + p.feats_per_cta - 1) / p.feats_per_cta);
    const int key = dseg.C * 100 + (f32 ? 10 : 0) + (dseg.K1 == 10 ? 0 : 1);
    cudaError_t e;
    switch (key) {
#define RING_CASE(CC, FF, AA) case CC * 100 + FF * 10 + AA: e = launch_stream<CC, FF ? 1 : 3, AA, FF == 1, kOutRing>(tm, p, grid, st); break;
        RING_CASE(1, 0, 0) RING_CASE(2, 0, 0) RING_CASE(3, 0, 0) RING_CASE(1, 0, 1) RING_CASE(2, 0, 1) RING_CASE(3, 0, 1)
        RING_CASE(1, 1, 0) RING_CASE(2, 1, 0) RING_CASE(3, 1, 0) RING_CASE(1, 1, 1) RING_CASE(2, 1, 1) RING_CASE(3, 1, 1)
#undef RING_CASE
        default: *err = "no feature-ring instantiation for this channel count"; return -1;
    }
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    int *list = flags + P, *count = list + P;
    tc_compact_flags_kernel<<<(unsigned)((P + 255) / 256), 256, 0, st>>>(flags, (int)P, list, count);
    if (cudaGetLastError() != cudaSuccess) { *err = "flag compaction launch"; return -1; }
    return 2;
}

// Whole recordings (b2cnn_score_record): `rows` staged rows, each of dseg.W samples (first feature at sample 0) and
// dseg.L features, into feats[row * sB + position] (sB >= dseg.L), then the exact re-computation of every row the
// tensor-core kernel flagged.  flags [rows] (zeroed by the caller) | list [rows] | count.  Returns the launch count.
int tc_row_features(const TcState &s, const Dims &dseg, const ConvWeights &cw, const void *x, int64_t pitch, int dtype,
                    int64_t rows, float *feats, int64_t sB, int *flags, int num_sms, cudaStream_t st, const char **err) {
    const bool f32 = dtype == B2CNN_DTYPE_F32;
    CUtensorMap tm;
    if (make_tmap(dseg, x, pitch, rows, f32, &tm, err) != 0) return -1;
    TcFusedParams p;
    memset(&p, 0, sizeof p);
    p.feats = feats; p.sB = sB; p.sP = 1; p.nanflag = flags;
    p.bmats = reinterpret_cast<const uint8_t *>(s.d_bmats);
    p.B = (int)rows; p.W = dseg.W; p.L = dseg.L;
    p.tiles_per_cta = tiles_per_cta_for(dseg);
    p.feats_per_cta = 2 * kTcBlocks * p.tiles_per_cta - 4;
    fill_epilogue(p, dseg, cw);
    dim3 grid((unsigned)((rows + kTcM - 1) / kTcM), (dseg.L + p.feats_per_cta - 1) / p.feats_per_cta);
    const int key = dseg.C * 100 + (f32 ? 10 : 0) + (dseg.K1 == 10 ? 0 : 1);
    cudaError_t e;
    switch (key) {
#define ROW_CASE(CC, FF, AA) case CC * 100 + FF * 10 + AA: e = launch_stream<CC, FF ? 1 : 3, AA, FF == 1, kOutFeatures>(tm, p, grid, st); break;
        ROW_CASE(1, 0, 0) ROW_CASE(2, 0, 0) ROW_CASE(3, 0, 0) ROW_CASE(1, 0, 1) ROW_CASE(2, 0, 1) ROW_CASE(3, 0, 1)
        ROW_CASE(1, 1, 0) ROW_CASE(2, 1, 0) ROW_CASE(3, 1, 0) ROW_CASE(1, 1, 1) ROW_CASE(2, 1, 1) ROW_CASE(3, 1, 1)
#undef ROW_CASE
        default: *err = "no feature-row instantiation for this channel count"; return -1;
    }
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    int *list = flags + rows, *count = list + rows;
    tc_compact_flags_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, st>>>(flags, (int)rows, list, count);
    if (cudaGetLastError() != cudaSuccess) { *err = "flag compaction launch"; return -1; }
    // flagged rows (a NaN or inf sample): every feature of the row again, exact fp32 (the generic front end)
    const int n = launch_frontend_generic_listed(dseg, cw, x, dtype, rows, feats, sB, 1, list, count, st, num_sms, err);
    return n < 0 ? n : 2 + n;
}

}  // namespace b2cnn

// b2cnn_tc_fused.cuh -- the streaming front end on sm_90a (included by b2cnn_tc.cu): conv1 -> pool1 -> tanh ->
// conv2 -> pool2 -> tanh for 128 windows x one position range per CTA, the features either written out
// (OUT = kOutFeatures) or multiplied on chip into the LSTM layer-0 input projection (OUT = kOutGates):
//
//      gates[w, g] += sum_p  f[w, p] * W_ih_l0[g, p]           (bin/models.py:30, layer 0)
//
// conv1 of bf16 windows is the banded-Toeplitz GEMM described in b2cnn_tc.cu, on wgmma: per 8-position block,
// two m64n32k16 row halves x C channels x SPLITS weight pieces, A = the TMA tile (SWIZZLE_128B, the block's
// 16-sample slice selected by a 16n-byte descriptor offset), B = the band-matrix piece, D in registers.  The
// accumulator fragment (two windows x 16 values per thread) is turned into thread == window through an 18 KB
// shared-memory transpose; the next block's MMAs run while the epilogue of this one computes.  fp32 windows
// (F32IN) evaluate conv1 in exact fp32 FMAs straight from the tile instead (32-sample boxes, 3 blocks per tile).
//
// Epilogue, thread == window: each thread streams through its window's positions in order, so pool1 -> tanh ->
// conv2 -> pool2 -> tanh are register-local sliding windows; tanh is 1 - 2/(1+2^(2x log2 e)) on MUFU.EX2 +
// MUFU.RCP with the bias folded into the exponent FMA; pooling runs BEFORE the activation (monotone) with
// max.NaN so NaNs propagate exactly like ATen's max_pool1d.  conv2 consumes r = (1 - tanh)/2 (weights
// pre-multiplied by -2, the bias absorbs sum(w)).
//
// Projection: the two features of a step are split into three bf16 pieces and stored into a [128 x 16]
// K-major A tile per piece; every 16 positions the warpgroup issues 2 row halves x 6 m64n64k16 MMAs (piece
// pairs hh hm mh hl lh mm: fp32-equivalent products) against the packed W_ih chunk, accumulating the 64 gate
// pre-activations in registers over the CTA's whole range.  They leave once, as partial[range][window][64].
//
// CTA = 192 threads: warps 0-3 the consumer warpgroup, warp 4 the TMA producer of the window tiles, warp 5 the
// producer of the W_ih chunks (1-D bulk copies).
#pragma once

namespace b2cnn {

constexpr int kHpThreads = 192;
constexpr int kHpTStride = 36;                    // floats per window row of the accumulator transpose (conflict-free float4 reads)
constexpr int kHpTBytes = kTcM * kHpTStride * 4;
constexpr int kHpPieceBytes = kTcM * 16 * 2;      // one bf16 piece of the projection A operand
constexpr int kFuWChunkBytes = 3 * 64 * 16 * 2;   // 3 pieces x (64 gates x 16 positions) bf16
constexpr int kSfBlocks = 3;                      // fp32 windows: 8-position blocks per 32-sample tile
constexpr int kSfAdv = 24;
constexpr int kOutFeatures = 0, kOutGates = 1;

struct TcFusedParams {
    float *partial;           // [n_ranges][B][64]                 (kOutGates)
    float *feats;             // feats[b * sB + p * sP]            (kOutFeatures)
    int64_t sB, sP;
    int *nanflag;             // [B]
    int *list, *count;        // flagged windows: list[atomicAdd(count, 1)] = b (first flagger only)
    const uint8_t *bmats;     // conv1 band matrices [C][SPLITS][1 KB]
    const uint8_t *wpack;     // [n_ranges][chunks_per_cta][kFuWChunkBytes]
    int B, W, L;
    int tiles_per_cta, feats_per_cta, chunks_per_cta;
    float w1[kTcMaxC][10][kCMid];   // conv1 weights w1[o][c][k] (fp32 windows)
    float w9[kTcMaxC][kCMid];       // tap k=9 of conv1 (bf16 windows, MyCNN5: it does not fit the 16-sample slice)
    float b1s[kCMid];               // conv1 bias * 2 log2 e
    float w2n[kCMid][5];            // -2 * conv2 weights
    float b2s;                      // (conv2 bias + sum of conv2 weights) * 2 log2 e
};

__host__ __device__ constexpr size_t hp_smem_bytes(int C, int SPLITS, bool f32in, int out) {
    return 1024 + (size_t)2 * C * kTcABytes + (f32in ? 0 : (size_t)C * SPLITS * kTcBBytes + kHpTBytes) +
           (out == kOutGates ? (size_t)2 * kFuWChunkBytes + 3 * kHpPieceBytes : 0) + 8 * 8;
}

// ARCH 0: MyCNN5 geometry (K1=10, pool(3,2)) -- bin/models.py.
// ARCH 1: MyCNN2/3/4 geometry (K1=5, pool(2,2)) -- bin/explore_torch copy.ipynb:189-277: every tap fits the
//         16-sample slice (no tap-9 patch), pooling pairs stay inside a block (no carry), and a step emits
//         features 2j-2, 2j-1 instead of 2j-3, 2j-2.
template <int C, int SPLITS, int ARCH, bool F32IN, int OUT>
__global__ void __launch_bounds__(kHpThreads, 1)
tc_stream_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ TcFusedParams p) {
    constexpr int K1 = ARCH == 0 ? 10 : 5;
    constexpr int kBlocks = F32IN ? kSfBlocks : kTcBlocks;
    constexpr int kAdv = F32IN ? kSfAdv : kTcAdv;
    constexpr int FOFF = ARCH == 0 ? 3 : 2;           // step j emits features 2j-FOFF, 2j-FOFF+1
    extern __shared__ uint8_t smem_raw[];
    // [2 stages][C][16 KB] | bands | transpose | W ring [2][6 KB] | A pieces [3][4 KB] | barriers
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t *sA = smem;
    uint8_t *sBm = sA + 2 * C * kTcABytes;
    float *sT = reinterpret_cast<float *>(sBm + (F32IN ? 0 : C * SPLITS * kTcBBytes));
    uint8_t *sW = reinterpret_cast<uint8_t *>(sT) + (F32IN ? 0 : kHpTBytes);
    uint8_t *sPc = sW + (OUT == kOutGates ? 2 * kFuWChunkBytes : 0);
    uint64_t *bars = reinterpret_cast<uint64_t *>(sPc + (OUT == kOutGates ? 3 * kHpPieceBytes : 0));
    const uint32_t bar_full = smem_u32(bars + 0), bar_empty = smem_u32(bars + 2);
    const uint32_t bar_wfull = smem_u32(bars + 4), bar_wempty = smem_u32(bars + 6);
    auto sA_of = [&](int s, int c) -> uint8_t * { return sA + (size_t)(s * C + c) * kTcABytes; };

    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
    const int lane = threadIdx.x & 31;
    const int b0 = blockIdx.x * kTcM;
    const int p0 = blockIdx.y * p.feats_per_cta;
    const int nfeat = min(p.feats_per_cta, p.L - p0);
    const int nsteps = OUT == kOutGates ? (nfeat + FOFF - 1) / 2 + 1 : (nfeat + 4) / 2;
    const int ntiles = (nsteps + kBlocks - 1) / kBlocks;
    const int J = ntiles * kBlocks;                   // steps actually run
    const int nchunks = (J + 7) / 8;
    const int T0 = p0 * 4;                            // first conv1 position == first sample

    if (!F32IN)
        for (int i = threadIdx.x; i < C * SPLITS * kTcBBytes / 16; i += kHpThreads)
            reinterpret_cast<uint4 *>(sBm)[i] = reinterpret_cast<const uint4 *>(p.bmats)[i];
    if (threadIdx.x == 0) {
        for (int i = 0; i < 2; ++i) {
            mbar_init(bar_full + 8 * i, 1);
            mbar_init(bar_empty + 8 * i, 4);
            mbar_init(bar_wfull + 8 * i, 1);
            mbar_init(bar_wempty + 8 * i, 4);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    fence_proxy_async();                              // band matrices visible to the tensor core
    __syncthreads();

    if (warp == 4) {
        // ===================== TMA producer: window tiles =====================
        if (lane == 0) {
            for (int i = 0; i < ntiles; ++i) {
                const int s = i & 1, ph = (i >> 1) & 1;
                mbar_wait(bar_empty + 8 * s, ph ^ 1);
                mbar_expect_tx(bar_full + 8 * s, C * kTcABytes);
#pragma unroll
                for (int c = 0; c < C; ++c) tma_load_3d(smem_u32(sA_of(s, c)), &tmap, T0 + kAdv * i, c, b0, bar_full + 8 * s);
            }
        }
    } else if (warp == 5) {
        // ===================== producer of the packed W_ih chunks =====================
        if (OUT == kOutGates && lane == 0) {
            const uint8_t *wsrc = p.wpack + (size_t)blockIdx.y * p.chunks_per_cta * kFuWChunkBytes;
            for (int m = 0; m < nchunks; ++m) {
                const int u = m & 1;
                mbar_wait(bar_wempty + 8 * u, ((m >> 1) & 1) ^ 1);
                mbar_expect_tx(bar_wfull + 8 * u, kFuWChunkBytes);
                bulk_load_1d(smem_u32(sW + u * kFuWChunkBytes), wsrc + (size_t)m * kFuWChunkBytes, kFuWChunkBytes, bar_wfull + 8 * u);
            }
        }
    } else {
        // ===================== consumer warpgroup: thread == window =====================
        const int row = threadIdx.x;
        const int b = b0 + row;
        const bool row_ok = b < p.B;
        const uint32_t swz = (uint32_t)(row & 7);     // SWIZZLE_128B: 16-byte chunk ^= row % 8
        float acc[2][16];                             // conv1 accumulators of one block (two m64 row halves)
        float gacc[2][32];                            // gate pre-activations (two m64 row halves)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[h][i] = 0.f;
#pragma unroll
            for (int i = 0; i < 32; ++i) gacc[h][i] = 0.f;
        }
        float pm6[kCMid], pm7[kCMid], ah[4][kCMid], c2c = 0.f, nan_probe = 0.f;
#pragma unroll
        for (int o = 0; o < kCMid; ++o) {
            pm6[o] = 0.f; pm7[o] = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) ah[i][o] = 0.f;
        }
        float *fout = p.feats + (int64_t)b * p.sB + (int64_t)p0 * p.sP;

        auto issue_conv1 = [&](int s, int n) {
            const uint64_t bdesc0 = gdesc_none_kmajor(smem_u32(sBm), 128, 256);
            wgmma_fence();
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int c = 0; c < C; ++c) {
                    const uint64_t adesc = gdesc_sw128_kmajor(smem_u32(sA_of(s, c)) + h * 64 * 128 + 16 * n);
#pragma unroll
                    for (int sp = 0; sp < SPLITS; ++sp)
                        wgmma_m64n32(acc[h], adesc, bdesc0 + (uint64_t)((c * SPLITS + sp) * (kTcBBytes >> 4)), (c | sp) != 0);
                }
            wgmma_commit();
        };
        if (!F32IN) {
            mbar_wait(bar_full, 0);
            issue_conv1(0, 0);
        }

#pragma unroll 1
        for (int j = 0; j < J; ++j) {
            const int i = j / kBlocks, n = j - i * kBlocks, s = i & 1;
            float D[32];                              // conv1 pre-activations of block j: D[shift * 4 + out channel]
            if constexpr (!F32IN) {
                if constexpr (ARCH == 0) {
                    // tap 9 of the previous block's position 7: sample 8n + 8 of this tile
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        const uint16_t raw = *reinterpret_cast<const uint16_t *>(sA_of(s, c) + row * 128 + (((uint32_t)(n + 1) ^ swz) << 4));
                        const float xv = __uint_as_float((uint32_t)raw << 16);
#pragma unroll
                        for (int o = 0; o < kCMid; ++o) pm7[o] = fmaf(p.w9[c][o], xv, pm7[o]);
                    }
                }
                wgmma_wait<0>();
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 16; e += 2) {
                        const int r = 64 * h + 16 * warp + (lane >> 2) + 8 * ((e >> 1) & 1);
                        const int col = 8 * (e >> 2) + 2 * (lane & 3);
                        *reinterpret_cast<float2 *>(sT + r * kHpTStride + col) = make_float2(acc[h][e], acc[h][e + 1]);
                    }
                wg_bar();
                if (n == kBlocks - 1 && lane == 0) mbar_arrive(bar_empty + 8 * s);   // stage fully consumed
                if (j + 1 < J) {                      // the next block's MMAs overlap this block's epilogue
                    const int i2 = (j + 1) / kBlocks, n2 = j + 1 - i2 * kBlocks;
                    if (n2 == 0) mbar_wait(bar_full + 8 * (i2 & 1), (i2 >> 1) & 1);
                    issue_conv1(i2 & 1, n2);
                }
#pragma unroll
                for (int k = 0; k < 32; k += 4) {
                    const float4 v = *reinterpret_cast<const float4 *>(sT + row * kHpTStride + k);
                    D[k] = v.x; D[k + 1] = v.y; D[k + 2] = v.z; D[k + 3] = v.w;
                }
                wg_bar();                             // transpose buffer free for the next block
            } else {
                // conv1 of block j on the CUDA cores, exact fp32, from the 16 samples at tile offset 8n
                if (n == 0) mbar_wait(bar_full + 8 * s, (i >> 1) & 1);
#pragma unroll
                for (int k = 0; k < 32; ++k) D[k] = 0.f;
#pragma unroll 1
                for (int c = 0; c < C; ++c) {
                    float xs[16];
#pragma unroll
                    for (int j4 = 0; j4 < 4; ++j4) {
                        const float4 v = *reinterpret_cast<const float4 *>(sA_of(s, c) + row * 128 + (((uint32_t)(2 * n + j4) ^ swz) << 4));
                        xs[4 * j4 + 0] = v.x; xs[4 * j4 + 1] = v.y; xs[4 * j4 + 2] = v.z; xs[4 * j4 + 3] = v.w;
                    }
                    if constexpr (ARCH == 0) {
#pragma unroll
                        for (int o = 0; o < kCMid; ++o) pm7[o] = fmaf(p.w1[c][9][o], xs[8], pm7[o]);
                    }
#pragma unroll
                    for (int k = 0; k < K1; ++k)
#pragma unroll
                        for (int sft = 0; sft < 8; ++sft)
                            if (sft + k < 16) {
#pragma unroll
                                for (int o = 0; o < kCMid; ++o) D[sft * 4 + o] = fmaf(p.w1[c][k][o], xs[sft + k], D[sft * 4 + o]);
                            }
                }
                if (n == kBlocks - 1) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_empty + 8 * s);
                }
            }
            // ---- pool1 on pre-activations, then r = (1 - tanh(+bias)) / 2: a1 positions of this block
            float an[4][kCMid];
#pragma unroll
            for (int o = 0; o < kCMid; ++o) {
                if constexpr (ARCH == 0) {
                    an[0][o] = sig_fold(max3_nan(pm6[o], pm7[o], D[0 * 4 + o]), p.b1s[o]);
                    an[1][o] = sig_fold(max3_nan(D[0 * 4 + o], D[1 * 4 + o], D[2 * 4 + o]), p.b1s[o]);
                    an[2][o] = sig_fold(max3_nan(D[2 * 4 + o], D[3 * 4 + o], D[4 * 4 + o]), p.b1s[o]);
                    an[3][o] = sig_fold(max3_nan(D[4 * 4 + o], D[5 * 4 + o], D[6 * 4 + o]), p.b1s[o]);
                    pm6[o] = D[6 * 4 + o];
                    pm7[o] = D[7 * 4 + o];
                } else {
#pragma unroll
                    for (int r = 0; r < 4; ++r) an[r][o] = sig_fold(max_nan(D[(2 * r) * 4 + o], D[(2 * r + 1) * 4 + o]), p.b1s[o]);
                }
            }
            // ---- conv2 over the previous block's and this block's a1 (no bias yet)
            float c2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int c = 0; c < kCMid; ++c) {
                const float A8[8] = {ah[0][c], ah[1][c], ah[2][c], ah[3][c], an[0][c], an[1][c], an[2][c], an[3][c]};
#pragma unroll
                for (int k = 0; k < 5; ++k)
#pragma unroll
                    for (int r = 0; r < 4; ++r) c2[r] = fmaf(p.w2n[c][k], A8[r + k], c2[r]);
            }
#pragma unroll
            for (int c = 0; c < kCMid; ++c)
#pragma unroll
                for (int r = 0; r < 4; ++r) ah[r][c] = an[r][c];
            // ---- pool2 + tanh(+bias): the two features of step j
            float f0, f1;
            if constexpr (ARCH == 0) {
                f0 = tanh_fold(max3_nan(c2c, c2[0], c2[1]), p.b2s);
                f1 = tanh_fold(max3_nan(c2[1], c2[2], c2[3]), p.b2s);
                c2c = c2[3];
            } else {
                f0 = tanh_fold(max_nan(c2[0], c2[1]), p.b2s);
                f1 = tanh_fold(max_nan(c2[2], c2[3]), p.b2s);
            }
            if constexpr (OUT == kOutFeatures) {
                nan_probe = fmaf(f0, 0.f, nan_probe);
                nan_probe = fmaf(f1, 0.f, nan_probe);
                const int pr0 = 2 * j - FOFF;
                if (row_ok) {
                    if (pr0 >= 0 && pr0 < nfeat) fout[(int64_t)pr0 * p.sP] = f0;
                    if (pr0 + 1 >= 0 && pr0 + 1 < nfeat) fout[(int64_t)(pr0 + 1) * p.sP] = f1;
                }
            } else {
                // three bf16 pieces of (f0, f1) -> word kk of this window's row of the A tiles
                const int kk = j & 7, m = j >> 3, u = m & 1;
                const uint32_t h = pack_bf16x2(f0, f1);
                const float r1x = f0 - __uint_as_float(h << 16), r1y = f1 - __uint_as_float(h & 0xffff0000u);
                const uint32_t md = pack_bf16x2(r1x, r1y);
                const uint32_t lo = pack_bf16x2(r1x - __uint_as_float(md << 16), r1y - __uint_as_float(md & 0xffff0000u));
                uint8_t *arow = sPc + (row >> 3) * 256 + (row & 7) * 16;
                auto put = [&](int col, uint32_t w0, uint32_t w1, uint32_t w2) {
                    const int off = (col >> 2) * 128 + (col & 3) * 4;
                    *reinterpret_cast<uint32_t *>(arow + off) = w0;
                    *reinterpret_cast<uint32_t *>(arow + kHpPieceBytes + off) = w1;
                    *reinterpret_cast<uint32_t *>(arow + 2 * kHpPieceBytes + off) = w2;
                };
                put(kk, h, md, lo);
                if (kk == 7 || j == J - 1) {
                    for (int z = kk + 1; z < 8; ++z) put(z, 0u, 0u, 0u);
                    fence_proxy_async();
                    wg_bar();
                    mbar_wait(bar_wfull + 8 * u, (m >> 1) & 1);
                    const uint32_t pa = smem_u32(sPc), pw = smem_u32(sW + u * kFuWChunkBytes);
                    wgmma_fence();
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        // piece pairs (feature piece, weight piece) with fp + wp <= 2: hh hm mh hl lh mm
                        constexpr int kAp[6] = {0, 0, 1, 0, 2, 1}, kWp[6] = {0, 1, 0, 2, 0, 1};
#pragma unroll
                        for (int q = 0; q < 6; ++q)
                            wgmma_m64n64(gacc[hh], gdesc_none_kmajor(pa + kAp[q] * kHpPieceBytes + hh * 2048, 128, 256),
                                         gdesc_none_kmajor(pw + kWp[q] * 2048, 128, 256));
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_wempty + 8 * u);
                    wg_bar();                         // A tiles free for the next chunk
                }
            }
        }

        if constexpr (OUT == kOutFeatures) {
            if (row_ok && nan_probe != nan_probe) p.nanflag[b] = 1;
        } else {
            // gate pre-activations of this CTA's position range -> partial[range][window][64].  A NaN feature (a NaN / inf
            // sample met a zero of the band matrix, or a real NaN) makes every gate it is multiplied into NaN -- zero weights
            // included -- so the sums themselves are the probe.
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int e2 = 0; e2 < 2; ++e2) {
                    const int r = 64 * hh + 16 * warp + (lane >> 2) + 8 * e2;
                    const int bb = b0 + r;
                    bool bad = false;
#pragma unroll
                    for (int e = 0; e < 32; ++e)
                        if (((e >> 1) & 1) == e2) bad |= gacc[hh][e] != gacc[hh][e];
                    if (bb < p.B) {
                        float *dst = p.partial + ((int64_t)blockIdx.y * p.B + bb) * kGates + 2 * (lane & 3);
#pragma unroll
                        for (int e = 2 * e2; e < 32; e += 4)
                            *reinterpret_cast<float2 *>(dst + 8 * (e >> 2)) = make_float2(gacc[hh][e], gacc[hh][e + 1]);
                        // up to n_ranges CTAs (and four threads of one) may flag the same window: the first appends it
                        if (bad && atomicExch(&p.nanflag[bb], 1) == 0) p.list[atomicAdd(p.count, 1)] = bb;
                    }
                }
        }
    }
}

// W_ih_l0 [64][L] fp32 -> per (range, 16-position chunk) three bf16 pieces in GMMA K-major
// no-swizzle core-matrix order (byte = (g/8)*256 + (k/8)*128 + (g%8)*16 + (k%8)*2 per piece).
// Chunk m of a range covers relative features 16m-foff .. 16m-foff+15 (the stream emits 2j-foff, 2j-foff+1 at
// step j); positions outside the range or beyond L get zero weights, which also masks the
// stream's warm-up / tail garbage.
__global__ void tc_pack_wih_kernel(const float *__restrict__ wih, uint8_t *__restrict__ out, int L, int feats_per_cta,
                                   int chunks_per_cta, int n_ranges, int foff) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)n_ranges * chunks_per_cta * 1024;
    if (e >= total) return;
    const int k = (int)(e & 15), g = (int)((e >> 4) & 63);
    const int64_t cm = e >> 10;
    const int m = (int)(cm % chunks_per_cta), pr = (int)(cm / chunks_per_cta);
    const int prel = 16 * m - foff + k;
    const int pos = pr * feats_per_cta + prel;
    float w = 0.f;
    if (prel >= 0 && prel < feats_per_cta && pos < L) w = wih[(int64_t)g * L + pos];
    uint16_t *base = reinterpret_cast<uint16_t *>(out + (size_t)cm * kFuWChunkBytes);
    const int off = (g / 8) * 128 + (k / 8) * 64 + (g % 8) * 8 + (k % 8);
#pragma unroll
    for (int piece = 0; piece < 3; ++piece) {
        const __nv_bfloat16 hb = __float2bfloat16_rn(w);
        base[piece * 1024 + off] = __bfloat16_as_ushort(hb);
        w -= __bfloat162float(hb);
    }
}

}  // namespace b2cnn

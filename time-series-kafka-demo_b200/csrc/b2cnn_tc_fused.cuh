// b2cnn_tc_fused.cuh -- the streaming front end on sm_90a (included by b2cnn_tc.cu): conv1 -> pool1 -> tanh ->
// conv2 -> pool2 -> tanh for 128 windows x one position range per CTA, the features either written out
// (OUT = kOutFeatures) or multiplied on chip into the LSTM layer-0 input projection (OUT = kOutGates):
//
//      gates[w, g] += sum_p  f[w, p] * W_ih_l0[g, p]           (bin/models.py:30, layer 0)
//
// conv1 of bf16 windows is the banded-Toeplitz GEMM described in b2cnn_tc.cu, on wgmma: per 8-position block,
// two m64n32k16 row halves x C channels x SPLITS weight pieces, A in registers (one ldmatrix.x4 per row half and
// channel of the block's 16-sample slice of the TMA tile: 32-sample boxes, SWIZZLE_64B, 3 blocks per tile, shared by
// the SPLITS pieces), B = the band-matrix piece, D in registers.  The band matrices' columns are ordered so that each
// lane of the accumulator fragment holds all 8 shifts of one conv1 channel for its four windows: pool1 and the
// activation run there, register-local, and only the pooled a1 (16 floats per window) cross to thread == window through
// a double-buffered 2 x 8 KB shared-memory exchange (XOR-swizzled, conflict-free both ways, one barrier per block); the
// next block's MMAs run while the epilogue of this one computes.  The three blocks of a tile are
// unrolled, so their addresses are the tile's plus immediates.  About 100 KB of shared memory and 128 registers per
// thread at launch let two CTAs share an SM, so each SM sub-partition has two consumer warps to interleave;
// setmaxnreg then gives the consumer warpgroup 232 of them and the producer warpgroup 24.  fp32 windows (F32IN) evaluate conv1 in exact fp32
// FMAs straight from the tile instead (the same 32-sample boxes as 128-byte SWIZZLE_128B rows; one CTA per SM).
//
// Epilogue, thread == window (after the a1 exchange for bf16 windows): each thread streams through its window's
// positions in order, so conv2 -> pool2 -> tanh (fp32 windows: pool1 -> tanh first) are register-local sliding
// windows; tanh is 1 - 2/(1+2^(2x log2 e)) on MUFU.EX2 + MUFU.RCP with the bias folded into the exponent FMA; pooling
// runs BEFORE the activation (monotone) with max.NaN so NaNs propagate exactly like ATen's max_pool1d.  conv2
// consumes r = (1 - tanh)/2 (weights pre-multiplied by -2, the bias absorbs sum(w)).
//
// Projection: the two features of a step are split into three bf16 pieces and stored into a [128 x 16]
// K-major A tile per piece; every 16 positions the warpgroup issues 2 row halves x 6 m64n64k16 MMAs (piece
// pairs hh hm mh hl lh mm: fp32-equivalent products) against the packed W_ih chunk, accumulating the 64 gate
// pre-activations in registers over the CTA's whole range.  They leave once, as partial[range][window][64].  The A
// tiles are double-buffered, so a chunk's MMAs are retired a block later by the wait that retires the next conv1,
// instead of draining the tensor pipe at every chunk.
//
// CTA = 256 threads for bf16 windows, 192 for fp32: warps 0-3 the consumer warpgroup, warp 4 the TMA producer of the
// window tiles, warp 5 the producer of the W_ih chunks (1-D bulk copies), warps 6-7 (bf16) idle.
#pragma once

namespace b2cnn {

// bf16 windows: two full warpgroups, so that setmaxnreg can move registers from the producer warpgroup (warps 4-7,
// 6 and 7 idle) to the consumer one; fp32 windows: 192 threads
__host__ __device__ constexpr int hp_threads(bool f32in) { return f32in ? 192 : 256; }
constexpr int kHpProducerRegs = 24, kHpConsumerRegs = 232;   // 128 x 24 + 128 x 232 = 256 x 128: two CTAs per SM
// a1 exchange (bf16 windows), double-buffered by block parity: per window row the 16 pooled activations of a block,
// 16-byte chunk o = channel o's 4 positions, stored at chunk o ^ (r / 2) % 4.  Both sides are conflict-free: an STS.128
// quarter-warp writes two whole adjacent 64-byte rows, and an LDS.128 quarter-warp reads 8 rows whose
// (r % 2, (r / 2) % 4) pairs are all distinct.
constexpr int kHpXStride = 16;
constexpr int kHpXBuf = kTcM * kHpXStride * 4;
constexpr int kHpXBytes = 2 * kHpXBuf;
constexpr int kHpPieceBytes = kTcM * 16 * 2;      // one bf16 piece of the projection A operand
constexpr int kFuWChunkBytes = 3 * 64 * 16 * 2;   // 3 pieces x (64 gates x 16 positions) bf16
// kOutRing: the features of a sliding-window scorer's new segment (b2cnn_slide.cu) into its position-major
// feature ring, feats[((ring_slot0 + p) mod ring_cap) * sP + b]: thread == window, so a warp stores 32
// consecutive floats per position.
constexpr int kOutFeatures = 0, kOutGates = 1, kOutRing = 2;

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
    int ring_slot0, ring_cap;       // kOutRing: ring slot of feature 0, slots in the ring
};

__host__ __device__ constexpr size_t hp_smem_bytes(int C, int SPLITS, bool f32in, int out) {
    return 1024 + (size_t)2 * C * kTcM * (f32in ? kTcF32ARow : kTcARow) + (f32in ? 0 : (size_t)C * SPLITS * kTcBBytes + kHpXBytes) +
           (out == kOutGates ? (size_t)2 * kFuWChunkBytes + 2 * 3 * kHpPieceBytes : 0) + 8 * 8;
}

// ARCH 0: MyCNN5 geometry (K1=10, pool(3,2)) -- bin/models.py.
// ARCH 1: MyCNN2/3/4 geometry (K1=5, pool(2,2)) -- bin/explore_torch copy.ipynb:189-277: every tap fits the
//         16-sample slice (no tap-9 patch), pooling pairs stay inside a block (no carry), and a step emits
//         features 2j-2, 2j-1 instead of 2j-3, 2j-2.
template <int C, int SPLITS, int ARCH, bool F32IN, int OUT>
__global__ void __launch_bounds__(hp_threads(F32IN), F32IN ? 1 : 2)
tc_stream_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ TcFusedParams p) {
    constexpr int K1 = ARCH == 0 ? 10 : 5;
    constexpr int kBlocks = kTcBlocks;
    constexpr int kARow = F32IN ? kTcF32ARow : kTcARow;
    constexpr int kABytes = kTcM * kARow;             // one channel of one stage
    constexpr int FOFF = ARCH == 0 ? 3 : 2;           // step j emits features 2j-FOFF, 2j-FOFF+1
    extern __shared__ uint8_t smem_raw[];
    // [2 stages][C][8 KB bf16 | 16 KB fp32] | bands | a1 exchange [2][8 KB] | W ring [2][6 KB] | A pieces [2][3][4 KB] |
    // barriers, aligned by an offset from smem_raw, not by rounding the generic address as an integer: the compiler then
    // still knows every pointer below is shared memory and emits 32-bit LDS / STS instead of 64-bit generic LD / ST
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t *sA = smem;
    uint8_t *sBm = sA + 2 * C * kABytes;
    uint8_t *sX = sBm + (F32IN ? 0 : C * SPLITS * kTcBBytes);
    uint8_t *sW = sX + (F32IN ? 0 : kHpXBytes);
    uint8_t *sPc = sW + (OUT == kOutGates ? 2 * kFuWChunkBytes : 0);
    uint64_t *bars = reinterpret_cast<uint64_t *>(sPc + (OUT == kOutGates ? 2 * 3 * kHpPieceBytes : 0));
    const uint32_t bar_full = smem_u32(bars + 0), bar_empty = smem_u32(bars + 2);
    const uint32_t bar_wfull = smem_u32(bars + 4), bar_wempty = smem_u32(bars + 6);
    auto sA_of = [&](int s, int c) -> uint8_t * { return sA + (size_t)(s * C + c) * kABytes; };

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
        for (int i = threadIdx.x; i < C * SPLITS * kTcBBytes / 16; i += hp_threads(F32IN))
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

    // bf16 windows: the consumer's conv1 A fragments stay live across the epilogue, so it needs more than the 128
    // registers per thread of two 256-thread CTAs; the producers need far fewer.  Each setmaxnreg opens its own branch,
    // so that ptxas allocates each role's code under its own limit.
    if (warp >= 4) {
        if constexpr (!F32IN) setmaxnreg_dec<kHpProducerRegs>();
        if (warp == 4) {
            // ===================== TMA producer: window tiles =====================
            if (lane == 0) {
                for (int i = 0; i < ntiles; ++i) {
                    const int s = i & 1, ph = (i >> 1) & 1;
                    mbar_wait(bar_empty + 8 * s, ph ^ 1);
                    mbar_expect_tx(bar_full + 8 * s, C * kABytes);
#pragma unroll
                    for (int c = 0; c < C; ++c) tma_load_3d(smem_u32(sA_of(s, c)), &tmap, T0 + kTcAdv * i, c, b0, bar_full + 8 * s);
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
        }
    } else {
        // ===================== consumer warpgroup: thread == window =====================
        if constexpr (!F32IN) setmaxnreg_inc<kHpConsumerRegs>();
        const int row = threadIdx.x;
        const int b = b0 + row;
        const bool row_ok = b < p.B;
        // 16-byte chunk k of a row sits at chunk k ^ swz: SWIZZLE_64B (bf16) k ^ (row / 2) % 4, SWIZZLE_128B (fp32) k ^ row % 8
        const uint32_t swz = F32IN ? (uint32_t)(row & 7) : (uint32_t)((row >> 1) & 3);
        // bf16 windows: lane l of the conv1 accumulator fragment holds every shift of out channel q = l % 4 for four
        // windows, rows 64 h + 16 warp + l / 4 + 8 e (row halves h, fragment row groups e), acc[h][4 (s / 2) + 2 e + s % 2]
        // for shift s (b2cnn_tc.cu packs the band matrices so).  Pool1 and the activation run there; only the pooled a1
        // cross to thread == window.  Rows are 64 bytes and every window of a lane has the same (r / 2) % 4 == l / 8, so
        // the lane writes chunk q ^ (l / 8) at x_w plus an immediate per window; a thread reads its own row's chunk o at
        // x_r ^ 16 o.  Block j uses buffer j % 2.
        const int q = lane & 3;
        const uint32_t x_w = smem_u32(sX) + (uint32_t)(16 * warp + (lane >> 2)) * (kHpXStride * 4) + 16 * (q ^ (lane >> 3));
        const uint32_t x_r = smem_u32(sX) + (uint32_t)row * (kHpXStride * 4) + 16 * swz;
        // the lane's own conv1 constants, in registers for the whole loop
        const float b1q = p.b1s[q];
        float w9q[C];
#pragma unroll
        for (int c = 0; c < C; ++c) w9q[c] = p.w9[c][q];
        float acc[2][16];                             // conv1 accumulators of one block (two m64 row halves)
        float gacc[2][32];                            // gate pre-activations (two m64 row halves)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[h][i] = 0.f;
#pragma unroll
            for (int i = 0; i < 32; ++i) gacc[h][i] = 0.f;
        }
        // conv1 positions 6 and 7 of the previous block: fp32 windows per out channel o of the thread's window, bf16
        // windows per window 2 h + e of the lane's out channel q
        float pm6[kCMid], pm7[kCMid], ah[4][kCMid], c2c = 0.f, nan_probe = 0.f;
#pragma unroll
        for (int o = 0; o < kCMid; ++o) {
            pm6[o] = 0.f; pm7[o] = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) ah[i][o] = 0.f;
        }
        float *fout = p.feats + (int64_t)b * p.sB + (int64_t)p0 * p.sP;

        // conv1's A operand from registers: per (row half h, channel c) one ldmatrix.x4 loads this warp's 16 rows of the
        // block's 16-sample slice (chunks n, n+1 of the tile) and all SPLITS weight pieces multiply that one fragment,
        // so the tile is read once instead of once per piece.  Lane l gives the address of row (l & 7) + 8 ((l >> 3) & 1)
        // of chunk n + (l >> 4): matrices (rows 0-7, 8-15) x (chunk n, n+1) = a0..a3 of the m16k16 fragment.  Its
        // SWIZZLE_64B term (row / 2) % 4 depends on l only.  The fragments stay live until the wait that retires the MMAs.
        uint32_t afr[2][C][4];
        const uint32_t a_lane = smem_u32(sA) + (uint32_t)(16 * warp + (lane & 7) + 8 * ((lane >> 3) & 1)) * kARow;
        const uint32_t a_swz = (lane >> 1) & 3, a_k = lane >> 4;
        // chunk (n + a_k) ^ a_swz of a 64-byte row: blocks 0 and 2 at a_b02 ^ 16 n, block 1 ((1 + a_k) == 1 << a_k) at a_b1
        const uint32_t a_b02 = a_lane | ((a_k ^ a_swz) << 4), a_b1 = a_lane | (((1u << a_k) ^ a_swz) << 4);
        // tap 9 of block n for the lane's four windows: chunk (n + 1) ^ (lane / 8) of their rows (SWIZZLE_64B), t9 ^ 16 (n + 1)
        // plus an immediate per window.  The 8 rows a warp reads get 8 distinct banks; a quad's lanes share an address.
        const uint32_t t9 = smem_u32(sA) + (uint32_t)(16 * warp + (lane >> 2)) * kARow + ((uint32_t)(lane >> 3) << 4);
        // B descriptor built once: a block's MMAs only add (start address offset) >> 4 to it
        const uint64_t bdesc0 = gdesc_none_kmajor(smem_u32(sBm), 128, 256);
        auto issue_conv1 = [&](int s, int n) {
            const uint32_t a_sn = (n == 1 ? a_b1 : a_b02 ^ (uint32_t)(16 * n)) + (uint32_t)(s * C * kABytes);
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int c = 0; c < C; ++c) ldmatrix_x4(afr[h][c], a_sn + (uint32_t)(c * kABytes + h * 64 * kARow));
            wgmma_fence();
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int c = 0; c < C; ++c)
#pragma unroll
                    for (int sp = 0; sp < SPLITS; ++sp)
                        wgmma_m64n32_rs(acc[h], afr[h][c], bdesc0 + (uint64_t)((c * SPLITS + sp) * (kTcBBytes >> 4)), (c | sp) != 0);
            wgmma_commit();
        };
        // the projection of chunk m (A pieces in buffer m & 1, W_ih in ring slot m & 1).  Its K-major no-swizzle
        // descriptors (LBO 128, SBO 256 bytes) differ only in the start-address field of their low word, so an MMA
        // adds its buffer, piece, row half and W slot offsets (>> 4) to one 32-bit base.  The caller has made every
        // warp's pieces visible.
        auto issue_proj = [&](int m) {
            const int u = m & 1;
            mbar_wait(bar_wfull + 8 * u, (m >> 1) & 1);
            const uint32_t pa = smem_u32(sPc) + u * 3 * kHpPieceBytes, pw = smem_u32(sW) + u * kFuWChunkBytes;
            auto desc = [](uint32_t addr) { return ((uint64_t)(256 >> 4) << 32) | ((addr >> 4) + (uint32_t)((128 >> 4) << 16)); };
            wgmma_fence();
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                // piece pairs (feature piece, weight piece) with fp + wp <= 2: hh hm mh hl lh mm
                constexpr int kAp[6] = {0, 0, 1, 0, 2, 1}, kWp[6] = {0, 1, 0, 2, 0, 1};
#pragma unroll
                for (int q = 0; q < 6; ++q)
                    wgmma_m64n64(gacc[hh], desc(pa + (uint32_t)(kAp[q] * kHpPieceBytes + hh * 2048)), desc(pw + (uint32_t)(kWp[q] * 2048)));
            }
            wgmma_commit();
        };
        // A chunk that ends at step jc inside the range is projected without draining the tensor pipe: bf16 windows issue
        // it at step jc + 1 behind that step's barrier and the next block's conv1, and the wait of step jc + 2 retires
        // both; fp32 windows issue it at the end of step jc and retire it at step jc + 1, after the CUDA-core conv1.  The
        // step that retires it gives its W slot back.  The range's last chunk is projected after the loop.
        constexpr int kLag = F32IN ? 1 : 2;
        // word col of this window's row of the three A tiles of buffer u
        uint8_t *const prow = sPc + (row >> 3) * 256 + (row & 7) * 16;
        auto put_pieces = [&](int u, int col, uint32_t w0, uint32_t w1, uint32_t w2) {
            uint8_t *const a = prow + u * 3 * kHpPieceBytes + (col >> 2) * 128 + (col & 3) * 4;
            *reinterpret_cast<uint32_t *>(a) = w0;
            *reinterpret_cast<uint32_t *>(a + kHpPieceBytes) = w1;
            *reinterpret_cast<uint32_t *>(a + 2 * kHpPieceBytes) = w2;
        };
        auto release_w = [&](int j) {
            if (OUT == kOutGates && j >= kLag && ((j - kLag) & 7) == 7 && lane == 0) mbar_arrive(bar_wempty + 8 * (((j - kLag) >> 3) & 1));
        };
        if (!F32IN) {
            mbar_wait(bar_full, 0);
            issue_conv1(0, 0);
        }

        // step j = kBlocks i + n: block n of tile i (stage i & 1).  bf16 windows run the blocks of a tile unrolled, n a
        // compile-time constant, so a block's tile, ldmatrix and tap-9 addresses are the tile's plus immediates.
        auto step = [&](const int j, const int i, const int n) {
            const int s = i & 1;
            float an[4][kCMid];                       // a1 of block j, thread == window: an[position][channel]
            if constexpr (!F32IN) {
                // tap 9 of the previous block's position 7 (sample 8n + 8 of this tile), added while the MMAs run, in
                // the same order over c as the fp32 path
                if constexpr (ARCH == 0) {
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int e = 0; e < 2; ++e)
#pragma unroll
                            for (int c = 0; c < C; ++c) {
                                const uint32_t raw = ld_shared_u16((t9 ^ (uint32_t)(16 * (n + 1))) +
                                                                   (uint32_t)((s * C + c) * kABytes + (64 * h + 8 * e) * kARow));
                                pm7[2 * h + e] = fmaf(w9q[c], __uint_as_float(raw << 16), pm7[2 * h + e]);
                            }
                }
                wgmma_wait<0>();                      // conv1 of this block (and the projection issued at step j - 1)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int c = 0; c < C; ++c) wgmma_keep(afr[h][c]);
                release_w(j);
                // ---- pool1 on pre-activations in the fragment layout: window 2 h + e, channel q, position r
                float m[2][2][4];
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float *d = acc[h] + 2 * e;   // shift t at d[4 (t / 2) + t % 2]
                        const int w = 2 * h + e;
                        if constexpr (ARCH == 0) {
                            m[h][e][0] = max3_nan(pm6[w], pm7[w], d[0]);
                            m[h][e][1] = max3_nan(d[0], d[1], d[4]);
                            m[h][e][2] = max3_nan(d[4], d[5], d[8]);
                            m[h][e][3] = max3_nan(d[8], d[9], d[12]);
                            pm6[w] = acc_copy(d[12]);
                            pm7[w] = acc_copy(d[13]);
                        } else {
#pragma unroll
                            for (int r = 0; r < 4; ++r) m[h][e][r] = max_nan(d[4 * r], d[4 * r + 1]);
                        }
                    }
                // acc is free once the maxima and the carries are taken: the next block's MMAs run on the tensor core
                // during this block's activations and the rest of its epilogue (issued after the barrier instead, behind
                // the projection, the step measured about 3 % slower)
                if (n < kBlocks - 1) {
                    issue_conv1(s, n + 1);
                } else if (i + 1 < ntiles) {          // (J is a whole number of tiles)
                    mbar_wait(bar_full + 8 * (s ^ 1), ((i + 1) >> 1) & 1);
                    issue_conv1(s ^ 1, 0);
                }
                // ---- r = (1 - tanh(+bias)) / 2, then the exchange: 4 positions of channel q per window and STS.128
                const uint32_t xb = (uint32_t)(((i + n) & 1) * kHpXBuf);
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        st_shared_v4(x_w + xb + (uint32_t)((64 * h + 8 * e) * kHpXStride * 4), sig_fold(m[h][e][0], b1q),
                                     sig_fold(m[h][e][1], b1q), sig_fold(m[h][e][2], b1q), sig_fold(m[h][e][3], b1q));
                // One barrier per block.  It publishes block j's a1 (buffer j % 2) and every warp's projection pieces of
                // step j - 1.  A warp writes buffer j % 2 again at block j + 2, after barrier j + 1, which every warp
                // reaches only after reading its block-j row, so the buffer needs no second barrier.
                wg_bar();
                if (n == kBlocks - 1 && lane == 0) mbar_arrive(bar_empty + 8 * s);   // stage fully consumed
                // the chunk that ended at step j - 1, its pieces published by the barrier above, behind the next conv1;
                // the next step's wait retires both
                if (OUT == kOutGates && (j & 7) == 0 && j > 0) issue_proj((j >> 3) - 1);
#pragma unroll
                for (int o = 0; o < kCMid; ++o) {
                    const float4 v = ld_shared_v4((x_r ^ (uint32_t)(16 * o)) + xb);
                    an[0][o] = v.x; an[1][o] = v.y; an[2][o] = v.z; an[3][o] = v.w;
                }
            } else {
                // conv1 of block j on the CUDA cores, exact fp32, from the 16 samples at tile offset 8n
                float D[32];                          // conv1 pre-activations of block j: D[shift * 4 + out channel]
                if (n == 0) mbar_wait(bar_full + 8 * s, (i >> 1) & 1);
#pragma unroll
                for (int k = 0; k < 32; ++k) D[k] = 0.f;
#pragma unroll 1
                for (int c = 0; c < C; ++c) {
                    float xs[16];
#pragma unroll
                    for (int j4 = 0; j4 < 4; ++j4) {
                        const float4 v = *reinterpret_cast<const float4 *>(sA_of(s, c) + row * kARow + (((uint32_t)(2 * n + j4) ^ swz) << 4));
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
                if constexpr (OUT == kOutGates) {
                    wgmma_wait<0>();                  // the projection issued at the end of step j - 1, if any
                    release_w(j);
                }
                if (n == kBlocks - 1) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_empty + 8 * s);
                }
                // ---- pool1 on pre-activations, then r = (1 - tanh(+bias)) / 2: a1 positions of this block
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
            } else if constexpr (OUT == kOutRing) {
                nan_probe = fmaf(f0, 0.f, nan_probe);
                nan_probe = fmaf(f1, 0.f, nan_probe);
                const int pr0 = 2 * j - FOFF;
                if (row_ok) {
                    // p0 + pr < L <= ring_cap and ring_slot0 < ring_cap: one subtraction wraps the slot
                    int slot = p.ring_slot0 + p0 + pr0;
                    if (slot >= p.ring_cap) slot -= p.ring_cap;
                    if (pr0 >= 0 && pr0 < nfeat) p.feats[(int64_t)slot * p.sP + b] = f0;
                    if (++slot == p.ring_cap) slot = 0;
                    if (pr0 + 1 >= 0 && pr0 + 1 < nfeat) p.feats[(int64_t)slot * p.sP + b] = f1;
                }
            } else {
                // three bf16 pieces of (f0, f1) -> word kk of this window's row of chunk m's A tiles (buffer m & 1)
                const int kk = j & 7, m = j >> 3;
                const uint32_t h = pack_bf16x2(f0, f1);
                const float r1x = f0 - __uint_as_float(h << 16), r1y = f1 - __uint_as_float(h & 0xffff0000u);
                const uint32_t md = pack_bf16x2(r1x, r1y);
                const uint32_t lo = pack_bf16x2(r1x - __uint_as_float(md << 16), r1y - __uint_as_float(md & 0xffff0000u));
                // chunk m's buffer was last read by chunk m - 2's projection, which every warp retired before it passed the
                // barrier that published chunk m - 1, so the pieces need no barrier after the MMAs
                put_pieces(m & 1, kk, h, md, lo);
                if (kk == 7) {
                    fence_proxy_async();
                    if (F32IN && j < J - 1) {
                        wg_bar();
                        issue_proj(m);
                    }
                }
            }
        };
        if constexpr (F32IN) {
#pragma unroll 1
            for (int j = 0; j < J; ++j) step(j, j / kBlocks, j % kBlocks);
        } else {
#pragma unroll 1
            for (int i = 0; i < ntiles; ++i)
#pragma unroll
                for (int n = 0; n < kBlocks; ++n) step(kBlocks * i + n, i, n);
        }

        if constexpr (OUT != kOutGates) {
            if (row_ok && nan_probe != nan_probe) p.nanflag[b] = 1;
        } else {
            // the range's last chunk, whole or partial: zero the words of the steps it does not have
            for (int z = ((J - 1) & 7) + 1; z < 8; ++z) put_pieces(((J - 1) >> 3) & 1, z, 0u, 0u, 0u);
            fence_proxy_async();
            wg_bar();
            issue_proj((J - 1) >> 3);
            wgmma_wait<0>();
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

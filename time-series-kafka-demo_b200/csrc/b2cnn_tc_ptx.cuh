// b2cnn_tc_ptx.cuh -- inline-PTX wrappers for TMA, mbarrier and wgmma (warpgroup MMA) on sm_90a,
// and the GMMA shared-memory descriptor encodings used by b2cnn_tc*.cu.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2cnn {

constexpr float k2Log2e = 2.8853900817779268f;

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
            : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    } while (!done);
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap *tm, int c0, int c1, int c2, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(dst), "l"(tm), "r"(c0), "r"(c1), "r"(c2), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *tm, int c0, int c1, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(dst), "l"(tm), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// register reallocation between warpgroups (every warp of a warpgroup executes the same one)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// named barrier of the consumer warpgroup (id 1, 128 threads): barrier 0 stays __syncthreads()
__device__ __forceinline__ void wg_bar() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// shared-memory accesses by 32-bit shared address (for addresses built with XOR swizzles)
__device__ __forceinline__ void st_shared_v4(uint32_t addr, float x, float y, float z, float w) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(x), "f"(y), "f"(z), "f"(w) : "memory");
}
__device__ __forceinline__ uint32_t ld_shared_u16(uint32_t addr) {
    uint16_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ float4 ld_shared_v4(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}

// max_nan: b2cnn_internal.cuh
__device__ __forceinline__ float max3_nan(float a, float b, float c) { return max_nan(max_nan(a, b), c); }
// tanh(m + bias) with bias pre-multiplied by 2 log2 e:  1 - 2 / (1 + 2^(2 log2e (m + bias)))
__device__ __forceinline__ float tanh_fold(float m, float bias_scaled) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(fmaf(m, k2Log2e, bias_scaled)));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
    return fmaf(-2.0f, r, 1.0f);
}
// r = 1 / (1 + 2^(2 log2e (m + bias))): tanh(m + bias) == 1 - 2 r.  conv2 consumes r directly (its weights are
// pre-multiplied by -2 and its bias absorbs sum(w)), saving the final FMA.  2^a = inf gives r = 0 without a clamp.
__device__ __forceinline__ float sig_fold(float m, float bias_scaled) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(fmaf(m, k2Log2e, bias_scaled)));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
    return r;
}
// two floats -> packed bf16x2 (round to nearest even): low half = lo_elem, high half = hi_elem
__device__ __forceinline__ uint32_t pack_bf16x2(float lo_elem, float hi_elem) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
    return r;
}

// ------------------------------------------------------------------------------------------
// wgmma (sm_90a): D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, A and B bf16 K-major in shared memory
// (m64n32: A in registers), D fp32 in registers.
// Fragment of D held by thread t of the warpgroup (warp w = t / 32, lane l): element i of the N/2 registers is
// row 16 w + l / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (l % 4) + i % 2.
// ------------------------------------------------------------------------------------------
// GMMA shared-memory descriptor: start >> 4 | LBO >> 4 << 16 | SBO >> 4 << 32 | layout << 62 (0 = no swizzle).
// No swizzle, K-major core matrices (8 rows x 16 bytes): LBO = K-adjacent core matrices, SBO = M/N-adjacent ones
__device__ __forceinline__ uint64_t gdesc_none_kmajor(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// the "+f" operands tie the accumulator registers to every wgmma and to the wait that follows.  A in registers:
// a[0..3] is thread t's m16k16 bf16 fragment of rows 16 w .. 16 w + 15 (the mma.m16n8k16 A layout, as ldmatrix_x4
// below loads it).  A wgmma reads a[] asynchronously: the registers must not change until the wait that retires it
// (wgmma_keep ties them to that wait).
__device__ __forceinline__ void wgmma_m64n32_rs(float *d, const uint32_t *a, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, %21, 0;\n"
        " wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate) : "memory");
}
// keeps the A fragment registers of in-flight wgmmas alive (and unmodified) up to this point: place after the wait
__device__ __forceinline__ void wgmma_keep(uint32_t *a) {
    asm volatile("" : "+r"(a[0]), "+r"(a[1]), "+r"(a[2]), "+r"(a[3]) :: "memory");
}
// an accumulator value copied out at this point, ahead of the next wgmma that overwrites its register.  A plain
// assignment of a value carried to the next block may be sunk past that wgmma's issue; it then reads an in-flight
// accumulator, and ptxas serializes every wgmma of the kernel (C7511).
__device__ __forceinline__ float acc_copy(float x) {
    float y;
    asm volatile("mov.b32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// four 8x8 b16 matrices from shared memory; lanes 8i .. 8i+7 give the row addresses of matrix i, which lands in r[i]
__device__ __forceinline__ void ldmatrix_x4(uint32_t *r, uint32_t saddr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(saddr) : "memory");
}
// always accumulates: D += A * B
__device__ __forceinline__ void wgmma_m64n64(float *d, uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, 1, 0;\n"
        " wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,"
        "%30,%31}, %32, %33, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc) : "memory");
}

}  // namespace b2cnn

// Thin inline-PTX layer over the Hopper (sm_90a) tensor-core path used by the fused kernels:
// wgmma.mma_async (operands in shared memory, fp32 accumulators in the registers of a warpgroup),
// mbarriers, bulk async copies (TMA 1-D) and the proxy fences between them.
//
// Operand layout (both A and B are K-major, SWIZZLE_NONE "interleaved" canonical layout):
//   the matrix is cut into 8-row x 16-byte core matrices, each stored as 128 contiguous bytes;
//   core matrices that are neighbours along M/N are SBO = 128 B apart, neighbours along K are
//   LBO = rows * 16 B apart.  Element (r, k) of a [rows, K] 16-bit matrix therefore lives at
//       (k / 8) * rows * 16  +  (r / 8) * 128  +  (r % 8) * 16  +  (k % 8) * 2      bytes,
//   i.e. for a fixed 8-wide k-chunk all rows form one contiguous slab of rows * 16 bytes.  A
//   thread that owns row r writes its 8 consecutive k-values with ONE 16-byte st.shared and a
//   warp (32 consecutive rows) writes 512 contiguous bytes -> conflict-free epilogue stores, and
//   a weight K-chunk is one contiguous range that a single cp.async.bulk can fetch.
// The same canonical layout is a wgmma operand (SWIZZLE_NONE descriptors), so the data formats of
// the kernels are independent of which tensor-core generation consumes them.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace tc05 {

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}

// ---- descriptors -----------------------------------------------------------------------------
// 64-bit shared-memory matrix descriptor of wgmma (layout type 0 = no swizzle, base offset 0):
//   [0,14) start address >> 4, [16,30) LBO >> 4, [32,46) SBO >> 4.
// K-major operands: LBO = distance of the two 8-element K core matrices, SBO = distance of 8-row groups.
// MN-major operands: LBO = distance of 8-sample (K) groups, SBO = distance of 8-element MN groups.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}

// ---- warpgroup MMA (sm_90a wgmma) -------------------------------------------------------------------
// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, both operands in shared memory, fp32 accumulators in the registers of the
// 128 threads of the issuing warpgroup (all of them execute it).  TA / TB = 1: the operand is MN-major (transposed).
// Accumulator fragment: thread t = 32 w + l holds d[4 j + 2 h + e] = D[16 w + l / 4 + 8 h][8 j + 2 (l % 4) + e].
template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_m64n16k16(float (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate) {
    if constexpr (BF16)
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                     : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
    else
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                     : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}

template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32k16(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
    if constexpr (BF16)
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                     : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
    else
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                     : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}

template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
    if constexpr (BF16)
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                     : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
    else
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                     : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}
// generic-proxy smem writes -> visible to the async proxy (tensor core / TMA reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// named barrier over the `threads` threads that use barrier `id` (1..15)
__device__ __forceinline__ void named_sync(uint32_t id, uint32_t threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// fragment row / column of accumulator element i of thread `t` of a warpgroup (see the layout above)
__device__ __forceinline__ int frag_row(int t, int i) { return ((t >> 5) << 4) + ((t & 31) >> 2) + (((i >> 1) & 1) << 3); }
__device__ __forceinline__ int frag_col(int t, int i) { return ((i >> 2) << 3) + ((t & 3) << 1) + (i & 1); }

// ---- mbarrier ----------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// For waits that are NOT on the critical path (producers running ahead): back off with nanosleep so
// the spinning warps do not steal issue slots from the warps doing the epilogue math on the same SMSP.
__device__ __forceinline__ void mbar_wait_backoff(uint64_t *bar, uint32_t parity, uint32_t ns = 256) {
    while (!mbar_try_wait(bar, parity)) __nanosleep(ns);
}

// ---- 1-D bulk async copy global -> shared (TMA engine), completion on an mbarrier -------------
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// ---- 16-bit packing ----------------------------------------------------------------------------
template <bool BF16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
    if constexpr (BF16) {
        __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t *>(&v);
    } else {
        __half2 v = __floats2half2_rn(a, b);
        return *reinterpret_cast<uint32_t *>(&v);
    }
}
template <bool BF16>
__device__ __forceinline__ float2 unpack2(uint32_t u) {
    if constexpr (BF16) {
        return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162 *>(&u));
    } else {
        return __half22float2(*reinterpret_cast<__half2 *>(&u));
    }
}

// byte offset of the 16-byte chunk holding elements (r, 8*kc .. 8*kc+7) of a [rows, K] operand
__host__ __device__ __forceinline__ constexpr uint32_t chunk_off(uint32_t rows, uint32_t r, uint32_t kc) {
    return kc * rows * 16u + (r >> 3) * 128u + (r & 7u) * 16u;
}

}  // namespace tc05

// Tensor-core self test: C[128, N] = A[128, K] * B[N, K]^T (fp32 accumulate) through exactly the
// shared-memory operand layouts and descriptors that the fused kernels use with wgmma (tc05.cuh).
// Used by tests/ to validate the operand layout on hardware.
#include "common.cuh"
#include "tc05.cuh"

namespace {

template <bool BF16>
__global__ void __launch_bounds__(128)
tc_selftest_kernel(const float *__restrict__ a, const float *__restrict__ b, float *__restrict__ c, int N, int K,
                   int variant)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *sA = smem;
    uint8_t *sB = smem + 130 * K * 2;
    const int tid = threadIdx.x;

    const int KC = K / 8;
    // variant 2 (layout of the convolution kernel, rendercnn.cu): A holds 130 rows per 8-column chunk -- a pixel row with a
    // one-pixel halo on either side -- and the operand starts ONE ROW (16 B) into it: a tap of a 3x3 convolution is the same
    // buffer read through a shifted start address.  Row r of `a` sits at buffer row r + 1; rows 0 and 129 are zero.
    if (variant == 2)
        for (int i = tid; i < 130 * KC; i += 128) *reinterpret_cast<uint4 *>(sA + i * 16) = make_uint4(0u, 0u, 0u, 0u);
    __syncthreads();
    for (int i = tid; i < 128 * KC; i += 128) {
        const int r = i / KC, kc = i % KC;
        const float *src = a + (size_t)r * K + kc * 8;
        uint4 v;
        v.x = tc05::pack2<BF16>(src[0], src[1]);
        v.y = tc05::pack2<BF16>(src[2], src[3]);
        v.z = tc05::pack2<BF16>(src[4], src[5]);
        v.w = tc05::pack2<BF16>(src[6], src[7]);
        *reinterpret_cast<uint4 *>(sA + (variant == 2 ? (uint32_t)(kc * 130 + r + 1) * 16u : tc05::chunk_off(128, r, kc))) = v;
    }
    for (int i = tid; i < N * KC; i += 128) {
        const int r = i / KC, kc = i % KC;
        const float *src = b + (size_t)r * K + kc * 8;
        uint4 v;
        v.x = tc05::pack2<BF16>(src[0], src[1]);
        v.y = tc05::pack2<BF16>(src[2], src[3]);
        v.z = tc05::pack2<BF16>(src[4], src[5]);
        v.w = tc05::pack2<BF16>(src[6], src[7]);
        *reinterpret_cast<uint4 *>(sB + tc05::chunk_off(N, r, kc)) = v;
    }
    tc05::fence_proxy_async_smem();
    __syncthreads();

    // one warpgroup: two 64-row blocks x 16-column slices of C, K in 16-wide steps
    const uint32_t lboA = (variant == 2 ? 130 : 128) * 16, lboB = N * 16, sbo = 128;
    for (int rb = 0; rb < 2; rb++) {
        for (int n0 = 0; n0 < N; n0 += 16) {
            float d[8];
            for (int kk = 0; kk < K / 16; kk++) {
                const uint32_t a0 = tc05::smem_u32(sA) + (variant == 2 ? 16u : 0u) + kk * 2 * lboA + rb * 1024;
                const uint32_t b0 = tc05::smem_u32(sB) + kk * 2 * lboB + n0 * 16;
                uint64_t da, db;
                if (variant == 1) {      // LBO / SBO meaning swapped (diagnostic)
                    da = tc05::make_smem_desc(a0, sbo, lboA);
                    db = tc05::make_smem_desc(b0, sbo, lboB);
                } else {
                    da = tc05::make_smem_desc(a0, lboA, sbo);
                    db = tc05::make_smem_desc(b0, lboB, sbo);
                }
                tc05::wgmma_fence();
                tc05::wgmma_m64n16k16<BF16, 0, 0>(d, da, db, kk > 0 ? 1u : 0u);
                tc05::wgmma_commit();
                tc05::wgmma_wait<0>();
                tc05::wgmma_fence_acc(d);
            }
#pragma unroll
            for (int i = 0; i < 8; i++)
                c[(size_t)(rb * 64 + tc05::frag_row(tid, i)) * N + n0 + tc05::frag_col(tid, i)] = d[i];
        }
    }
}

}  // namespace

extern "C" int sdb_tc_selftest(const float *d_a, const float *d_b, float *d_c, int32_t N, int32_t K,
                               int32_t use_bf16, int32_t variant, void *stream)
{
    if (!d_a || !d_b || !d_c) return SDB_EINVAL;
    if (N < 16 || N > 256 || N % 16 || K < 16 || K > 256 || K % 16) return SDB_EINVAL;
    const size_t smem = (size_t)130 * K * 2 + (size_t)N * K * 2 + 64;
    if (use_bf16) {
        SDB_CUDA(cudaFuncSetAttribute(tc_selftest_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        tc_selftest_kernel<true><<<1, 128, smem, (cudaStream_t)stream>>>(d_a, d_b, d_c, N, K, variant);
    } else {
        SDB_CUDA(cudaFuncSetAttribute(tc_selftest_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        tc_selftest_kernel<false><<<1, 128, smem, (cudaStream_t)stream>>>(d_a, d_b, d_c, N, K, variant);
    }
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}


// ---- MN-major operands (diagnostic for the planned weight-gradient kernel) ---------------------------------------------
// C[F=128, G] = X^T Y with X [S=128 samples, 128], Y [S=128, G]: the SAMPLES are the reduction dimension, and X / Y sit in
// shared memory exactly as the fused kernels keep activations: [feature chunk of 8][128 sample rows][8 features] (16 B per
// row), read by wgmma with both operands transposed (MN-major).  Read as an MMA operand with M (or N) = features and K = samples this is an MN-major canonical layout: 8 features
// contiguous, the 8 samples of a core matrix 16 B apart, next 8 samples +128 B, next 8 features +2048 B.
// variant 0: LBO = 128 (K direction), SBO = 2048 (MN direction); variant 1: swapped.
namespace {
__global__ void __launch_bounds__(128)
tc_selftest_mn_kernel(const float *__restrict__ x, const float *__restrict__ y, float *__restrict__ c, int G, int variant)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *sX = smem;
    uint8_t *sY = smem + 128 * 128 * 2;
    const int tid = threadIdx.x;
    for (int i = tid; i < 128 * 16; i += 128) {           // X: 128 samples x 16 feature chunks
        const int r = i / 16, kc = i % 16;
        const float *src = x + (size_t)r * 128 + kc * 8;
        *reinterpret_cast<uint4 *>(sX + tc05::chunk_off(128, r, kc)) =
            make_uint4(tc05::pack2<true>(src[0], src[1]), tc05::pack2<true>(src[2], src[3]), tc05::pack2<true>(src[4], src[5]),
                       tc05::pack2<true>(src[6], src[7]));
    }
    for (int i = tid; i < 128 * (G / 8); i += 128) {
        const int r = i / (G / 8), kc = i % (G / 8);
        const float *src = y + (size_t)r * G + kc * 8;
        *reinterpret_cast<uint4 *>(sY + tc05::chunk_off(128, r, kc)) =
            make_uint4(tc05::pack2<true>(src[0], src[1]), tc05::pack2<true>(src[2], src[3]), tc05::pack2<true>(src[4], src[5]),
                       tc05::pack2<true>(src[6], src[7]));
    }
    tc05::fence_proxy_async_smem();
    __syncthreads();
    const uint32_t kdir = 128, mndir = 128 * 16;
    const uint32_t lbo = variant == 0 ? kdir : mndir, sbo = variant == 0 ? mndir : kdir;
    for (int rb = 0; rb < 2; rb++) {                       // features 64 rb .. 64 rb + 63 = 8 chunks of 8
        for (int n0 = 0; n0 < G; n0 += 16) {
            float d[8];
            for (int kk = 0; kk < 8; kk++) {              // 16 samples per MMA
                const uint64_t da = tc05::make_smem_desc(tc05::smem_u32(sX) + rb * 8 * mndir + kk * 256, lbo, sbo);
                const uint64_t db = tc05::make_smem_desc(tc05::smem_u32(sY) + (n0 / 8) * mndir + kk * 256, lbo, sbo);
                tc05::wgmma_fence();
                tc05::wgmma_m64n16k16<true, 1, 1>(d, da, db, kk > 0 ? 1u : 0u);
                tc05::wgmma_commit();
                tc05::wgmma_wait<0>();
                tc05::wgmma_fence_acc(d);
            }
#pragma unroll
            for (int i = 0; i < 8; i++)
                c[(size_t)(rb * 64 + tc05::frag_row(tid, i)) * G + n0 + tc05::frag_col(tid, i)] = d[i];
        }
    }
}
}  // namespace

extern "C" int sdb_tc_selftest_mn(const float *d_x, const float *d_y, float *d_c, int32_t G, int32_t variant, void *stream)
{
    if (!d_x || !d_y || !d_c) return SDB_EINVAL;
    if (G < 16 || G > 256 || G % 16) return SDB_EINVAL;
    const size_t smem = (size_t)128 * 128 * 2 + (size_t)128 * G * 2 + 64;
    SDB_CUDA(cudaFuncSetAttribute(tc_selftest_mn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    tc_selftest_mn_kernel<<<1, 128, smem, (cudaStream_t)stream>>>(d_x, d_y, d_c, G, variant);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}

// Weight gradients of the per-pixel networks on the Hopper tensor cores (sm_90a, wgmma):  dW[n_out, k_in] = sum over samples of
// dZ[sample, n_out] * A[sample, k_in]  -- the backward of nn.Linear / ModLinear (imaginaire/model_utils/layers.py:247-269,
// :92-126) and of SKYMLP's layers (generators/gancraft_base.py:150-169) under torch.autograd in the reference.
//
// The SAMPLES are the reduction dimension.  The forward / gradient-chain kernels leave their bf16 records as MMA-ready
// tiles (rf_common.cuh: rec_chunk):  [work item][8-column chunk][128 sample rows][8 columns]  = 16 B per (row, chunk),
// 2 KB per chunk, so one item of an array is ONE contiguous range that a single 1-D bulk copy (TMA engine) drops into shared
// memory, where it IS a canonical MN-major, no-swizzle wgmma operand with K = samples: 8 columns contiguous, the 8
// samples of a core matrix 16 B apart, K-adjacent core matrices +128 B (LBO), MN-adjacent ones +2048 B (SBO)
// (operand form verified by sdb_tc_selftest_mn).  No transpose, no zero-filled padding, no library GEMM.
//
// Work decomposition: the output of every layer is cut into M-tiles of 128 rows of n_out ("jobs"); a job's samples are
// split over several CTAs (interleaved items, so the CTAs of the two M-tiles of a layer stream the same A tiles at the same
// time and the second read hits L2).  One CTA = one job x one split: fp32 accumulators [128 x k_in] stay in the registers of
// two warpgroups (64 rows each) for the whole reduction, then are added to the (zeroed) gradient with red.global.add.
// Thread 0 issues the bulk copies (2-stage ring, 100 KB per stage) one item ahead of the MMAs.
// Bound: HBM -- per sample and M-tile 800 B in, 17.8 MFLOP per 128-sample item against ~2.3 us of load time per SM.
#include "rf_common.cuh"
#include "wgrad.cuh"

namespace rf {

namespace {
constexpr int kWgStages = 2;
constexpr int kWgThreads = 256;
constexpr uint32_t kChunkBytes = kRows * 16;                  // 2048: one 8-column chunk of a 128-sample item
constexpr uint32_t kWgABytes = (kActCols / 8) * kChunkBytes;  // 69,632: the widest A tile (272 columns)
constexpr uint32_t kWgZBytes = 16 * kChunkBytes;              // 32,768: 128 columns of dZ
constexpr uint32_t kWgStageBytes = kWgABytes + kWgZBytes;
constexpr uint32_t kWgSmem = kWgStages * kWgStageBytes + 256;

struct WgParams {
    WgJob job[kWgMaxJobs];
    int n_jobs;
    const int32_t *view;         // device: {first, count} live ray tiles of the recorded pass (nullptr: every item up to cap_items exists)
    int items_per_live;
    long long cap_items;
};

__global__ void __launch_bounds__(kWgThreads, 1)
wgrad_kernel(const WgParams prm)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + kWgStages * kWgStageBytes);      // full[2], empty[2]
    const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127;

    // which (job, split) is this CTA?
    int j = 0, split = blockIdx.x;
    while (j < prm.n_jobs && split >= prm.job[j].nsplit) { split -= prm.job[j].nsplit; j++; }
    if (j >= prm.n_jobs) return;
    WgJob jb = prm.job[j];
    const long long n_items = prm.view ? (long long)__ldg(prm.view + 1) * prm.items_per_live : prm.cap_items;
    if (prm.view) jb.A += (size_t)__ldg(prm.view) * prm.items_per_live * jb.a_chunks * (kChunkBytes / 2);      // A: this image's record items
    const long long my_items = split < n_items ? (n_items - split + jb.nsplit - 1) / jb.nsplit : 0;

    // dZ chunks the job does not own stay zero for the whole kernel (M-tiles narrower than 128 rows: fc_out_c, fc_sigma)
    for (int s = 0; s < kWgStages; s++) {
        uint4 *z = reinterpret_cast<uint4 *>(smem + s * kWgStageBytes + kWgABytes);
        for (uint32_t i = tid; i < kWgZBytes / 16; i += kWgThreads) z[i] = make_uint4(0u, 0u, 0u, 0u);
    }
    if (tid == 0) {
        for (int s = 0; s < kWgStages; s++) { tc05::mbar_init(&bars[s], 1); tc05::mbar_init(&bars[kWgStages + s], 2); }
        tc05::fence_mbar_init();
    }
    tc05::fence_proxy_async_smem();
    __syncthreads();
    if (my_items == 0) return;
    const uint32_t a_bytes = (uint32_t)jb.a_chunks * kChunkBytes, z_bytes = (uint32_t)jb.z_chunks * kChunkBytes;
    auto load = [&](long long n) {           // one bulk copy per operand and item into stage n % 2
        const int s = (int)(n % kWgStages);
        if (n >= kWgStages) tc05::mbar_wait(&bars[kWgStages + s], (uint32_t)((n / kWgStages - 1) & 1));
        const long long item = split + n * jb.nsplit;
        uint8_t *sA = smem + s * kWgStageBytes, *sZ = sA + kWgABytes;
        tc05::mbar_arrive_expect_tx(&bars[s], a_bytes + z_bytes);
        tc05::bulk_g2s(sA, reinterpret_cast<const uint8_t *>(jb.A) + (size_t)item * a_bytes, a_bytes, &bars[s]);
        tc05::bulk_g2s(sZ, reinterpret_cast<const uint8_t *>(jb.Z) + ((size_t)item * jb.z_chunks_total + jb.z_chunk0) * kChunkBytes,
                       z_bytes, &bars[s]);
    };
    if (tid == 0) load(0);

    // warpgroup wg accumulates output rows 64 wg .. 64 wg + 63: D[64 x N] += Zpart^T [64 x 128 samples] * A [128 samples x N],
    // 16 samples per step, N in 16-column slices (k_in = 272 = 17 slices); both operands MN-major
    const int N = jb.a_chunks * 8;
    const bool rows_live = wg * 8 < jb.z_chunks;           // warpgroup-uniform: rows past the job's M-tile stay zero
    float acc[kActCols / 16][8];
#pragma unroll
    for (int q = 0; q < kActCols / 16; q++)
#pragma unroll
        for (int i = 0; i < 8; i++) acc[q][i] = 0.0f;
    for (long long n = 0; n < my_items; n++) {
        const int s = (int)(n % kWgStages);
        if (tid == 0 && n + 1 < my_items) load(n + 1);     // the other stage: free once both warpgroups finished item n - 1
        tc05::mbar_wait(&bars[s], (uint32_t)((n / kWgStages) & 1));
        if (rows_live) {
            const uint32_t sA = tc05::smem_u32(smem + s * kWgStageBytes), sZ = sA + kWgABytes;
            tc05::wgmma_fence();
#pragma unroll 1
            for (int kk = 0; kk < kRows / 16; kk++) {
                const uint64_t dz = tc05::make_smem_desc(sZ + wg * 8 * kChunkBytes + kk * 256, 128, kChunkBytes);
#pragma unroll
                for (int q = 0; q < kActCols / 16; q++)
                    if (16 * q < N)
                        tc05::wgmma_m64n16k16<true, 1, 1>(acc[q], dz, tc05::make_smem_desc(sA + 2 * q * kChunkBytes + kk * 256, 128, kChunkBytes), 1u);
            }
            tc05::wgmma_commit();
            tc05::wgmma_wait<0>();
#pragma unroll
            for (int q = 0; q < kActCols / 16; q++) tc05::wgmma_fence_acc(acc[q]);
        }
        tc05::named_sync(1 + wg, 128);
        if (t == 0) tc05::mbar_arrive(&bars[kWgStages + s]);       // this warpgroup is done reading the stage
    }
    // ---- accumulators -> gradient ----
    if (!rows_live) return;
#pragma unroll
    for (int q = 0; q < kActCols / 16; q++) {
        if (16 * q >= N) break;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int row = wg * 64 + tc05::frag_row(t, i);
            if (row < jb.rows) atomicAdd(jb.out + (size_t)(jb.row0 + row) * jb.ld_out + 16 * q + tc05::frag_col(t, i), acc[q][i]);
        }
    }
}
}  // namespace

// Splits: CTAs are handed out in proportion to the bytes a job streams per item, one CTA per SM over the whole list.
int launch_wgrad(WgJob *jobs, int n_jobs, const int32_t *d_view, int items_per_live, long long cap_items, cudaStream_t st)
{
    if (n_jobs < 1 || n_jobs > kWgMaxJobs) return SDB_EINVAL;
    if (cap_items <= 0) return SDB_OK;
    const long long n_items = cap_items;
    WgParams prm{};
    prm.n_jobs = n_jobs;
    prm.view = d_view;
    prm.items_per_live = items_per_live;
    prm.cap_items = cap_items;
    double total = 0.0;
    for (int i = 0; i < n_jobs; i++) {
        const WgJob &jb = jobs[i];
        if (!jb.A || !jb.Z || !jb.out || jb.a_chunks < 1 || jb.a_chunks > kActCols / 8 || (jb.a_chunks * 8) % 16 != 0 ||
            jb.z_chunks < 1 || jb.z_chunks > 16 || jb.z_chunk0 + jb.z_chunks > jb.z_chunks_total || jb.rows < 1 || jb.rows > 128)
            return SDB_EINVAL;
        total += jb.a_chunks + jb.z_chunks;
    }
    const int sms = sdb_num_sms();
    int used = 0;
    for (int i = 0; i < n_jobs; i++) {
        int ns = (int)((double)sms * (jobs[i].a_chunks + jobs[i].z_chunks) / total);
        if (ns < 1) ns = 1;
        if ((long long)ns > n_items) ns = (int)n_items;
        jobs[i].nsplit = ns;
        used += ns;
        prm.job[i] = jobs[i];
    }
    SDB_CUDA(cudaFuncSetAttribute(wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kWgSmem));
    wgrad_kernel<<<used, kWgThreads, kWgSmem, st>>>(prm);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}

}  // namespace rf
